// Micro-benchmarks of the warp primitives the sort / binning kernels lean on (development aid).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/ubench tools/ubench.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

#define ITERS 512

template <int OP>
__global__ void lat_kernel(int K, uint32_t seed, long long* out_cycles, uint32_t* sink, uint32_t* gbuf) {
    __shared__ uint32_t sm[4096];
    const int lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < 4096; i += blockDim.x) sm[i] = i;
    __syncthreads();
    uint32_t v = (uint32_t)(lane % K) + seed;       // K distinct values in the warp
    uint32_t acc = seed;
    float f = 1.0f + lane + seed;
    const long long t0 = clock64();
#pragma unroll 1
    for (int it = 0; it < ITERS; ++it) {
        if (OP == 0) { acc += __match_any_sync(0xffffffffu, v + (acc == 0xdeadbeefu)); }
        if (OP == 1) {   // ballot-based 8-bit match
            const uint32_t d = v + (acc == 0xdeadbeefu);
            uint32_t peers = 0xffffffffu;
#pragma unroll
            for (int b = 0; b < 8; ++b) { const uint32_t m = __ballot_sync(0xffffffffu, (d >> b) & 1u); peers &= ((d >> b) & 1u) ? m : ~m; }
            acc += peers;
        }
        if (OP == 2) { acc += __shfl_sync(0xffffffffu, acc, (lane + 1) & 31); }
        if (OP == 3) { acc += __ballot_sync(0xffffffffu, (acc + lane) & 1u); }
        if (OP == 4) { acc += __reduce_or_sync(0xffffffffu, acc + lane); }
        if (OP == 5) { acc += atomicAdd(&sm[(lane * 33 + (acc & 1u)) & 4095], 1u); }            // ATOMS w/ return, spread
        if (OP == 6) { atomicAdd(&sm[(lane * 33 + it) & 4095], 1u); }                              // RED.shared no return
        if (OP == 7) { const uint32_t a = (lane * 33 + (acc & 1u)) & 4095; const uint32_t o = sm[a]; sm[a] = o + 1; acc += o; __syncwarp(); }
        if (OP == 8) { f = __frcp_rd(f) + 1.0f; }
        if (OP == 9) { acc = (acc + 1000003u) / (v | 1u) + seed; }
        if (OP == 10) { f = __fdividef(1.0f, f) + 1.0f; }
        if (OP == 11) { acc += __popc(__ballot_sync(0xffffffffu, acc > (uint32_t)lane)) + __ffs(acc); }
        if (OP == 12) { acc += gbuf[(acc & 1023u) * 32 + lane]; }                                  // dependent L2/L1 load
        if (OP == 13) { acc += __ldcg(gbuf + ((acc & 1023u) * 32 + lane)); }                       // dependent L2 load
    }
    const long long t1 = clock64();
    if (threadIdx.x == 0 && blockIdx.x == 0) *out_cycles = t1 - t0;
    sink[blockIdx.x * blockDim.x + threadIdx.x] = acc + (uint32_t)f + sm[lane];
}

// throughput of warp-wide scattered 4-byte stores: every lane its own 32B sector vs coalesced
__global__ void store_kernel(uint32_t* buf, size_t words, int scattered, int reps) {
    const size_t gw = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    const size_t nwarps = (size_t)gridDim.x * (blockDim.x >> 5);
    for (int r = 0; r < reps; ++r) {
        size_t idx;
        if (scattered) idx = (((gw * 2654435761ull + (size_t)r * 40503ull) * 32 + lane) * 12345701ull) % (words / 8) * 8;    // random sector per lane
        else idx = ((gw + (size_t)r * nwarps) * 32 + lane) % words;
        buf[idx] = (uint32_t)r;
    }
}

template <int OP>
void run_lat(const char* name, int K, long long* d_cyc, uint32_t* d_sink, uint32_t* gbuf) {
    lat_kernel<OP><<<1, 32>>>(K, 0, d_cyc, d_sink, gbuf);
    lat_kernel<OP><<<1, 32>>>(K, 0, d_cyc, d_sink, gbuf);
    long long c = 0;
    cudaMemcpy(&c, d_cyc, 8, cudaMemcpyDeviceToHost);
    // throughput flavour: 16 warps on one SM
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    lat_kernel<OP><<<132, 512>>>(K, 0, d_cyc, d_sink, gbuf);
    cudaEventRecord(e0);
    lat_kernel<OP><<<132, 512>>>(K, 0, d_cyc, d_sink, gbuf);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
    long long c16 = 0;
    cudaMemcpy(&c16, d_cyc, 8, cudaMemcpyDeviceToHost);
    printf("{\"op\": \"%s\", \"K\": %d, \"cyc_per_iter_1warp\": %.1f, \"cyc_per_iter_16warps_per_SM\": %.1f, \"ms_132x16warps\": %.4f}\n", name, K,
           (double)c / ITERS, (double)c16 / ITERS, ms);
}

int main() {
    long long* d_cyc; uint32_t* d_sink; uint32_t* gbuf;
    cudaMalloc(&d_cyc, 8); cudaMalloc(&d_sink, 132 * 512 * 4); cudaMalloc(&gbuf, 1024 * 32 * 4);
    cudaMemset(gbuf, 0, 1024 * 32 * 4);
    for (int K : {1, 4, 16, 32}) run_lat<0>("match_any", K, d_cyc, d_sink, gbuf);
    for (int K : {1, 32}) run_lat<1>("ballot_match_8bit", K, d_cyc, d_sink, gbuf);
    run_lat<2>("shfl", 32, d_cyc, d_sink, gbuf);
    run_lat<3>("ballot", 32, d_cyc, d_sink, gbuf);
    run_lat<4>("redux_or", 32, d_cyc, d_sink, gbuf);
    run_lat<5>("atoms_return_spread", 32, d_cyc, d_sink, gbuf);
    run_lat<6>("red_shared_spread", 32, d_cyc, d_sink, gbuf);
    run_lat<7>("lds_sts_syncwarp", 32, d_cyc, d_sink, gbuf);
    run_lat<8>("frcp_rd", 32, d_cyc, d_sink, gbuf);
    run_lat<9>("udiv32", 32, d_cyc, d_sink, gbuf);
    run_lat<10>("fdividef", 32, d_cyc, d_sink, gbuf);
    run_lat<11>("ballot_popc_ffs", 32, d_cyc, d_sink, gbuf);
    run_lat<12>("dependent_ld_global", 32, d_cyc, d_sink, gbuf);
    run_lat<13>("dependent_ldcg", 32, d_cyc, d_sink, gbuf);

    const size_t words = (size_t)64 << 20;     // 256 MB
    uint32_t* big; cudaMalloc(&big, words * 4);
    for (int scattered = 0; scattered <= 1; ++scattered) {
        cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
        const int reps = 64;
        store_kernel<<<132 * 8, 256>>>(big, words, scattered, reps);
        cudaEventRecord(e0);
        store_kernel<<<132 * 8, 256>>>(big, words, scattered, reps);
        cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
        const double n = (double)132 * 8 * 8 * 32 * reps;
        printf("{\"op\": \"store_%s\", \"stores\": %.0f, \"ms\": %.4f, \"Gstores_per_s\": %.2f}\n", scattered ? "scattered_sector_per_lane" : "coalesced", n, ms, n / ms / 1e6);
    }
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { printf("cuda error %s\n", cudaGetErrorString(e)); return 1; }
    return 0;
}
