// Visibility of the per-pixel shading (include/r3dg_b200.h, PIXEL SHADING; DESIGN.md §4.29): N rays from the surface
// point of every valid pixel, around its unit normal, through the LBVH of the scene's Gaussians.  The ray of (pixel,
// sample i) is the one r3dg_bvh_trace_opacity traces for origin points_p, direction rotate_from_z(n^, fib_sample(i, N))
// and origin offset 0.05, so T is the same bits.  Compiled with the bake's flags (bvh.cu).
#include "bvh.cuh"
#include "importance.cuh"
#include "kernels.h"

namespace r3dg {

#define PT_THREADS 128
#define PT_TILE 8                   // pixels are numbered in PT_TILE x PT_TILE tiles: neighbouring rays, nearby surface points
#define PT_ORIGIN_OFFSET 0.05f      // bvh/__init__.py:63

// The bake's persistent trace loop (bvh_trace_kernel, kept as written there so that its SASS is unchanged) with the
// ray setup as a parameter.  `setup(ray, o, d, out)` starts ray `ray`, or returns false for a ray that is not traced
// (a masked pixel's, whose T it writes, or one outside the image); such rays do not hold a lane: the refill repeats
// until every lane has a ray or the rays are exhausted.  Stop rule and hit rule are the bake's: T < 0.9 writes 0.
template <class S>
__device__ __forceinline__ void trace_opacity_rays(const S& setup, long long num_rays, int NI, const float4* __restrict__ packets,
                                                   float* __restrict__ T_out, unsigned long long* counter,
                                                   int (*sStack)[PT_THREADS]) {
    const int tid = threadIdx.x, lane = tid & 31;
    SplitStack<PT_THREADS> st;
    st.sh = sStack; st.tid = tid; st.sp = 0;
    bool has_ray = false, exhausted = false;
    long long out = 0;
    float ox = 0, oy = 0, oz = 0, dx = 0, dy = 0, dz = 0, ix = 0, iy = 0, iz = 0, T = 1.0f;
    while (true) {
        while (true) {                                   // refill idle lanes from the global ray counter (warp-aggregated)
            const unsigned want = __ballot_sync(0xffffffffu, !has_ray && !exhausted);
            if (!want) break;
            const int leader = __ffs(want) - 1;
            unsigned long long base = 0;
            if (lane == leader) base = atomicAdd(counter, (unsigned long long)__popc(want));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (!has_ray && !exhausted) {
                const long long ray = (long long)base + __popc(want & ((1u << lane) - 1u));
                if (ray >= num_rays) {
                    exhausted = true;
                } else if (setup(ray, ox, oy, oz, dx, dy, dz, out)) {
                    ix = div_(1.0f, dx); iy = div_(1.0f, dy); iz = div_(1.0f, dz);
                    has_ray = true; T = 1.0f;
                    st.sp = 0; st.push(NI == 0 ? -1 : 0);         // root (a lone leaf when P == 1)
                }
            }
        }
        if (!__any_sync(0xffffffffu, has_ray)) break;
        // ---- a bounded burst of traversal steps, ended early once 8+ lanes can be refilled (the bake's policy) ----
#pragma unroll 1
        for (int step = 0; step < 32; ++step) {
            if (step > 0 && (step & 3) == 0 && __popc(__ballot_sync(0xffffffffu, !has_ray && !exhausted)) >= 8) break;
            if (!has_ray) continue;
            const int node = st.pop();
            if (node >= 0) {
                const float4* p = packets + (size_t)node * 4;
                const float4 p0 = p[0], p1 = p[1], p2 = p[2], p3 = p[3];
                const int l = __float_as_int(p0.x), r = __float_as_int(p0.y);
                const float lmax = ray_box_tmax(p0.z, p0.w, p1.x, p1.y, p1.z, p1.w, ox, oy, oz, ix, iy, iz);
                const float rmax = ray_box_tmax(p2.x, p2.y, p2.z, p2.w, p3.x, p3.y, ox, oy, oz, ix, iy, iz);
                if (lmax > rmax) {                                    // far child first
                    if (lmax > 0) st.push(l);
                    if (rmax > 0) st.push(r);
                } else {
                    if (rmax > 0) st.push(r);
                    if (lmax > 0) st.push(l);
                }
            } else {
                const LeafRecord q = load_leaf(packets + (size_t)(NI - node - 1) * 4);   // leaf slot = -node - 1
                float t, power;
                if (gaussian_hit(q, ox, oy, oz, dx, dy, dz, t, power)) {
                    const float alpha = q.op * __expf(power);
                    T *= 1 - alpha;
                    if (T < 0.9f) {                                   // the bake's stop rule
                        T_out[out] = 0.0f;
                        has_ray = false;
                    }
                }
            }
            if (has_ray && st.sp == 0) {
                T_out[out] = T;
                has_ray = false;
            }
        }
    }
}

// Ray r = (cell r / N, sample r % N); cell c of view v = c / cells is pixel (c % 64) of tile (c % cells) / 64, tiles
// in rows of tiles_x.  Output T[v,i,p].
struct PixelRays {
    int N, W, H, tiles_x;
    long long cells;                 // PT_TILE^2 * tiles per view
    const float *normal, *points;    // [V,3,H,W]
    const uint8_t* mask;             // [V,H,W] or NULL
    const float3* smp;               // the N canonical samples
    float* T;
    __device__ __forceinline__ bool operator()(long long ray, float& ox, float& oy, float& oz, float& dx, float& dy, float& dz,
                                               long long& out) const {
        const long long cell = ray / N;
        const int i = (int)(ray - cell * N);
        const long long v = cell / cells;
        const long long c = cell - v * cells;
        const long long tile = c / (PT_TILE * PT_TILE);
        const int w = (int)(c - tile * (PT_TILE * PT_TILE));
        const int px = (int)(tile % tiles_x) * PT_TILE + w % PT_TILE, py = (int)(tile / tiles_x) * PT_TILE + w / PT_TILE;
        if (px >= W || py >= H) return false;
        const size_t HW = (size_t)H * W, p = (size_t)py * W + px;
        out = ((long long)v * N + i) * (long long)HW + (long long)p;
        if (mask && !mask[v * HW + p]) { T[out] = 0.0f; return false; }
        const float* nb = normal + 3 * v * HW + p;
        const float3 n = unit_normal(nb[0], nb[HW], nb[2 * HW]);
        const float3 d = rotate_from_z(n.x, n.y, n.z, smp[i]);
        dx = d.x; dy = d.y; dz = d.z;
        const float* pb = points + 3 * v * HW + p;
        ox = add_(pb[0], mul_(dx, PT_ORIGIN_OFFSET)); oy = add_(pb[HW], mul_(dy, PT_ORIGIN_OFFSET)); oz = add_(pb[2 * HW], mul_(dz, PT_ORIGIN_OFFSET));
        return true;
    }
};

// The same rays along the importance sampler's directions (include/r3dg_b200.h, IMPORTANCE SAMPLING): sample i of
// pixel p = y W + x is importance_sample(q = p), with the GGX frame of viewdir campos_v - point_p and the pixel's
// roughness when the sampler has GGX samples.
struct ImportancePixelRays {
    int N, W, H, tiles_x;
    long long cells;
    const float *normal, *points, *roughness, *campos;   // roughness [V,1,H,W], campos [V,3]: read when n_ggx > 0
    const uint8_t* mask;
    ImportanceSampler s;
    float* T;
    __device__ __forceinline__ bool operator()(long long ray, float& ox, float& oy, float& oz, float& dx, float& dy, float& dz,
                                               long long& out) const {
        const long long cell = ray / N;
        const int i = (int)(ray - cell * N);
        const long long v = cell / cells;
        const long long c = cell - v * cells;
        const long long tile = c / (PT_TILE * PT_TILE);
        const int w = (int)(c - tile * (PT_TILE * PT_TILE));
        const int px = (int)(tile % tiles_x) * PT_TILE + w % PT_TILE, py = (int)(tile / tiles_x) * PT_TILE + w / PT_TILE;
        if (px >= W || py >= H) return false;
        const size_t HW = (size_t)H * W, p = (size_t)py * W + px;
        out = ((long long)v * N + i) * (long long)HW + (long long)p;
        if (mask && !mask[v * HW + p]) { T[out] = 0.0f; return false; }
        const float* nb = normal + 3 * v * HW + p;
        const float3 n = unit_normal(nb[0], nb[HW], nb[2 * HW]);
        const float* pb = points + 3 * v * HW + p;
        GgxFrame f{};
        if (s.n_ggx > 0)
            f = ggx_frame(n, sub_(campos[3 * v], pb[0]), sub_(campos[3 * v + 1], pb[HW]), sub_(campos[3 * v + 2], pb[2 * HW]),
                          roughness[v * HW + p]);
        float area;
        const float3 d = importance_sample(s, (uint32_t)p, i, n, f, area);
        dx = d.x; dy = d.y; dz = d.z;
        ox = add_(pb[0], mul_(dx, PT_ORIGIN_OFFSET)); oy = add_(pb[HW], mul_(dy, PT_ORIGIN_OFFSET)); oz = add_(pb[2 * HW], mul_(dz, PT_ORIGIN_OFFSET));
        return true;
    }
};

__global__ void __launch_bounds__(PT_THREADS) bvh_pixel_importance_kernel(int P, long long num_rays, ImportancePixelRays rays,
                                                                          const float* __restrict__ table,
                                                                          const float4* __restrict__ packets, unsigned long long* counter) {
    __shared__ int sStack[TRACE_STACK_SH][PT_THREADS];
    rays.s.t = EnvTable(table);
    trace_opacity_rays(rays, num_rays, P - 1, packets, rays.T, counter, sStack);
}

__global__ void __launch_bounds__(PT_THREADS) bvh_pixel_trace_kernel(int P, long long num_rays, PixelRays rays,
                                                                     const float4* __restrict__ packets, unsigned long long* counter) {
    __shared__ int sStack[TRACE_STACK_SH][PT_THREADS];
    extern __shared__ float3 sSample[];
    for (int i = threadIdx.x; i < rays.N; i += PT_THREADS) sSample[i] = fib_sample(i, rays.N);
    __syncthreads();
    rays.smp = sSample;
    trace_opacity_rays(rays, num_rays, P - 1, packets, rays.T, counter, sStack);
}

}  // namespace r3dg

using namespace r3dg;
extern "C" {

size_t r3dg_bvh_trace_pixels_tmp_bytes(int P) { return bvh_packets_bytes(P); }

int r3dg_bvh_trace_pixels(const r3dg_pixel_args* a, int P, const int32_t* nodes, const float* aabbs, const float* means3D,
                          const float* covs3D, const float* opacities, const float* normals, float* T, void* tmp,
                          size_t tmp_bytes, r3dg_stream_t stream_) {
    if (!a || a->V < 1 || a->V > R3DG_MAX_VIEWS || a->H < 1 || a->W < 1 || a->N < 1 || P < 1) return R3DG_ERR_BAD_ARG;
    if (!a->normal || !a->points || !nodes || !aabbs || !means3D || !covs3D || !opacities || !normals || !T || !tmp)
        return R3DG_ERR_BAD_ARG;
    if (tmp_bytes < bvh_packets_bytes(P)) return R3DG_ERR_BAD_ARG;
    if ((size_t)a->N * sizeof(float3) > BAKE_SAMPLE_SMEM) return R3DG_ERR_UNSUPPORTED;
    if ((long long)a->V * a->H * a->W > 0x7fffffffLL) return R3DG_ERR_UNSUPPORTED;
    const cudaStream_t stream = (cudaStream_t)stream_;
    unsigned long long* counter = (unsigned long long*)tmp;
    float4* packets = (float4*)((char*)tmp + 256);
    R3DG_CUDA_TRY(cudaMemsetAsync(counter, 0, 8, stream));
    const int rc = launch_bvh_pack(P, nodes, aabbs, means3D, covs3D, opacities, normals, packets, stream);
    if (rc != 0) return rc;
    if (a->sampler_table && (a->n_env < 0 || a->n_ggx < 0 || (long long)a->N - a->n_env - a->n_ggx < 1)) return R3DG_ERR_BAD_ARG;
    if (a->sampler_table && a->n_ggx > 0 && (!a->roughness || !a->campos)) return R3DG_ERR_BAD_ARG;
    const int tiles_x = (a->W + PT_TILE - 1) / PT_TILE, tiles_y = (a->H + PT_TILE - 1) / PT_TILE;
    const PixelRays rays{a->N, a->W, a->H, tiles_x, (long long)tiles_x * tiles_y * PT_TILE * PT_TILE, a->normal, a->points,
                         a->mask, nullptr, T};
    const long long num_rays = (long long)a->V * rays.cells * a->N;
    const long long want = (num_rays + PT_THREADS - 1) / PT_THREADS;
    const int blocks = (int)(want < (long long)num_sms() * 16 ? want : (long long)num_sms() * 16);
    if (a->sampler_table) {
        ImportancePixelRays ir{a->N, a->W, a->H, tiles_x, rays.cells, a->normal, a->points, a->roughness, a->campos, a->mask,
                               ImportanceSampler{}, T};
        ir.s.T = a->sampler_transform; ir.s.N = a->N; ir.s.n_env = a->n_env; ir.s.n_ggx = a->n_ggx; ir.s.seed = a->seed;
        bvh_pixel_importance_kernel<<<blocks, PT_THREADS, 0, stream>>>(P, num_rays, ir, a->sampler_table, packets, counter);
    } else {
        bvh_pixel_trace_kernel<<<blocks, PT_THREADS, (size_t)a->N * sizeof(float3), stream>>>(P, num_rays, rays, packets, counter);
    }
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // extern "C"
