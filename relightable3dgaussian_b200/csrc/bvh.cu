// Stage 3b of the hot path: LBVH over the Gaussians' 3-sigma boxes and the opacity ray trace that
// bakes per-Gaussian visibility (reference bvh/: __init__.py:29-71, src/construct.cu:147-266,
// src/trace.cu:196-287, include/utility.cuh:35-111; kernels K17-K22 of SURVEY.md §2.3).
//
// Design notes
//  * build: no thrust temporaries or host round trips — scene bounds by ordered-int atomics, Morton
//    keys sorted with the library's own one-sweep radix sort (stable => the reference's
//    (morton, index) order), Karras internal nodes, bottom-up refit with fenced flags.  Every
//    result is integer or min/max arithmetic, so nodes / aabbs / morton are bit-identical to the
//    reference's.
//  * trace: the reference reads a 20 B node, then two 24 B child boxes from another array, then
//    four per-Gaussian arrays at a leaf, from a per-thread local-memory stack.  Here the tree is
//    re-packed once per trace call into 64 B internal packets {children, both child boxes} and
//    64 B leaf records {mean, inverse covariance, opacity, normal} stored in Morton order, so one
//    aligned 4x16 B fetch serves a whole traversal step; the top 20 stack levels live in shared memory
//    (deeper ones spill to a local array: 10 KB instead of 32 KB per CTA); warps are
//    persistent and refill finished lanes from a global ray counter (ray-stack compaction), so the
//    early exit at T < 0.9 does not idle lanes.  Per ray the visiting order (far child pushed
//    first) is the reference's, hence the product order of (1 - alpha) too.
#include <cstdio>
#include "bvh.cuh"
#include "kernels.h"

namespace r3dg {

// ---- leaf boxes: bvh/__init__.py:31-57 + build_rotation (utils/general_utils.py:82-103), restated
// with torch's op-by-op fp32 rounding (explicit intrinsics: no contraction) ----------------------
__global__ void __launch_bounds__(256) bvh_leaf_aabb_kernel(int P, const float* __restrict__ means3D,
                                                            const float* __restrict__ scales,
                                                            const float* __restrict__ rotations,
                                                            int32_t* __restrict__ nodes, float* __restrict__ aabbs) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int NI = P - 1;
    if (i < NI) {      // internal node init (bvh/__init__.py:32-37)
        int32_t* n = nodes + (size_t)i * 5;
        n[0] = -1; n[1] = -1; n[2] = -1; n[3] = -1; n[4] = 0;
        float* b = aabbs + (size_t)i * 6;
        b[0] = 100000.f; b[1] = 100000.f; b[2] = 100000.f; b[3] = -100000.f; b[4] = -100000.f; b[5] = -100000.f;
    }
    if (i >= P) return;
    {
        int32_t* n = nodes + (size_t)(NI + i) * 5;
        n[0] = -1; n[1] = -1; n[2] = -1; n[3] = -1; n[4] = 1;
    }
    const float4 rq = *reinterpret_cast<const float4*>(rotations + 4 * (size_t)i);
    const float norm = sqrt_(add_(add_(add_(mul_(rq.x, rq.x), mul_(rq.y, rq.y)), mul_(rq.z, rq.z)), mul_(rq.w, rq.w)));
    const float r = div_(rq.x, norm), x = div_(rq.y, norm), y = div_(rq.z, norm), z = div_(rq.w, norm);
    float R[3][3];
    R[0][0] = sub_(1.f, mul_(2.f, add_(mul_(y, y), mul_(z, z)))); R[0][1] = mul_(2.f, sub_(mul_(x, y), mul_(r, z))); R[0][2] = mul_(2.f, add_(mul_(x, z), mul_(r, y)));
    R[1][0] = mul_(2.f, add_(mul_(x, y), mul_(r, z))); R[1][1] = sub_(1.f, mul_(2.f, add_(mul_(x, x), mul_(z, z)))); R[1][2] = mul_(2.f, sub_(mul_(y, z), mul_(r, x)));
    R[2][0] = mul_(2.f, sub_(mul_(x, z), mul_(r, y))); R[2][1] = mul_(2.f, add_(mul_(y, z), mul_(r, x))); R[2][2] = sub_(1.f, mul_(2.f, add_(mul_(x, x), mul_(y, y))));
    const float sa = mul_(3.f, scales[3 * (size_t)i]), sb = mul_(3.f, scales[3 * (size_t)i + 1]), sc = mul_(3.f, scales[3 * (size_t)i + 2]);
    float* out = aabbs + (size_t)(NI + i) * 6;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float m = means3D[3 * (size_t)i + k];
        const float ta = mul_(R[k][0], sa), tb = mul_(R[k][1], sb), tc = mul_(R[k][2], sc);
        const float pa = add_(m, ta), ma = sub_(m, ta);
        const float c8[8] = {add_(add_(pa, tb), tc), sub_(add_(pa, tb), tc), add_(sub_(pa, tb), tc), sub_(sub_(pa, tb), tc),
                             add_(add_(ma, tb), tc), sub_(add_(ma, tb), tc), add_(sub_(ma, tb), tc), sub_(sub_(ma, tb), tc)};
        float lo = c8[0], hi = c8[0];
#pragma unroll
        for (int j = 1; j < 8; ++j) { lo = fminf(lo, c8[j]); hi = fmaxf(hi, c8[j]); }
        out[k] = lo; out[3 + k] = hi;
    }
}

// ---- build -----------------------------------------------------------------------------------
struct BvhTmp {                 // layout of the caller-provided build workspace
    size_t header, bounds, leafcopy, flags, bin, total;
    SortLayout bl;
    __host__ BvhTmp(int P) : bl(P < 1 ? 1 : P) {
        size_t off = 0;
        header = off;   off = align_up(off + sizeof(GeomHeader), 256);
        bounds = off;   off = align_up(off + 6 * 4, 256);
        leafcopy = off; off = align_up(off + (size_t)P * 24, 256);
        flags = off;    off = align_up(off + (size_t)P * 4, 256);
        bin = off;      off = align_up(off + bl.total, 256);
        total = off;
    }
};

__device__ __forceinline__ int f2ord(float f) { const int b = __float_as_int(f); return b >= 0 ? b : b ^ 0x7fffffff; }
__device__ __forceinline__ float ord2f(int o) { return __int_as_float(o >= 0 ? o : o ^ 0x7fffffff); }

__global__ void bvh_init_kernel(GeomHeader* h, int* bounds, int P) {
    if (threadIdx.x == 0) {
        h->num_rendered = (uint32_t)P; h->depth_or = 0x3fffffffu; h->depth_nor = 0x3fffffffu;   // sort all 30 Morton bits
        for (int k = 0; k < 3; ++k) { bounds[k] = f2ord(100000.f); bounds[3 + k] = f2ord(-100000.f); }   // construct.cu:159-162
    }
}

__global__ void __launch_bounds__(256) bvh_bounds_kernel(int P, const float* __restrict__ leaf, int* bounds, float* __restrict__ leafcopy) {
    float lo[3] = {3.0e38f, 3.0e38f, 3.0e38f}, hi[3] = {-3.0e38f, -3.0e38f, -3.0e38f};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float a = leaf[6 * (size_t)i + k], b = leaf[6 * (size_t)i + 3 + k];
            leafcopy[6 * (size_t)i + k] = a; leafcopy[6 * (size_t)i + 3 + k] = b;
            lo[k] = fminf(lo[k], a); hi[k] = fmaxf(hi[k], b);
        }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[k] = fminf(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], o));
            hi[k] = fmaxf(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], o));
        }
        if ((threadIdx.x & 31) == 0) { atomicMin(&bounds[k], f2ord(lo[k])); atomicMax(&bounds[3 + k], f2ord(hi[k])); }
    }
}

__device__ __forceinline__ uint32_t expand_bits(uint32_t v) {
    v = (v * 0x00010001u) & 0xFF0000FFu;
    v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u;
    v = (v * 0x00000005u) & 0x49249249u;
    return v;
}

// construct.cu:23-51: 30-bit Morton code of the leaf-box centroid normalised to the scene box
__global__ void __launch_bounds__(256) bvh_morton_kernel(int P, const float* __restrict__ leaf, const int* __restrict__ bounds,
                                                         uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    uint32_t code[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float wl = ord2f(bounds[k]), wu = ord2f(bounds[3 + k]);
        float c = (float)((double)add_(leaf[6 * (size_t)i + 3 + k], leaf[6 * (size_t)i + k]) * 0.5);
        c = sub_(c, wl);
        c = div_(c, sub_(wu, wl));
        c = fminf(fmaxf(mul_(c, 1024.0f), 0.0f), 1023.0f);
        code[k] = expand_bits((uint32_t)c);
    }
    keys[i] = code[0] * 4 + code[1] * 2 + code[2];
    vals[i] = (uint32_t)i;
}

__global__ void __launch_bounds__(256) bvh_leaves_kernel(int P, const GeomHeader* __restrict__ h,
                                                         const uint32_t* __restrict__ ka, const uint32_t* __restrict__ kb,
                                                         const uint32_t* __restrict__ va, const uint32_t* __restrict__ vb,
                                                         const float* __restrict__ leafcopy, int32_t* __restrict__ nodes,
                                                         float* __restrict__ aabbs, uint64_t* __restrict__ morton) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const bool in_b = (h->sort_exec & 1u) != 0;
    const uint64_t m = in_b ? kb[i] : ka[i];   // 30-bit code, widened
    const uint32_t idx = in_b ? vb[i] : va[i];
    morton[i] = (m << 31) | idx;                                    // construct.cu:184-192 (31, not 32)
    nodes[(size_t)(P - 1 + i) * 5 + 3] = (int32_t)idx;               // construct.cu:196-201
    float* dst = aabbs + (size_t)(P - 1 + i) * 6;
    const float* src = leafcopy + (size_t)idx * 6;
#pragma unroll
    for (int k = 0; k < 6; ++k) dst[k] = src[k];                    // leaves reordered like stable_sort_by_key's zip
}

__device__ __forceinline__ int common_upper_bits(uint64_t a, uint64_t b) { return __clzll((long long)(a ^ b)); }

// construct.cu:53-145,203-227
__global__ void __launch_bounds__(256) bvh_internal_kernel(int P, const uint64_t* __restrict__ code, int32_t* nodes) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P - 1) return;
    const int n = P;
    int lo, hi;
    if (idx == 0) { lo = 0; hi = n - 1; }
    else {
        const uint64_t self = code[idx];
        const int Ld = common_upper_bits(self, code[idx - 1]), Rd = common_upper_bits(self, code[idx + 1]);
        const int d = (Rd > Ld) ? 1 : -1;
        const int dmin = min(Ld, Rd);
        int l_max = 2, delta = -1;
        long long it = (long long)idx + d * l_max;
        if (0 <= it && it < n) delta = common_upper_bits(self, code[it]);
        while (delta > dmin) {
            l_max <<= 1;
            it = (long long)idx + (long long)d * l_max;
            delta = -1;
            if (0 <= it && it < n) delta = common_upper_bits(self, code[it]);
        }
        int l = 0, t = l_max >> 1;
        while (t > 0) {
            it = (long long)idx + (long long)(l + t) * d;
            delta = -1;
            if (0 <= it && it < n) delta = common_upper_bits(self, code[it]);
            if (delta > dmin) l += t;
            t >>= 1;
        }
        const int j = idx + l * d;
        lo = min(idx, j); hi = max(idx, j);
    }
    int gamma;
    {
        const uint64_t fc = code[lo], lc = code[hi];
        if (fc == lc) gamma = (lo + hi) >> 1;
        else {
            const int dn = common_upper_bits(fc, lc);
            int split = lo, stride = hi - lo;
            do {
                stride = (stride + 1) >> 1;
                const int middle = split + stride;
                if (middle < hi && common_upper_bits(fc, code[middle]) > dn) split = middle;
            } while (stride > 1);
            gamma = split;
        }
    }
    int32_t* node = nodes + (size_t)idx * 5;
    int l = gamma, r = gamma + 1;
    if (lo == gamma) l += P - 1;
    if (hi == gamma + 1) r += P - 1;
    node[1] = l; node[2] = r; node[3] = -1;
    nodes[(size_t)l * 5] = idx;
    nodes[(size_t)r * 5] = idx;
}

// construct.cu:229-265 with the missing fences added
__global__ void __launch_bounds__(256) bvh_refit_kernel(int P, int32_t* nodes, float* aabbs, int* flags) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    int32_t num = 1;
    int32_t parent = nodes[(size_t)(P - 1 + i) * 5];
    while (parent != -1) {
        atomicAdd(nodes + (size_t)parent * 5 + 4, num);
        __threadfence();
        const int old = atomicCAS(flags + parent, 0, 1);
        if (old == 0) return;
        __threadfence();
        int32_t* pn = nodes + (size_t)parent * 5;
        const float* lb = aabbs + (size_t)pn[1] * 6;
        const float* rb = aabbs + (size_t)pn[2] * 6;
        float* pb = aabbs + (size_t)parent * 6;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            pb[k] = fminf(__ldcg(lb + k), __ldcg(rb + k));
            pb[3 + k] = fmaxf(__ldcg(lb + 3 + k), __ldcg(rb + 3 + k));
        }
        num = atomicAdd(nodes + (size_t)parent * 5 + 4, 0);
        parent = pn[0];
    }
}

// ---- trace ------------------------------------------------------------------------------------
// packets: the layout of bvh.cuh (LeafRecord)
__global__ void __launch_bounds__(256) bvh_pack_kernel(int P, const int32_t* __restrict__ nodes, const float* __restrict__ aabbs,
                                                       const float* __restrict__ means3D, const float* __restrict__ covs3D,
                                                       const float* __restrict__ opacities, const float* __restrict__ normals,
                                                       float4* __restrict__ packets) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int NI = P - 1;
    if (i < NI) {
        const int32_t* n = nodes + (size_t)i * 5;
        const int l = n[1], r = n[2];
        const float* lb = aabbs + (size_t)l * 6;
        const float* rb = aabbs + (size_t)r * 6;
        const int le = l >= NI ? -(l - NI + 1) : l, re = r >= NI ? -(r - NI + 1) : r;
        float4* p = packets + (size_t)i * 4;
        p[0] = make_float4(__int_as_float(le), __int_as_float(re), lb[0], lb[1]);
        p[1] = make_float4(lb[2], lb[3], lb[4], lb[5]);
        p[2] = make_float4(rb[0], rb[1], rb[2], rb[3]);
        p[3] = make_float4(rb[4], rb[5], 0.f, 0.f);
    }
    if (i < P) {
        const int g = nodes[(size_t)(NI + i) * 5 + 3];
        const float* mu = means3D + 3 * (size_t)g; const float* ci = covs3D + 6 * (size_t)g; const float* nr = normals + 3 * (size_t)g;
        float4* p = packets + (size_t)(NI + i) * 4;
        p[0] = make_float4(mu[0], mu[1], mu[2], ci[0]);
        p[1] = make_float4(ci[1], ci[2], ci[3], ci[4]);
        p[2] = make_float4(ci[5], opacities[g], nr[0], nr[1]);
        p[3] = make_float4(nr[2], 0.f, 0.f, 0.f);
    }
}

// phase != nullptr: random_rotate=True — theta_i += phase[g] * 2 * pi with phase = torch.rand(P) drawn by the caller
__global__ void __launch_bounds__(256) sample_dirs_kernel(int P, int N, const float* __restrict__ normals,
                                                          const float* __restrict__ phase,
                                                          float* __restrict__ dirs, float* __restrict__ areas) {
    extern __shared__ float3 sSample[];
    for (int i = threadIdx.x; i < N; i += blockDim.x) sSample[i] = fib_sample(i, N);
    __syncthreads();
    const long long total = (long long)P * N;
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < total; r += (long long)gridDim.x * blockDim.x) {
        const long long g = r / N;
        const int i = (int)(r - g * N);
        float3 smp = sSample[i];
        if (phase) {          // theta = rand * 2 * pi + delta * idx  (graphics_utils.py:24-25)
            const float rad = sqrt_(sub_(1.0f, mul_(smp.z, smp.z)));
            const float theta = add_(mul_(mul_(phase[g], 2.0f), 3.141592653589793f), mul_(2.399963229728653f, (float)i));
            smp.x = mul_(sinf(theta), rad); smp.y = mul_(cosf(theta), rad);
        }
        const float3 d = rotate_from_z(normals[3 * g], normals[3 * g + 1], normals[3 * g + 2], smp);
        dirs[3 * r] = d.x; dirs[3 * r + 1] = d.y; dirs[3 * r + 2] = d.z;
        if (areas) areas[r] = 6.283185307179586f;                 // ones * 2 * pi
    }
}

#define TRACE_THREADS 128
// BAKE = false: explicit rays (rays_o [num_rays / o_group, 3], rays_d [num_rays, 3]) — trace_bvh_opacity.
// BAKE = true : the visibility bake: ray r = (leaf slot first_slot + r / N, sample r % N); the Gaussian is the
//   slot's object (Morton order => neighbouring warps walk neighbouring subtrees), the origin its mean, the
//   direction is generated HERE from its normal (never read from HBM) and written once to `dirs_out` together
//   with the constant area; results land at the Gaussian's own row g * N + i.
template <bool BAKE>
__global__ void __launch_bounds__(TRACE_THREADS) bvh_trace_kernel(int P, long long num_rays, const float4* __restrict__ packets,
                                                                  const float* __restrict__ rays_o, int o_group, float o_offset,
                                                                  const float* __restrict__ rays_d, int32_t* __restrict__ num_contributes,
                                                                  float* __restrict__ rendered_opacity, unsigned long long* counter,
                                                                  int N, int first_slot, const int32_t* __restrict__ nodes,
                                                                  float* __restrict__ dirs_out, float* __restrict__ areas_out) {
    __shared__ int sStack[TRACE_STACK_SH][TRACE_THREADS];
    extern __shared__ float3 sSample[];
    int lStack[TRACE_STACK - TRACE_STACK_SH];
    const int tid = threadIdx.x, lane = tid & 31;
    const int NI = P - 1;
    if (BAKE) {
        for (int i = tid; i < N; i += TRACE_THREADS) sSample[i] = fib_sample(i, N);
        __syncthreads();
    }
    auto push = [&](int& sp, int v) {
        if (sp < TRACE_STACK_SH) sStack[sp][tid] = v;
        else if (sp < TRACE_STACK) lStack[sp - TRACE_STACK_SH] = v;
        else { printf("WARNING TOO BIG\n"); return; }           // the reference's own message (bvh/include/trace.cuh:24-29; it then writes
                                                           // past its array) — here the push is dropped, nothing out of bounds
        ++sp;
    };
    auto pop = [&](int& sp) {
        --sp;
        return sp < TRACE_STACK_SH ? sStack[sp][tid] : lStack[sp - TRACE_STACK_SH];
    };
    bool has_ray = false, exhausted = false;
    long long ray = 0, out = 0;
    int sp = 0, count = 0;
    float ox = 0, oy = 0, oz = 0, dx = 0, dy = 0, dz = 0, ix = 0, iy = 0, iz = 0, T = 1.0f;
    while (true) {
        // ---- refill idle lanes from the global ray counter (warp-aggregated) -------------------
        const unsigned want = __ballot_sync(0xffffffffu, !has_ray && !exhausted);
        if (want) {
            const int leader = __ffs(want) - 1;
            unsigned long long base = 0;
            if (lane == leader) base = atomicAdd(counter, (unsigned long long)__popc(want));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (!has_ray && !exhausted) {
                ray = (long long)base + __popc(want & ((1u << lane) - 1u));
                if (ray < num_rays) {
                    if (BAKE) {
                        const long long slot = ray / N;
                        const int i = (int)(ray - slot * N);
                        const float4* q = packets + (size_t)(NI + first_slot + slot) * 4;     // the slot's own leaf record
                        const float4 q0 = q[0], q2 = q[2], q3 = q[3];
                        const long long g = nodes[(size_t)(NI + first_slot + slot) * 5 + 3];
                        const float3 d = rotate_from_z(q2.z, q2.w, q3.x, sSample[i]);
                        dx = d.x; dy = d.y; dz = d.z;
                        ox = q0.x; oy = q0.y; oz = q0.z;
                        out = g * N + i;
                        if (dirs_out) { dirs_out[3 * out] = dx; dirs_out[3 * out + 1] = dy; dirs_out[3 * out + 2] = dz; }
                        if (areas_out) areas_out[out] = 6.283185307179586f;
                    } else {
                        dx = rays_d[3 * ray]; dy = rays_d[3 * ray + 1]; dz = rays_d[3 * ray + 2];
                        const long long oi = ray / o_group;
                        ox = rays_o[3 * oi]; oy = rays_o[3 * oi + 1]; oz = rays_o[3 * oi + 2];
                        out = ray;
                    }
                    if (o_offset != 0.0f) {                    // rays_o + rays_d * 0.05 (bvh/__init__.py:63), torch op order
                        ox = add_(ox, mul_(dx, o_offset)); oy = add_(oy, mul_(dy, o_offset)); oz = add_(oz, mul_(dz, o_offset));
                    }
                    ix = div_(1.0f, dx); iy = div_(1.0f, dy); iz = div_(1.0f, dz);
                    has_ray = true; T = 1.0f; count = 0;
                    sp = 0; push(sp, NI == 0 ? -1 : 0);        // root (a lone leaf when P == 1)
                } else {
                    exhausted = true;
                }
            }
        }
        if (!__any_sync(0xffffffffu, has_ray)) break;
        // ---- a bounded burst of traversal steps, then look for idle lanes again.  The burst ends early as soon as a
        // quarter of the warp has finished its ray (checked every 4 steps: rays that hit T < 0.9 quickly would otherwise
        // idle their lanes for the rest of the burst — ncu: 12.5 of 32 lanes active with 93 % blocked rays) ----------
#pragma unroll 1
        for (int step = 0; step < 32; ++step) {
            if (step > 0 && (step & 3) == 0 && __popc(__ballot_sync(0xffffffffu, !has_ray && !exhausted)) >= 8) break;   // 8+ lanes can be refilled
            if (!has_ray) continue;
            const int node = pop(sp);
            if (node >= 0) {
                const float4* p = packets + (size_t)node * 4;
                const float4 p0 = p[0], p1 = p[1], p2 = p[2], p3 = p[3];
                const int l = __float_as_int(p0.x), r = __float_as_int(p0.y);
                const float lmax = ray_box_tmax(p0.z, p0.w, p1.x, p1.y, p1.z, p1.w, ox, oy, oz, ix, iy, iz);
                const float rmax = ray_box_tmax(p2.x, p2.y, p2.z, p2.w, p3.x, p3.y, ox, oy, oz, ix, iy, iz);
                if (lmax > rmax) {                                    // trace.cu:258-272: far child first
                    if (lmax > 0) push(sp, l);
                    if (rmax > 0) push(sp, r);
                } else {
                    if (rmax > 0) push(sp, r);
                    if (lmax > 0) push(sp, l);
                }
            } else {
                const float4* p = packets + (size_t)(NI - node - 1) * 4;    // leaf slot = -node - 1
                const float4 q0 = p[0], q1 = p[1], q2 = p[2], q3 = p[3];
                const float mx = q0.x, my = q0.y, mz = q0.z, c0 = q0.w, c1 = q1.x, c2 = q1.y, c3 = q1.z, c4 = q1.w, c5 = q2.x;
                const float op = q2.y, nx = q2.z, ny = q2.w, nz = q3.x;
                bool live = !(op < 1.f / 255.f) && !(nx * dx + ny * dy + nz * dz > 0);
                if (live) {
                    const float m0 = mx - ox, m1 = my - oy, m2 = mz - oz;
                    const float t1 = c0 * m0 * dx + c1 * m0 * dy + c2 * m0 * dz + c1 * m1 * dx + c3 * m1 * dy + c4 * m1 * dz +
                                     c2 * m2 * dx + c4 * m2 * dy + c5 * m2 * dz;
                    const float t2 = c0 * dx * dx + c1 * dx * dy + c2 * dx * dz + c1 * dy * dx + c3 * dy * dy + c4 * dy * dz +
                                     c2 * dz * dx + c4 * dz * dy + c5 * dz * dz;
                    const float t = t1 / t2;
                    if (!(t < 0.01f)) {
                        const float e0 = mx - (ox + t * dx), e1 = my - (oy + t * dy), e2 = mz - (oz + t * dz);
                        const float power = -0.5f * (e0 * e0 * c0 + e1 * e1 * c3 + e2 * e2 * c5 + 2 * e0 * e1 * c1 + 2 * e0 * e2 * c2 + 2 * e1 * e2 * c4);
                        if (!(power > 0)) {
                            count += 1;
                            const float alpha = op * __expf(power);
                            T *= 1 - alpha;
                            if (T < 0.9f) {                          // trace.cu:251-254
                                rendered_opacity[out] = 0.0f;
                                if (num_contributes) num_contributes[out] = 0;
                                has_ray = false;
                            }
                        }
                    }
                }
            }
            if (has_ray && sp == 0) {
                if (num_contributes) num_contributes[out] = count;
                rendered_opacity[out] = T;
                has_ray = false;
            }
        }
    }
}

// ---- host launchers -----------------------------------------------------------------------
size_t bvh_build_tmp_bytes(int P) { return BvhTmp(P).total; }
size_t bvh_packets_bytes(int P) { return (size_t)(2 * (size_t)(P < 1 ? 1 : P)) * 64 + 256; }

int launch_bvh_leaf_aabbs(int P, const float* means3D, const float* scales, const float* rotations,
                          int32_t* nodes, float* aabbs, cudaStream_t stream) {
    if (P <= 0) return 0;
    bvh_leaf_aabb_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, means3D, scales, rotations, nodes, aabbs);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_bvh_build(int P, int32_t* nodes, float* aabbs, uint64_t* morton, void* tmp_, size_t tmp_bytes,
                     int num_sms, cudaStream_t stream) {
    if (P <= 0) return 0;
    const BvhTmp t(P);
    if (tmp_bytes < t.total) return R3DG_ERR_BAD_ARG;
    char* tmp = (char*)tmp_;
    GeomHeader* h = (GeomHeader*)(tmp + t.header);
    int* bounds = (int*)(tmp + t.bounds);
    float* leafcopy = (float*)(tmp + t.leafcopy);
    int* flags = (int*)(tmp + t.flags);
    char* bin = tmp + t.bin;
    float* leaf = aabbs + (size_t)(P - 1) * 6;
    R3DG_CUDA_TRY(cudaMemsetAsync(h, 0, sizeof(GeomHeader), stream));
    R3DG_CUDA_TRY(cudaMemsetAsync(flags, 0, (size_t)P * 4, stream));
    bvh_init_kernel<<<1, 32, 0, stream>>>(h, bounds, P);
    bvh_bounds_kernel<<<num_sms * 4, 256, 0, stream>>>(P, leaf, bounds, leafcopy);
    bvh_morton_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, leafcopy, bounds, (uint32_t*)(bin + t.bl.keys_a), (uint32_t*)(bin + t.bl.vals_a));
    int rc = launch_sort(h, bin, t.bl, P, num_sms, stream);          // 30-bit keys: 4 passes of 8 bits
    if (rc != 0) return rc;
    bvh_leaves_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, h, (const uint32_t*)(bin + t.bl.keys_a), (const uint32_t*)(bin + t.bl.keys_b),
                                                           (const uint32_t*)(bin + t.bl.vals_a), (const uint32_t*)(bin + t.bl.vals_b),
                                                           leafcopy, nodes, aabbs, morton);
    if (P > 1) bvh_internal_kernel<<<(P - 1 + 255) / 256, 256, 0, stream>>>(P, morton, nodes);
    bvh_refit_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, nodes, aabbs, flags);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

static int trace_blocks(long long num_rays, int num_sms) {
    const long long want = (num_rays + TRACE_THREADS - 1) / TRACE_THREADS;
    return (int)(want < (long long)num_sms * 16 ? want : (long long)num_sms * 16);
}

int launch_bvh_trace(int P, long long num_rays, const int32_t* nodes, const float* aabbs, const float* rays_o,
                     int o_group, float o_offset, const float* rays_d, const float* means3D, const float* covs3D,
                     const float* opacities, const float* normals, int32_t* num_contributes, float* rendered_opacity,
                     void* packets_, size_t packets_bytes, int num_sms, cudaStream_t stream) {
    if (P <= 0 || num_rays <= 0) return 0;
    if (packets_bytes < bvh_packets_bytes(P) || o_group < 1) return R3DG_ERR_BAD_ARG;
    unsigned long long* counter = (unsigned long long*)packets_;
    float4* packets = (float4*)((char*)packets_ + 256);
    R3DG_CUDA_TRY(cudaMemsetAsync(counter, 0, 8, stream));
    bvh_pack_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, nodes, aabbs, means3D, covs3D, opacities, normals, packets);
    bvh_trace_kernel<false><<<trace_blocks(num_rays, num_sms), TRACE_THREADS, 0, stream>>>(
        P, num_rays, packets, rays_o, o_group, o_offset, rays_d, num_contributes, rendered_opacity, counter, 1, 0, nodes, nullptr, nullptr);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_bvh_pack(int P, const int32_t* nodes, const float* aabbs, const float* means3D, const float* covs3D,
                    const float* opacities, const float* normals, float4* packets, cudaStream_t stream) {
    bvh_pack_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, nodes, aabbs, means3D, covs3D, opacities, normals, packets);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_sample_dirs(int P, int N, const float* normals, const float* phase, float* dirs, float* areas, int num_sms, cudaStream_t stream) {
    if (P <= 0 || N <= 0) return 0;
    if ((size_t)N * sizeof(float3) > 48 * 1024) return R3DG_ERR_UNSUPPORTED;          // N <= 4096
    const long long total = (long long)P * N;
    const long long want = (total + 255) / 256;
    const int blocks = (int)(want < (long long)num_sms * 16 ? want : (long long)num_sms * 16);
    sample_dirs_kernel<<<blocks, 256, (size_t)N * sizeof(float3), stream>>>(P, N, normals, phase, dirs, areas);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_bvh_bake(int P, int first_slot, int count, int N, const int32_t* nodes, const float* aabbs, const float* means3D,
                    const float* covs3D, const float* opacities, const float* normals, float o_offset,
                    int32_t* num_contributes, float* visibility, float* dirs, float* areas, void* packets_,
                    size_t packets_bytes, int num_sms, cudaStream_t stream) {
    if (P <= 0 || count <= 0 || N <= 0) return 0;
    if (packets_bytes < bvh_packets_bytes(P) || first_slot < 0 || first_slot + count > P) return R3DG_ERR_BAD_ARG;
    if ((size_t)N * sizeof(float3) > BAKE_SAMPLE_SMEM) return R3DG_ERR_UNSUPPORTED;
    unsigned long long* counter = (unsigned long long*)packets_;
    float4* packets = (float4*)((char*)packets_ + 256);
    R3DG_CUDA_TRY(cudaMemsetAsync(counter, 0, 8, stream));
    bvh_pack_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, nodes, aabbs, means3D, covs3D, opacities, normals, packets);
    const long long num_rays = (long long)count * N;
    bvh_trace_kernel<true><<<trace_blocks(num_rays, num_sms), TRACE_THREADS, (size_t)N * sizeof(float3), stream>>>(
        P, num_rays, packets, nullptr, 1, o_offset, nullptr, num_contributes, visibility, counter, N, first_slot, nodes, dirs, areas);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace r3dg
