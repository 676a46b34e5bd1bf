// Shadow transmittance of point and directional lights through the LBVH (include/r3dg_b200.h, LIGHTS; DESIGN.md
// §4.26).  One ray per (Gaussian, light): the visibility bake's packed tree, persistent warps refilled from a global
// ray counter, traversal order (far child pushed first), slab test and hit rule, compiled with the bake's flags so
// that a directional light's T is the bake's product bit for bit wherever the bake keeps it (T >= 0.9).  Differences
// from the bake: a subtree is skipped when the ray's segment [0, t_max] misses its box (exact, because a hit must also
// meet its own leaf box within the segment), hits need peak t < (1 - 1e-5) t_max, and the ray stops at T < 1e-4 instead of 0.9.
// Spot and rect lights (SHAPED LIGHTS; DESIGN.md §4.28) trace the same point-light rays towards a spot's position or
// a rect's hashed stratified samples, in bvh_shaped_lights_kernel.  The per-pixel lights (PIXEL LIGHTS; DESIGN.md
// §4.30) trace the same rays from every valid pixel's surface point, in bvh_pixel_lights_kernel.
#include <cmath>
#include "bvh.cuh"
#include "kernels.h"
#include "lights.cuh"

namespace r3dg {

#define LT_THREADS 128
#define LIGHT_T_MIN 1e-4f           // a shadow ray stops once its transmittance falls below this
// A hit's peak t must lie below (1 - 1e-5) t_max: a Gaussian whose peak is at the light (the light at its centre) is
// then clearly not a hit, instead of a tie that fp32 rounding decides
#define LIGHT_T_MAX_MARGIN (1.0f - 1e-5f)
#define PL_TILE 8                   // pixels are numbered in PL_TILE x PL_TILE tiles, as pixel_trace.cu's PT_TILE

// The shaped lights' persistent trace loop: bvh_lights_kernel's loop (kept as written there, so that its SASS is
// unchanged) with the ray setup as a parameter.  `setup(ray, ...)` starts ray `ray` of the launch: its
// direction d, origin o, segment tseg, hit bound thit and output index out (S: a ray source, inlined).  A source
// with S::kDeclines may return false for a ray it does not trace (a masked pixel's, whose T it writes, or one outside
// the image); such rays hold no lane: the refill repeats until every lane has a ray or the rays are exhausted.
template <class S>
__device__ __forceinline__ void trace_shadow_rays(const S& setup, long long num_rays, int NI, const float4* __restrict__ packets,
                                                  float* __restrict__ shadows, unsigned long long* counter,
                                                  int (*sStack)[LT_THREADS]) {
    const int tid = threadIdx.x, lane = tid & 31;
    SplitStack<LT_THREADS> st;
    st.sh = sStack; st.tid = tid; st.sp = 0;
    bool has_ray = false, exhausted = false;
    long long out = 0;
    float ox = 0, oy = 0, oz = 0, dx = 0, dy = 0, dz = 0, ix = 0, iy = 0, iz = 0, tseg = 0, thit = 0, T = 1.0f;
    while (true) {
        // ---- refill idle lanes from the global ray counter (warp-aggregated), as the bake does ----
        while (true) {
            const unsigned want = __ballot_sync(0xffffffffu, !has_ray && !exhausted);
            if (want) {
                const int leader = __ffs(want) - 1;
                unsigned long long base = 0;
                if (lane == leader) base = atomicAdd(counter, (unsigned long long)__popc(want));
                base = __shfl_sync(0xffffffffu, base, leader);
                if (!has_ray && !exhausted) {
                    const long long ray = (long long)base + __popc(want & ((1u << lane) - 1u));
                    if (ray < num_rays) {
                        if (setup(ray, ox, oy, oz, dx, dy, dz, tseg, thit, out)) {
                            ix = div_(1.0f, dx); iy = div_(1.0f, dy); iz = div_(1.0f, dz);
                            has_ray = true; T = 1.0f;
                            st.sp = 0; st.push(NI == 0 ? -1 : 0);         // root (a lone leaf when P == 1)
                        }
                    } else {
                        exhausted = true;
                    }
                }
            }
            if (!S::kDeclines || !want) break;
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
                const float lmax = ray_box_tmax<true>(p0.z, p0.w, p1.x, p1.y, p1.z, p1.w, ox, oy, oz, ix, iy, iz, tseg);
                const float rmax = ray_box_tmax<true>(p2.x, p2.y, p2.z, p2.w, p3.x, p3.y, ox, oy, oz, ix, iy, iz, tseg);
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
                if (gaussian_hit(q, ox, oy, oz, dx, dy, dz, t, power) && t < thit) {
                    const float alpha = q.op * __expf(power);
                    T *= 1 - alpha;
                    if (T < LIGHT_T_MIN) {
                        shadows[out] = T;
                        has_ray = false;
                    }
                }
            }
            if (has_ray && st.sp == 0) {
                shadows[out] = T;
                has_ray = false;
            }
        }
    }
}

// A ray towards the point `target` from the Gaussian (mx, my, mz): l as light_dir's, o = m + 0.05 l, the segment
// |target - o| and its hit bound, all rounded op by op
__device__ __forceinline__ void ray_to_point(const float* target, float mx, float my, float mz, float& ox, float& oy,
                                             float& oz, float& dx, float& dy, float& dz, float& tseg, float& thit) {
    const LightDir ld = light_dir(1, target, mx, my, mz);
    dx = ld.l[0]; dy = ld.l[1]; dz = ld.l[2];
    ox = add_(mx, mul_(dx, LIGHT_ORIGIN_OFFSET));
    oy = add_(my, mul_(dy, LIGHT_ORIGIN_OFFSET));
    oz = add_(mz, mul_(dz, LIGHT_ORIGIN_OFFSET));
    const float e0 = sub_(target[0], ox), e1 = sub_(target[1], oy), e2 = sub_(target[2], oz);
    tseg = sqrt_(add_(add_(mul_(e0, e0), mul_(e1, e1)), mul_(e2, e2)));
    thit = mul_(tseg, LIGHT_T_MAX_MARGIN);
}

// Ray r = (leaf slot r / K, light r % K): neighbouring lanes start from neighbouring Gaussians (Morton order).
__global__ void __launch_bounds__(LT_THREADS) bvh_lights_kernel(int P, int K, const uint32_t point_mask, const float* __restrict__ vec,
                                                                const float4* __restrict__ packets,
                                                                const int32_t* __restrict__ nodes, float* __restrict__ shadows,
                                                                unsigned long long* counter) {
    __shared__ int sStack[TRACE_STACK_SH][LT_THREADS];
    __shared__ float sVec[3 * R3DG_MAX_LIGHTS];
    const int tid = threadIdx.x, lane = tid & 31;
    for (int i = tid; i < 3 * K; i += LT_THREADS) sVec[i] = vec[i];
    __syncthreads();
    const int NI = P - 1;
    const long long num_rays = (long long)P * K;
    SplitStack<LT_THREADS> st;
    st.sh = sStack; st.tid = tid; st.sp = 0;
    bool has_ray = false, exhausted = false;
    long long out = 0;
    float ox = 0, oy = 0, oz = 0, dx = 0, dy = 0, dz = 0, ix = 0, iy = 0, iz = 0, tseg = 0, thit = 0, T = 1.0f;
    while (true) {
        // ---- refill idle lanes from the global ray counter (warp-aggregated), as the bake does ----
        const unsigned want = __ballot_sync(0xffffffffu, !has_ray && !exhausted);
        if (want) {
            const int leader = __ffs(want) - 1;
            unsigned long long base = 0;
            if (lane == leader) base = atomicAdd(counter, (unsigned long long)__popc(want));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (!has_ray && !exhausted) {
                const long long ray = (long long)base + __popc(want & ((1u << lane) - 1u));
                if (ray < num_rays) {
                    const long long slot = ray / K;
                    const int j = (int)(ray - slot * K);
                    const LeafRecord self = load_leaf(packets + (size_t)(NI + slot) * 4);
                    const int kind = (point_mask >> j) & 1;
                    const LightDir ld = light_dir(kind, sVec + 3 * j, self.mx, self.my, self.mz);
                    dx = ld.l[0]; dy = ld.l[1]; dz = ld.l[2];
                    ox = add_(self.mx, mul_(dx, LIGHT_ORIGIN_OFFSET));
                    oy = add_(self.my, mul_(dy, LIGHT_ORIGIN_OFFSET));
                    oz = add_(self.mz, mul_(dz, LIGHT_ORIGIN_OFFSET));
                    if (kind == 0) {
                        tseg = INFINITY; thit = INFINITY;
                    } else {
                        const float e0 = sub_(sVec[3 * j], ox), e1 = sub_(sVec[3 * j + 1], oy), e2 = sub_(sVec[3 * j + 2], oz);
                        tseg = sqrt_(add_(add_(mul_(e0, e0), mul_(e1, e1)), mul_(e2, e2)));
                        thit = mul_(tseg, LIGHT_T_MAX_MARGIN);
                    }
                    out = (long long)nodes[(size_t)(NI + slot) * 5 + 3] * K + j;
                    ix = div_(1.0f, dx); iy = div_(1.0f, dy); iz = div_(1.0f, dz);
                    has_ray = true; T = 1.0f;
                    st.sp = 0; st.push(NI == 0 ? -1 : 0);         // root (a lone leaf when P == 1)
                } else {
                    exhausted = true;
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
                const float lmax = ray_box_tmax<true>(p0.z, p0.w, p1.x, p1.y, p1.z, p1.w, ox, oy, oz, ix, iy, iz, tseg);
                const float rmax = ray_box_tmax<true>(p2.x, p2.y, p2.z, p2.w, p3.x, p3.y, ox, oy, oz, ix, iy, iz, tseg);
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
                if (gaussian_hit(q, ox, oy, oz, dx, dy, dz, t, power) && t < thit) {
                    const float alpha = q.op * __expf(power);
                    T *= 1 - alpha;
                    if (T < LIGHT_T_MIN) {
                        shadows[out] = T;
                        has_ray = false;
                    }
                }
            }
            if (has_ray && st.sp == 0) {
                shadows[out] = T;
                has_ray = false;
            }
        }
    }
}

// The lights' ray targets in shared memory: sL [K][9] = pos, and u, v of a rect; column c of a Gaussian or pixel
// belongs to light sRay[c] >> 8 (its sample sRay[c] & 255), 1 column per light and M^2 per rect, in light order
__device__ __forceinline__ void stage_light_rays(int K, int M, uint32_t rect_mask, const float* __restrict__ pos,
                                                 const float* __restrict__ a, const float* __restrict__ b, float* sL,
                                                 uint16_t* sRay) {
    const int tid = threadIdx.x;
    for (int i = tid; i < 3 * K; i += LT_THREADS) {
        const int j = i / 3, c = i - 3 * j;
        const bool rect = (rect_mask >> j) & 1;
        sL[9 * j + c] = pos[i];
        sL[9 * j + 3 + c] = rect ? a[i] : 0.f;
        sL[9 * j + 6 + c] = rect ? b[i] : 0.f;
    }
    if (tid == 0) {
        int col = 0;
        for (int j = 0; j < K; ++j) {
            const int n = ((rect_mask >> j) & 1) ? M * M : 1;
            for (int q = 0; q < n; ++q) sRay[col++] = (uint16_t)((j << 8) | q);
        }
    }
    __syncthreads();
}

// Spot and rect lights.  Ray r = (leaf slot r / R, column r % R); column c belongs to light sRay[c] >> 8 (its sample
// sRay[c] & 255).  A spot's ray is a point light's at pos, a rect sample's the same towards its y_q.
struct ShapedRays {
    static constexpr bool kDeclines = false;
    int NI, R, M;
    uint32_t rect_mask, seed;
    const float* sL;                 // [K][9]: pos, u (or the axis), v
    const uint16_t* sRay;
    const float4* packets;
    const int32_t* nodes;
    __device__ __forceinline__ bool operator()(long long ray, float& ox, float& oy, float& oz, float& dx, float& dy, float& dz,
                                               float& tseg, float& thit, long long& out) const {
        const long long slot = ray / R;
        const int col = (int)(ray - slot * R);
        const LeafRecord self = load_leaf(packets + (size_t)(NI + slot) * 4);
        const int g = nodes[(size_t)(NI + slot) * 5 + 3];
        const int j = sRay[col] >> 8, q = sRay[col] & 255;
        const float* L = sL + 9 * j;
        float y[3];
        if ((rect_mask >> j) & 1) {
            float s, t;
            rect_sample(L, L + 3, L + 6, M, rect_hash(seed, (uint32_t)g, (uint32_t)j), q, s, t, y);
        } else {
            y[0] = L[0]; y[1] = L[1]; y[2] = L[2];
        }
        ray_to_point(y, self.mx, self.my, self.mz, ox, oy, oz, dx, dy, dz, tseg, thit);
        out = (long long)g * R + col;
        return true;
    }
};

__global__ void __launch_bounds__(LT_THREADS) bvh_shaped_lights_kernel(int P, int K, int R, int M, uint32_t rect_mask, uint32_t seed,
                                                                       const float* __restrict__ pos, const float* __restrict__ a,
                                                                       const float* __restrict__ b,
                                                                       const float4* __restrict__ packets,
                                                                       const int32_t* __restrict__ nodes,
                                                                       float* __restrict__ shadows, unsigned long long* counter) {
    __shared__ int sStack[TRACE_STACK_SH][LT_THREADS];
    __shared__ float sL[9 * R3DG_MAX_LIGHTS];
    __shared__ uint16_t sRay[R3DG_MAX_SHAPED_RAYS];
    stage_light_rays(K, M, rect_mask, pos, a, b, sL, sRay);
    const int NI = P - 1;
    const ShapedRays setup{NI, R, M, rect_mask, seed, sL, sRay, packets, nodes};
    trace_shadow_rays(setup, (long long)P * R, NI, packets, shadows, counter, sStack);
}

// Per-pixel lights (PIXEL LIGHTS).  Ray r = (cell r / R, column r % R); cell c of view v = c / cells is pixel (c % 64)
// of tile (c % cells) / 64, tiles in rows of tiles_x (pixel_trace.cu's numbering).  Column c is a directional light's
// ray (dir_mask), a rect sample's towards y_q with the pixel's index p in the hash, or a point light's or spot's
// towards pos.  Output T[v,c,p].
struct PixelLightRays {
    static constexpr bool kDeclines = true;
    int R, M, W, H, tiles_x;
    uint32_t dir_mask, rect_mask, seed;
    long long cells;                 // PT_TILE^2 * tiles per view
    const float* sL;
    const uint16_t* sRay;
    const float* points;             // [V,3,H,W]
    const uint8_t* mask;             // [V,H,W] or NULL
    float* T;
    __device__ __forceinline__ bool operator()(long long ray, float& ox, float& oy, float& oz, float& dx, float& dy, float& dz,
                                               float& tseg, float& thit, long long& out) const {
        const long long cell = ray / R;
        const int col = (int)(ray - cell * R);
        const long long v = cell / cells;
        const long long c = cell - v * cells;
        const long long tile = c / (PL_TILE * PL_TILE);
        const int w = (int)(c - tile * (PL_TILE * PL_TILE));
        const int px = (int)(tile % tiles_x) * PL_TILE + w % PL_TILE, py = (int)(tile / tiles_x) * PL_TILE + w / PL_TILE;
        if (px >= W || py >= H) return false;
        const size_t HW = (size_t)H * W, p = (size_t)py * W + px;
        out = ((long long)v * R + col) * (long long)HW + (long long)p;
        if (mask && !mask[v * HW + p]) { T[out] = 0.0f; return false; }
        const float* pb = points + 3 * v * HW + p;
        const float mx = pb[0], my = pb[HW], mz = pb[2 * HW];
        const int j = sRay[col] >> 8, q = sRay[col] & 255;
        const float* L = sL + 9 * j;
        if ((dir_mask >> j) & 1) {                       // bvh_lights_kernel's directional ray
            const LightDir ld = light_dir(0, L, mx, my, mz);
            dx = ld.l[0]; dy = ld.l[1]; dz = ld.l[2];
            ox = add_(mx, mul_(dx, LIGHT_ORIGIN_OFFSET));
            oy = add_(my, mul_(dy, LIGHT_ORIGIN_OFFSET));
            oz = add_(mz, mul_(dz, LIGHT_ORIGIN_OFFSET));
            tseg = INFINITY; thit = INFINITY;
        } else if ((rect_mask >> j) & 1) {
            float s, t, y[3];
            rect_sample(L, L + 3, L + 6, M, rect_hash(seed, (uint32_t)p, (uint32_t)j), q, s, t, y);
            ray_to_point(y, mx, my, mz, ox, oy, oz, dx, dy, dz, tseg, thit);
        } else {
            ray_to_point(L, mx, my, mz, ox, oy, oz, dx, dy, dz, tseg, thit);
        }
        return true;
    }
};

__global__ void __launch_bounds__(LT_THREADS) bvh_pixel_lights_kernel(int P, int K, long long num_rays, PixelLightRays rays,
                                                                      const float* __restrict__ pos, const float* __restrict__ a,
                                                                      const float* __restrict__ b,
                                                                      const float4* __restrict__ packets,
                                                                      unsigned long long* counter) {
    __shared__ int sStack[TRACE_STACK_SH][LT_THREADS];
    __shared__ float sL[9 * R3DG_MAX_LIGHTS];
    __shared__ uint16_t sRay[R3DG_MAX_SHAPED_RAYS];
    stage_light_rays(K, rays.M, rays.rect_mask, pos, a, b, sL, sRay);
    rays.sL = sL; rays.sRay = sRay;
    trace_shadow_rays(rays, num_rays, P - 1, packets, rays.T, counter, sStack);
}

// ---- host launcher ------------------------------------------------------------------------
size_t bvh_lights_tmp_bytes(int P) { return bvh_packets_bytes(P); }

int launch_bvh_lights(int P, int K, const int32_t* kind, const float* vec, const int32_t* nodes, const float* aabbs,
                      const float* means3D, const float* covs3D, const float* opacities, const float* normals, float* shadows,
                      void* tmp, size_t tmp_bytes, int num_sms, cudaStream_t stream, bool* launched) {
    *launched = false;
    if (P < 0 || !lights_valid(K, kind)) return R3DG_ERR_BAD_ARG;
    if (P == 0 || K == 0) return 0;
    if (!vec || !nodes || !aabbs || !means3D || !covs3D || !opacities || !normals || !shadows || !tmp) return R3DG_ERR_BAD_ARG;
    if (tmp_bytes < bvh_lights_tmp_bytes(P)) return R3DG_ERR_BAD_ARG;
    unsigned long long* counter = (unsigned long long*)tmp;
    float4* packets = (float4*)((char*)tmp + 256);
    R3DG_CUDA_TRY(cudaMemsetAsync(counter, 0, 8, stream));
    const int rc = launch_bvh_pack(P, nodes, aabbs, means3D, covs3D, opacities, normals, packets, stream);
    if (rc != 0) return rc;
    const long long num_rays = (long long)P * K;
    const long long want = (num_rays + LT_THREADS - 1) / LT_THREADS;
    const int blocks = (int)(want < (long long)num_sms * 16 ? want : (long long)num_sms * 16);
    bvh_lights_kernel<<<blocks, LT_THREADS, 0, stream>>>(P, K, point_mask(K, kind), vec, packets, nodes, shadows, counter);
    R3DG_CUDA_TRY(cudaGetLastError());
    *launched = true;
    return 0;
}

int shaped_num_rays(int K, const int32_t* kind, int M) { return shaped_rays(K, kind, M); }

int launch_bvh_shaped_lights(const r3dg_shaped_light_args* a, const int32_t* nodes, const float* aabbs, const float* covs3D,
                             const float* opacities, float* shadows, void* tmp, size_t tmp_bytes, int num_sms,
                             cudaStream_t stream, bool* launched) {
    *launched = false;
    if (!a || a->P < 0) return R3DG_ERR_BAD_ARG;
    const int R = shaped_rays(a->K, a->kind, a->M);
    if (R < 0) return R3DG_ERR_BAD_ARG;
    if (a->P == 0 || a->K == 0) return 0;
    const uint32_t rm = rect_mask(a->K, a->kind);
    if (!a->pos || (rm && (!a->a || !a->b)) || !nodes || !aabbs || !a->means3D || !covs3D || !opacities || !a->normals ||
        !shadows || !tmp)
        return R3DG_ERR_BAD_ARG;
    if (tmp_bytes < bvh_lights_tmp_bytes(a->P)) return R3DG_ERR_BAD_ARG;
    unsigned long long* counter = (unsigned long long*)tmp;
    float4* packets = (float4*)((char*)tmp + 256);
    R3DG_CUDA_TRY(cudaMemsetAsync(counter, 0, 8, stream));
    const int rc = launch_bvh_pack(a->P, nodes, aabbs, a->means3D, covs3D, opacities, a->normals, packets, stream);
    if (rc != 0) return rc;
    const long long num_rays = (long long)a->P * R;
    const long long want = (num_rays + LT_THREADS - 1) / LT_THREADS;
    const int blocks = (int)(want < (long long)num_sms * 16 ? want : (long long)num_sms * 16);
    bvh_shaped_lights_kernel<<<blocks, LT_THREADS, 0, stream>>>(a->P, a->K, R, a->M, rm, a->seed, a->pos, a->a, a->b, packets,
                                                                nodes, shadows, counter);
    R3DG_CUDA_TRY(cudaGetLastError());
    *launched = true;
    return 0;
}

}  // namespace r3dg

using namespace r3dg;
extern "C" {

size_t r3dg_bvh_trace_pixel_lights_tmp_bytes(int P) { return bvh_lights_tmp_bytes(P); }

int r3dg_bvh_trace_pixel_lights(const r3dg_pixel_light_args* a, int P, const int32_t* nodes, const float* aabbs,
                                const float* means3D, const float* covs3D, const float* opacities, const float* normals,
                                float* T, void* tmp, size_t tmp_bytes, r3dg_stream_t stream_) {
    PixelLightSet ls;
    const int err = pixel_light_set(a, false, ls);
    if (err != 0) return err;
    if (P < 1 || !nodes || !aabbs || !means3D || !covs3D || !opacities || !normals || !T || !tmp) return R3DG_ERR_BAD_ARG;
    if (tmp_bytes < bvh_lights_tmp_bytes(P)) return R3DG_ERR_BAD_ARG;
    if (a->K == 0) return 0;                             // T [V,0,H,W] is empty
    const cudaStream_t stream = (cudaStream_t)stream_;
    unsigned long long* counter = (unsigned long long*)tmp;
    float4* packets = (float4*)((char*)tmp + 256);
    R3DG_CUDA_TRY(cudaMemsetAsync(counter, 0, 8, stream));
    const int rc = launch_bvh_pack(P, nodes, aabbs, means3D, covs3D, opacities, normals, packets, stream);
    if (rc != 0) return rc;
    const int tiles_x = (a->W + PL_TILE - 1) / PL_TILE, tiles_y = (a->H + PL_TILE - 1) / PL_TILE;
    const long long cells = (long long)tiles_x * tiles_y * PL_TILE * PL_TILE;
    const PixelLightRays rays{ls.R, a->M, a->W, a->H, tiles_x, ls.dir_mask, ls.rect_mask, a->seed, cells, nullptr, nullptr,
                              a->points, a->mask, T};
    const long long num_rays = (long long)a->V * cells * ls.R;
    const long long want = (num_rays + LT_THREADS - 1) / LT_THREADS;
    const int blocks = (int)(want < (long long)num_sms() * 16 ? want : (long long)num_sms() * 16);
    bvh_pixel_lights_kernel<<<blocks, LT_THREADS, 0, stream>>>(P, a->K, num_rays, rays, a->pos, a->a, a->b, packets, counter);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // extern "C"
