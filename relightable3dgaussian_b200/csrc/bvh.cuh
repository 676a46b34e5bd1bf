// Device pieces shared by the BVH traces of bvh.cu (visibility), indirect.cu (radiance) and lights_trace.cu (shadows):
// the packed tree layout, the incident-direction generator, the slab test, the hit rule and the split ray stack.
#pragma once
#include <cstdio>
#include "common.cuh"

namespace r3dg {

// ---- packed tree (written once per trace call by bvh_pack_kernel, bvh.cu) -------------------------------
// packets: [NI] internal {l, r, lbox[6], rbox[6], pad[2]} then [P] leaf {mean3, cinv6, opacity, normal3, pad3}
// child encoding: >= 0 internal node index; < 0 leaf slot  -(slot + 1)   (slot = Morton-order position)
struct LeafRecord {
    float mx, my, mz;                   // mean
    float c0, c1, c2, c3, c4, c5;       // inverse covariance (xx, xy, xz, yy, yz, zz)
    float op;                           // opacity
    float nx, ny, nz;                   // normal
};
__device__ __forceinline__ LeafRecord load_leaf(const float4* __restrict__ p) {
    const float4 q0 = p[0], q1 = p[1], q2 = p[2], q3 = p[3];
    return LeafRecord{q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, q3.x};
}

// Slab test of utility.cuh:35-82.  The reference divides (b - o) / d six times per box; here the three reciprocals
// 1/d are formed ONCE per ray (IEEE, so zero components still give +-inf and 0 * inf = NaN exactly where the
// reference's 0 / 0 does) and each slab distance is one multiply: ~12 instructions per box instead of ~60.  A product
// by the rounded reciprocal can differ from the quotient in the last bit, which only matters when a ray grazes a box
// exactly; the tests bound the resulting visibility flip rate against the reference's own kernels (<= 1e-3).
// Returns the exit distance, or -1 for a miss; a child is visited when the result is > 0.
// SEG (the light traces, lights_trace.cu): -1 also when the box is entered beyond tseg, so a result > 0 means the
// segment [0, tseg] of the ray meets the box; with tseg = +inf it is the plain test.
template <bool SEG = false>
__device__ __forceinline__ float ray_box_tmax(float b0, float b1, float b2, float b3, float b4, float b5,
                                              float ox, float oy, float oz, float ix, float iy, float iz, float tseg = 0.f) {
    float tmin = mul_(sub_(b0, ox), ix), tmax = mul_(sub_(b3, ox), ix);
    if (tmin > tmax) { const float t = tmin; tmin = tmax; tmax = t; }
    float tymin = mul_(sub_(b1, oy), iy), tymax = mul_(sub_(b4, oy), iy);
    if (tymin > tymax) { const float t = tymin; tymin = tymax; tymax = t; }
    if (tmin > tymax || tymin > tmax) return -1.0f;
    if (tymin > tmin) tmin = tymin;
    if (tymax < tmax) tmax = tymax;
    float tzmin = mul_(sub_(b2, oz), iz), tzmax = mul_(sub_(b5, oz), iz);
    if (tzmin > tzmax) { const float t = tzmin; tzmin = tzmax; tzmax = t; }
    if (tmin > tzmax || tzmin > tmax) return -1.0f;
    if (tzmax < tmax) tmax = tzmax;
    if (SEG) {
        if (tzmin > tmin) tmin = tzmin;
        if (tmin > tseg) return -1.0f;
    }
    return tmax;
}

// The visibility trace's hit rule for the Gaussian of leaf record `q` on ray (o, d): opacity >= 1/255, not
// back-facing, peak t >= 0.01 and power <= 0.  Same arithmetic as bvh_trace_kernel, so the bakes and the light
// traces see one hit set.
__device__ __forceinline__ bool gaussian_hit(const LeafRecord& q, float ox, float oy, float oz, float dx, float dy, float dz,
                                             float& t, float& power) {
    if ((q.op < 1.f / 255.f) || (q.nx * dx + q.ny * dy + q.nz * dz > 0)) return false;
    const float c0 = q.c0, c1 = q.c1, c2 = q.c2, c3 = q.c3, c4 = q.c4, c5 = q.c5;
    const float m0 = q.mx - ox, m1 = q.my - oy, m2 = q.mz - oz;
    const float t1 = c0 * m0 * dx + c1 * m0 * dy + c2 * m0 * dz + c1 * m1 * dx + c3 * m1 * dy + c4 * m1 * dz +
                     c2 * m2 * dx + c4 * m2 * dy + c5 * m2 * dz;
    const float t2 = c0 * dx * dx + c1 * dx * dy + c2 * dx * dz + c1 * dy * dx + c3 * dy * dy + c4 * dy * dz +
                     c2 * dz * dx + c4 * dz * dy + c5 * dz * dz;
    t = t1 / t2;
    if (t < 0.01f) return false;
    const float e0 = q.mx - (ox + t * dx), e1 = q.my - (oy + t * dy), e2 = q.mz - (oz + t * dz);
    power = -0.5f * (e0 * e0 * c0 + e1 * e1 * c3 + e2 * e2 * c5 + 2 * e0 * e1 * c1 + 2 * e0 * e2 * c2 + 2 * e1 * e2 * c4);
    return !(power > 0);
}

// ---- incident-direction sampling (reference utils/graphics_utils.py:9-37 fibonacci_sphere_sampling with
// random_rotate=False — the bake always samples deterministically, scene/gaussian_model.py:324 — and
// utils/sh_utils.py:36-68 rotation_between_z), restated with torch's op-by-op fp32 rounding -------------
// Canonical sample i of N (the [1,3,N] `z_samples` tensor of the reference): computed per CTA into shared
// memory by whoever needs it; identical for every Gaussian.
__device__ __forceinline__ float3 fib_sample(int i, int N) {
    const float idx = (float)i;
    // z = (1 - 2*idx/(2N-1)).clamp_min(sin(10 deg));  rad = sqrt(1 - z**2);  theta = delta*idx
    const float z = fmaxf(sub_(1.0f, div_(mul_(2.0f, idx), (float)(2 * N - 1))), 0.17364817766693033f);
    const float rad = sqrt_(sub_(1.0f, mul_(z, z)));
    const float theta = mul_(2.399963229728653f, idx);          // pi * (3 - sqrt(5))
    return make_float3(mul_(sinf(theta), rad), mul_(cosf(theta), rad), z);
}
// R(normal) @ sample, then F.normalize: the rotation taking +z to `normal` (Rodrigues from z; -I when n.z + 1 <= 0).
// With v = (-n.y, n.x, 0) the reference's nine entries reduce exactly (x + 0 == x, -0 - x == -x in IEEE) to the ones below.
__device__ __forceinline__ float3 rotate_from_z(float nx, float ny, float nz, float3 s) {
    float r00, r01, r02, r10, r11, r12, r20, r21, r22;
    const float zp1 = add_(nz, 1.0f);
    if (zp1 > 0.0f) {
        const float v1 = -ny, v2 = nx, c = fmaxf(zp1, 1e-7f);
        const float v11 = mul_(v1, v1), v22 = mul_(v2, v2), v12 = mul_(v1, v2);
        r00 = add_(1.0f, div_(-v22, c)); r01 = div_(v12, c);             r02 = v2;
        r10 = div_(v12, c);             r11 = add_(1.0f, div_(-v11, c)); r12 = -v1;
        r20 = -v2;                      r21 = v1;                        r22 = add_(1.0f, div_(sub_(-v22, v11), c));
    } else {
        r00 = r11 = r22 = -1.0f; r01 = r02 = r10 = r12 = r20 = r21 = 0.0f;
    }
    // the [P,3,3] @ [1,3,N] matmul: K = 3 accumulated in order (fp32 FMA chain, as cuBLAS sgemm does)
    const float x = fma_(r02, s.z, fma_(r01, s.y, mul_(r00, s.x)));
    const float y = fma_(r12, s.z, fma_(r11, s.y, mul_(r10, s.x)));
    const float z = fma_(r22, s.z, fma_(r21, s.y, mul_(r20, s.x)));
    const float nrm = fmaxf(sqrt_(fma_(z, z, fma_(y, y, mul_(x, x)))), 1e-12f);   // F.normalize eps
    return make_float3(div_(x, nrm), div_(y, nrm), div_(z, nrm));
}
// F.normalize(n) op by op: n / max(sqrt((x*x + y*y) + z*z), 1e-12).  The per-pixel trace and shading rotate the
// samples to this unit normal (a rasterized normal is a blend, not unit length).
__device__ __forceinline__ float3 unit_normal(float x, float y, float z) {
    const float nn = fmaxf(sqrt_(add_(add_(mul_(x, x), mul_(y, y)), mul_(z, z))), 1e-12f);
    return make_float3(div_(x, nn), div_(y, nn), div_(z, nn));
}
// The bake's sample table holds N float3 in dynamic shared memory; a larger N is refused (R3DG_ERR_UNSUPPORTED).
#define BAKE_SAMPLE_SMEM (32 * 1024)

// ---- per-ray traversal stack: the top TRACE_STACK_SH levels in shared memory (one column per thread), deeper
// ones in a per-thread local array; a push beyond TRACE_STACK is dropped with the reference's own warning
// (bvh/include/trace.cuh:24-29; it then writes past its array) ---------------------------------------------
#define TRACE_STACK 64          // total per-ray stack capacity (the reference's local array is 64 too, trace.cuh)
#define TRACE_STACK_SH 20       // entries kept in shared memory; deeper levels spill to a per-thread local array
template <int THREADS>
struct SplitStack {
    int (*sh)[THREADS];                              // __shared__ int [TRACE_STACK_SH][THREADS]
    int local[TRACE_STACK - TRACE_STACK_SH];
    int tid, sp;
    __device__ __forceinline__ void push(int v) {
        if (sp < TRACE_STACK_SH) sh[sp][tid] = v;
        else if (sp < TRACE_STACK) local[sp - TRACE_STACK_SH] = v;
        else { printf("WARNING TOO BIG\n"); return; }
        ++sp;
    }
    __device__ __forceinline__ int pop() {
        --sp;
        return sp < TRACE_STACK_SH ? sh[sp][tid] : local[sp - TRACE_STACK_SH];
    }
};

}  // namespace r3dg
