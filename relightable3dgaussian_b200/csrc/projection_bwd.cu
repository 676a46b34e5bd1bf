// Stage 1 backward: computeCov2DCUDA (reference K11, backward.cu:144-276) and preprocessCUDA
// backward (K12, backward.cu:348-398, SH backward :20-139, cov3D backward :280-343) fused into a
// single per-Gaussian kernel.
//
// Design notes
//  * one pass over the Gaussians instead of two kernels + ten zero-fill memsets: every output row
//    (including the rows of culled Gaussians) is written here exactly once, so the caller hands
//    in uninitialised memory (the reference zero-fills 320 MB at P=1M, rasterize_points.cu:183-192);
//  * the input gradient is one packed [RECF] row per Gaussian produced by the compositor;
//  * cov3D is recomputed from scale/rotation instead of being stored and re-read.
#include "common.cuh"
#include "detacc.cuh"
#include "kernels.h"

namespace r3dg {

struct ProjBwdParams {
    int P, S, D, M, W, H, recf;
    const float *means3D, *shs, *colors_precomp, *scales, *rotations, *cov3D_precomp, *viewmatrix,
        *projmatrix, *campos;
    float scale_modifier, tan_fovx, tan_fovy, h_x, h_y;
    bool antialiasing;          // the record's opacity slot holds o rho (projection.cu): differentiate rho too
    const float* rec;
    const float* grad;
    const uint8_t* clamped;     // bits 0-2: SH colour clamped, kComposited: the row is live (read and differentiated)
    float *dL_dmeans2D, *dL_dcolors, *dL_dopacity, *dL_dmeans3D, *dL_dfeatures, *dL_dcov3D, *dL_dsh,
        *dL_dscales, *dL_drotations;
    float* dL_dsh_factor;       // [P,3] gated dL_dRGB (multi-GPU exchange, sh_exchange.cu); dL_dsh may then be NULL
    DetAcc det;                 // DET: the gradient rows as fixed-point accumulators (composite_bwd.cu), read instead of grad
    size_t det_row0;            // DET: the view's first row in `det` (several views: v * P)
    const uint32_t* det_scale;  // DET: the view's scale words of the colour / feature and geometry slots (composite_bwd.cu)
    // several views, views after the first: add this view's gradient to what the earlier views wrote (fp32, view order)
    // instead of writing it — acc for the gradients summed over the views, acc_colors / acc_features for dL_dcolors /
    // dL_dfeatures when those inputs are shared (per-view inputs get per-view rows: no accumulation)
    bool acc, acc_colors, acc_features;
    // CAM: this view's [kCamGradFloats][gridDim.x] partial sums of the camera gradients (column-major: one column per CTA)
    float* cam_work;
};
static_assert(kCamGradThreads == 128, "cam_grad_blocks() counts projection-backward CTAs");

// out = x, or out += x when `acc` (the left fold of several views' gradients)
__device__ __forceinline__ void put(float* out, float x, bool acc) { *out = acc ? *out + x : x; }

__device__ __forceinline__ void cov3d_plain(const float* s3, float mod, const float* q, float* c6,
                                            float R[3][3], float s[3]) {
    const float r = q[0], x = q[1], y = q[2], z = q[3];
    // glm column-major R[c][r] (backward.cu:289-293)
    R[0][0] = 1.f - 2.f * (y * y + z * z); R[0][1] = 2.f * (x * y - r * z); R[0][2] = 2.f * (x * z + r * y);
    R[1][0] = 2.f * (x * y + r * z); R[1][1] = 1.f - 2.f * (x * x + z * z); R[1][2] = 2.f * (y * z - r * x);
    R[2][0] = 2.f * (x * z - r * y); R[2][1] = 2.f * (y * z + r * x); R[2][2] = 1.f - 2.f * (x * x + y * y);
    s[0] = mod * s3[0]; s[1] = mod * s3[1]; s[2] = mod * s3[2];
    float M[3][3];
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int rr = 0; rr < 3; ++rr) M[c][rr] = s[rr] * R[c][rr];
    // Sigma[c][r] = dot(M col r, M col c)
    c6[0] = M[0][0] * M[0][0] + M[0][1] * M[0][1] + M[0][2] * M[0][2];
    c6[1] = M[0][0] * M[1][0] + M[0][1] * M[1][1] + M[0][2] * M[1][2];
    c6[2] = M[0][0] * M[2][0] + M[0][1] * M[2][1] + M[0][2] * M[2][2];
    c6[3] = M[1][0] * M[1][0] + M[1][1] * M[1][1] + M[1][2] * M[1][2];
    c6[4] = M[1][0] * M[2][0] + M[1][1] * M[2][1] + M[1][2] * M[2][2];
    c6[5] = M[2][0] * M[2][0] + M[2][1] * M[2][1] + M[2][2] * M[2][2];
}

// The SH basis (backward.cu:20-139) at the unit view direction (x, y, z) for degree D, and its derivatives; zero above
// (D + 1)^2.  One definition for the projection backward and the appearance-only backward, so that both compute the
// same dL/dsh bits.
__device__ __forceinline__ void sh_basis(int D, float x, float y, float z, float (&w)[16], float (&wx)[16], float (&wy)[16],
                                         float (&wz)[16]) {
#pragma unroll
    for (int k = 0; k < 16; ++k) { w[k] = 0.f; wx[k] = 0.f; wy[k] = 0.f; wz[k] = 0.f; }
    const float C1 = 0.4886025119029199f;
    w[0] = 0.28209479177387814f;
    if (D > 0) {
        w[1] = -C1 * y; w[2] = C1 * z; w[3] = -C1 * x;
        wy[1] = -C1; wz[2] = C1; wx[3] = -C1;
        if (D > 1) {
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            const float c20 = 1.0925484305920792f, c21 = -1.0925484305920792f, c22 = 0.31539156525252005f,
                        c23 = -1.0925484305920792f, c24 = 0.5462742152960396f;
            w[4] = c20 * xy; w[5] = c21 * yz; w[6] = c22 * (2.f * zz - xx - yy); w[7] = c23 * xz; w[8] = c24 * (xx - yy);
            wx[4] = c20 * y;  wy[4] = c20 * x;
            wy[5] = c21 * z;  wz[5] = c21 * y;
            wx[6] = c22 * 2.f * -x; wy[6] = c22 * 2.f * -y; wz[6] = c22 * 2.f * 2.f * z;
            wx[7] = c23 * z;  wz[7] = c23 * x;
            wx[8] = c24 * 2.f * x; wy[8] = c24 * 2.f * -y;
            if (D > 2) {
                const float c30 = -0.5900435899266435f, c31 = 2.890611442640554f, c32 = -0.4570457994644658f,
                            c33 = 0.3731763325901154f, c34 = -0.4570457994644658f, c35 = 1.445305721320277f,
                            c36 = -0.5900435899266435f;
                w[9] = c30 * y * (3.f * xx - yy); w[10] = c31 * xy * z; w[11] = c32 * y * (4.f * zz - xx - yy);
                w[12] = c33 * z * (2.f * zz - 3.f * xx - 3.f * yy); w[13] = c34 * x * (4.f * zz - xx - yy);
                w[14] = c35 * z * (xx - yy); w[15] = c36 * x * (xx - 3.f * yy);
                wx[9] = c30 * 3.f * 2.f * xy;  wy[9] = c30 * 3.f * (xx - yy);
                wx[10] = c31 * yz;             wy[10] = c31 * xz;            wz[10] = c31 * xy;
                wx[11] = c32 * -2.f * xy;      wy[11] = c32 * (-3.f * yy + 4.f * zz - xx); wz[11] = c32 * 4.f * 2.f * yz;
                wx[12] = c33 * -3.f * 2.f * xz; wy[12] = c33 * -3.f * 2.f * yz; wz[12] = c33 * 3.f * (2.f * zz - xx - yy);
                wx[13] = c34 * (-3.f * xx + 4.f * zz - yy); wy[13] = c34 * -2.f * xy; wz[13] = c34 * 4.f * 2.f * xz;
                wx[14] = c35 * 2.f * xz;       wy[14] = c35 * -2.f * yz;     wz[14] = c35 * (xx - yy);
                wx[15] = c36 * 3.f * (xx - yy); wy[15] = c36 * -3.f * 2.f * xy;
            }
        }
    }
}

// The view direction of a Gaussian (backward.cu:20-139): d = m - cam, its squares, |d|^2 and the unit vector (x, y, z).
// |d|^2 is three rounded products and two rounded sums in this order — explicit, so that the compiler cannot contract
// it differently in the projection backward (where the squares have other uses) and in the appearance-only backward:
// both compute the same direction, and so the same dL/dsh bits.
struct ViewDir { float dx, dy, dz, xx, yy, zz, sum2, x, y, z; };
__device__ __forceinline__ ViewDir view_dir(const float* m, const float* cam) {
    ViewDir d;
    d.dx = m[0] - cam[0]; d.dy = m[1] - cam[1]; d.dz = m[2] - cam[2];
    d.xx = __fmul_rn(d.dx, d.dx); d.yy = __fmul_rn(d.dy, d.dy); d.zz = __fmul_rn(d.dz, d.dz);
    d.sum2 = __fadd_rn(__fadd_rn(d.xx, d.yy), d.zz);
    const float len = sqrtf(d.sum2);
    d.x = d.dx / len; d.y = d.dy / len; d.z = d.dz / len;
    return d;
}

#define PROJ_THREADS 128
#define SLAB_LD (PROJ_THREADS + 1)
// DET (deterministic mode): the packed gradient row is read from the fixed-point accumulators and converted on load.
// CAM (camera gradients): every thread also stages its Gaussian's 35 camera-gradient terms in a [35][SLAB_LD] slab
// behind the SH slab, and the CTA writes their sums in a fixed order to its column of p.cam_work.
template <bool DET = false, bool CAM = false>
__global__ void __launch_bounds__(PROJ_THREADS, 5) projection_bwd_kernel(const ProjBwdParams p) {
    // SH rows (192 B at M=16) travel through shared memory: the CTA's [128][3M] slab of shs is ONE contiguous
    // 24 KB block, fetched by a single TMA-unit bulk copy (cp.async.bulk, mbarrier-signalled) into a row-major
    // slab; every thread turns its row into dL/dsh in place (16-byte vector accesses) and ONE bulk store writes the
    // slab back (zeros for rows that are not live).  Rows that are not 16-byte multiples (SH degree 0 / 2) or ragged /
    // unaligned tails use the transposed slab s[k * SLAB_LD + t] with 4-byte LDGSTS copies and a coalesced write-back
    // loop.
    // Only LIVE rows — some pixel composited them in the forward pass (kComposited) — read anything: every other row's
    // gradients are exactly zero, and it writes +0 to its outputs without reading its gradient row, parameters or SH.
    // A CTA whose rows are all live fetches its SH slab with the one bulk copy; otherwise each live row is fetched on its
    // own (one bulk copy per row, or the transposed LDGSTS loads of the live rows only).
    extern __shared__ __align__(16) float sSH[];
    __shared__ float sV[16], sPr[16], sCam[3];
    __shared__ uint32_t sLive[PROJ_THREADS / 32];
    __shared__ __align__(8) uint64_t sBar;
    const int rowf_ = 3 * p.M, base_ = blockIdx.x * PROJ_THREADS;
    const unsigned slab_bytes = (unsigned)min(PROJ_THREADS, p.P - base_) * (unsigned)rowf_ * 4u;
    const bool bulk = p.shs && (rowf_ & 3) == 0 && (slab_bytes & 15u) == 0 &&
                      (reinterpret_cast<uintptr_t>(p.shs + (size_t)base_ * rowf_) & 15) == 0 &&
                      (!p.dL_dsh || (reinterpret_cast<uintptr_t>(p.dL_dsh + (size_t)base_ * rowf_) & 15) == 0);
    if (threadIdx.x == 0 && bulk) { mbar_init(&sBar, 1); fence_proxy_async_smem(); }
    if (threadIdx.x < 16) { sV[threadIdx.x] = p.viewmatrix[threadIdx.x]; sPr[threadIdx.x] = p.projmatrix[threadIdx.x]; }
    if (threadIdx.x < 3) sCam[threadIdx.x] = p.campos[threadIdx.x];
    const int idx_raw = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in_range = idx_raw < p.P;
    const int idx = in_range ? idx_raw : p.P - 1;      // clamp: out-of-range threads only help with the slab
    const unsigned cl = in_range ? p.clamped[idx] : 0u;
    const bool live = (cl & kComposited) != 0;         // composited => visible
    const uint32_t live_warp = __ballot_sync(0xffffffffu, live);
    if ((threadIdx.x & 31) == 0) sLive[threadIdx.x >> 5] = live_warp;
    const int nlive = __syncthreads_count(live);
    const int rowf = 3 * p.M, block_base = blockIdx.x * PROJ_THREADS;
    const int nvalid = min(PROJ_THREADS, p.P - block_base);
    float* sG = sSH + (p.shs ? rowf * SLAB_LD : 0) + threadIdx.x;   // CAM: this thread's terms at sG[k * SLAB_LD]
    if constexpr (CAM) {
#pragma unroll
        for (int k = 0; k < kCamGradFloats; ++k) sG[k * SLAB_LD] = 0.f;   // rows that are not live add nothing
    }
    // the thread's own rows are requested before the cooperative slab load so that both are in flight together
    const float4* g4 = reinterpret_cast<const float4*>(p.grad + (size_t)idx * p.recf);
    float4 gA = make_float4(0, 0, 0, 0), gB = gA, gC = gA, q4 = gA;
    float m3[3] = {0, 0, 0}, s3[3] = {0, 0, 0}, aa_op = 0.f;
    if (live) {
        if (p.antialiasing) aa_op = p.rec[(size_t)idx * p.recf + 5];   // the forward's compensated opacity o rho
        if constexpr (DET) {
            const size_t r0 = (p.det_row0 + idx) * p.recf;
            const int eg = det_scale_exp(p.det_scale[1]), ea = det_scale_exp(p.det_scale[0]);
            gA = make_float4(det_load(p.det, r0, eg), det_load(p.det, r0 + 1, eg), det_load(p.det, r0 + 2, eg), det_load(p.det, r0 + 3, eg));
            gB = make_float4(det_load(p.det, r0 + 4, eg), det_load(p.det, r0 + 5, eg), det_load(p.det, r0 + 6, eg), 0.0f);
            gC = make_float4(det_load(p.det, r0 + 8, ea), det_load(p.det, r0 + 9, ea), det_load(p.det, r0 + 10, ea), 0.0f);
        } else {
            gA = g4[0]; gB = g4[1]; gC = g4[2];
        }
        m3[0] = p.means3D[3 * (size_t)idx]; m3[1] = p.means3D[3 * (size_t)idx + 1]; m3[2] = p.means3D[3 * (size_t)idx + 2];
        if (!p.cov3D_precomp) {
            q4 = *reinterpret_cast<const float4*>(p.rotations + 4 * (size_t)idx);
            s3[0] = p.scales[3 * (size_t)idx]; s3[1] = p.scales[3 * (size_t)idx + 1]; s3[2] = p.scales[3 * (size_t)idx + 2];
        }
    }
    const bool fetch_sh = p.shs && nlive > 0;          // (CTA-uniform)
    if (fetch_sh) {  // asynchronous copy of the live rows of the slab, overlapped with the covariance chain below
        if (bulk) {
            const unsigned row_bytes = (unsigned)rowf * 4u;
            if (nlive == nvalid) {                     // every row: the one contiguous slab
                if (threadIdx.x == 0) { mbar_arrive_expect_tx(&sBar, slab_bytes); bulk_copy_g2s(sSH, p.shs + (size_t)block_base * rowf, slab_bytes, &sBar); }
            } else {
                // one copy per live row into its slab row; a copy may land before thread 0 announces the bytes (the
                // barrier's transaction count may go negative), the phase completes only after that single arrival
                if (threadIdx.x == 0) mbar_arrive_expect_tx(&sBar, (unsigned)nlive * row_bytes);
                if (live) bulk_copy_g2s(sSH + (size_t)threadIdx.x * rowf, p.shs + (size_t)idx * rowf, row_bytes, &sBar);
            }
        } else {
            load_rows_transposed_async(sSH, SLAB_LD, p.shs + (size_t)block_base * rowf, nvalid, rowf, PROJ_THREADS,
                                       nlive == nvalid ? nullptr : sLive);
            cp_async_commit();
        }
    }
    const float* V = sV;
    const float* proj = sPr;

    float dmean2[3] = {0, 0, 0}, dcol[3] = {0, 0, 0}, dop = 0, dmean3[3] = {0, 0, 0}, dfac[3] = {0, 0, 0};
    float dcov[6] = {0, 0, 0, 0, 0, 0}, dscale[3] = {0, 0, 0}, drot[4] = {0, 0, 0, 0};

    // feature gradients: straight copy-out of the packed row (a row that is not live adds nothing to earlier views')
    if (p.S > 0 && in_range && (live || !p.acc_features)) {
        float* df = p.dL_dfeatures + (size_t)idx * p.S;
        for (int c = 0; c < p.S; ++c) {
            if constexpr (DET) put(df + c, live ? det_load(p.det, (p.det_row0 + idx) * p.recf + 11 + c, det_scale_exp(p.det_scale[0])) : 0.0f, p.acc_features);
            else put(df + c, live ? p.grad[(size_t)idx * p.recf + 11 + c] : 0.0f, p.acc_features);
        }
    }
    if (live) {
        dmean2[0] = gA.x; dmean2[1] = gA.y; dmean2[2] = gA.z; dop = gA.w;
        dcol[0] = gC.x; dcol[1] = gC.y; dcol[2] = gC.z;
        const float mx = m3[0], my = m3[1], mz = m3[2];
        const float dcx = gB.x, dcy = gB.y, dcz = gB.z;      // dL/d conic a,b,c
        float c6[6], R[3][3], s[3];
        const bool have_sr = p.scales != nullptr;
        if (p.cov3D_precomp) {
#pragma unroll
            for (int i = 0; i < 6; ++i) c6[i] = p.cov3D_precomp[6 * (size_t)idx + i];
        } else {
            const float q[4] = {q4.x, q4.y, q4.z, q4.w};
            cov3d_plain(s3, p.scale_modifier, q, c6, R, s);
        }
        // ---- computeCov2DCUDA (backward.cu:144-276) -------------------------------------------
        float t[3] = {V[0] * mx + V[4] * my + V[8] * mz + V[12], V[1] * mx + V[5] * my + V[9] * mz + V[13],
                      V[2] * mx + V[6] * my + V[10] * mz + V[14]};
        const float limx = 1.3f * p.tan_fovx, limy = 1.3f * p.tan_fovy;
        const float txtz = t[0] / t[2], tytz = t[1] / t[2];
        t[0] = fminf(limx, fmaxf(-limx, txtz)) * t[2];
        t[1] = fminf(limy, fmaxf(-limy, tytz)) * t[2];
        const float x_grad_mul = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
        const float y_grad_mul = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
        const float h_x = p.h_x, h_y = p.h_y;
        // J (glm columns): J0 = (h_x/tz, 0, -(h_x tx)/tz^2), J1 = (0, h_y/tz, -(h_y ty)/tz^2), J2 = 0
        const float J00 = h_x / t[2], J02 = -(h_x * t[0]) / (t[2] * t[2]);
        const float J11 = h_y / t[2], J12 = -(h_y * t[1]) / (t[2] * t[2]);
        // W (glm columns) = rows of the 3x3 of the stored view matrix: W[k][r] = V[4r + k]
        // T = W * J : T[c][r] = sum_k W[k][r] * J[c][k]
        float T0[3], T1[3];            // T[0][r], T[1][r]; T[2][r] = 0
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            T0[r] = V[4 * r + 0] * J00 + V[4 * r + 2] * J02;
            T1[r] = V[4 * r + 1] * J11 + V[4 * r + 2] * J12;
        }
        const float Vrk[3][3] = {{c6[0], c6[1], c6[2]}, {c6[1], c6[3], c6[4]}, {c6[2], c6[4], c6[5]}};
        float VT0[3], VT1[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            VT0[r] = Vrk[r][0] * T0[0] + Vrk[r][1] * T0[1] + Vrk[r][2] * T0[2];
            VT1[r] = Vrk[r][0] * T1[0] + Vrk[r][1] * T1[1] + Vrk[r][2] * T1[2];
        }
        const float a0 = T0[0] * VT0[0] + T0[1] * VT0[1] + T0[2] * VT0[2];
        const float c0 = T1[0] * VT1[0] + T1[1] * VT1[1] + T1[2] * VT1[2];
        const float a = a0 + 0.3f;
        const float b = T1[0] * VT0[0] + T1[1] * VT0[1] + T1[2] * VT0[2];
        const float c = c0 + 0.3f;
        const float denom = a * c - b * b;
        // antialiased mode: r = det0 / det1 (0 for det0 <= 0) of the forward's rho = sqrt(max(r, 2.5e-5)); the record
        // holds o rho and dop = dL/d(o rho)
        float aa_r = 0.f;
        if (p.antialiasing) {
            const float det0 = a0 * c0 - b * b;
            aa_r = det0 > 0.f ? det0 / denom : 0.f;
        }
        float dL_da = 0, dL_db = 0, dL_dc = 0;
        const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
        if (denom2inv != 0) {
            dL_da = denom2inv * (-c * c * dcx + 2 * b * c * dcy + (denom - a * c) * dcz);
            dL_dc = denom2inv * (-a * a * dcz + 2 * a * b * dcy + (denom - a * c) * dcx);
            dL_db = denom2inv * 2 * (b * c * dcx - (denom + 2 * b * b) * dcy + a * b * dcz);
            if (p.antialiasing && aa_r > 2.5e-5f) {     // (uniform) rho's path: dL/dr = dL/d(o rho) (o rho) / (2 r)
                const float inv1 = 1.0f / denom, gr = dop * aa_op / (2.0f * aa_r) * (inv1 * inv1);
                dL_da = __fadd_rn(dL_da, gr * (0.3f * (c0 * c + b * b)));
                dL_dc = __fadd_rn(dL_dc, gr * (0.3f * (a0 * a + b * b)));
                dL_db = __fadd_rn(dL_db, gr * (-2.0f * b * (0.3f * (a0 + c0) + 0.09f)));
            }
            dcov[0] = (T0[0] * T0[0] * dL_da + T0[0] * T1[0] * dL_db + T1[0] * T1[0] * dL_dc);
            dcov[3] = (T0[1] * T0[1] * dL_da + T0[1] * T1[1] * dL_db + T1[1] * T1[1] * dL_dc);
            dcov[5] = (T0[2] * T0[2] * dL_da + T0[2] * T1[2] * dL_db + T1[2] * T1[2] * dL_dc);
            dcov[1] = 2 * T0[0] * T0[1] * dL_da + (T0[0] * T1[1] + T0[1] * T1[0]) * dL_db + 2 * T1[0] * T1[1] * dL_dc;
            dcov[2] = 2 * T0[0] * T0[2] * dL_da + (T0[0] * T1[2] + T0[2] * T1[0]) * dL_db + 2 * T1[0] * T1[2] * dL_dc;
            dcov[4] = 2 * T0[2] * T0[1] * dL_da + (T0[1] * T1[2] + T0[2] * T1[1]) * dL_db + 2 * T1[1] * T1[2] * dL_dc;
        }
        if (p.antialiasing) dop = __fmul_rn(dop, sqrtf(fmaxf(aa_r, 2.5e-5f)));   // dL/do = rho dL/d(o rho)
        float dT0[3], dT1[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float t0v = T0[0] * Vrk[k][0] + T0[1] * Vrk[k][1] + T0[2] * Vrk[k][2];
            const float t1v = T1[0] * Vrk[k][0] + T1[1] * Vrk[k][1] + T1[2] * Vrk[k][2];
            dT0[k] = 2 * t0v * dL_da + t1v * dL_db;
            dT1[k] = 2 * t1v * dL_dc + t0v * dL_db;
        }
        // W[c][r] = V[4r + c]
        const float dL_dJ00 = V[0] * dT0[0] + V[4] * dT0[1] + V[8] * dT0[2];
        const float dL_dJ02 = V[2] * dT0[0] + V[6] * dT0[1] + V[10] * dT0[2];
        const float dL_dJ11 = V[1] * dT1[0] + V[5] * dT1[1] + V[9] * dT1[2];
        const float dL_dJ12 = V[2] * dT1[0] + V[6] * dT1[1] + V[10] * dT1[2];
        const float tz = 1.f / t[2], tz2 = tz * tz, tz3 = tz2 * tz;
        const float dL_dtx = x_grad_mul * -h_x * tz2 * dL_dJ02;
        const float dL_dty = y_grad_mul * -h_y * tz2 * dL_dJ12;
        const float dL_dtz = -h_x * tz2 * dL_dJ00 - h_y * tz2 * dL_dJ11 + (2 * h_x * t[0]) * tz3 * dL_dJ02 +
                             (2 * h_y * t[1]) * tz3 * dL_dJ12;
        const float gz = dL_dtz + dmean2[2];                     // depth gradient joins here (backward.cu:269)
        dmean3[0] = V[0] * dL_dtx + V[1] * dL_dty + V[2] * gz;
        dmean3[1] = V[4] * dL_dtx + V[5] * dL_dty + V[6] * gz;
        dmean3[2] = V[8] * dL_dtx + V[9] * dL_dty + V[10] * gz;
        // ---- preprocessCUDA backward (backward.cu:372-389) ------------------------------------
        const float m_w = 1.0f / ((proj[3] * mx + proj[7] * my + proj[11] * mz + proj[15]) + 0.0000001f);
        const float mul1 = (proj[0] * mx + proj[4] * my + proj[8] * mz + proj[12]) * m_w * m_w;
        const float mul2 = (proj[1] * mx + proj[5] * my + proj[9] * mz + proj[13]) * m_w * m_w;
        dmean3[0] += (proj[0] * m_w - proj[3] * mul1) * dmean2[0] + (proj[1] * m_w - proj[3] * mul2) * dmean2[1];
        dmean3[1] += (proj[4] * m_w - proj[7] * mul1) * dmean2[0] + (proj[5] * m_w - proj[7] * mul2) * dmean2[1];
        dmean3[2] += (proj[8] * m_w - proj[11] * mul1) * dmean2[0] + (proj[9] * m_w - proj[11] * mul2) * dmean2[1];
        if constexpr (CAM) {
            // viewmatrix: t_k = sum_j [m,1]_j V[4j + k] (k < 3) gives dL/dt (x) [m,1]; the 3x3 block also enters
            // T = W J directly (T0[r] = V[4r] J00 + V[4r + 2] J02, T1[r] = V[4r + 1] J11 + V[4r + 2] J12).  Column 3 is
            // never read.
            const float mt[4] = {mx, my, mz, 1.f};
            const float dt[3] = {dL_dtx, dL_dty, gz};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float d0 = dt[0] * mt[j], d1 = dt[1] * mt[j], d2 = dt[2] * mt[j];
                if (j < 3) { d0 += dT0[j] * J00; d1 += dT1[j] * J11; d2 += dT0[j] * J02 + dT1[j] * J12; }
                sG[(4 * j + 0) * SLAB_LD] = d0; sG[(4 * j + 1) * SLAB_LD] = d1; sG[(4 * j + 2) * SLAB_LD] = d2;
            }
            // projmatrix: ndc = (h_0, h_1) / (h_3 + 1e-7) with h_k = sum_j [m,1]_j P[4j + k]; column 2 is never read
            const float dh0 = dmean2[0] * m_w, dh1 = dmean2[1] * m_w, dh3 = -(dmean2[0] * mul1 + dmean2[1] * mul2);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                sG[(16 + 4 * j + 0) * SLAB_LD] = dh0 * mt[j];
                sG[(16 + 4 * j + 1) * SLAB_LD] = dh1 * mt[j];
                sG[(16 + 4 * j + 3) * SLAB_LD] = dh3 * mt[j];
            }
        }

        // ---- cov3D -> scale / rotation (backward.cu:280-343) ----------------------------------
        if (have_sr) {
            const float r = p.rotations[4 * (size_t)idx], x = p.rotations[4 * (size_t)idx + 1],
                        y = p.rotations[4 * (size_t)idx + 2], z = p.rotations[4 * (size_t)idx + 3];
            if (p.cov3D_precomp) {   // not reachable through the reference wrapper, kept for safety
                const float q[4] = {r, x, y, z};
                const float s3[3] = {p.scales[3 * (size_t)idx], p.scales[3 * (size_t)idx + 1], p.scales[3 * (size_t)idx + 2]};
                float tmp[6];
                cov3d_plain(s3, p.scale_modifier, q, tmp, R, s);
            }
            float Mm[3][3];
#pragma unroll
            for (int cc = 0; cc < 3; ++cc)
#pragma unroll
                for (int rr = 0; rr < 3; ++rr) Mm[cc][rr] = s[rr] * R[cc][rr];
            const float dSig[3][3] = {{dcov[0], 0.5f * dcov[1], 0.5f * dcov[2]},
                                      {0.5f * dcov[1], dcov[3], 0.5f * dcov[4]},
                                      {0.5f * dcov[2], 0.5f * dcov[4], dcov[5]}};
            float dMt[3][3];       // dL_dMt[c][r] = dL_dM[r][c], dL_dM = 2 * M * dL_dSigma
#pragma unroll
            for (int cc = 0; cc < 3; ++cc)
#pragma unroll
                for (int rr = 0; rr < 3; ++rr)
                    dMt[rr][cc] = 2.0f * (Mm[0][rr] * dSig[cc][0] + Mm[1][rr] * dSig[cc][1] + Mm[2][rr] * dSig[cc][2]);
#pragma unroll
            for (int k = 0; k < 3; ++k) dscale[k] = R[0][k] * dMt[k][0] + R[1][k] * dMt[k][1] + R[2][k] * dMt[k][2];
#pragma unroll
            for (int k = 0; k < 3; ++k)
#pragma unroll
                for (int rr = 0; rr < 3; ++rr) dMt[k][rr] *= s[k];
            drot[0] = 2 * z * (dMt[0][1] - dMt[1][0]) + 2 * y * (dMt[2][0] - dMt[0][2]) + 2 * x * (dMt[1][2] - dMt[2][1]);
            drot[1] = 2 * y * (dMt[1][0] + dMt[0][1]) + 2 * z * (dMt[2][0] + dMt[0][2]) + 2 * r * (dMt[1][2] - dMt[2][1]) - 4 * x * (dMt[2][2] + dMt[1][1]);
            drot[2] = 2 * x * (dMt[1][0] + dMt[0][1]) + 2 * r * (dMt[2][0] - dMt[0][2]) + 2 * z * (dMt[1][2] + dMt[2][1]) - 4 * y * (dMt[2][2] + dMt[0][0]);
            drot[3] = 2 * r * (dMt[0][1] - dMt[1][0]) + 2 * x * (dMt[2][0] + dMt[0][2]) + 2 * y * (dMt[1][2] + dMt[2][1]) - 4 * z * (dMt[1][1] + dMt[0][0]);
        }
    }
    // the SH slab was requested asynchronously at the top; it is first needed here
    if (fetch_sh) {
        if (bulk) mbar_wait(&sBar, 0);
        else { cp_async_wait_all(); __syncthreads(); }
    }
    if (live) {
        // ---- SH backward (backward.cu:20-139) -------------------------------------------------
        if (p.shs) {
            const ViewDir vd = view_dir(m3, sCam);
            const float dox = vd.dx, doy = vd.dy, doz = vd.dz, x = vd.x, y = vd.y, z = vd.z;
            float* slab = sSH + threadIdx.x;                 // element (k, c) at slab[(3k + c) * SLAB_LD]
            const float dRGB[3] = {(cl & 1u) ? 0.f : dcol[0], (cl & 2u) ? 0.f : dcol[1], (cl & 4u) ? 0.f : dcol[2]};
            dfac[0] = dRGB[0]; dfac[1] = dRGB[1]; dfac[2] = dRGB[2];
            float w[16], wx[16], wy[16], wz[16];   // basis and its derivatives w.r.t. x,y,z
            sh_basis(p.D, x, y, z, w, wx, wy, wz);
            const int ncoef = (p.D + 1) * (p.D + 1);
            float ddx = 0.f, ddy = 0.f, ddz = 0.f;
            if (bulk) {
                // row-major slab: 4 coefficients (12 floats = three 16-byte vectors) at a time, read, used, overwritten
                float4* row4 = reinterpret_cast<float4*>(sSH + (size_t)threadIdx.x * rowf);
#pragma unroll
                for (int kb = 0; kb < 4; ++kb) {
                    if (4 * kb < p.M) {
                        float v[12];
#pragma unroll
                        for (int i = 0; i < 3; ++i) { const float4 t4 = row4[3 * kb + i]; v[4 * i] = t4.x; v[4 * i + 1] = t4.y; v[4 * i + 2] = t4.z; v[4 * i + 3] = t4.w; }
#pragma unroll
                        for (int kk = 0; kk < 4; ++kk) {
                            const int k = 4 * kb + kk;
                            const bool act = k < ncoef;
                            const float s0 = act ? v[3 * kk] : 0.f, s1 = act ? v[3 * kk + 1] : 0.f, s2 = act ? v[3 * kk + 2] : 0.f;
                            const float dotc = s0 * dRGB[0] + s1 * dRGB[1] + s2 * dRGB[2];
                            ddx += wx[k] * dotc; ddy += wy[k] * dotc; ddz += wz[k] * dotc;
                            v[3 * kk] = act ? w[k] * dRGB[0] : 0.f; v[3 * kk + 1] = act ? w[k] * dRGB[1] : 0.f; v[3 * kk + 2] = act ? w[k] * dRGB[2] : 0.f;
                        }
                        if (p.dL_dsh) {
#pragma unroll
                            for (int i = 0; i < 3; ++i) row4[3 * kb + i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
                        }
                    }
                }
            } else {
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                if (k < p.M) {
                    const bool act = k < ncoef;
                    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
                    if (act) { s0 = slab[(3 * k) * SLAB_LD]; s1 = slab[(3 * k + 1) * SLAB_LD]; s2 = slab[(3 * k + 2) * SLAB_LD]; }
                    const float dotc = s0 * dRGB[0] + s1 * dRGB[1] + s2 * dRGB[2];
                    ddx += wx[k] * dotc; ddy += wy[k] * dotc; ddz += wz[k] * dotc;
                    if (p.dL_dsh) {
                        slab[(3 * k) * SLAB_LD] = act ? w[k] * dRGB[0] : 0.f;        // in place: sh -> dL/dsh
                        slab[(3 * k + 1) * SLAB_LD] = act ? w[k] * dRGB[1] : 0.f;
                        slab[(3 * k + 2) * SLAB_LD] = act ? w[k] * dRGB[2] : 0.f;
                    }
                }
            }
            }
            // dnormvdv (auxiliary.h:105-116)
            const float sum2 = vd.sum2;
            const float invsum32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
            const float ddir[3] = {(+sum2 - vd.xx) * ddx - doy * dox * ddy - doz * dox * ddz,
                                   -dox * doy * ddx + (sum2 - vd.yy) * ddy - doz * doy * ddz,
                                   -dox * doz * ddx - doy * doz * ddy + (sum2 - vd.zz) * ddz};
            // explicit FMAs: the contraction of `dmean3 += ddir * invsum32` must not depend on whether the product
            // has a second use (CAM), so that dL/dmeans3D is the same with and without camera gradients
            dmean3[0] = __fmaf_rn(ddir[0], invsum32, dmean3[0]);
            dmean3[1] = __fmaf_rn(ddir[1], invsum32, dmean3[1]);
            dmean3[2] = __fmaf_rn(ddir[2], invsum32, dmean3[2]);
            if constexpr (CAM) {            // campos: the view direction is mean - campos
#pragma unroll
                for (int k = 0; k < 3; ++k) sG[(32 + k) * SLAB_LD] = -(ddir[k] * invsum32);
            }
        }
    } else if (p.shs && p.dL_dsh) {
        if (bulk) {
            if ((int)threadIdx.x < nvalid) {
                float4* row4 = reinterpret_cast<float4*>(sSH + (size_t)threadIdx.x * rowf);
                for (int i = 0; i < rowf / 4; ++i) row4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        } else {
            for (int k = 0; k < rowf; ++k) sSH[k * SLAB_LD + threadIdx.x] = 0.f;
        }
    }
    if (p.shs && p.dL_dsh) {                        // write-back of the dL/dsh slab
        float* dst = p.dL_dsh + (size_t)block_base * rowf;
        if (bulk) {
            fence_proxy_async_smem();               // this thread's generic-proxy stores -> visible to the bulk-copy engine
            __syncthreads();
            if (threadIdx.x == 0) { bulk_copy_s2g(dst, sSH, slab_bytes); bulk_wait_read_all(); }
        } else {
            __syncthreads();
            const int total = nvalid * rowf;
            if ((rowf & 3) == 0) {
                float4* dst4 = reinterpret_cast<float4*>(dst);
                for (int i4 = threadIdx.x; i4 < total / 4; i4 += PROJ_THREADS) {
                    const int i = 4 * i4, t = i / rowf, k = i - t * rowf;
                    dst4[i4] = make_float4(sSH[(k + 0) * SLAB_LD + t], sSH[(k + 1) * SLAB_LD + t],
                                           sSH[(k + 2) * SLAB_LD + t], sSH[(k + 3) * SLAB_LD + t]);
                }
            } else {
                for (int i = threadIdx.x; i < total; i += PROJ_THREADS) {
                    const int t = i / rowf, k = i - t * rowf;
                    dst[i] = sSH[k * SLAB_LD + t];
                }
            }
        }
    }
    if constexpr (CAM) {
        // the CTA's sum of each term: warp w takes terms w, w + 4, ...; each lane adds rows lane, +32, +64, +96 in that
        // order, then a butterfly over the lanes — a fixed order, so equal gradient rows give equal bits
        __syncthreads();
        const float* col = sSH + (p.shs ? rowf * SLAB_LD : 0);
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        for (int k = warp; k < kCamGradFloats; k += PROJ_THREADS / 32) {
            const float* r = col + k * SLAB_LD;
            float s = ((r[lane] + r[lane + 32]) + r[lane + 64]) + r[lane + 96];
#pragma unroll
            for (int m = 16; m > 0; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
            if (lane == 0) p.cam_work[(size_t)k * gridDim.x + blockIdx.x] = s;
        }
    }
    if (!in_range) return;
#pragma unroll
    for (int k = 0; k < 3; ++k) p.dL_dmeans2D[3 * (size_t)idx + k] = dmean2[k];
    if (p.dL_dsh_factor) {
#pragma unroll
        for (int k = 0; k < 3; ++k) p.dL_dsh_factor[3 * (size_t)idx + k] = dfac[k];
    }
    if (live || !p.acc_colors) {
#pragma unroll
        for (int k = 0; k < 3; ++k) put(p.dL_dcolors + 3 * (size_t)idx + k, dcol[k], p.acc_colors);
    }
    if (!live && p.acc) return;                     // later views: a row that is not live adds nothing
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        put(p.dL_dmeans3D + 3 * (size_t)idx + k, dmean3[k], p.acc);
        put(p.dL_dscales + 3 * (size_t)idx + k, dscale[k], p.acc);
    }
    put(p.dL_dopacity + idx, dop, p.acc);
#pragma unroll
    for (int k = 0; k < 6; ++k) put(p.dL_dcov3D + 6 * (size_t)idx + k, dcov[k], p.acc);
    float4* drot4 = reinterpret_cast<float4*>(p.dL_drotations + 4 * (size_t)idx);
    if (p.acc) {
        const float4 o = *drot4;
        *drot4 = make_float4(o.x + drot[0], o.y + drot[1], o.z + drot[2], o.w + drot[3]);
    } else {
        *drot4 = make_float4(drot[0], drot[1], drot[2], drot[3]);
    }
}

// One CTA per (column k, view v): the sum of the column's nblk partials work[(v * width + k) * nblk + i] in a fixed
// order (each thread adds i = t, t + 256, ... in turn, then a butterfly per warp, then the 8 warps in order), written
// to the output segment column k falls in.
__global__ void __launch_bounds__(256) cam_grad_sum_kernel(const float* __restrict__ work, int nblk, const CamGradOut o) {
    __shared__ float part[8];
    const int k = blockIdx.x, v = blockIdx.y, width = gridDim.x;
    const float* col = work + ((size_t)v * width + k) * nblk;
    float s = 0.f;
    for (int i = threadIdx.x; i < nblk; i += 256) s += col[i];
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = part[0];
#pragma unroll
        for (int w = 1; w < 8; ++w) t += part[w];
        const int k1 = o.n[0], k2 = o.n[0] + o.n[1];
        if (k < k1) o.out[0][(size_t)v * o.n[0] + k] = t;
        else if (k < k2) o.out[1][(size_t)v * o.n[1] + (k - k1)] = t;
        else o.out[2][(size_t)v * o.n[2] + (k - k2)] = t;
    }
}

int launch_cam_grad_sum(const float* work, int nblk, int V, const CamGradOut& o, cudaStream_t stream) {
    const int width = o.n[0] + o.n[1] + o.n[2];
    cam_grad_sum_kernel<<<dim3(width, V), 256, 0, stream>>>(work, nblk, o);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_projection_backward(const r3dg_raster_bwd_args& a, const RasterBuffers& b, int v, cudaStream_t stream) {
    ProjBwdParams p;
    float tan_fovx = a.tan_fovx, tan_fovy = a.tan_fovy, cx = 0.f, cy = 0.f;
    view_cam(b.V, a.view_cams, v, tan_fovx, tan_fovy, cx, cy);
    const size_t r = (size_t)v * a.P;                 // view v's rows of the per-view inputs and outputs
    const bool later = v > 0;
    p.P = a.P; p.S = a.S; p.D = a.D; p.M = a.M; p.W = a.W; p.H = a.H; p.recf = b.recf;
    p.means3D = a.means3D; p.shs = a.shs; p.scales = a.scales;
    p.colors_precomp = a.colors_precomp && a.colors_per_view ? a.colors_precomp + 3 * r : a.colors_precomp;
    p.rotations = a.rotations; p.cov3D_precomp = a.cov3D_precomp; p.viewmatrix = a.viewmatrix + 16 * v;
    p.projmatrix = a.projmatrix + 16 * v; p.campos = a.campos + 3 * v;
    p.scale_modifier = a.scale_modifier; p.tan_fovx = tan_fovx; p.tan_fovy = tan_fovy;
    p.h_y = a.H / (2.0f * tan_fovy); p.h_x = a.W / (2.0f * tan_fovx);
    p.antialiasing = a.antialiasing != 0;
    p.rec = b.rec; p.grad = b.grad; p.clamped = b.clamped;
    p.dL_dmeans2D = a.dL_dmeans2D + 3 * r; p.dL_dopacity = a.dL_dopacity;
    p.dL_dcolors = a.colors_per_view ? a.dL_dcolors + 3 * r : a.dL_dcolors;
    p.dL_dfeatures = a.features_per_view ? a.dL_dfeatures + (size_t)a.S * r : a.dL_dfeatures;
    p.dL_dmeans3D = a.dL_dmeans3D; p.dL_dcov3D = a.dL_dcov3D;
    p.dL_dscales = a.dL_dscales; p.dL_drotations = a.dL_drotations;
    // several views: each writes its rank-1 SH factor, dL_dsh is rebuilt from them afterwards (r3dg_raster_backward)
    p.dL_dsh = b.V > 1 ? nullptr : a.dL_dsh;
    p.dL_dsh_factor = a.dL_dsh_factor ? a.dL_dsh_factor + 3 * r : nullptr;
    p.det = det_acc(a.det_work, (size_t)b.V * a.P * b.recf);
    p.det_row0 = r;
    p.det_scale = a.deterministic ? raster_det_scale(b) + 2 * v : nullptr;
    p.acc = later;
    p.acc_colors = later && !a.colors_per_view;
    p.acc_features = later && !a.features_per_view;
    const size_t sh_smem = a.shs ? (size_t)3 * a.M * SLAB_LD * sizeof(float) : 0;
    const int blocks = (a.P + PROJ_THREADS - 1) / PROJ_THREADS;
    // camera gradients (r3dg_raster_backward checked that all three outputs and the workspace are given): view v's
    // partials follow the earlier views' in the workspace
    const bool cam = a.dL_dviewmatrix != nullptr;
    p.cam_work = cam ? (float*)a.cam_work + (size_t)v * kCamGradFloats * blocks : nullptr;
    const size_t cam_smem = sh_smem + (size_t)kCamGradFloats * SLAB_LD * sizeof(float);
    if (cam && a.deterministic) projection_bwd_kernel<true, true><<<blocks, PROJ_THREADS, cam_smem, stream>>>(p);
    else if (cam) projection_bwd_kernel<false, true><<<blocks, PROJ_THREADS, cam_smem, stream>>>(p);
    else if (a.deterministic) projection_bwd_kernel<true><<<blocks, PROJ_THREADS, sh_smem, stream>>>(p);
    else projection_bwd_kernel<<<blocks, PROJ_THREADS, sh_smem, stream>>>(p);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

// ---- appearance-only backward (r3dg_raster_backward with every geometry output NULL) ---------------------------------
// The compositor (composite_bwd_kernel<GEOM = false>) left one row of nc = 4 * num_groups(S) channel gradients
// {r, g, b, f0, ...} per view and Gaussian.  One thread per Gaussian walks the views in order and writes what
// projection_bwd_kernel writes for the same outputs, with the same arithmetic: per-view rows, or the fp32 left fold over
// the views of shared inputs (a row that is not live adds nothing to the earlier views'); with `shs`, the colour
// gradient gated by the clamp flags becomes the SH factor, or (one view) the dense dL/dsh from the same basis.  Only
// live rows read anything: their packed row, their clamp flags, their mean and the view's campos.
struct AppBwdParams {
    int P, S, D, M, V, nc;
    const float *means3D, *campos;
    const uint8_t* clamped;     // [V][P]: bits 0-2 SH colour clamped, kComposited
    const float* grad;          // [V * P][nc]
    DetAcc det;                 // DET: the same rows as fixed-point accumulators, read instead of grad
    const uint32_t* det_scale;  // DET: per view, the scale word of the rows (composite_bwd.cu; [2 v], colour / feature)
    float *dL_dcolors, *dL_dfeatures, *dL_dsh, *dL_dsh_factor;   // each may be NULL (not requested)
    bool sh, colors_per_view, features_per_view;
};

// The feature rows of the CTA's Gaussians are one contiguous range per view: the CTA writes it element by element
// (coalesced), the rest is one thread per Gaussian.
template <bool DET>
__global__ void __launch_bounds__(128) appearance_bwd_kernel(const AppBwdParams p) {
    auto load = [&](size_t row, int c) -> float {
        if constexpr (DET) return det_load(p.det, row * p.nc + c, det_scale_exp(p.det_scale[2 * (row / p.P)]));
        else return p.grad[row * p.nc + c];
    };
    const int g0 = blockIdx.x * blockDim.x;
    if (p.dL_dfeatures && p.S > 0) {
        const int n = min((int)blockDim.x, p.P - g0) * p.S;
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const int gi = g0 + i / p.S, c = i - (i / p.S) * p.S;
            for (int v = 0; v < p.V; ++v) {
                const size_t r = (size_t)v * p.P + gi;
                const bool live = (p.clamped[r] & kComposited) != 0, acc = v > 0 && !p.features_per_view;
                if (live || !acc) put(p.dL_dfeatures + (p.features_per_view ? r : (size_t)gi) * p.S + c,
                                      live ? load(r, 3 + c) : 0.0f, acc);
            }
        }
    }
    // the colour rows are read only for dL_dcolors, the SH factors or the dense dL/dsh (not in the stage-2 case, where
    // only dL_dfeatures is requested)
    if (!p.dL_dcolors && !(p.sh && (p.dL_dsh_factor || p.dL_dsh))) return;          // (grid-uniform)
    // one view's dense dL/dsh: each thread fills its row of the CTA's slab s[k * SLAB_LD + t] (conflict-free), and the
    // CTA writes the slab's contiguous range of dL_dsh with coalesced stores, as projection_bwd_kernel's write-back
    extern __shared__ float sOut[];
    const int g = g0 + threadIdx.x, rowf = 3 * p.M;
    float m3[3] = {0.f, 0.f, 0.f};
    bool have_m3 = false;
    for (int v = 0; g < p.P && v < p.V; ++v) {
        const size_t r = (size_t)v * p.P + g;
        const unsigned cl = p.clamped[r];
        const bool live = (cl & kComposited) != 0;
        float dcol[3] = {0.f, 0.f, 0.f};
        if (live) {
#pragma unroll
            for (int k = 0; k < 3; ++k) dcol[k] = load(r, k);
        }
        if (p.dL_dcolors) {
            const bool acc = v > 0 && !p.colors_per_view;
            if (live || !acc) {
                float* dc = p.dL_dcolors + 3 * (p.colors_per_view ? r : (size_t)g);
#pragma unroll
                for (int k = 0; k < 3; ++k) put(dc + k, dcol[k], acc);
            }
        }
        if (!p.sh) continue;
        const float dRGB[3] = {(cl & 1u) ? 0.f : dcol[0], (cl & 2u) ? 0.f : dcol[1], (cl & 4u) ? 0.f : dcol[2]};
        if (p.dL_dsh_factor) {
#pragma unroll
            for (int k = 0; k < 3; ++k) p.dL_dsh_factor[3 * r + k] = live ? dRGB[k] : 0.f;
        }
        if (!p.dL_dsh) continue;                       // (one view only: several views rebuild it from the factors)
        float w[16], wx[16], wy[16], wz[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) w[k] = 0.f;
        if (live) {
            if (!have_m3) {
                m3[0] = p.means3D[3 * (size_t)g]; m3[1] = p.means3D[3 * (size_t)g + 1]; m3[2] = p.means3D[3 * (size_t)g + 2];
                have_m3 = true;
            }
            const ViewDir vd = view_dir(m3, p.campos + 3 * v);
            sh_basis(p.D, vd.x, vd.y, vd.z, w, wx, wy, wz);
        }
        const int ncoef = (p.D + 1) * (p.D + 1);
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            if (k < p.M) {
                const bool act = live && k < ncoef;
#pragma unroll
                for (int c = 0; c < 3; ++c) sOut[(3 * k + c) * SLAB_LD + threadIdx.x] = act ? w[k] * dRGB[c] : 0.f;
            }
        }
    }
    if (!p.dL_dsh || !p.sh) return;                     // (grid-uniform)
    __syncthreads();
    const int total = min((int)blockDim.x, p.P - g0) * rowf;
    float* dst = p.dL_dsh + (size_t)g0 * rowf;
    if ((rowf & 3) == 0 && (reinterpret_cast<uintptr_t>(p.dL_dsh) & 15) == 0) {
        float4* dst4 = reinterpret_cast<float4*>(dst);
        for (int i4 = threadIdx.x; i4 < total / 4; i4 += blockDim.x) {
            const int i = 4 * i4, t = i / rowf, k = i - t * rowf;
            dst4[i4] = make_float4(sOut[(k + 0) * SLAB_LD + t], sOut[(k + 1) * SLAB_LD + t], sOut[(k + 2) * SLAB_LD + t],
                                   sOut[(k + 3) * SLAB_LD + t]);
        }
    } else {
        for (int i = threadIdx.x; i < total; i += blockDim.x) {
            const int t = i / rowf, k = i - t * rowf;
            dst[i] = sOut[k * SLAB_LD + t];
        }
    }
}

int launch_appearance_backward(const r3dg_raster_bwd_args& a, const RasterBuffers& b, cudaStream_t stream) {
    AppBwdParams p;
    p.P = a.P; p.S = a.S; p.D = a.D; p.M = a.M; p.V = b.V; p.nc = composite_bwd_row_floats(a.S, false);
    p.means3D = a.means3D; p.campos = a.campos;
    p.clamped = b.clamped; p.grad = b.grad;
    p.det = det_acc(a.det_work, (size_t)b.V * a.P * p.nc);
    p.det_scale = a.deterministic ? raster_det_scale(b) : nullptr;
    p.dL_dcolors = a.dL_dcolors; p.dL_dfeatures = a.dL_dfeatures;
    p.dL_dsh = b.V > 1 ? nullptr : a.dL_dsh;       // several views: from the factors afterwards (r3dg_raster_backward)
    p.dL_dsh_factor = a.dL_dsh_factor;
    p.sh = a.shs != nullptr;
    p.colors_per_view = a.colors_per_view != 0; p.features_per_view = a.features_per_view != 0;
    static_assert(PROJ_THREADS == 128, "the dL/dsh slab holds one CTA of 128 rows");
    const int blocks = (a.P + 127) / 128;
    const size_t smem = p.sh && p.dL_dsh ? (size_t)3 * a.M * SLAB_LD * sizeof(float) : 0;
    if (a.deterministic) appearance_bwd_kernel<true><<<blocks, 128, smem, stream>>>(p);
    else appearance_bwd_kernel<false><<<blocks, 128, smem, stream>>>(p);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace r3dg
