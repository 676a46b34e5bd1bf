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
    const int* radii_rec;       // unused (radius is read from the record)
    const float* rec;
    const float* grad;
    const uint8_t* clamped;
    float *dL_dmeans2D, *dL_dcolors, *dL_dopacity, *dL_dmeans3D, *dL_dfeatures, *dL_dcov3D, *dL_dsh,
        *dL_dscales, *dL_drotations;
    float* dL_dsh_factor;       // [P,3] gated dL_dRGB (multi-GPU exchange, sh_exchange.cu); dL_dsh may then be NULL
    DetAcc det;                 // DET: the gradient rows as fixed-point accumulators (composite_bwd.cu), read instead of grad
};

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

#define PROJ_THREADS 128
#define SLAB_LD (PROJ_THREADS + 1)
// DET (deterministic mode): the packed gradient row is read from the fixed-point accumulators and converted on load.
template <bool DET = false>
__global__ void __launch_bounds__(PROJ_THREADS, 5) projection_bwd_kernel(const ProjBwdParams p) {
    // SH rows (192 B at M=16) travel through shared memory: the CTA's [128][3M] slab of shs is ONE contiguous
    // 24 KB block, fetched by a single TMA-unit bulk copy (cp.async.bulk, mbarrier-signalled) into a row-major
    // slab; every thread turns its row into dL/dsh in place (16-byte vector accesses) and ONE bulk store writes the
    // slab back (zeros for culled rows).  Rows that are not 16-byte multiples (SH degree 0 / 2) or ragged / unaligned
    // tails use the transposed slab s[k * SLAB_LD + t] with 4-byte LDGSTS copies and a coalesced write-back loop.
    extern __shared__ __align__(16) float sSH[];
    __shared__ float sV[16], sPr[16], sCam[3];
    __shared__ __align__(8) uint64_t sBar;
    const int rowf_ = 3 * p.M, base_ = blockIdx.x * PROJ_THREADS;
    const unsigned slab_bytes = (unsigned)min(PROJ_THREADS, p.P - base_) * (unsigned)rowf_ * 4u;
    const bool bulk = p.shs && (rowf_ & 3) == 0 && (slab_bytes & 15u) == 0 &&
                      (reinterpret_cast<uintptr_t>(p.shs + (size_t)base_ * rowf_) & 15) == 0 &&
                      (!p.dL_dsh || (reinterpret_cast<uintptr_t>(p.dL_dsh + (size_t)base_ * rowf_) & 15) == 0);
    if (threadIdx.x == 0 && bulk) { mbar_init(&sBar, 1); fence_proxy_async_smem(); }
    if (threadIdx.x < 16) { sV[threadIdx.x] = p.viewmatrix[threadIdx.x]; sPr[threadIdx.x] = p.projmatrix[threadIdx.x]; }
    if (threadIdx.x < 3) sCam[threadIdx.x] = p.campos[threadIdx.x];
    __syncthreads();
    const int idx_raw = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in_range = idx_raw < p.P;
    const int idx = in_range ? idx_raw : p.P - 1;      // clamp: out-of-range threads only help with the slab
    const int rowf = 3 * p.M, block_base = blockIdx.x * PROJ_THREADS;
    const int nvalid = min(PROJ_THREADS, p.P - block_base);
    // the thread's own rows are requested before the cooperative slab load so that both are in flight
    // together (nothing can be hoisted across the barrier below by the compiler)
    const float4* g4 = reinterpret_cast<const float4*>(p.grad + (size_t)idx * p.recf);
    const bool visible = in_range && p.radii_rec[idx] > 0;
    float4 gA = make_float4(0, 0, 0, 0), gB = gA, gC = gA, q4 = gA;
    float m3[3] = {0, 0, 0}, s3[3] = {0, 0, 0};
    unsigned cl = 0;
    if (visible) {
        if constexpr (DET) {
            const size_t r0 = (size_t)idx * p.recf;
            gA = make_float4(det_load(p.det, r0), det_load(p.det, r0 + 1), det_load(p.det, r0 + 2), det_load(p.det, r0 + 3));
            gB = make_float4(det_load(p.det, r0 + 4), det_load(p.det, r0 + 5), det_load(p.det, r0 + 6), 0.0f);
            gC = make_float4(det_load(p.det, r0 + 8), det_load(p.det, r0 + 9), det_load(p.det, r0 + 10), 0.0f);
        } else {
            gA = g4[0]; gB = g4[1]; gC = g4[2];
        }
        m3[0] = p.means3D[3 * (size_t)idx]; m3[1] = p.means3D[3 * (size_t)idx + 1]; m3[2] = p.means3D[3 * (size_t)idx + 2];
        if (!p.cov3D_precomp) {
            q4 = *reinterpret_cast<const float4*>(p.rotations + 4 * (size_t)idx);
            s3[0] = p.scales[3 * (size_t)idx]; s3[1] = p.scales[3 * (size_t)idx + 1]; s3[2] = p.scales[3 * (size_t)idx + 2];
        }
        if (p.shs) cl = p.clamped[idx];
    }
    if (p.shs) {     // asynchronous copy of the slab, overlapped with the covariance chain below
        if (bulk) {
            if (threadIdx.x == 0) { mbar_arrive_expect_tx(&sBar, slab_bytes); bulk_copy_g2s(sSH, p.shs + (size_t)block_base * rowf, slab_bytes, &sBar); }
        } else {
            load_rows_transposed_async(sSH, SLAB_LD, p.shs + (size_t)block_base * rowf, nvalid, rowf, PROJ_THREADS);
            cp_async_commit();
        }
    }
    const float* V = sV;
    const float* proj = sPr;
    // (visibility comes from tiles_touched: the record row of a culled Gaussian is never written)

    float dmean2[3] = {0, 0, 0}, dcol[3] = {0, 0, 0}, dop = 0, dmean3[3] = {0, 0, 0}, dfac[3] = {0, 0, 0};
    float dcov[6] = {0, 0, 0, 0, 0, 0}, dscale[3] = {0, 0, 0}, drot[4] = {0, 0, 0, 0};

    // feature gradients: straight copy-out of the packed row
    if (p.S > 0 && in_range) {
        float* df = p.dL_dfeatures + (size_t)idx * p.S;
        for (int c = 0; c < p.S; ++c) {
            if constexpr (DET) df[c] = visible ? det_load(p.det, (size_t)idx * p.recf + 11 + c) : 0.0f;
            else df[c] = visible ? p.grad[(size_t)idx * p.recf + 11 + c] : 0.0f;
        }
    }
    if (visible) {
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
        const float a = (T0[0] * VT0[0] + T0[1] * VT0[1] + T0[2] * VT0[2]) + 0.3f;
        const float b = T1[0] * VT0[0] + T1[1] * VT0[1] + T1[2] * VT0[2];
        const float c = (T1[0] * VT1[0] + T1[1] * VT1[1] + T1[2] * VT1[2]) + 0.3f;
        const float denom = a * c - b * b;
        float dL_da = 0, dL_db = 0, dL_dc = 0;
        const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
        if (denom2inv != 0) {
            dL_da = denom2inv * (-c * c * dcx + 2 * b * c * dcy + (denom - a * c) * dcz);
            dL_dc = denom2inv * (-a * a * dcz + 2 * a * b * dcy + (denom - a * c) * dcx);
            dL_db = denom2inv * 2 * (b * c * dcx - (denom + 2 * b * b) * dcy + a * b * dcz);
            dcov[0] = (T0[0] * T0[0] * dL_da + T0[0] * T1[0] * dL_db + T1[0] * T1[0] * dL_dc);
            dcov[3] = (T0[1] * T0[1] * dL_da + T0[1] * T1[1] * dL_db + T1[1] * T1[1] * dL_dc);
            dcov[5] = (T0[2] * T0[2] * dL_da + T0[2] * T1[2] * dL_db + T1[2] * T1[2] * dL_dc);
            dcov[1] = 2 * T0[0] * T0[1] * dL_da + (T0[0] * T1[1] + T0[1] * T1[0]) * dL_db + 2 * T1[0] * T1[1] * dL_dc;
            dcov[2] = 2 * T0[0] * T0[2] * dL_da + (T0[0] * T1[2] + T0[2] * T1[0]) * dL_db + 2 * T1[0] * T1[2] * dL_dc;
            dcov[4] = 2 * T0[2] * T0[1] * dL_da + (T0[1] * T1[2] + T0[2] * T1[1]) * dL_db + 2 * T1[1] * T1[2] * dL_dc;
        }
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
    if (p.shs) {
        if (bulk) mbar_wait(&sBar, 0);
        else { cp_async_wait_all(); __syncthreads(); }
    }
    if (visible) {
        // ---- SH backward (backward.cu:20-139) -------------------------------------------------
        if (p.shs) {
            const float dox = m3[0] - sCam[0], doy = m3[1] - sCam[1], doz = m3[2] - sCam[2];
            const float len = sqrtf(dox * dox + doy * doy + doz * doz);
            const float x = dox / len, y = doy / len, z = doz / len;
            float* slab = sSH + threadIdx.x;                 // element (k, c) at slab[(3k + c) * SLAB_LD]
            const float dRGB[3] = {(cl & 1u) ? 0.f : dcol[0], (cl & 2u) ? 0.f : dcol[1], (cl & 4u) ? 0.f : dcol[2]};
            dfac[0] = dRGB[0]; dfac[1] = dRGB[1]; dfac[2] = dRGB[2];
            float w[16], wx[16], wy[16], wz[16];   // basis and its derivatives w.r.t. x,y,z
#pragma unroll
            for (int k = 0; k < 16; ++k) { w[k] = 0.f; wx[k] = 0.f; wy[k] = 0.f; wz[k] = 0.f; }
            const float C1 = 0.4886025119029199f;
            w[0] = 0.28209479177387814f;
            if (p.D > 0) {
                w[1] = -C1 * y; w[2] = C1 * z; w[3] = -C1 * x;
                wy[1] = -C1; wz[2] = C1; wx[3] = -C1;
                if (p.D > 1) {
                    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                    const float c20 = 1.0925484305920792f, c21 = -1.0925484305920792f, c22 = 0.31539156525252005f,
                                c23 = -1.0925484305920792f, c24 = 0.5462742152960396f;
                    w[4] = c20 * xy; w[5] = c21 * yz; w[6] = c22 * (2.f * zz - xx - yy); w[7] = c23 * xz; w[8] = c24 * (xx - yy);
                    wx[4] = c20 * y;  wy[4] = c20 * x;
                    wy[5] = c21 * z;  wz[5] = c21 * y;
                    wx[6] = c22 * 2.f * -x; wy[6] = c22 * 2.f * -y; wz[6] = c22 * 2.f * 2.f * z;
                    wx[7] = c23 * z;  wz[7] = c23 * x;
                    wx[8] = c24 * 2.f * x; wy[8] = c24 * 2.f * -y;
                    if (p.D > 2) {
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
            const float sum2 = dox * dox + doy * doy + doz * doz;
            const float invsum32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
            dmean3[0] += ((+sum2 - dox * dox) * ddx - doy * dox * ddy - doz * dox * ddz) * invsum32;
            dmean3[1] += (-dox * doy * ddx + (sum2 - doy * doy) * ddy - doz * doy * ddz) * invsum32;
            dmean3[2] += (-dox * doz * ddx - doy * doz * ddy + (sum2 - doz * doz) * ddz) * invsum32;
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
    if (!in_range) return;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        p.dL_dmeans2D[3 * (size_t)idx + k] = dmean2[k];
        p.dL_dcolors[3 * (size_t)idx + k] = dcol[k];
        p.dL_dmeans3D[3 * (size_t)idx + k] = dmean3[k];
        p.dL_dscales[3 * (size_t)idx + k] = dscale[k];
    }
    p.dL_dopacity[idx] = dop;
    if (p.dL_dsh_factor) {
#pragma unroll
        for (int k = 0; k < 3; ++k) p.dL_dsh_factor[3 * (size_t)idx + k] = dfac[k];
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) p.dL_dcov3D[6 * (size_t)idx + k] = dcov[k];
    *reinterpret_cast<float4*>(p.dL_drotations + 4 * (size_t)idx) = make_float4(drot[0], drot[1], drot[2], drot[3]);
}

int launch_projection_backward(const r3dg_raster_bwd_args& a, const GeomLayout& gl, cudaStream_t stream) {
    char* geom = (char*)a.geom;
    ProjBwdParams p;
    p.P = a.P; p.S = a.S; p.D = a.D; p.M = a.M; p.W = a.W; p.H = a.H; p.recf = gl.recf;
    p.means3D = a.means3D; p.shs = a.shs; p.colors_precomp = a.colors_precomp; p.scales = a.scales;
    p.rotations = a.rotations; p.cov3D_precomp = a.cov3D_precomp; p.viewmatrix = a.viewmatrix;
    p.projmatrix = a.projmatrix; p.campos = a.campos;
    p.scale_modifier = a.scale_modifier; p.tan_fovx = a.tan_fovx; p.tan_fovy = a.tan_fovy;
    p.h_y = a.H / (2.0f * a.tan_fovy); p.h_x = a.W / (2.0f * a.tan_fovx);
    p.radii_rec = (const int*)(geom + gl.tiles_touched);   // tiles_touched > 0  <=>  radii > 0
    p.rec = (const float*)(geom + gl.rec);
    p.grad = (const float*)(geom + gl.grad);
    p.clamped = (const uint8_t*)(geom + gl.clamped);
    p.dL_dmeans2D = a.dL_dmeans2D; p.dL_dcolors = a.dL_dcolors; p.dL_dopacity = a.dL_dopacity;
    p.dL_dmeans3D = a.dL_dmeans3D; p.dL_dfeatures = a.dL_dfeatures; p.dL_dcov3D = a.dL_dcov3D;
    p.dL_dsh = a.dL_dsh; p.dL_dscales = a.dL_dscales; p.dL_drotations = a.dL_drotations;
    p.dL_dsh_factor = a.dL_dsh_factor;
    p.det = det_acc(a.det_work, (size_t)a.P * gl.recf);
    const size_t sh_smem = a.shs ? (size_t)3 * a.M * SLAB_LD * sizeof(float) : 0;
    const int blocks = (a.P + PROJ_THREADS - 1) / PROJ_THREADS;
    if (a.deterministic) projection_bwd_kernel<true><<<blocks, PROJ_THREADS, sh_smem, stream>>>(p);
    else projection_bwd_kernel<<<blocks, PROJ_THREADS, sh_smem, stream>>>(p);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace r3dg
