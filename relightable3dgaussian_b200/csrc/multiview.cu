// Multi-view consistency losses of PGSR (Chen et al., 2024): a geometric term (reproject each pixel's depth into a
// neighbouring view and back, penalise the pixel error) and a photometric term (warp a 7x7 grey patch with the
// homography of the pixel's plane, penalise 1 - NCC against the neighbour's grey image), for B (reference, neighbour)
// pairs of rendered views.  The semantics are stated in include/r3dg_b200.h (r3dg_multiview_*) and multiview.py.
//   forward : ONE kernel (a CTA owns a 16x16 pixel tile of one pair, stages the reference grey tile with a 3-pixel
//             halo, one thread per pixel evaluates both terms and the CTA writes fp64 (sum, count) partials) + ONE
//             fixed-order reduction that writes the per-pair losses and counts on the device;
//   backward: ONE kernel that recomputes the forward per pixel (nothing per tap is saved) and adds dL/ddepth and
//             dL/dnormal at the pixel and dL/ddepth of the neighbour at the four bilinear taps of the reprojected
//             pixel: float atomics into zeroed outputs by default; in deterministic mode a first launch of the same
//             kernel that only measures the largest |term| of each gradient, then fixed-point accumulators
//             (detacc.cuh) and ONE pass that reads them back, so repeated references and shared neighbours sum in an
//             order-independent way.
// Arithmetic is IEEE fp32: divisions and square roots are the correctly rounded forms (no fast-math intrinsics);
// nvcc contracts multiply-adds into FMAs.  exp(-phi) is expf (max 2 ulp).
#include "common.cuh"
#include "detacc.cuh"
#include "kernels.h"
#include "reduce.cuh"

namespace r3dg {
namespace {

constexpr int TS = 16;                 // pixel tile edge; one thread per pixel
constexpr int NT = TS * TS;
constexpr int HALO = 3;                // 7x7 patch
constexpr int ST = TS + 2 * HALO;      // staged grey tile edge
constexpr float kMinZ = 1e-6f;         // Y.z, X'.z, |d| and h.z thresholds
constexpr float kNormEps = 1e-12f;     // F.normalize's eps
constexpr float kNccEps = 1e-8f;
constexpr float kMaxCost = 0.9f;       // photo-valid: 1 - NCC below this

struct MvPair {
    int r, n;
    float fxr, fyr, cxr, cyr, fxn, fyn, cxn, cyn;
};
struct MvParams {
    int B, V, H, W;
    float tau;
    MvPair pair[R3DG_MAX_VIEWS];
};

// the pair's ref -> neighbour rigid transform (R, t) and the reference view's world -> camera rotation Rr, from the
// row-vector view matrices (cam_j = sum_i world_i V[i][j] + V[3][j])
struct MvCam {
    float R[9], t[3], Rr[9];
};

__device__ __forceinline__ void make_cam(const float* __restrict__ vr, const float* __restrict__ vn, MvCam& c) {
    float Rn[9], tr[3], tn[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            c.Rr[j * 3 + i] = vr[i * 4 + j];
            Rn[j * 3 + i] = vn[i * 4 + j];
        }
        tr[i] = vr[12 + i];
        tn[i] = vn[12 + i];
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int k = 0; k < 3; ++k)
            c.R[i * 3 + k] = Rn[i * 3 + 0] * c.Rr[k * 3 + 0] + Rn[i * 3 + 1] * c.Rr[k * 3 + 1] + Rn[i * 3 + 2] * c.Rr[k * 3 + 2];
    }
#pragma unroll
    for (int i = 0; i < 3; ++i)
        c.t[i] = tn[i] - (c.R[i * 3 + 0] * tr[0] + c.R[i * 3 + 1] * tr[1] + c.R[i * 3 + 2] * tr[2]);
}

// Bilinear sample of plane p [H,W] at pixel coordinates (u, v), align-corners, zero padding (grid_sample), and its
// derivatives in u and v.  Outside [-1, W) x [-1, H) every tap is outside the image: 0 with zero derivatives.
__device__ __forceinline__ float bilinear(const float* __restrict__ p, int H, int W, float u, float v, float& du,
                                          float& dv, float* wt = nullptr, int* idx = nullptr) {
    if (!(u >= -1.f && u < (float)W && v >= -1.f && v < (float)H)) {
        du = dv = 0.f;
        if (wt) { wt[0] = wt[1] = wt[2] = wt[3] = 0.f; }
        return 0.f;
    }
    const float fx0 = floorf(u), fy0 = floorf(v);
    const int x0 = (int)fx0, y0 = (int)fy0;
    const float ax = u - fx0, ay = v - fy0, bx = 1.f - ax, by = 1.f - ay;
    const bool inx0 = x0 >= 0, inx1 = x0 + 1 < W, iny0 = y0 >= 0, iny1 = y0 + 1 < H;
    const size_t row0 = (size_t)y0 * W, row1 = row0 + W;
    const float v00 = (inx0 && iny0) ? __ldg(p + row0 + x0) : 0.f;
    const float v10 = (inx1 && iny0) ? __ldg(p + row0 + x0 + 1) : 0.f;
    const float v01 = (inx0 && iny1) ? __ldg(p + row1 + x0) : 0.f;
    const float v11 = (inx1 && iny1) ? __ldg(p + row1 + x0 + 1) : 0.f;
    du = by * (v10 - v00) + ay * (v11 - v01);
    dv = bx * (v01 - v00) + ax * (v11 - v10);
    const float w00 = bx * by, w10 = ax * by, w01 = bx * ay, w11 = ax * ay;
    if (wt) {
        wt[0] = (inx0 && iny0) ? w00 : 0.f; wt[1] = (inx1 && iny0) ? w10 : 0.f;
        wt[2] = (inx0 && iny1) ? w01 : 0.f; wt[3] = (inx1 && iny1) ? w11 : 0.f;
        idx[0] = y0 * W + x0;
    }
    return w00 * v00 + w10 * v10 + w01 * v01 + w11 * v11;
}

// Gradient sink of the backward: float atomics into zeroed outputs, or fixed-point accumulators (deterministic mode),
// or (measure) the largest |term| of each class in this thread, to size the accumulators' exponents.
// Accumulator layout: depth [V][H*W], then normal [V][3][H*W].
struct Sink {
    float* dd;           // dL_ddepth  [V,H,W]
    float* dn;           // dL_dnormal [V,3,H,W]
    DetAcc acc;
    int ed, en;          // fixed-point exponents of the depth and the normal class
    bool det, measure;
    size_t VHW;
    uint32_t md, mn;     // measure: the thread's largest |term| (float bits) of each class
    __device__ __forceinline__ void depth(size_t i, float x) {
        if (measure) md = max(md, det_abs_bits(x));
        else if (det) det_add(acc, i, x, ed);
        else atomicAdd(dd + i, x);
    }
    __device__ __forceinline__ void normal(size_t i, float x) {
        if (measure) mn = max(mn, det_abs_bits(x));
        else if (det) det_add(acc, VHW + i, x, en);
        else atomicAdd(dn + i, x);
    }
};

// One pixel (x, y) of pair b, both terms.  Forward: acc[0..3] += (w phi, 1) if geo-valid, (w c, 1) if photo-valid.
// Backward (BWD): the pixel's gradient, scaled by sg = dL/dgeo / max(count, 1) and sp likewise, into `sink`.
template <bool BWD>
__device__ __forceinline__ void mv_pixel(const MvParams& prm, const MvPair& pr, const MvCam& cam, int x, int y,
                                         const float* __restrict__ depth, const float* __restrict__ normal,
                                         const float* __restrict__ gray, const float* sgray, int lx, int ly,
                                         double* acc, float sg, float sp, Sink& sink) {
    const int H = prm.H, W = prm.W;
    const size_t HW = (size_t)H * W, o = (size_t)y * W + x;
    const float* dr = depth + (size_t)pr.r * HW;
    const float* dnb = depth + (size_t)pr.n * HW;
    const float D = __ldg(dr + o);
    if (!(D > 0.f)) return;
    const float* R = cam.R;
    const float* t = cam.t;
    const float ux = ((float)x - pr.cxr) / pr.fxr, uy = ((float)y - pr.cyr) / pr.fyr;
    const float X0 = D * ux, X1 = D * uy, X2 = D;
    const float Y0 = R[0] * X0 + R[1] * X1 + R[2] * X2 + t[0];
    const float Y1 = R[3] * X0 + R[4] * X1 + R[5] * X2 + t[1];
    const float Y2 = R[6] * X0 + R[7] * X1 + R[8] * X2 + t[2];
    if (!(Y2 > kMinZ)) return;
    const float qx = pr.fxn * (Y0 / Y2) + pr.cxn, qy = pr.fyn * (Y1 / Y2) + pr.cyn;
    if (!(qx >= 0.f && qx <= (float)(W - 1) && qy >= 0.f && qy <= (float)(H - 1))) return;
    float dDq_x, dDq_y, wt[4];
    int i00;
    const float Dn = bilinear(dnb, H, W, qx, qy, dDq_x, dDq_y, wt, &i00);
    if (!(Dn > 0.f)) return;
    const float unx = (qx - pr.cxn) / pr.fxn, uny = (qy - pr.cyn) / pr.fyn;
    const float Z0 = Dn * unx - t[0], Z1 = Dn * uny - t[1], Z2 = Dn - t[2];
    const float P0 = R[0] * Z0 + R[3] * Z1 + R[6] * Z2;
    const float P1 = R[1] * Z0 + R[4] * Z1 + R[7] * Z2;
    const float P2 = R[2] * Z0 + R[5] * Z1 + R[8] * Z2;
    if (!(P2 > kMinZ)) return;
    const float ex = (pr.fxr * (P0 / P2) + pr.cxr) - (float)x, ey = (pr.fyr * (P1 / P2) + pr.cyr) - (float)y;
    const float phi = sqrtf(ex * ex + ey * ey);
    if (!(phi < prm.tau)) return;
    const float w = expf(-phi);
    if (!BWD) { acc[0] += (double)(w * phi); acc[1] += 1.0; }

    // ---- photometric term: the homography of the pixel's plane in the reference camera
    const float* Rr = cam.Rr;
    const float nw0 = __ldg(normal + (size_t)pr.r * 3 * HW + o), nw1 = __ldg(normal + ((size_t)pr.r * 3 + 1) * HW + o),
                nw2 = __ldg(normal + ((size_t)pr.r * 3 + 2) * HW + o);
    const float v0 = Rr[0] * nw0 + Rr[1] * nw1 + Rr[2] * nw2;
    const float v1 = Rr[3] * nw0 + Rr[4] * nw1 + Rr[5] * nw2;
    const float v2 = Rr[6] * nw0 + Rr[7] * nw1 + Rr[8] * nw2;
    const float len = sqrtf(v0 * v0 + v1 * v1 + v2 * v2), den_n = fmaxf(len, kNormEps);
    const float nc0 = v0 / den_n, nc1 = v1 / den_n, nc2 = v2 / den_n;
    const float d = nc0 * X0 + nc1 * X1 + nc2 * X2;
    bool photo = fabsf(d) > kMinZ;
    float Hm[9], m[3] = {0.f, 0.f, 0.f};
    float Sa = 0.f, Sb = 0.f, Saa = 0.f, Sbb = 0.f, Sab = 0.f;
    if (photo) {
        m[0] = nc0 / d; m[1] = nc1 / d; m[2] = nc2 / d;
        float A[9];                                       // A = (R + t m^T) K_r^-1
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const float M0 = R[i * 3 + 0] + t[i] * m[0], M1 = R[i * 3 + 1] + t[i] * m[1], M2 = R[i * 3 + 2] + t[i] * m[2];
            A[i * 3 + 0] = M0 / pr.fxr;
            A[i * 3 + 1] = M1 / pr.fyr;
            A[i * 3 + 2] = M2 - A[i * 3 + 0] * pr.cxr - A[i * 3 + 1] * pr.cyr;
        }
#pragma unroll
        for (int j = 0; j < 3; ++j) {                     // H = K_n A
            Hm[0 * 3 + j] = pr.fxn * A[0 * 3 + j] + pr.cxn * A[2 * 3 + j];
            Hm[1 * 3 + j] = pr.fyn * A[1 * 3 + j] + pr.cyn * A[2 * 3 + j];
            Hm[2 * 3 + j] = A[2 * 3 + j];
        }
        const float* gnb = gray + (size_t)pr.n * HW;
#pragma unroll 7
        for (int k = 0; k < 49; ++k) {
            const int ky = k / 7 - HALO, kx = k % 7 - HALO;
            const float px = (float)(x + kx), py = (float)(y + ky);
            const float hz = Hm[6] * px + Hm[7] * py + Hm[8];
            if (!(hz > kMinZ)) { photo = false; break; }
            const float hx = Hm[0] * px + Hm[1] * py + Hm[2], hy = Hm[3] * px + Hm[4] * py + Hm[5];
            float du, dv;
            const float b = bilinear(gnb, H, W, hx / hz, hy / hz, du, dv);
            const float a = sgray[(ly + HALO + ky) * ST + lx + HALO + kx];
            Sa += a; Sb += b; Saa += a * a; Sbb += b * b; Sab += a * b;
        }
    }
    float ma = 0.f, mb = 0.f, cov = 0.f, va = 0.f, den = 1.f, ncc = 0.f;
    if (photo) {
        ma = Sa / 49.f; mb = Sb / 49.f;
        cov = Sab / 49.f - ma * mb;
        va = Saa / 49.f - ma * ma;
        const float vb = Sbb / 49.f - mb * mb;
        den = sqrtf(va * vb + kNccEps);
        ncc = cov / den;
        const float c = fminf(fmaxf(1.f - ncc, 0.f), 2.f);
        photo = c < kMaxCost;
        if (!BWD && photo) { acc[2] += (double)(w * c); acc[3] += 1.0; }
    }
    if (!BWD) return;

    // ---- backward: geometric chain p' <- X' <- (D', q) <- Y <- X <- D, and D' -> the neighbour's taps
    float gX0 = 0.f, gX1 = 0.f, gX2 = 0.f;
    {
        const float gs = sg * w;
        const float gex = phi > 0.f ? gs * ex / phi : 0.f, gey = phi > 0.f ? gs * ey / phi : 0.f;
        const float gP0 = gex * pr.fxr / P2, gP1 = gey * pr.fyr / P2;
        const float gP2 = -(gP0 * P0 + gP1 * P1) / P2;
        const float gZ0 = R[0] * gP0 + R[1] * gP1 + R[2] * gP2;
        const float gZ1 = R[3] * gP0 + R[4] * gP1 + R[5] * gP2;
        const float gZ2 = R[6] * gP0 + R[7] * gP1 + R[8] * gP2;
        const float gDn = gZ0 * unx + gZ1 * uny + gZ2;
        const float gqx = Dn * gZ0 / pr.fxn + gDn * dDq_x, gqy = Dn * gZ1 / pr.fyn + gDn * dDq_y;
        if (gDn != 0.f) {
            const size_t base = (size_t)pr.n * HW + i00;
            if (wt[0] != 0.f) sink.depth(base, gDn * wt[0]);
            if (wt[1] != 0.f) sink.depth(base + 1, gDn * wt[1]);
            if (wt[2] != 0.f) sink.depth(base + W, gDn * wt[2]);
            if (wt[3] != 0.f) sink.depth(base + W + 1, gDn * wt[3]);
        }
        const float gY0 = gqx * pr.fxn / Y2, gY1 = gqy * pr.fyn / Y2;
        const float gY2 = -(gY0 * Y0 + gY1 * Y1) / Y2;
        gX0 = R[0] * gY0 + R[3] * gY1 + R[6] * gY2;
        gX1 = R[1] * gY0 + R[4] * gY1 + R[7] * gY2;
        gX2 = R[2] * gY0 + R[5] * gY1 + R[8] * gY2;
    }

    // ---- photometric chain: b_k <- h_k <- H <- (n_c, d) <- (normal, X); zero in the clamp's flat region
    if (photo && 1.f - ncc >= 0.f) {
        const float gncc = -(sp * w);
        const float cA = gncc / (49.f * den), cB = -gncc * cov * va / (49.f * den * den * den);
        float gH[9];
#pragma unroll
        for (int i = 0; i < 9; ++i) gH[i] = 0.f;
        const float* gnb = gray + (size_t)pr.n * HW;
#pragma unroll 7
        for (int k = 0; k < 49; ++k) {
            const int ky = k / 7 - HALO, kx = k % 7 - HALO;
            const float px = (float)(x + kx), py = (float)(y + ky);
            const float hz = Hm[6] * px + Hm[7] * py + Hm[8];
            const float hx = Hm[0] * px + Hm[1] * py + Hm[2], hy = Hm[3] * px + Hm[4] * py + Hm[5];
            const float u = hx / hz, v = hy / hz;
            float du, dv;
            const float b = bilinear(gnb, H, W, u, v, du, dv);
            const float a = sgray[(ly + HALO + ky) * ST + lx + HALO + kx];
            const float gb = cA * (a - ma) + cB * (b - mb);
            const float gu = gb * du, gv = gb * dv;
            const float ghx = gu / hz, ghy = gv / hz, ghz = -(gu * u + gv * v) / hz;
            gH[0] += ghx * px; gH[1] += ghx * py; gH[2] += ghx;
            gH[3] += ghy * px; gH[4] += ghy * py; gH[5] += ghy;
            gH[6] += ghz * px; gH[7] += ghz * py; gH[8] += ghz;
        }
        // H = K_n A: dL/dA = K_n^T dL/dH; A = M K_r^-1: dL/dM; M = R + t m^T: dL/dm_j = sum_i dL/dM[i][j] t_i
        float gA[9];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            gA[0 * 3 + j] = pr.fxn * gH[0 * 3 + j];
            gA[1 * 3 + j] = pr.fyn * gH[1 * 3 + j];
            gA[2 * 3 + j] = pr.cxn * gH[0 * 3 + j] + pr.cyn * gH[1 * 3 + j] + gH[2 * 3 + j];
        }
        float gm0 = 0.f, gm1 = 0.f, gm2 = 0.f;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const float gM0 = (gA[i * 3 + 0] - gA[i * 3 + 2] * pr.cxr) / pr.fxr;
            const float gM1 = (gA[i * 3 + 1] - gA[i * 3 + 2] * pr.cyr) / pr.fyr;
            const float gM2 = gA[i * 3 + 2];
            gm0 += gM0 * t[i]; gm1 += gM1 * t[i]; gm2 += gM2 * t[i];
        }
        // m = n_c / d, d = n_c . X
        const float gd = -(gm0 * m[0] + gm1 * m[1] + gm2 * m[2]) / d;
        const float gn0 = gm0 / d + gd * X0, gn1 = gm1 / d + gd * X1, gn2 = gm2 / d + gd * X2;
        gX0 += gd * nc0; gX1 += gd * nc1; gX2 += gd * nc2;
        // n_c = v / max(|v|, eps), v = Rr n_world
        float gv0, gv1, gv2;
        if (len > kNormEps) {
            const float dot = nc0 * gn0 + nc1 * gn1 + nc2 * gn2;
            gv0 = (gn0 - nc0 * dot) / len; gv1 = (gn1 - nc1 * dot) / len; gv2 = (gn2 - nc2 * dot) / len;
        } else {
            gv0 = gn0 / kNormEps; gv1 = gn1 / kNormEps; gv2 = gn2 / kNormEps;
        }
        const size_t nb = (size_t)pr.r * 3 * HW + o;
        sink.normal(nb, Rr[0] * gv0 + Rr[3] * gv1 + Rr[6] * gv2);
        sink.normal(nb + HW, Rr[1] * gv0 + Rr[4] * gv1 + Rr[7] * gv2);
        sink.normal(nb + 2 * HW, Rr[2] * gv0 + Rr[5] * gv1 + Rr[8] * gv2);
    }
    const float gD = gX0 * ux + gX1 * uy + gX2;
    if (gD != 0.f) sink.depth((size_t)pr.r * HW + o, gD);
}

// the CTA's pair, camera and staged reference grey tile (zero outside the image)
__device__ __forceinline__ void mv_setup(const MvParams& prm, const float* __restrict__ gray,
                                         const float* __restrict__ view, MvCam& cam, float* sgray) {
    const MvPair& pr = prm.pair[blockIdx.z];
    if (threadIdx.x == 0) make_cam(view + 16 * pr.r, view + 16 * pr.n, cam);
    const float* g = gray + (size_t)pr.r * prm.H * prm.W;
    const int gx0 = blockIdx.x * TS - HALO, gy0 = blockIdx.y * TS - HALO;
    for (int i = threadIdx.x; i < ST * ST; i += NT) {
        const int gy = gy0 + i / ST, gx = gx0 + i % ST;
        sgray[i] = (gy >= 0 && gy < prm.H && gx >= 0 && gx < prm.W) ? __ldg(g + (size_t)gy * prm.W + gx) : 0.f;
    }
    __syncthreads();
}

__global__ void __launch_bounds__(NT) mv_fwd_kernel(const __grid_constant__ MvParams prm, const float* __restrict__ depth,
                                                    const float* __restrict__ normal, const float* __restrict__ gray,
                                                    const float* __restrict__ view, double* __restrict__ partial) {
    __shared__ float sgray[ST * ST];
    __shared__ MvCam cam;
    mv_setup(prm, gray, view, cam, sgray);
    const int lx = threadIdx.x % TS, ly = threadIdx.x / TS;
    const int x = blockIdx.x * TS + lx, y = blockIdx.y * TS + ly;
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    Sink none = {};
    if (x < prm.W && y < prm.H)
        mv_pixel<false>(prm, prm.pair[blockIdx.z], cam, x, y, depth, normal, gray, sgray, lx, ly, acc, 0.f, 0.f, none);
    cta_partials<NT, 4>(acc, partial + 4 * (((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x));
}

// geo[b] = S_geo / max(n_geo, 1), photo[b] likewise, counts[b] = (n_geo, n_photo); one CTA per pair, fixed order
__global__ void __launch_bounds__(kReduceNT) mv_reduce_kernel(const double* __restrict__ partial, long long per,
                                                              float* __restrict__ geo, float* __restrict__ photo,
                                                              int* __restrict__ counts) {
    __shared__ double s[4][kReduceNT];
    const double* p = partial + (size_t)blockIdx.x * per * 4;
    double a[4] = {0.0, 0.0, 0.0, 0.0};
    for (long long i = threadIdx.x; i < per; i += kReduceNT) {
#pragma unroll
        for (int k = 0; k < 4; ++k) a[k] += p[4 * i + k];
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) s[k][threadIdx.x] = a[k];
    __syncthreads();
    for (int o = kReduceNT / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) {
#pragma unroll
            for (int k = 0; k < 4; ++k) s[k][threadIdx.x] += s[k][threadIdx.x + o];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        geo[blockIdx.x] = (float)(s[0][0] / fmax(s[1][0], 1.0));
        photo[blockIdx.x] = (float)(s[2][0] / fmax(s[3][0], 1.0));
        counts[2 * blockIdx.x] = (int)s[1][0];
        counts[2 * blockIdx.x + 1] = (int)s[3][0];
    }
}

// the per-pair cotangent scales sg = dL/dgeo / max(n_geo, 1), sp likewise
__device__ __forceinline__ float pair_scale(const float* __restrict__ g, const int* __restrict__ counts, int b, int k) {
    return __ldg(g + b) / (float)max(__ldg(counts + 2 * b + k), 1);
}

// The fixed-point exponents of the depth and the normal class (e[0], e[1]).  Every term is linear in one of the
// pairs' |sg|, |sp|, so the exponent starts from the largest of them.  A term can still be far larger than its
// cotangent: a normal shorter than kNormEps carries 1 / kNormEps = 1e12 in its gradient, and Y.z, X'.z or |d| near
// their 1e-6 thresholds divide.  So each class's exponent is raised until its largest |term|, measured by the
// backward's first launch (tmax[0], tmax[1]), lies inside the accumulator range 2^R3DG_DET_RANGE_LOG2; it is unchanged
// when the terms already fit.  Computed by warp 0 of each CTA (every CTA gets the same values).
__device__ __forceinline__ void det_exponent(int B, const float* __restrict__ dgeo, const float* __restrict__ dphoto,
                                             const int* __restrict__ counts, const uint32_t* __restrict__ tmax, int* e) {
    if (threadIdx.x < 32) {
        uint32_t mx = 0u;
        for (int b = threadIdx.x; b < B; b += 32)
            mx = max(mx, max(det_abs_bits(pair_scale(dgeo, counts, b, 0)), det_abs_bits(pair_scale(dphoto, counts, b, 1))));
        mx = __reduce_max_sync(0xffffffffu, mx);
        if (threadIdx.x < 2) {
            const int ec = det_scale_exp(mx);
            const uint32_t t = tmax[threadIdx.x], tb = t >> 23;    // 0 < tb < 255: a finite, normal largest term
            e[threadIdx.x] = (tb == 0u || tb >= 255u) ? ec : max(ec, det_scale_exp(t) - (R3DG_DET_RANGE_LOG2 - 1));
        }
    }
}

__global__ void __launch_bounds__(NT) mv_bwd_kernel(const __grid_constant__ MvParams prm, const float* __restrict__ depth,
                                                    const float* __restrict__ normal, const float* __restrict__ gray,
                                                    const float* __restrict__ view, const float* __restrict__ dgeo,
                                                    const float* __restrict__ dphoto, const int* __restrict__ counts,
                                                    const Sink sink_arg, uint32_t* __restrict__ tmax) {
    __shared__ float sgray[ST * ST];
    __shared__ MvCam cam;
    __shared__ int s_e[2];
    if (sink_arg.det) det_exponent(prm.B, dgeo, dphoto, counts, tmax, s_e);
    mv_setup(prm, gray, view, cam, sgray);
    Sink sink = sink_arg;
    if (sink.det) { sink.ed = s_e[0]; sink.en = s_e[1]; }
    const int b = blockIdx.z;
    const float sg = pair_scale(dgeo, counts, b, 0), sp = pair_scale(dphoto, counts, b, 1);
    const int lx = threadIdx.x % TS, ly = threadIdx.x / TS;
    const int x = blockIdx.x * TS + lx, y = blockIdx.y * TS + ly;
    if (x < prm.W && y < prm.H && (sg != 0.f || sp != 0.f))
        mv_pixel<true>(prm, prm.pair[b], cam, x, y, depth, normal, gray, sgray, lx, ly, nullptr, sg, sp, sink);
    if (sink.measure) {                                       // every thread of the CTA gets here
        det_max_bits(tmax, sink.md);
        det_max_bits(tmax + 1, sink.mn);
    }
}

// deterministic mode: the accumulators read back into dL_ddepth and dL_dnormal (every element written)
__global__ void __launch_bounds__(256) mv_det_read_kernel(int B, size_t VHW, const float* __restrict__ dgeo,
                                                          const float* __restrict__ dphoto, const int* __restrict__ counts,
                                                          const uint32_t* __restrict__ tmax, DetAcc acc,
                                                          float* __restrict__ dd, float* __restrict__ dn) {
    __shared__ int s_e[2];
    det_exponent(B, dgeo, dphoto, counts, tmax, s_e);
    __syncthreads();
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < 4 * VHW; i += (size_t)gridDim.x * blockDim.x) {
        const float v = det_load(acc, i, i < VHW ? s_e[0] : s_e[1]);
        if (i < VHW) dd[i] = v;
        else dn[i - VHW] = v;
    }
}

int check_args(const r3dg_multiview_args* a, MvParams& prm, bool bwd) {
    if (!a) return R3DG_ERR_BAD_ARG;
    if (a->V <= 0 || a->H <= 0 || a->W <= 0 || a->B <= 0 || a->B > R3DG_MAX_VIEWS) return R3DG_ERR_BAD_ARG;
    if ((long long)a->V * 4 * a->H * a->W >= (1LL << 40) || (long long)a->H * a->W >= (1LL << 31) ||
        (a->H + TS - 1) / TS > 65535)
        return R3DG_ERR_UNSUPPORTED;
    if (!a->depth || !a->normal || !a->gray || !a->viewmatrix || !a->pair_cams || !a->pairs) return R3DG_ERR_BAD_ARG;
    if (!(a->pixel_noise_threshold >= 0.f)) return R3DG_ERR_BAD_ARG;
    prm.B = a->B; prm.V = a->V; prm.H = a->H; prm.W = a->W;
    prm.tau = a->pixel_noise_threshold;
    for (int b = 0; b < a->B; ++b) {
        const int r = a->pairs[2 * b], n = a->pairs[2 * b + 1];
        if (r < 0 || r >= a->V || n < 0 || n >= a->V) return R3DG_ERR_BAD_ARG;
        const float* c = a->pair_cams + 8 * b;
        for (int k = 0; k < 8; ++k)
            if (!std::isfinite(c[k])) return R3DG_ERR_BAD_ARG;
        if (!(c[0] > 0.f && c[1] > 0.f && c[4] > 0.f && c[5] > 0.f)) return R3DG_ERR_BAD_ARG;
        MvPair& p = prm.pair[b];
        p.r = r; p.n = n;
        p.fxr = (float)(a->W / (2.0 * c[0])); p.fyr = (float)(a->H / (2.0 * c[1])); p.cxr = c[2]; p.cyr = c[3];
        p.fxn = (float)(a->W / (2.0 * c[4])); p.fyn = (float)(a->H / (2.0 * c[5])); p.cxn = c[6]; p.cyn = c[7];
    }
    if (!bwd) {
        if (!a->geo || !a->photo || !a->counts || !a->work || a->work_bytes < multiview_work_bytes(a->B, a->H, a->W))
            return R3DG_ERR_BAD_ARG;
    } else {
        if (!a->dL_dgeo || !a->dL_dphoto || !a->counts || !a->dL_ddepth || !a->dL_dnormal) return R3DG_ERR_BAD_ARG;
        if (a->deterministic && (!a->det_work || a->det_work_bytes < multiview_det_bytes(a->V, a->H, a->W)))
            return R3DG_ERR_BAD_ARG;
    }
    return 0;
}

dim3 tile_grid(int B, int H, int W) { return dim3((W + TS - 1) / TS, (H + TS - 1) / TS, B); }

}  // namespace

size_t multiview_work_bytes(int B, int H, int W) {
    if (B <= 0 || B > R3DG_MAX_VIEWS || H <= 0 || W <= 0 || (long long)H * W >= (1LL << 31)) return 0;
    const dim3 g = tile_grid(B, H, W);
    return ((size_t)g.x * g.y * g.z * 4 * sizeof(double) + 255) & ~(size_t)255;
}

size_t multiview_det_bytes(int V, int H, int W) {
    if (V <= 0 || H <= 0 || W <= 0 || (long long)H * W >= (1LL << 31)) return 0;
    return det_bytes((size_t)V * 4 * H * W) + 256;          // the accumulators, then the two largest-term words
}

int launch_multiview_forward(const r3dg_multiview_args* a, cudaStream_t stream) {
    MvParams prm;
    const int rc = check_args(a, prm, false);
    if (rc != 0) return rc;
    const dim3 g = tile_grid(a->B, a->H, a->W);
    double* partial = (double*)a->work;
    mv_fwd_kernel<<<g, NT, 0, stream>>>(prm, a->depth, a->normal, a->gray, a->viewmatrix, partial);
    R3DG_CUDA_TRY(cudaGetLastError());
    mv_reduce_kernel<<<a->B, kReduceNT, 0, stream>>>(partial, (long long)g.x * g.y, a->geo, a->photo, a->counts);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_multiview_backward(const r3dg_multiview_args* a, cudaStream_t stream) {
    MvParams prm;
    const int rc = check_args(a, prm, true);
    if (rc != 0) return rc;
    const size_t HW = (size_t)a->H * a->W, VHW = (size_t)a->V * HW;
    Sink sink = {};
    sink.dd = a->dL_ddepth;
    sink.dn = a->dL_dnormal;
    sink.det = a->deterministic != 0;
    sink.VHW = VHW;
    const dim3 grid = tile_grid(a->B, a->H, a->W);
    uint32_t* tmax = nullptr;
    if (sink.det) {
        sink.acc = det_acc(a->det_work, 4 * VHW);
        tmax = (uint32_t*)((char*)a->det_work + det_bytes(4 * VHW));
        R3DG_CUDA_TRY(cudaMemsetAsync(a->det_work, 0, det_bytes(4 * VHW) + 2 * sizeof(uint32_t), stream));
        Sink measure = sink;
        measure.det = false;
        measure.measure = true;
        mv_bwd_kernel<<<grid, NT, 0, stream>>>(prm, a->depth, a->normal, a->gray, a->viewmatrix, a->dL_dgeo,
                                               a->dL_dphoto, a->counts, measure, tmax);
        R3DG_CUDA_TRY(cudaGetLastError());
    } else {
        R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_ddepth, 0, VHW * sizeof(float), stream));
        R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_dnormal, 0, 3 * VHW * sizeof(float), stream));
    }
    mv_bwd_kernel<<<grid, NT, 0, stream>>>(prm, a->depth, a->normal, a->gray, a->viewmatrix, a->dL_dgeo, a->dL_dphoto,
                                           a->counts, sink, tmax);
    R3DG_CUDA_TRY(cudaGetLastError());
    if (sink.det) {
        const size_t n = 4 * VHW;
        const unsigned blocks = (unsigned)std::min<size_t>((n + 255) / 256, 132 * 16);
        mv_det_read_kernel<<<blocks, 256, 0, stream>>>(a->B, VHW, a->dL_dgeo, a->dL_dphoto, a->counts, tmax, sink.acc,
                                                       a->dL_ddepth, a->dL_dnormal);
        R3DG_CUDA_TRY(cudaGetLastError());
    }
    return 0;
}

}  // namespace r3dg
