// Similarity transforms of Gaussian models, K objects per launch (include/r3dg_b200.h, COMPOSE; DESIGN.md §4.27).
//
// Design notes
//  * tiles: each object's rows are cut into tiles of CP_ROWS rows; a CTA owns one tile, so every tile lies inside one
//    object and every CTA applies one pose.  The host lays the tiles out from the offsets (ComposeTiles).
//  * pose: each CTA builds its object's R and D^l (l = 1..4) in fp64 from the generated table
//    (D^l = A_l^-1 [Y_lm(R^T u_k)]) and keeps them in shared memory as fp32.  That is a few hundred fp64 operations
//    per CTA, so no separate launch and no D buffer between the forward and the backward.
//  * SH rows: a [P,(L+1)^2-1,C] tile is contiguous in global memory.  It is read into shared memory with unit-stride
//    loads, and each thread then produces output elements at unit stride (element e of the tile: row e / W,
//    coefficient and channel from e % W), reading the 2l+1 inputs of its band from shared memory, so both the loads
//    and the stores are coalesced whatever the row width.
//  * backward: the same walk with D^T gives dL/dsh; dL/dD = sum over rows and channels of dL/dsh'_l sh_l^T is
//    summed per CTA by one thread per D entry in a fixed row order.  The small per-row tensors (xyz, normal,
//    rotation, scaling) are one thread per row; their pose terms are summed over the CTA by a warp butterfly and
//    the warps' rows in warp order.  Each CTA writes one partial row; compose_finish_kernel sums an object's tiles
//    in a fixed order and chains dL/dD into dL/dR in fp64.  No atomics: every output is bitwise reproducible.
#include "kernels.h"
#include "sh_rotation_table.cuh"

namespace r3dg {

#define CP_THREADS 256
#define CP_WARPS (CP_THREADS / 32)
#define CP_ROWS 128
#define CP_NSH 3
#define CP_ND 164                          // sum over l = 1..4 of (2l+1)^2
#define CP_NPOSE 18                        // dR 9, dq 4, dt 3, ds (through xyz) 1, dlog s 1
#define CP_G (CP_NPOSE + CP_ND)            // floats per partial row
#define CP_MAX_W 72                        // widest SH row: L = 4, C = 3

// Row and tile layout of the objects (host-computed, passed by value)
struct ComposeTiles {
    int K;
    int row[R3DG_MAX_OBJECTS + 1];         // offsets
    int tile[R3DG_MAX_OBJECTS + 1];        // first tile of each object; tile[K] = number of tiles
};

// ---- the real SH basis, band l only, for T = double or a forward-mode dual number ---------------------------------
struct Dual3 {
    double v, d[3];
};
__device__ __forceinline__ Dual3 operator+(const Dual3& a, const Dual3& b) {
    return {a.v + b.v, {a.d[0] + b.d[0], a.d[1] + b.d[1], a.d[2] + b.d[2]}};
}
__device__ __forceinline__ Dual3 operator-(const Dual3& a, const Dual3& b) {
    return {a.v - b.v, {a.d[0] - b.d[0], a.d[1] - b.d[1], a.d[2] - b.d[2]}};
}
__device__ __forceinline__ Dual3 operator*(const Dual3& a, const Dual3& b) {
    return {a.v * b.v, {a.d[0] * b.v + a.v * b.d[0], a.d[1] * b.v + a.v * b.d[1], a.d[2] * b.v + a.v * b.d[2]}};
}
__device__ __forceinline__ Dual3 operator*(double s, const Dual3& a) { return {s * a.v, {s * a.d[0], s * a.d[1], s * a.d[2]}}; }
__device__ __forceinline__ Dual3 operator-(const Dual3& a, double s) { return {a.v - s, {a.d[0], a.d[1], a.d[2]}}; }
__device__ __forceinline__ Dual3 operator+(const Dual3& a, double s) { return {a.v + s, {a.d[0], a.d[1], a.d[2]}}; }

template <typename T>
__device__ void sh_band(int l, const T& x, const T& y, const T& z, T* out) {
    const T xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    if (l == 1) {
        const double c = 0.4886025119029199;
        out[0] = -c * y; out[1] = c * z; out[2] = -c * x;
    } else if (l == 2) {
        out[0] = 1.0925484305920792 * xy; out[1] = -1.0925484305920792 * yz;
        out[2] = 0.31539156525252005 * ((2.0 * zz - xx) - yy);
        out[3] = -1.0925484305920792 * xz; out[4] = 0.5462742152960396 * (xx - yy);
    } else if (l == 3) {
        out[0] = -0.5900435899266435 * (y * (3.0 * xx - yy));
        out[1] = 2.890611442640554 * (xy * z);
        out[2] = -0.4570457994644658 * (y * ((4.0 * zz - xx) - yy));
        out[3] = 0.3731763325901154 * (z * ((2.0 * zz - 3.0 * xx) - 3.0 * yy));
        out[4] = -0.4570457994644658 * (x * ((4.0 * zz - xx) - yy));
        out[5] = 1.445305721320277 * (z * (xx - yy));
        out[6] = -0.5900435899266435 * (x * (xx - 3.0 * yy));
    } else {
        out[0] = 2.5033429417967046 * (xy * (xx - yy));
        out[1] = -1.7701307697799304 * (yz * (3.0 * xx - yy));
        out[2] = 0.9461746957575601 * (xy * (7.0 * zz - 1.0));
        out[3] = -0.6690465435572892 * (yz * (7.0 * zz - 3.0));
        out[4] = 0.10578554691520431 * (zz * (35.0 * zz - 30.0) + 3.0);
        out[5] = -0.6690465435572892 * (xz * (7.0 * zz - 3.0));
        out[6] = 0.47308734787878004 * ((xx - yy) * (7.0 * zz - 1.0));
        out[7] = -1.7701307697799304 * (xz * (xx - 3.0 * yy));
        out[8] = 0.6258357354491761 * (xx * (xx - 3.0 * yy) - yy * (3.0 * xx - yy));
    }
}

// band of table row / rest coefficient index k (0-based over the rest coefficients: band l holds k = l^2-1 .. l^2+2l-1)
__device__ __forceinline__ int band_of(int k) {
    int l = 1;
    while ((l + 1) * (l + 1) <= k + 1) ++l;
    return l;
}

// D^l starts at entry doff(l) of the packed D^1..D^4 (row-major, (2l+1)^2 entries each); entry e lies in band dband_of(e)
__device__ __forceinline__ int doff(int l) { return l == 1 ? 0 : l == 2 ? 9 : l == 3 ? 34 : 83; }
__device__ __forceinline__ int dband_of(int e) { return e < 9 ? 1 : e < 34 ? 2 : e < 83 ? 3 : 4; }

// q^ = q / |q| and R(q^) (build_rotation), in fp64
__device__ __forceinline__ void pose_rotation(const float* q4, double* qn, double* R) {
    const double w0 = q4[0], x0 = q4[1], y0 = q4[2], z0 = q4[3];
    const double n = sqrt(w0 * w0 + x0 * x0 + y0 * y0 + z0 * z0);
    const double r = w0 / n, x = x0 / n, y = y0 / n, z = z0 / n;
    qn[0] = r; qn[1] = x; qn[2] = y; qn[3] = z;
    R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - r * z); R[2] = 2 * (x * z + r * y);
    R[3] = 2 * (x * y + r * z); R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - r * x);
    R[6] = 2 * (x * z - r * y); R[7] = 2 * (y * z + r * x); R[8] = 1 - 2 * (x * x + y * y);
}

struct PoseSmem {
    float R[9], q[4], t[3], s, logs;
    float D[CP_ND];
    double B[CP_ND];
    int k, r0, nrows;
};

// The CTA's object and rows, and its pose with D^1..D^4, in shared memory.
__device__ void load_pose(const r3dg_compose_args& a, const ComposeTiles& T, PoseSmem& ps) {
    const int b = blockIdx.x;
    int k = 0;
    while (k + 1 < T.K && T.tile[k + 1] <= b) ++k;
    const int tid = threadIdx.x;
    double qn[4], R[9];
    pose_rotation(a.quat + 4 * k, qn, R);
    if (tid < 24) {                                   // B_l[k][m] = Y_lm(R^T u_k), one direction per thread
        const int l = band_of(tid), n = 2 * l + 1, kk = tid - (l * l - 1);
        const double* u = SHROT_DIRS[tid];
        const double v[3] = {R[0] * u[0] + R[3] * u[1] + R[6] * u[2], R[1] * u[0] + R[4] * u[1] + R[7] * u[2],
                             R[2] * u[0] + R[5] * u[1] + R[8] * u[2]};
        double y[9];
        sh_band<double>(l, v[0], v[1], v[2], y);
        for (int m = 0; m < n; ++m) ps.B[doff(l) + kk * n + m] = y[m];
    } else if (tid == 32) {
        for (int i = 0; i < 9; ++i) ps.R[i] = (float)R[i];
        for (int i = 0; i < 4; ++i) ps.q[i] = (float)qn[i];
        for (int i = 0; i < 3; ++i) ps.t[i] = a.translation[3 * k + i];
        ps.s = a.scale[k];
        ps.logs = logf(ps.s);
        ps.k = k;
        ps.r0 = T.row[k] + (b - T.tile[k]) * CP_ROWS;
        ps.nrows = min(CP_ROWS, T.row[k + 1] - ps.r0);
    }
    __syncthreads();
    if (tid < CP_ND) {                                // D_l = A_l^-1 B_l
        const int l = dband_of(tid), n = 2 * l + 1, off = doff(l), e = tid - off, i = e / n, j = e - i * n;
        double d = 0.0;
        for (int kk = 0; kk < n; ++kk) d += SHROT_AINV[off + i * n + kk] * ps.B[off + kk * n + j];
        ps.D[tid] = (float)d;
    }
    __syncthreads();
}

__device__ __forceinline__ int sh_width(const r3dg_compose_args& a, int i) {
    const int L = a.sh_degree[i];
    return ((L + 1) * (L + 1) - 1) * a.sh_channels[i];
}

// Tile element e of an SH tensor of width W and C channels: out = sum_j M[i][j] in[j] over its band (M = D) or
// sum_j M[j][i] in[j] (M = D^T).
template <bool TRANSPOSE>
__device__ __forceinline__ float rotate_element(const float* tile, int e, int W, int C, const float* D) {
    const int row = e / W, r = e - row * W, kc = r / C, ch = r - kc * C;
    const int l = band_of(kc), n = 2 * l + 1, i = kc - (l * l - 1), off = l * l - 1;
    const float* Dl = D + doff(l);
    const float* in = tile + row * W + off * C + ch;
    float acc = 0.f;
    for (int j = 0; j < n; ++j) acc = fmaf(TRANSPOSE ? Dl[j * n + i] : Dl[i * n + j], in[j * C], acc);
    return acc;
}

// Tile of rows [r0, r0 + nrows) of an SH tensor of width W into shared memory, unit stride
__device__ __forceinline__ void stage_tile(const float* __restrict__ src, size_t r0, int nrows, int W, float* dst) {
    const float* s = src + r0 * W;
    for (int e = threadIdx.x; e < nrows * W; e += CP_THREADS) dst[e] = s[e];
}

__global__ void __launch_bounds__(CP_THREADS) compose_fwd_kernel(const r3dg_compose_args a, const ComposeTiles T) {
    extern __shared__ float tile[];
    __shared__ PoseSmem ps;
    load_pose(a, T, ps);
    const size_t r0 = ps.r0;
    const int nrows = ps.nrows, tid = threadIdx.x;
    if (tid < nrows) {
        const size_t p = r0 + tid;
        const float* R = ps.R;
        const float x[3] = {a.xyz[3 * p], a.xyz[3 * p + 1], a.xyz[3 * p + 2]};
        const float n[3] = {a.normal[3 * p], a.normal[3 * p + 1], a.normal[3 * p + 2]};
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const float rx = fmaf(R[3 * i + 2], x[2], fmaf(R[3 * i + 1], x[1], R[3 * i] * x[0]));
            a.xyz_out[3 * p + i] = fmaf(ps.s, rx, ps.t[i]);
            a.normal_out[3 * p + i] = fmaf(R[3 * i + 2], n[2], fmaf(R[3 * i + 1], n[1], R[3 * i] * n[0]));
            a.scaling_out[3 * p + i] = a.scaling[3 * p + i] + ps.logs;
        }
        const float qw = ps.q[0], qx = ps.q[1], qy = ps.q[2], qz = ps.q[3];
        const float rw = a.rotation[4 * p], rx = a.rotation[4 * p + 1], ry = a.rotation[4 * p + 2], rz = a.rotation[4 * p + 3];
        a.rotation_out[4 * p] = qw * rw - qx * rx - qy * ry - qz * rz;
        a.rotation_out[4 * p + 1] = qw * rx + qx * rw + qy * rz - qz * ry;
        a.rotation_out[4 * p + 2] = qw * ry - qx * rz + qy * rw + qz * rx;
        a.rotation_out[4 * p + 3] = qw * rz + qx * ry - qy * rx + qz * rw;
    }
    for (int i = 0; i < a.n_sh; ++i) {
        const int W = sh_width(a, i), C = a.sh_channels[i];
        if (W == 0) continue;
        __syncthreads();                                 // the previous tensor's readers are done with the tile
        stage_tile(a.sh[i], r0, nrows, W, tile);
        __syncthreads();
        float* out = a.sh_out[i] + r0 * W;
        for (int e = tid; e < nrows * W; e += CP_THREADS) out[e] = rotate_element<false>(tile, e, W, C, ps.D);
    }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// partial: [tiles][CP_G] = the tile's (dR, dq, dt, ds through xyz, dlog s, dD)
__global__ void __launch_bounds__(CP_THREADS) compose_bwd_kernel(const r3dg_compose_args a, const ComposeTiles T,
                                                                 float* __restrict__ partial) {
    extern __shared__ float tile[];                      // [2][nrows * W]: the input rows, then their output cotangents
    __shared__ PoseSmem ps;
    __shared__ float sRed[CP_WARPS][CP_NPOSE];
    load_pose(a, T, ps);
    const size_t r0 = ps.r0;
    const int nrows = ps.nrows, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float pose[CP_NPOSE];
#pragma unroll
    for (int i = 0; i < CP_NPOSE; ++i) pose[i] = 0.f;
    if (tid < nrows) {
        const size_t p = r0 + tid;
        const float* R = ps.R;
        const float s = ps.s;
        const float x[3] = {a.xyz[3 * p], a.xyz[3 * p + 1], a.xyz[3 * p + 2]};
        const float n[3] = {a.normal[3 * p], a.normal[3 * p + 1], a.normal[3 * p + 2]};
        const float gx[3] = {a.dL_dxyz_out[3 * p], a.dL_dxyz_out[3 * p + 1], a.dL_dxyz_out[3 * p + 2]};
        const float gn[3] = {a.dL_dnormal_out[3 * p], a.dL_dnormal_out[3 * p + 1], a.dL_dnormal_out[3 * p + 2]};
#pragma unroll
        for (int j = 0; j < 3; ++j) {               // dx = s R^T gx, dn = R^T gn
            a.dL_dxyz[3 * p + j] = s * fmaf(R[6 + j], gx[2], fmaf(R[3 + j], gx[1], R[j] * gx[0]));
            a.dL_dnormal[3 * p + j] = fmaf(R[6 + j], gn[2], fmaf(R[3 + j], gn[1], R[j] * gn[0]));
        }
#pragma unroll
        for (int i = 0; i < 3; ++i) {
#pragma unroll
            for (int j = 0; j < 3; ++j) pose[3 * i + j] = fmaf(s * gx[i], x[j], gn[i] * n[j]);   // dR = s gx x^T + gn n^T
            const float rx = fmaf(R[3 * i + 2], x[2], fmaf(R[3 * i + 1], x[1], R[3 * i] * x[0]));
            pose[13 + i] = gx[i];
            pose[16] = fmaf(gx[i], rx, pose[16]);
            const float gs = a.dL_dscaling_out[3 * p + i];
            a.dL_dscaling[3 * p + i] = gs;
            pose[17] += gs;
        }
        const float qw = ps.q[0], qx = ps.q[1], qy = ps.q[2], qz = ps.q[3];
        const float rw = a.rotation[4 * p], rx = a.rotation[4 * p + 1], ry = a.rotation[4 * p + 2], rz = a.rotation[4 * p + 3];
        const float gw = a.dL_drotation_out[4 * p], gxq = a.dL_drotation_out[4 * p + 1], gy = a.dL_drotation_out[4 * p + 2],
                    gz = a.dL_drotation_out[4 * p + 3];
        a.dL_drotation[4 * p] = qw * gw + qx * gxq + qy * gy + qz * gz;             // L(q)^T g
        a.dL_drotation[4 * p + 1] = -qx * gw + qw * gxq + qz * gy - qy * gz;
        a.dL_drotation[4 * p + 2] = -qy * gw - qz * gxq + qw * gy + qx * gz;
        a.dL_drotation[4 * p + 3] = -qz * gw + qy * gxq - qx * gy + qw * gz;
        pose[9] = rw * gw + rx * gxq + ry * gy + rz * gz;                           // R(r)^T g
        pose[10] = -rx * gw + rw * gxq - rz * gy + ry * gz;
        pose[11] = -ry * gw + rz * gxq + rw * gy - rx * gz;
        pose[12] = -rz * gw - ry * gxq + rx * gy + rw * gz;
    }
#pragma unroll
    for (int i = 0; i < CP_NPOSE; ++i) {
        const float v = warp_sum(pose[i]);
        if (lane == 0) sRed[warp][i] = v;
    }
    // dD entry tid (band l, row i, column j): sum over the tile's rows and channels of g'[row][i][c] sh[row][j][c]
    float dD = 0.f;
    for (int t = 0; t < a.n_sh; ++t) {
        const int W = sh_width(a, t), C = a.sh_channels[t], L = a.sh_degree[t];
        if (W == 0) continue;
        float* sh_s = tile;
        float* g_s = tile + nrows * W;
        __syncthreads();
        stage_tile(a.sh[t], r0, nrows, W, sh_s);
        stage_tile(a.dL_dsh_out[t], r0, nrows, W, g_s);
        __syncthreads();
        float* out = a.dL_dsh[t] + r0 * W;
        for (int e = tid; e < nrows * W; e += CP_THREADS) out[e] = rotate_element<true>(g_s, e, W, C, ps.D);
        if (tid < CP_ND) {
            const int l = dband_of(tid);
            if (l <= L) {
                const int n = 2 * l + 1, e = tid - doff(l), i = e / n, j = e - i * n, off = l * l - 1;
                const float* gi = g_s + (off + i) * C;
                const float* sj = sh_s + (off + j) * C;
                for (int row = 0; row < nrows; ++row)
                    for (int c = 0; c < C; ++c) dD = fmaf(gi[row * W + c], sj[row * W + c], dD);
            }
        }
    }
    __syncthreads();
    float* out = partial + (size_t)blockIdx.x * CP_G;
    if (tid < CP_NPOSE) {
        float v = sRed[0][tid];
#pragma unroll
        for (int w = 1; w < CP_WARPS; ++w) v += sRed[w][tid];
        out[tid] = v;
    }
    if (tid < CP_ND) out[CP_NPOSE + tid] = dD;
}

// One CTA per object: its tiles' partials summed in tile order (lane-strided, then a fixed butterfly), then dL/dD
// chained into dL/dR in fp64: dL/dB_l = A_l^-T dL/dD_l, dL/dv_k = sum_m dL/dB_l[k][m] grad Y_lm(v_k) at
// v_k = R^T u_k, dL/dR[b][a] += dL/dv_k[a] u_k[b].
__global__ void __launch_bounds__(CP_THREADS) compose_finish_kernel(const r3dg_compose_args a, const ComposeTiles T,
                                                                    const float* __restrict__ partial) {
    __shared__ float sum[CP_G];
    __shared__ double dRk[24][9];
    const int k = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int t0 = T.tile[k], t1 = T.tile[k + 1];
    for (int i = warp; i < CP_G; i += CP_WARPS) {
        float x = 0.f;
        for (int b = t0 + lane; b < t1; b += 32) x += partial[(size_t)b * CP_G + i];
        x = warp_sum(x);
        if (lane == 0) sum[i] = x;
    }
    __syncthreads();
    double qn[4], R[9];
    pose_rotation(a.quat + 4 * k, qn, R);
    if (tid < 24) {
        const int l = band_of(tid), n = 2 * l + 1, kk = tid - (l * l - 1), off = doff(l);
        const double* u = SHROT_DIRS[tid];
        Dual3 v[3];
        for (int c = 0; c < 3; ++c) {
            v[c].v = R[c] * u[0] + R[3 + c] * u[1] + R[6 + c] * u[2];
            v[c].d[0] = v[c].d[1] = v[c].d[2] = 0.0;
            v[c].d[c] = 1.0;
        }
        Dual3 y[9];
        sh_band<Dual3>(l, v[0], v[1], v[2], y);
        double dv[3] = {0.0, 0.0, 0.0};
        for (int m = 0; m < n; ++m) {
            double dB = 0.0;                               // (A^-T dD)[kk][m] = sum_i A^-1[i][kk] dD[i][m]
            for (int i = 0; i < n; ++i) dB += SHROT_AINV[off + i * n + kk] * (double)sum[CP_NPOSE + off + i * n + m];
            for (int c = 0; c < 3; ++c) dv[c] += dB * y[m].d[c];
        }
        for (int b = 0; b < 3; ++b)
            for (int c = 0; c < 3; ++c) dRk[tid][3 * b + c] = dv[c] * u[b];
    }
    __syncthreads();
    if (tid < 9) {
        double d = sum[tid];
        for (int kk = 0; kk < 24; ++kk) d += dRk[kk][tid];
        a.dL_dR[9 * k + tid] = (float)d;
    } else if (tid < 13) {
        a.dL_dquat[4 * k + tid - 9] = sum[tid];
    } else if (tid < 16) {
        a.dL_dtranslation[3 * k + tid - 13] = sum[tid];
    } else if (tid == 16) {
        a.dL_dscale[k] = (float)((double)sum[16] + (double)sum[17] / (double)a.scale[k]);
    }
}

// ---- host launchers -----------------------------------------------------------------------
static int max_width(const r3dg_compose_args* a) {
    int w = 0;
    for (int i = 0; i < a->n_sh; ++i) w = max(w, ((a->sh_degree[i] + 1) * (a->sh_degree[i] + 1) - 1) * a->sh_channels[i]);
    return w;
}

size_t compose_work_bytes(int P, int K) {
    if (P <= 0 || K < 1 || K > R3DG_MAX_OBJECTS) return 0;
    return ((size_t)(P + CP_ROWS - 1) / CP_ROWS + K) * CP_G * sizeof(float);
}

// Validates everything both directions read; fills the tile layout.
static bool compose_args_valid(const r3dg_compose_args* a, ComposeTiles* T) {
    if (!a || a->P < 0 || a->K < 1 || a->K > R3DG_MAX_OBJECTS || !a->offsets) return false;
    if (!a->quat || !a->translation || !a->scale) return false;
    if (a->offsets[0] != 0 || a->offsets[a->K] != a->P) return false;
    for (int k = 0; k < a->K; ++k)
        if (a->offsets[k + 1] < a->offsets[k]) return false;
    if (a->n_sh < 0 || a->n_sh > R3DG_COMPOSE_MAX_SH) return false;
    for (int i = 0; i < a->n_sh; ++i) {
        if (a->sh_degree[i] < 0 || a->sh_degree[i] > 4 || (a->sh_channels[i] != 1 && a->sh_channels[i] != 3)) return false;
        if (a->P > 0 && a->sh_degree[i] > 0 && !a->sh[i]) return false;
    }
    if (a->P > 0 && (!a->xyz || !a->normal || !a->rotation || !a->scaling)) return false;
    T->K = a->K;
    T->tile[0] = 0;
    for (int k = 0; k <= a->K; ++k) T->row[k] = a->offsets[k];
    for (int k = 0; k < a->K; ++k) T->tile[k + 1] = T->tile[k] + (a->offsets[k + 1] - a->offsets[k] + CP_ROWS - 1) / CP_ROWS;
    return true;
}

template <typename Kern>
static int set_smem(Kern kern, size_t bytes) {
    if (bytes > 48 * 1024) R3DG_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    return 0;
}

int launch_compose_forward(const r3dg_compose_args* a, cudaStream_t stream, bool* launched) {
    *launched = false;
    ComposeTiles T;
    if (!compose_args_valid(a, &T)) return R3DG_ERR_BAD_ARG;
    if (a->P > 0 && (!a->xyz_out || !a->normal_out || !a->rotation_out || !a->scaling_out)) return R3DG_ERR_BAD_ARG;
    for (int i = 0; i < a->n_sh; ++i)
        if (a->P > 0 && a->sh_degree[i] > 0 && !a->sh_out[i]) return R3DG_ERR_BAD_ARG;
    if (a->P == 0) return 0;
    const size_t smem = (size_t)CP_ROWS * max_width(a) * sizeof(float);
    if (int rc = set_smem(compose_fwd_kernel, smem)) return rc;
    compose_fwd_kernel<<<T.tile[a->K], CP_THREADS, smem, stream>>>(*a, T);
    R3DG_CUDA_TRY(cudaGetLastError());
    *launched = true;
    return 0;
}

int launch_compose_backward(const r3dg_compose_args* a, cudaStream_t stream, bool* launched) {
    *launched = false;
    ComposeTiles T;
    if (!compose_args_valid(a, &T)) return R3DG_ERR_BAD_ARG;
    if (!a->dL_dR || !a->dL_dquat || !a->dL_dtranslation || !a->dL_dscale) return R3DG_ERR_BAD_ARG;
    if (a->P > 0 && (!a->dL_dxyz_out || !a->dL_dnormal_out || !a->dL_drotation_out || !a->dL_dscaling_out || !a->dL_dxyz ||
                     !a->dL_dnormal || !a->dL_drotation || !a->dL_dscaling))
        return R3DG_ERR_BAD_ARG;
    for (int i = 0; i < a->n_sh; ++i)
        if (a->P > 0 && a->sh_degree[i] > 0 && (!a->dL_dsh_out[i] || !a->dL_dsh[i])) return R3DG_ERR_BAD_ARG;
    const size_t need = compose_work_bytes(a->P, a->K);
    if (need > 0 && (!a->work || a->work_bytes < need)) return R3DG_ERR_BAD_ARG;
    if (a->P == 0) {
        R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_dR, 0, (size_t)a->K * 9 * sizeof(float), stream));
        R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_dquat, 0, (size_t)a->K * 4 * sizeof(float), stream));
        R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_dtranslation, 0, (size_t)a->K * 3 * sizeof(float), stream));
        R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_dscale, 0, (size_t)a->K * sizeof(float), stream));
        return 0;
    }
    const size_t smem = 2 * (size_t)CP_ROWS * max_width(a) * sizeof(float);
    if (int rc = set_smem(compose_bwd_kernel, smem)) return rc;
    float* partial = (float*)a->work;
    compose_bwd_kernel<<<T.tile[a->K], CP_THREADS, smem, stream>>>(*a, T, partial);
    compose_finish_kernel<<<a->K, CP_THREADS, 0, stream>>>(*a, T, partial);
    R3DG_CUDA_TRY(cudaGetLastError());
    *launched = true;
    return 0;
}

}  // namespace r3dg
