// Stage 2 backward: per-tile back-to-front re-traversal (reference K10, backward.cu:401-614).
//
// Design notes
//  * the reference issues 10+S global atomicAdds per contributing (pixel, Gaussian) pair.  Here a warp (8x4 pixels)
//    works in two phases per sub-batch of E staged entries.  Pixel phase (lane = pixel): alpha, the tests and the T / A
//    recurrences, and the two per-(entry, pixel) scalars every gradient component is linear in,  w = G dL_dalpha  and
//    dcc = alpha T,  written to shared planes.  Entry phase (lane = entry): each lane sums its entry's row over the
//    block's pixels with plain FMAs — the 6 centred moments of w (geometry), the cotangent dots of dcc (depth, colour,
//    features) — one shuffle per accumulator joins the pixel parts, and the finished rows are added from shared memory
//    by vector reductions that cover whole row segments (DESIGN.md §4.2);
//  * warps are autonomous (no CTA barrier; see composite.cu): each walks ONLY the entries whose
//    contributor bit the forward pass set for its pixel block, back to front from the block's
//    deepest last contributor — no culling test, no record fetch, no exp() for anything else;
//  * CTAs are launched in the order of the work the forward pass measured (cta_order_kernel): the kernel is bound by
//    per-warp latency and its heaviest warps (DESIGN.md §4.2);
//  * per-pixel state is register resident (template on channel groups); the reference keeps three
//    float[24] arrays in local memory and 36 KB of shared memory per CTA;
//  * gradients differ from the reference only by fp32 summation order (the reference's own
//    atomics make it run-to-run nondeterministic), tolerance 1e-3 relative.
#include <algorithm>
#include <cstring>
#include "common.cuh"
#include "detacc.cuh"
#include "kernels.h"

namespace r3dg {

struct CompositeBwdParams {
    int W, H, gx, gy, S, recf, backward_geometry;   // gy: tile rows of one view (see CompositeFwdParams)
    const uint2* ranges;
    const uint32_t* point_list;  // per-tile depth-sorted Gaussian ids (binning.cu)
    const uint32_t* cmask32;     // per-instance contributor masks written by the forward compositor
    const GeomHeader* header;
    const uint32_t* cta_order;   // CTA -> half tile (2 * tile + part), most backward work first (cta_order_kernel)
    const float* rec;
    const float* bg;
    const float* final_T;
    const int* n_contrib;
    const float *dL_dpix, *dL_dpix_o, *dL_dpix_d, *dL_dpix_f;
    float* grad;     // [P][recf], the composited rows zero-initialised (zero_composited_rows_kernel)
    DetAcc det;      // DET: the same rows as fixed-point accumulators (detacc.cuh), [P * recf], as grad
    const uint32_t* det_scale;   // DET: per view, the scale words of its colour / feature and geometry slots (det_scale_reduce)
    // ABS (absgrad): per row, sum_pixels |dL/dmean2D.x| and |dL/dmean2D.y|, [rows][2]: in the default mode the caller's
    // dL_dmeans2D_abs itself (its composited rows zeroed by zero_composited_rows_kernel), in DET mode fixed-point
    // accumulators of the geometry class behind the gradient rows' (det_abs)
    float* abs_grad;
    DetAcc det_abs;
    const float *dL_dpix_d2, *dL_dpix_m;   // DS: the cotangents of depth2 and of the median depth
    const int* median_pos;                 // DS: the forward's median entry per pixel (1-based list position, 0: none)
    const uint32_t* depth_bound;           // DS: per view, the forward's largest |d| of an accepted entry (float bits)
};

// Per warp (one 8x4 pixel block): the forward pass left one contributor bit per (instance, block).  The warp streams
// its tile's contributor bytes BACK TO FRONT, 128 instances per step, compacts the positions whose bit is set into a
// circular queue (warp scan) and processes batches of 32 of them: every staged entry is one that some pixel of the
// block composited in the forward pass — no culling test, no record fetch and no exp() for anything else.
// A batch is processed in sub-batches of E entries, each in two phases:
//  * pixel phase (lane = pixel): per entry G, alpha, the forward pass's tests, T and A in list order, then
//    w = G dL_dalpha  and  dcc = gate alpha T  into the planes sW / sC [entry][pixel] (row stride 33: conflict-free);
//  * entry phase (lane = entry): lane l sums entry l % E over pixel part l / E (E pixels, whole pixel rows) in a fixed
//    order.  Every row component is such a sum times per-entry factors:  the two dL/dmean2D slots from the per-pixel
//    terms  w (a dx + b dy)  and  w (c dy + b dx)  (a, b, c the conic), the conic slots from the centred moments
//    sum w dx^2, w dx dy, w dy^2,  the opacity slot from  sum w  (dx, dy the entry's mean minus the pixel centre,
//    exactly the pixel phase's: centred per pixel, so far-away Gaussians do not cancel), depth and channel slots from
//    sum dcc dL_dpix.
//    The parts are joined by shuffles, the rows are staged in shared memory (over the planes) and added by lanes that
//    cover contiguous float4 segments of them (red.global.add.v4.f32).  Geometry slot 7 and the padding channels
//    (>= 3 + S) are zero; a segment of padding channels only is not added.
// DET (deterministic mode): each real row component is added through the order-independent fixed-point primitive
// (detacc.cuh) into p.det instead of by a float atomic into p.grad, scaled by its view's exponent of the colour /
// feature slots or of the geometry slots (det_scale_reduce).  Everything else is the same code.
// GEOM = false (appearance-only backward, no geometry gradient requested): the same walk, CTA order and alpha / T
// arithmetic, but only the NC colour and feature components are formed — no dL/dalpha, no A recurrence, no geometry
// moments — into a narrower row of NC floats (channel c at slot c).  The channel sums run the same loop as with GEOM,
// so each added value, and in DET mode each row total, is bitwise the full kernel's.
// ABS (absgrad, GEOM only): the entry phase also sums the magnitudes of the pixels' two dL/dmean2D terms in the order
// of the signed sums, times |o| W/2 and |o| H/2, and adds the two totals to p.abs_grad (DET:
// p.det_abs, class exponent e_geo) once per entry.  Everything else, the gradient row included, is the same code.
// RD (ray-depth mode, GEOM only): an entry's depth at a pixel is d = tz - p.x dx - p.y dy (the record's appended depth
// plane p), in dL/dalpha too.  The entry phase also sums  dcc dL_dD dx  and  dcc dL_dD dy : the row's appended group
// gets dL/dp = -(those sums), and the dL/dmean2D slots get d's own term  -p dL/dtz  (times W/2, H/2), added after the
// alpha term, so that a zero depth cotangent leaves them as they are.  With ABS, the per-pixel magnitudes are those of
// the two terms together.
// DS (depth statistics, GEOM only): with g2, gm the pixel's cotangents of depth2 and of the median depth, dL/dalpha's
// per-pixel scalar gains  d^2 g2  and the entry's depth cotangent  dcc dL_dD  becomes  dcc (dL_dD + 2 d g2) + [the
// entry is the pixel's median] gm  wherever it enters: the dL/dtz slot and, with RD, the dL/dp sums and  -p dL/dtz.
// The median entry is the forward's (its stored list position), never re-derived from the recomputed T.
template <int NG, int NW, int MINB, bool DET = false, bool GEOM = true, bool ABS = false, bool RD = false, bool DS = false>
__global__ void __launch_bounds__(32 * NW, MINB) composite_bwd_kernel(const CompositeBwdParams p) {
    static_assert(GEOM || !ABS, "absgrad needs the geometry half of the backward");
    static_assert(GEOM || !RD, "the depth plane's gradient needs the geometry half of the backward");
    static_assert(GEOM || !DS, "the depth statistics' gradients need the geometry half of the backward");
    constexpr int NC = 4 * NG;              // padded channel count {r,g,b,f...}; gradient row = 8 geometry slots + NC
    constexpr int GOFF = GEOM ? 8 : 0;      // slot of channel 0 in the gradient row (GEOM = false: no geometry slots)
    constexpr int ROWF = GOFF + NC + (RD ? 4 : 0);   // floats per gradient row (p.recf with GEOM); RD: + dL/dp group
    constexpr int RG = 2 + NG;
    constexpr int RGX = RG + (RD ? 1 : 0);  // staged record groups: RD adds the depth plane (group RG)
    // entries per sub-batch: 16, or 8 from NG = 6 on (static shared memory stays under 48 KB); lane l of the entry
    // phase sums entry l % E over the E pixels of part l / E
    constexpr int E = NG <= 5 ? 16 : 8;
    constexpr int PS = 33;                  // plane row stride
    constexpr int SROW = 4 * ((ROWF / 4) | 1);   // staged row stride: an odd number of float4, conflict-free stores
    static_assert(E * SROW <= 2 * E * PS, "the staged rows overlay the planes");
    constexpr int UP = 2;                   // entries per step of the pixel phase (divides E)
    __shared__ float4 sRec[NW][RGX][32];
    __shared__ uint32_t sId[NW][32];
    __shared__ uint32_t sK[NW][32];
    __shared__ uint32_t sQ[NW][R3DG_QCAP];
    __shared__ __align__(16) float sPl[NW][2 * E * PS];   // sW = [0, E PS), sC = [E PS, 2 E PS); then the staged rows
    __shared__ float4 sCot[NW][NG][32];                   // per pixel of the block its NC channel cotangents
    __shared__ float sCotD[NW][32];                       // and its depth cotangent
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int PARTS = 8 / NW;
    static_assert(PARTS == 2, "bwd_work / cta_order are per half tile");
    const int cta = (int)p.cta_order[blockIdx.x];
    const int tile = cta / PARTS;
    const int wb = (cta % PARTS) * NW + warp;
    const int tx = tile % p.gx, tyv = tile / p.gx;
    const int view = tyv / p.gy, ty = tyv - view * p.gy;          // the view's image and its view-local tile row
    const int bx0 = tx * R3DG_TILE + (wb & 1) * 8, by0 = ty * R3DG_TILE + (wb >> 1) * 4;
    const int px = bx0 + (lane & 7), py = by0 + (lane >> 3);
    const bool inside = px < p.W && py < p.H;
    const float pxf = (float)px, pyf = (float)py;
    const uint2 range = p.ranges[tile];
    const uint32_t lo = range.x;
    const size_t HW = (size_t)p.H * p.W, pix = (size_t)p.W * py + px, vpix = (size_t)view * HW + pix;
    const float4* __restrict__ rec4 = reinterpret_cast<const float4*>(p.rec);
    const int rec4n = p.recf >> 2;
    const uint32_t* __restrict__ plist = p.point_list + lo;
    uint32_t* q = sQ[warp];

    const float T_final = inside ? p.final_T[vpix] : 0.0f;
    float T = T_final;
    const int last_contributor = inside ? p.n_contrib[vpix] : 0;
    // nothing behind the warp's deepest last contributor matters to this warp
    int total = last_contributor;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) total = max(total, __shfl_xor_sync(0xffffffffu, total, o));
    total = min(total, (int)(range.y - range.x));
    if (total == 0) return;

    float dpix[NC];                                          // cotangents of channels {r,g,b,f0..} at this lane's pixel
#pragma unroll
    for (int c = 0; c < NC; ++c) {
        if (!inside) dpix[c] = 0.0f;
        else if (c < 3) dpix[c] = p.dL_dpix[(size_t)(3 * view + c) * HW + pix];
        else dpix[c] = c - 3 < p.S ? p.dL_dpix_f[((size_t)view * p.S + (c - 3)) * HW + pix] : 0.0f;
    }
    // GEOM = false: the opacity and depth cotangents have no appearance gradient and are not read
    const float dpix_d = GEOM && inside ? p.dL_dpix_d[vpix] : 0.0f;
    const float dpix_o = GEOM && inside ? p.dL_dpix_o[vpix] : 0.0f;
#pragma unroll
    for (int g = 0; g < NG; ++g) sCot[warp][g][lane] = make_float4(dpix[4 * g], dpix[4 * g + 1], dpix[4 * g + 2], dpix[4 * g + 3]);
    sCotD[warp][lane] = dpix_d;                              // (read by the entry phase after the first __syncwarp)
    // DS: this lane's pixel's depth2 and median cotangents and its median entry's 0-based list position (-1: none).
    // The entry phase reads them by shuffles from the pixel's lane (the static shared memory is at its 48 KB limit).
    const float dpix_d2 = DS && inside ? p.dL_dpix_d2[vpix] : 0.0f;
    const float dpix_d2x2 = 2.0f * dpix_d2;
    const float dpix_m = DS && inside ? p.dL_dpix_m[vpix] : 0.0f;
    const int pix_med = DS && inside ? p.median_pos[vpix] - 1 : -1;
    const float* bg = p.bg + 3 * view;
    const float bg_dot = GEOM ? bg[0] * dpix[0] + bg[1] * dpix[1] + bg[2] * dpix[2] : 0.0f;
    const float ddelx_dx = 0.5f * p.W, ddely_dy = 0.5f * p.H;
    const bool geo = p.backward_geometry != 0;
    int e_app = 0, e_geo = 0;
    if constexpr (DET) { e_app = det_scale_exp(p.det_scale[2 * view]); e_geo = det_scale_exp(p.det_scale[2 * view + 1]); }
    // The reference keeps, per channel, the colour accumulated BEHIND the current entry (accum_rec[ch], backward.cu:
    // 541-566) only to form  dL_dalpha = sum_ch (c_ch - accum_rec[ch]) * dL_dpix[ch].  With D = sum_ch c_ch * dL_dpix[ch]
    // (the entry's own channels, depth and opacity terms included) the same quantity is  D - A  where the ONE scalar
    // A = sum_ch accum_rec[ch] * dL_dpix[ch] obeys the same recurrence  A <- alpha * D + (1 - alpha) * A : one FMA per
    // channel instead of four, and no per-channel state (20 registers at S = 16).  Gradients are compared at 1e-3.
    float A = 0.0f;

    // ---- contributor-mask stream, descending: word w holds instances [4w, 4w+4); lane takes word w_next - lane -------
    const uint32_t hi = lo + (uint32_t)total;                 // instances [lo, hi) matter
    const long long w_low = (long long)(lo >> 2);             // lowest word of the tile
    long long w_next = (long long)((hi - 1u) >> 2);           // highest word still to scan
    uint32_t m_nxt = (w_next - lane >= w_low) ? p.cmask32[w_next - lane] : 0u;
    int qhead = 0, qcount = 0;
    auto scan_step = [&]() {
        const long long w = w_next - lane;
        uint32_t flags = 0u;
        if (w >= w_low) {
            flags = (m_nxt >> wb) & 0x01010101u;
            const uint32_t e0 = (uint32_t)w << 2;
            if (e0 < lo) flags &= 0xffffffffu << (8 * (lo - e0));
            if (e0 + 4 > hi) flags &= 0xffffffffu >> (8 * (e0 + 4 - hi));
        }
        w_next -= 32;
        m_nxt = (w_next - lane >= w_low) ? p.cmask32[w_next - lane] : 0u;
        uint32_t tot;
        uint32_t slot = (uint32_t)(qhead + qcount) + warp_excl_scan(__popc(flags), lane, tot);
        const uint32_t rel = ((uint32_t)w << 2) - lo;
#pragma unroll
        for (int k = 3; k >= 0; --k)                                              // back to front inside the word too
            if (flags & (1u << (8 * k))) { q[slot & (R3DG_QCAP - 1)] = rel + k; ++slot; }
        qcount += (int)tot;
    };
    while (qcount < 64 && w_next >= w_low) scan_step();
    __syncwarp();

    uint32_t id_cur = 0u, k_cur = 0u;
    float4 r[RGX];
#pragma unroll
    for (int g = 0; g < RGX; ++g) r[g] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (lane < qcount) {
        k_cur = q[(qhead + lane) & (R3DG_QCAP - 1)];
        id_cur = plist[k_cur];
#pragma unroll
        for (int g = 0; g < RGX; ++g) r[g] = rec4[(size_t)id_cur * rec4n + g];
    }

    float* const sW = sPl[warp];
    float* const sC = sPl[warp] + E * PS;
    const int le = lane % E, part = lane / E;               // entry phase: entry and pixel part of this lane
    while (qcount > 0) {
        const int n = min(32, qcount);
        __syncwarp();
        // element offset of the Gaussian's gradient row (ABS: the row index itself, also that of its absgrad pair)
        sId[warp][lane] = ABS ? id_cur : id_cur * (uint32_t)(GEOM ? p.recf : NC);
        sK[warp][lane] = k_cur;                                        // 0-based list position == contributor index
#pragma unroll
        for (int g = 0; g < RGX; ++g) sRec[warp][g][lane] = r[g];
        qhead = (qhead + n) & (R3DG_QCAP - 1);
        qcount -= n;
        while (qcount < 64 && w_next >= w_low) scan_step();
        __syncwarp();
        if (lane < qcount) {
            k_cur = q[(qhead + lane) & (R3DG_QCAP - 1)];
            id_cur = plist[k_cur];
#pragma unroll
            for (int g = 0; g < RGX; ++g) r[g] = rec4[(size_t)id_cur * rec4n + g];
        }
#pragma unroll 1
        for (int j0 = 0; j0 < n; j0 += E) {
            const int ne = min(E, n - j0);
            __syncwarp();                                   // the previous sub-batch's staged rows are added
            // ---- pixel phase, steps of UP entries for instruction-level parallelism: (1) everything that depends only
            // on the entry — exp(), alpha, 1/(1-alpha), the entry's own cotangent dot D — for all UP entries; (2) the two
            // short recurrences T and A in list order; (3) the plane stores.  Entries past the sub-batch are evaluated
            // with their gate closed.
#pragma unroll 1
            for (int u0 = 0; u0 < ne; u0 += UP) {
                bool valid[UP];
                float G[UP], alpha[UP], inv[UP], D[UP];
#pragma unroll
                for (int u = 0; u < UP; ++u) {                              // (1)
                    const int j = min(j0 + u0 + u, n - 1);
                    const int k = (int)sK[warp][j];
                    const float4 a = sRec[warp][0][j];
                    const float4 b = sRec[warp][1][j];
                    const float dx = sub_(a.x, pxf), dy = sub_(a.y, pyf);
                    const float qd = fma_(dx, mul_(dx, a.z), mul_(dy, mul_(dy, b.x)));
                    const float power = fma_(qd, -0.5f, -mul_(dy, mul_(dx, a.w)));
                    G[u] = expf(power);
                    alpha[u] = fminf(0.99f, mul_(b.y, G[u]));
                    // the same three tests as the forward pass (identical arithmetic) + "not behind this pixel's last
                    // contributor"
                    valid[u] = u0 + u < ne && k < last_contributor && !(power > 0.0f) && !(alpha[u] < 1.0f / 255.0f);
                    // a skipped entry of a non-positive-definite conic can have power > 88: expf = inf, and the gated
                    // product w (0 * inf) would be NaN.  Composited entries have power <= 0, so G <= 1 is unchanged.
                    G[u] = valid[u] ? G[u] : 0.0f;
                    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(inv[u]) : "f"(1.0f - alpha[u]));   // 1 - alpha in [0.01, 1]: one MUFU
                    float d = 0.0f;
                    if constexpr (GEOM) {
                        float dep = b.z;
                        if constexpr (RD) {                                 // the forward's plane depth
                            const float4 pl = sRec[warp][RG][j];
                            dep = fmaf(-pl.y, dy, fmaf(-pl.x, dx, b.z));
                        }
                        d = fmaf(dep, dpix_d, dpix_o);                      // depth * dL_ddepth + 1 * dL_dopacity
                        if constexpr (DS) d = fmaf(dep * dep, dpix_d2, d);  // + depth^2 * dL_ddepth2
                        const float4 c0 = sRec[warp][2][j], t0 = sCot[warp][0][lane];
                        d = fmaf(c0.z, t0.z, fmaf(c0.y, t0.y, fmaf(c0.x, t0.x, d)));
                        // feature channels enter dL_dalpha only when backward_geometry is set (backward.cu:563-566)
                        if (geo) {
                            d = fmaf(c0.w, t0.w, d);
#pragma unroll
                            for (int g = 1; g < NG; ++g) {
                                const float4 c4 = sRec[warp][2 + g][j], t = sCot[warp][g][lane];
                                d = fmaf(c4.w, t.w, fmaf(c4.z, t.z, fmaf(c4.y, t.y, fmaf(c4.x, t.x, d))));
                            }
                        }
                    }
                    D[u] = d;
                }
#pragma unroll
                for (int u = 0; u < UP; ++u) {                              // (2) branch-free: lanes that did not composite
                    const float gate = valid[u] ? 1.0f : 0.0f;              // the entry contribute zeros and keep their state
                    const float Tn = T * inv[u];                            // T before this entry (backward.cu:533)
                    sC[(u0 + u) * PS + lane] = gate * alpha[u] * Tn;        // (3)
                    if constexpr (GEOM) {
                        const float dL_dalpha = gate * fmaf(D[u] - A, Tn, -(T_final * inv[u]) * bg_dot);
                        sW[(u0 + u) * PS + lane] = G[u] * dL_dalpha;
                        if (valid[u]) { A = fmaf(alpha[u], D[u] - A, A); T = Tn; } // A <- alpha D + (1 - alpha) A
                    } else if (valid[u]) {
                        T = Tn;
                    }
                }
            }
            __syncwarp();
            // ---- entry phase: lane sums entry le over pixels [part E, part E + E) (pixel rows of 8)
            const int je = min(j0 + le, n - 1);
            const float4 a = sRec[warp][0][je];
            const float4 b = sRec[warp][1][je];
            constexpr int ROWS = E / 8;
            float sw = 0.f, s0 = 0.f, s1 = 0.f, sxx = 0.f, sxy = 0.f, syy = 0.f, sd = 0.f, ax = 0.f, ay = 0.f;
            float sdx = 0.f, sdy = 0.f;                                     // RD: sums of dcc dL_dD dx, dcc dL_dD dy
            const float4 pl = RD ? sRec[warp][RGX - 1][je] : make_float4(0.f, 0.f, 0.f, 0.f);
            const int ke = DS ? (int)sK[warp][je] : 0;                     // DS: the entry's list position
            float sc[NC];
#pragma unroll
            for (int c = 0; c < NC; ++c) sc[c] = 0.0f;
#pragma unroll 1
            for (int rr = part * ROWS; rr < (part + 1) * ROWS; ++rr) {      // pixel rows of this lane's part
              const float dy = sub_(a.y, (float)(by0 + rr));
              const float* pw = sW + le * PS + 8 * rr;
              const float* pc = sC + le * PS + 8 * rr;
#pragma unroll 2                                                    // (more unrolling spills at 5 CTAs per SM)
              for (int i = 0; i < 8; ++i) {
                const int pb = 8 * rr + i;                                  // pixel of the block
                const float c = pc[i];
                if constexpr (GEOM) {
                    const float w = pw[i], dx = sub_(a.x, (float)(bx0 + i));   // the pixel phase's dx, dy
                    // the two dL/dmean2D terms per pixel (unfused: ABS sums their magnitudes in the same order, so that
                    // |signed sum| <= sum of magnitudes holds bit for bit); the conic terms from centred moments
                    const float t0 = mul_(w, fmaf(a.z, dx, mul_(a.w, dy))), t1 = mul_(w, fmaf(b.x, dy, mul_(a.w, dx)));
                    s0 = add_(s0, t0); s1 = add_(s1, t1);
                    const float wdx = w * dx, wdy = w * dy;
                    sw += w;
                    sxx = fmaf(wdx, dx, sxx); sxy = fmaf(wdx, dy, sxy); syy = fmaf(wdy, dy, syy);
                    // the entry's depth cotangent at the pixel: dcc dL_dD (DS: dcc (dL_dD + 2 d g2) + [median] gm)
                    float cot = sCotD[warp][pb], gm = 0.0f;
                    bool is_med = false;
                    if constexpr (DS) {
                        const float dd = RD ? fmaf(-pl.y, dy, fmaf(-pl.x, dx, b.z)) : b.z;   // the forward's d
                        cot = fmaf(dd, __shfl_sync(0xffffffffu, dpix_d2x2, pb), cot);
                        is_med = __shfl_sync(0xffffffffu, pix_med, pb) == ke;
                        gm = __shfl_sync(0xffffffffu, dpix_m, pb);
                    }
                    sd = fmaf(c, cot, sd);
                    if (DS && is_med) sd = add_(sd, gm);
                    if constexpr (RD) {
                        float cd = c * cot;
                        if (DS && is_med) cd = add_(cd, gm);
                        sdx = fmaf(cd, dx, sdx); sdy = fmaf(cd, dy, sdy);
                        if constexpr (ABS) {                                // the pixel's whole dL/dmean2D term / (W/2)
                            ax = add_(ax, fabsf(fmaf(b.y, t0, pl.x * cd))); ay = add_(ay, fabsf(fmaf(b.y, t1, pl.y * cd)));
                        }
                    } else if constexpr (ABS) {
                        ax = add_(ax, fabsf(t0)); ay = add_(ay, fabsf(t1));
                    }
                }
#pragma unroll
                for (int g = 0; g < NG; ++g) {
                    const float4 t = sCot[warp][g][pb];
                    sc[4 * g + 0] = fmaf(c, t.x, sc[4 * g + 0]);
                    sc[4 * g + 1] = fmaf(c, t.y, sc[4 * g + 1]);
                    sc[4 * g + 2] = fmaf(c, t.z, sc[4 * g + 2]);
                    sc[4 * g + 3] = fmaf(c, t.w, sc[4 * g + 3]);
                }
              }
            }
#pragma unroll
            for (int m = E; m < 32; m <<= 1) {                              // join the pixel parts
#pragma unroll
                for (int c = 0; c < NC; ++c) sc[c] += __shfl_xor_sync(0xffffffffu, sc[c], m);
                if constexpr (GEOM) {
                    sw += __shfl_xor_sync(0xffffffffu, sw, m);
                    s0 += __shfl_xor_sync(0xffffffffu, s0, m);
                    s1 += __shfl_xor_sync(0xffffffffu, s1, m);
                    sxx += __shfl_xor_sync(0xffffffffu, sxx, m);
                    sxy += __shfl_xor_sync(0xffffffffu, sxy, m);
                    syy += __shfl_xor_sync(0xffffffffu, syy, m);
                    sd += __shfl_xor_sync(0xffffffffu, sd, m);
                }
                if constexpr (RD) {
                    sdx += __shfl_xor_sync(0xffffffffu, sdx, m);
                    sdy += __shfl_xor_sync(0xffffffffu, sdy, m);
                }
                if constexpr (ABS) {
                    ax += __shfl_xor_sync(0xffffffffu, ax, m);
                    ay += __shfl_xor_sync(0xffffffffu, ay, m);
                }
            }
            float row[ROWF];
            if constexpr (GEOM) {
                const float o = b.y, ho = -0.5f * o;                        // dL_dG = o dL_dalpha
                row[0] = mul_(-(o * ddelx_dx), s0);                         // sum dL_dG dG_ddelx W/2
                row[1] = mul_(-(o * ddely_dy), s1);
                row[2] = sd;
                row[3] = sw;
                row[4] = ho * sxx; row[5] = ho * sxy; row[6] = ho * syy;
                row[7] = 0.0f;
                if constexpr (RD) {                                         // d's own dependence on the mean: -p dL/dtz
                    row[0] = fmaf(-(ddelx_dx * pl.x), sd, row[0]);
                    row[1] = fmaf(-(ddely_dy * pl.y), sd, row[1]);
                    row[GOFF + NC] = -sdx; row[GOFF + NC + 1] = -sdy;       // dL/dp = sum dcc dL_dD (pixel - mean)
                    row[GOFF + NC + 2] = 0.0f; row[GOFF + NC + 3] = 0.0f;
                }
            }
#pragma unroll
            for (int c = 0; c < NC; ++c) row[GOFF + c] = sc[c];
            if constexpr (ABS) {                                            // lane: pair component part & 1 of entry le
                if (part < 2 && le < ne) {
                    const float v = RD ? (part ? mul_(ddely_dy, ay) : mul_(ddelx_dx, ax))
                                       : (part ? mul_(fabsf(b.y) * ddely_dy, ay) : mul_(fabsf(b.y) * ddelx_dx, ax));
                    const size_t ai = 2 * (size_t)sId[warp][j0 + le] + part;
                    if constexpr (DET) det_add(p.det_abs, ai, v, e_geo);
                    else atomicAdd(p.abs_grad + ai, v);
                }
            }
            __syncwarp();                                                   // every lane has read the planes
            constexpr int CH = ROWF / 4, NPART = 32 / E;
#pragma unroll
            for (int c4 = 0; c4 < CH; ++c4)
                if (c4 % NPART == part)
                    *reinterpret_cast<float4*>(sPl[warp] + le * SROW + 4 * c4) =
                        make_float4(row[4 * c4], row[4 * c4 + 1], row[4 * c4 + 2], row[4 * c4 + 3]);
            __syncwarp();
            if constexpr (DET) {                                            // one fixed-point add per real component
#pragma unroll 1
                for (int i = lane; i < ne * ROWF; i += 32) {
                    const int e = i / ROWF, s = i - e * ROWF;
                    const bool plane = RD && s >= GOFF + NC;                // RD: the dL/dp group, geometry class
                    if ((GEOM && s == 7) || (!plane && s >= GOFF && s - GOFF >= 3 + p.S) || (plane && s >= GOFF + NC + 2)) continue;
                    const size_t row0 = ABS ? (size_t)sId[warp][j0 + e] * p.recf : (size_t)sId[warp][j0 + e];
                    det_add(p.det, row0 + s, sPl[warp][e * SROW + s], s < GOFF || plane ? e_geo : e_app);
                }
            } else {                                                        // 32 float4 segments per instruction
#pragma unroll 1
                for (int i = lane; i < ne * CH; i += 32) {
                    const int e = i / CH, c4 = i - e * CH;
                    if (4 * c4 >= GOFF && 4 * c4 - GOFF >= 3 + p.S && !(RD && 4 * c4 >= GOFF + NC)) continue;   // padding channels only
                    const size_t row0 = ABS ? (size_t)sId[warp][j0 + e] * p.recf : (size_t)sId[warp][j0 + e];
                    atomicAdd(reinterpret_cast<float4*>(p.grad + row0) + c4,
                              *reinterpret_cast<const float4*>(sPl[warp] + e * SROW + 4 * c4));
                }
            }
        }
    }
}

// DET: the largest |cotangent| of each of the V views as float bits, combined by atomicMax (exact, order-independent)
// into the zeroed scale words: scale[2 v] over the colour and feature planes, the cotangents of the colour / feature
// slots (dcc * dL_dpix); scale[2 v + 1] over those and the opacity and depth planes (the surface pull-back already
// added), every plane the geometry slots are linear in.  GEOM = false reads only the former.  The compositor and the
// kernels that read its rows take the class exponents from these words (det_scale_exp): a V-view call scales each
// view as its one-view call does.  Every thread of the first `nblocks` blocks calls it (256 threads each): one
// atomicMax per block and word.
// Depth statistics (p.depth_bound set): the cotangents of depth2 and of the median depth join the geometry class.  A
// depth2 term carries d^2 g2 (in dL/dalpha) or 2 d g2 (in the depth cotangent), so its plane enters as
// |g2| max(Z^2, 2 Z) with Z the view's largest |d| of an accepted entry (from the forward): scaled by the class
// exponent, every new term is then bounded as the flag-off ones are (DESIGN.md §4.21).  A product beyond fp32 enters
// as FLT_MAX (the exponent clamps at R3DG_DET_SCALE_MAX); a zero cotangent enters as 0, so that zero cotangents leave
// the exponent, and every bit of the result, as without the statistics.
__device__ void det_scale_reduce(const CompositeBwdParams& p, int V, bool geometry, int nblocks, uint32_t* __restrict__ scale) {
    __shared__ uint32_t s_max[2][8];
    const bool ds = geometry && p.depth_bound != nullptr;
    const size_t HW = (size_t)p.H * p.W, n_app = (size_t)(3 + p.S) * HW, n = n_app + (geometry ? (ds ? 4 : 2) * HW : 0);
    const size_t stride = (size_t)nblocks * blockDim.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int v = 0; v < V; ++v) {
        const float* col = p.dL_dpix + (size_t)v * 3 * HW;
        const float* feat = p.dL_dpix_f + (size_t)v * p.S * HW;
        uint32_t m_app = 0u, m_geo = 0u;
        float zf = 0.0f;                                         // DS: max(Z^2, 2 Z)
        if (ds) { const float z = __uint_as_float(p.depth_bound[v]); zf = fmaxf(z * z, 2.0f * z); }
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
            if (i < 3 * HW) m_app = max(m_app, det_abs_bits(col[i]));
            else if (i < n_app) m_app = max(m_app, det_abs_bits(feat[i - 3 * HW]));
            else if (i < n_app + HW) m_geo = max(m_geo, det_abs_bits(p.dL_dpix_o[(size_t)v * HW + (i - n_app)]));
            else if (i < n_app + 2 * HW) m_geo = max(m_geo, det_abs_bits(p.dL_dpix_d[(size_t)v * HW + (i - n_app - HW)]));
            else if (i < n_app + 3 * HW) {
                const float g = p.dL_dpix_d2[(size_t)v * HW + (i - n_app - 2 * HW)];
                const uint32_t b = g == 0.0f ? 0u : (g != g ? det_abs_bits(g) : det_abs_bits(fminf(fabsf(g) * zf, 3.40282347e38f)));
                m_geo = max(m_geo, b);
            } else {
                m_geo = max(m_geo, det_abs_bits(p.dL_dpix_m[(size_t)v * HW + (i - n_app - 3 * HW)]));
            }
        }
        m_geo = max(m_app, m_geo);
        m_app = __reduce_max_sync(0xffffffffu, m_app);
        m_geo = __reduce_max_sync(0xffffffffu, m_geo);
        if (lane == 0) { s_max[0][warp] = m_app; s_max[1][warp] = m_geo; }
        __syncthreads();
        if (warp == 0) {
            const uint32_t a = lane < 8 ? s_max[0][lane] : 0u, g = lane < 8 ? s_max[1][lane] : 0u;
            det_max_bits(scale + 2 * v, a);
            det_max_bits(scale + 2 * v + 1, g);
        }
        __syncthreads();
    }
}

// Zeroes the gradient rows the kernel above adds to: exactly the rows the forward pass composited (kComposited), since
// it walks only their contributor bits.  Every other row is neither written nor read in the backward, so ~80 % of the
// rows of a dense scene are never touched.  One thread per row.  DET: the row's accumulators in the three word planes
// and its flag bits, which are recf / 4 whole bytes (2 bits per accumulator, recf a multiple of 4); and, before that,
// the views' cotangent scale (det_scale_reduce) into the scale words the caller zeroed.  Absgrad (p.abs_grad or
// p.det_abs set): also the row's pair of absgrad sums; in DET mode their flag bits, 8 rows to a word, are zeroed whole
// by the first thread of each 8 rows (the flags of rows that are not composited are never read).
template <bool DET>
__global__ void __launch_bounds__(256) zero_composited_rows_kernel(size_t rows, int recf, const uint8_t* __restrict__ clamped,
                                                                   float* __restrict__ grad, const DetAcc det,
                                                                   const CompositeBwdParams p, int V, bool geometry, int nred) {
    const size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if constexpr (DET) {
        if ((int)blockIdx.x < nred) det_scale_reduce(p, V, geometry, nred, const_cast<uint32_t*>(p.det_scale));   // (block-uniform)
    }
    if constexpr (DET) {
        if (p.det_abs.words && (r & 7) == 0 && r < rows) p.det_abs.flags[r >> 3] = 0u;
    }
    if (r >= rows || !(clamped[r] & kComposited)) return;
    if constexpr (DET) {
        if (p.det_abs.words) {
#pragma unroll 1
            for (int plane = 0; plane < 3; ++plane)
                *reinterpret_cast<uint4*>(p.det_abs.words + plane * p.det_abs.n + 2 * r) = make_uint4(0u, 0u, 0u, 0u);
        }
#pragma unroll 1
        for (int plane = 0; plane < 3; ++plane) {
            uint4* w = reinterpret_cast<uint4*>(det.words + plane * det.n + r * recf);
            for (int i = 0; i < recf / 2; ++i) w[i] = make_uint4(0u, 0u, 0u, 0u);
        }
        uint8_t* f = reinterpret_cast<uint8_t*>(det.flags) + r * (recf / 4);
        for (int i = 0; i < recf / 4; ++i) f[i] = 0;
    } else {
        if (p.abs_grad) { p.abs_grad[2 * r] = 0.0f; p.abs_grad[2 * r + 1] = 0.0f; }
        float4* g = reinterpret_cast<float4*>(grad + r * recf);
        for (int i = 0; i < recf / 4; ++i) g[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

DetAcc raster_det_abs(const r3dg_raster_bwd_args& a, size_t rows, int recf) {
    return det_acc((char*)a.det_work + det_bytes(rows * recf), 2 * rows);   // behind r3dg_raster_(ray_depth_)bwd_det_bytes
}

uint32_t* raster_det_scale(const RasterBuffers& b) {
    return reinterpret_cast<uint32_t*>(b.grad - (size_t)b.row_base * b.recf);     // the whole call's grad region
}

// resident CTAs per SM the register allocation is pinned to, by channel groups NG: the most at which no instantiation
// (DET x GEOM x ABS) spills (DESIGN.md §4.2)
template <int NG> struct BwdOcc { static constexpr int v = NG <= 2 ? 5 : (NG <= 4 ? 4 : 3); };
// ray-depth mode (two more entry-phase sums and the depth plane): one CTA fewer where the count above spills
template <int NG> struct BwdOccRD { static constexpr int v = BwdOcc<NG>::v - (NG == 1 || NG == 2 || NG == 4 ? 1 : 0); };
// depth statistics (three more per-pixel planes read by the entry phase), without and with the ray-depth mode: fewer
// CTAs where the counts above spill
template <int NG, bool RD> struct BwdOccDS {
    static constexpr int v = RD ? BwdOccRD<NG>::v - (NG == 3 || NG == 7 ? 1 : 0) : BwdOcc<NG>::v - (NG == 2 || NG == 4 ? 1 : 0);
};
int g_bwd_ctas = 0;             // r3dg_tune("composite_bwd_ctas"): resident CTAs per SM (0 = whatever fits)
int composite_bwd_tune(const char* key, int value, int* previous) {
    if (strcmp(key, "composite_bwd_ctas") != 0) return R3DG_ERR_UNSUPPORTED;
    if (previous) *previous = g_bwd_ctas;
    if (value < 0 || value > 32) return R3DG_ERR_BAD_ARG;
    g_bwd_ctas = value;
    return 0;
}
template <int NG, bool DET, bool GEOM, bool ABS = false, bool RD = false, bool DS = false>
static void launch_bwd_kernel(const CompositeBwdParams& p, int tiles, cudaStream_t stream) {
    constexpr int minb = DS ? BwdOccDS<NG, RD>::v : (RD ? BwdOccRD<NG>::v : BwdOcc<NG>::v);
    constexpr auto kernel = composite_bwd_kernel<NG, 4, minb, DET, GEOM, ABS, RD, DS>;
    kernel<<<tiles * 2, 128, residency_pad<kernel>(g_bwd_ctas), stream>>>(p);    // two 4-warp CTAs per tile
}
template <int NG>
static void launch_bwd_ng(const CompositeBwdParams& p, int tiles, bool det, bool geometry, bool absgrad, bool rd,
                          bool ds, cudaStream_t stream) {
    if (geometry && ds) {                             // (absgrad implies geometry)
        if (rd) {
            if (absgrad) det ? launch_bwd_kernel<NG, true, true, true, true, true>(p, tiles, stream) : launch_bwd_kernel<NG, false, true, true, true, true>(p, tiles, stream);
            else det ? launch_bwd_kernel<NG, true, true, false, true, true>(p, tiles, stream) : launch_bwd_kernel<NG, false, true, false, true, true>(p, tiles, stream);
        } else {
            if (absgrad) det ? launch_bwd_kernel<NG, true, true, true, false, true>(p, tiles, stream) : launch_bwd_kernel<NG, false, true, true, false, true>(p, tiles, stream);
            else det ? launch_bwd_kernel<NG, true, true, false, false, true>(p, tiles, stream) : launch_bwd_kernel<NG, false, true, false, false, true>(p, tiles, stream);
        }
        return;
    }
    if (geometry && rd) {                             // (absgrad implies geometry)
        if (absgrad) det ? launch_bwd_kernel<NG, true, true, true, true>(p, tiles, stream) : launch_bwd_kernel<NG, false, true, true, true>(p, tiles, stream);
        else det ? launch_bwd_kernel<NG, true, true, false, true>(p, tiles, stream) : launch_bwd_kernel<NG, false, true, false, true>(p, tiles, stream);
        return;
    }
    if (absgrad) det ? launch_bwd_kernel<NG, true, true, true>(p, tiles, stream) : launch_bwd_kernel<NG, false, true, true>(p, tiles, stream);
    else if (geometry) det ? launch_bwd_kernel<NG, true, true>(p, tiles, stream) : launch_bwd_kernel<NG, false, true>(p, tiles, stream);
    else det ? launch_bwd_kernel<NG, true, false>(p, tiles, stream) : launch_bwd_kernel<NG, false, false>(p, tiles, stream);
}

int composite_bwd_row_floats(int S, bool geometry) { return geometry ? rec_floats(S) : 4 * num_groups(S); }

int launch_composite_backward(const r3dg_raster_bwd_args& a, const RasterBuffers& b, bool geometry, cudaStream_t stream) {
    CompositeBwdParams p;
    const int V = b.V;
    p.W = a.W; p.H = a.H; p.gx = b.gx; p.gy = b.gy; p.S = a.S; p.recf = b.recf;
    p.backward_geometry = a.backward_geometry;
    p.ranges = b.ranges;
    p.point_list = b.point_list; p.cmask32 = (const uint32_t*)b.cmask;
    p.header = b.header;
    p.cta_order = b.bwd_order;
    p.rec = b.rec;
    p.bg = a.background;
    p.final_T = b.final_T;
    p.dL_dpix = a.dL_dout_color; p.dL_dpix_o = a.dL_dout_opacity; p.dL_dpix_d = a.dL_dout_depth;
    p.dL_dpix_f = a.dL_dout_feature;
    // depth statistics (geometry only: the appearance-only backward reads neither cotangent)
    const bool ds = geometry && a.depth_stats != 0;
    p.dL_dpix_d2 = ds ? a.dL_dout_depth2 : nullptr; p.dL_dpix_m = ds ? a.dL_dout_median_depth : nullptr;
    p.median_pos = b.median_pos; p.depth_bound = ds ? b.depth_bound : nullptr;
    p.grad = b.grad;
    p.n_contrib = b.n_contrib;
    const bool det = a.deterministic != 0;
    const size_t rows = (size_t)V * a.P;
    const int gradf = geometry ? b.recf : composite_bwd_row_floats(a.S, false);   // the gradient row: b.recf, or NC without geometry
    p.det = det_acc(a.det_work, rows * gradf);
    p.det_scale = det ? raster_det_scale(b) : nullptr;
    // absgrad (geometry only; the appearance-only backward ignores dL_dmeans2D_abs): the default mode adds into the
    // output itself, DET mode into its own accumulators behind the gradient rows' in det_work
    const bool absgrad = geometry && a.dL_dmeans2D_abs != nullptr;
    p.abs_grad = absgrad && !det ? a.dL_dmeans2D_abs : nullptr;
    p.det_abs = absgrad && det ? raster_det_abs(a, rows, b.recf) : det_acc(nullptr, 0);
    // zeroed here, in the backward, so that every backward over one forward (retain_graph) starts from zero
    const int zblocks = (int)((rows + 255) / 256);
    if (det) {
        R3DG_CUDA_TRY(cudaMemsetAsync(const_cast<uint32_t*>(p.det_scale), 0, 2 * (size_t)V * sizeof(uint32_t), stream));
        const int nred = std::min(zblocks, 4 * num_sms());          // the blocks that also reduce the cotangent scale
        zero_composited_rows_kernel<true><<<zblocks, 256, 0, stream>>>(rows, gradf, b.clamped, p.grad, p.det, p, V, geometry, nred);
    } else {
        zero_composited_rows_kernel<false><<<zblocks, 256, 0, stream>>>(rows, gradf, b.clamped, p.grad, p.det, p, V, geometry, 0);
    }
    const int tiles = V * b.tiles;                    // the tall grid of all views
    int rc = launch_cta_order(b.bwd_work, b.bwd_order, 2 * tiles, stream);
    if (rc != 0) return rc;
    const bool rd = a.ray_depth != 0;
    switch (num_groups(a.S)) {
        case 1: launch_bwd_ng<1>(p, tiles, det, geometry, absgrad, rd, ds, stream); break;
        case 2: launch_bwd_ng<2>(p, tiles, det, geometry, absgrad, rd, ds, stream); break;
        case 3: launch_bwd_ng<3>(p, tiles, det, geometry, absgrad, rd, ds, stream); break;
        case 4: launch_bwd_ng<4>(p, tiles, det, geometry, absgrad, rd, ds, stream); break;
        case 5: launch_bwd_ng<5>(p, tiles, det, geometry, absgrad, rd, ds, stream); break;
        case 6: launch_bwd_ng<6>(p, tiles, det, geometry, absgrad, rd, ds, stream); break;
        case 7: launch_bwd_ng<7>(p, tiles, det, geometry, absgrad, rd, ds, stream); break;
        default: return R3DG_ERR_UNSUPPORTED;   // S > 24: reference backward limit (backward.cu:449)
    }
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace r3dg
