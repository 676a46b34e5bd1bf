// Stage 2 backward: per-tile back-to-front re-traversal (reference K10, backward.cu:401-614).
//
// Design notes
//  * the reference issues 10+S global atomicAdds per contributing (pixel, Gaussian) pair.  Here a
//    warp (8x4 pixels) first reduces its 32 per-pixel gradient rows with transposed butterflies
//    ("reduce-scatter": ~V shuffles for V values instead of 5V), after which every lane holds one
//    finished component and the warp adds the whole per-Gaussian gradient row with ONE reduction
//    instruction into a packed [P][RECF] row (2-4 sectors).  The colour / feature components are
//    all  (alpha T) * dL_dpix[c] : each lane keeps its dL_dpix in a lane-specific PERMUTED order,
//    so that what a lane sends and what it keeps at every butterfly level sit in fixed registers —
//    no select instructions (reduce_scatter_permuted); only the 7 geometry components pay them;
//  * warps are autonomous (no CTA barrier; see composite.cu): each walks ONLY the entries whose
//    contributor bit the forward pass set for its pixel block, back to front from the block's
//    deepest last contributor — no culling test, no record fetch, no exp() for anything else;
//  * CTAs are launched in the order of the work the forward pass measured (cta_order_kernel), and
//    the walk is laid out in rounds of U entries for instruction-level parallelism: the kernel is
//    bound by per-warp latency and its heaviest warps (DESIGN.md §4.2);
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

// entries per round of the backward walk (composite_bwd_kernel): 2 for S <= 5, 1 for S > 5 (twice the accumulators:
// registers)
template <int NG> struct BwdIlp { static constexpr int v = NG <= 2 ? 2 : 1; };

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
};

// Sum v[i] over the 32 lanes for every i in [0,N) (N power of two, 4 <= N <= 32) with a
// transposed butterfly; on return lane l holds the total of component (l >> (5 - log2 N)).
template <int N>
__device__ __forceinline__ float reduce_scatter(float (&v)[N], int lane) {
    int m = 16;
#pragma unroll
    for (int n = N; n > 1; n >>= 1) {
        const bool upper = (lane & m) != 0;
#pragma unroll
        for (int i = 0; i < n / 2; ++i) {
            const float send = upper ? v[i] : v[i + n / 2];
            const float keep = upper ? v[i + n / 2] : v[i];
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, m);
        }
        m >>= 1;
    }
    float r = v[0];
#pragma unroll
    for (int mm = 16 / N; mm > 0; mm >>= 1) r += __shfl_xor_sync(0xffffffffu, r, mm);
    return r;
}

// U independent reduce-scatters advanced level by level together: U shuffle chains in flight instead of one (the last
// levels of a single butterfly are one dependent SHFL -> FADD after the other).
template <int U, int N>
__device__ __forceinline__ void reduce_scatter_multi(float (&v)[U][N], int lane, float (&r)[U]) {
    int m = 16;
#pragma unroll
    for (int n = N; n > 1; n >>= 1) {
        const bool upper = (lane & m) != 0;
#pragma unroll
        for (int i = 0; i < n / 2; ++i) {
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const float send = upper ? v[u][i] : v[u][i + n / 2];
                const float keep = upper ? v[u][i + n / 2] : v[u][i];
                v[u][i] = keep + __shfl_xor_sync(0xffffffffu, send, m);
            }
        }
        m >>= 1;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) r[u] = v[u][0];
#pragma unroll
    for (int mm = 16 / N; mm > 0; mm >>= 1) {
#pragma unroll
        for (int u = 0; u < U; ++u) r[u] += __shfl_xor_sync(0xffffffffu, r[u], mm);
    }
}

// The same reduce-scatter without selects, for W values whose slot order the caller chose per lane: slot p of lane l
// must hold component  p ^ (~(l >> (5 - log2 W)) & (W - 1)).  At level n every lane sends slots [0, n/2) and keeps
// [n/2, n): with that order the kept slot i + n/2 and the partner's sent slot i are the same component.  On return
// lane l holds the total of component  l >> (5 - log2 W)  (as reduce_scatter).
template <int W>
__device__ __forceinline__ float reduce_scatter_permuted(float (&x)[W]) {
    int m = 16;
#pragma unroll
    for (int n = W; n > 1; n >>= 1) {
#pragma unroll
        for (int i = 0; i < n / 2; ++i) x[i] = x[i + n / 2] + __shfl_xor_sync(0xffffffffu, x[i], m);
        m >>= 1;
    }
    float r = x[0];
#pragma unroll
    for (int mm = 16 / W; mm > 0; mm >>= 1) r += __shfl_xor_sync(0xffffffffu, r, mm);
    return r;
}

template <int U, int W>
__device__ __forceinline__ void reduce_scatter_permuted_multi(float (&x)[U][W], float (&r)[U]) {
    int m = 16;
#pragma unroll
    for (int n = W; n > 1; n >>= 1) {
#pragma unroll
        for (int i = 0; i < n / 2; ++i) {
#pragma unroll
            for (int u = 0; u < U; ++u) x[u][i] = x[u][i + n / 2] + __shfl_xor_sync(0xffffffffu, x[u][i], m);
        }
        m >>= 1;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) r[u] = x[u][0];
#pragma unroll
    for (int mm = 16 / W; mm > 0; mm >>= 1) {
#pragma unroll
        for (int u = 0; u < U; ++u) r[u] += __shfl_xor_sync(0xffffffffu, r[u], mm);
    }
}

// Per warp (one 8x4 pixel block): the forward pass left one contributor bit per (instance, block).  The warp streams
// its tile's contributor bytes BACK TO FRONT, 128 instances per step, compacts the positions whose bit is set into a
// circular queue (warp scan) and processes batches of 32 of them: every staged entry is one that some pixel of the
// block composited in the forward pass — no culling test, no record fetch and no exp() for anything else.
// DET (deterministic mode): each finished row component is added through the order-independent fixed-point primitive
// (detacc.cuh) into p.det instead of by a float atomic into p.grad, scaled by its view's exponent of the colour /
// feature slots or of the geometry slots (det_scale_reduce).  Everything else is the same code.
// GEOM = false (appearance-only backward, no geometry gradient requested): the same walk, CTA order and alpha / T
// arithmetic, but only the NC colour and feature components are formed and reduced — no dL/dalpha, no A recurrence, no
// geometry butterfly — into a narrower row of NC floats (channel c at slot c).  Every channel component goes through the
// same butterfly as with GEOM, so each added value, and in DET mode each row total, is bitwise the full kernel's.
// ABS (absgrad, GEOM only): each lane also takes the magnitudes |v0[0]|, |v0[1]| of its pixel's two dL/dmean2D terms
// (0 on gated lanes) before the geometry butterfly sums the signed terms away; one more 2-wide butterfly reduces them
// over the warp's 32 pixels, and lanes 0 and 16 add the two totals to p.abs_grad (DET: p.det_abs, class exponent
// e_geo) once per entry.  Everything else, the gradient row included, is the same code.
template <int NG, int NW, int MINB, bool DET = false, bool GEOM = true, bool ABS = false>
__global__ void __launch_bounds__(32 * NW, MINB) composite_bwd_kernel(const CompositeBwdParams p) {
    static_assert(GEOM || !ABS, "absgrad needs the geometry half of the backward");
    constexpr int NC = 4 * NG;              // padded channel count {r,g,b,f...}; gradient row = 8 geometry slots + NC
    constexpr int GOFF = GEOM ? 8 : 0;      // slot of channel 0 in the gradient row (GEOM = false: no geometry slots)
    // the NC channel components are reduced in power-of-two chunks of 16 / 8 / 4 (select-free butterflies)
    constexpr int C16 = NC >= 16 ? 16 : 0, C8 = (NC - C16) >= 8 ? 8 : 0, C4 = NC - C16 - C8;
    constexpr int B8 = C16, B4 = C16 + C8;
    static_assert(C4 == 0 || C4 == 4, "channel groups come in fours");
    constexpr int RG = 2 + NG;
    constexpr int U = BwdIlp<NG>::v;                 // entries per round of the walk below
    __shared__ float4 sRec[NW][RG][32];
    __shared__ uint32_t sId[NW][32];
    __shared__ uint32_t sK[NW][32];
    __shared__ uint32_t sQ[NW][R3DG_QCAP];
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

    auto load_dpix = [&](int c) -> float {                   // cotangent of channel c of {r,g,b,f0..} at this lane's pixel
        if (!inside) return 0.0f;
        if (c < 3) return p.dL_dpix[(size_t)(3 * view + c) * HW + pix];
        return c - 3 < p.S ? p.dL_dpix_f[((size_t)view * p.S + (c - 3)) * HW + pix] : 0.0f;
    };
    float dpix[NC];
#pragma unroll
    for (int c = 0; c < NC; ++c) dpix[c] = load_dpix(c);
    // the same cotangents in this lane's butterfly slot order (reduce_scatter_permuted), one array per chunk
    float cst16[C16 ? C16 : 1], cst8[C8 ? C8 : 1], cst4[C4 ? C4 : 1];
    if constexpr (C16 > 0) {
        const int K = ~(lane >> 1) & 15;
#pragma unroll
        for (int i = 0; i < 16; ++i) cst16[i] = load_dpix(i ^ K);
    }
    if constexpr (C8 > 0) {
        const int K = ~(lane >> 2) & 7;
#pragma unroll
        for (int i = 0; i < 8; ++i) cst8[i] = load_dpix(B8 + (i ^ K));
    }
    if constexpr (C4 > 0) {
        const int K = ~(lane >> 3) & 3;
#pragma unroll
        for (int i = 0; i < 4; ++i) cst4[i] = load_dpix(B4 + (i ^ K));
    }
    // which finished component this lane adds to the Gaussian's gradient row: geometry slot lane >> 2 on lanes 0 mod 4,
    // the 16-chunk on odd lanes, the 8-chunk on lanes 2 mod 4, the 4-chunk on a free lane class (second instruction
    // only when all three chunks exist, NG == 7, and the geometry slots take lanes 0 mod 4; without them the 4-chunk
    // takes lanes 0 mod 8)
    constexpr bool C4_SECOND = GEOM && C16 > 0 && C8 > 0 && C4 > 0;
    constexpr int C4_CLASS = C16 > 0 ? (C8 > 0 ? 0 : 2) : 1;
    int my_sel = -1, my_off = 0;
    if ((lane & 3) == 0) { if (GEOM && (lane >> 2) != 7) { my_sel = 0; my_off = lane >> 2; } }
    else if (C16 > 0 && (lane & 1)) { my_sel = 1; my_off = GOFF + (lane >> 1); }
    else if (C8 > 0 && (lane & 3) == 2) { my_sel = 2; my_off = GOFF + B8 + (lane >> 2); }
    if (C4 > 0 && !C4_SECOND && (lane & 7) == C4_CLASS) { my_sel = 3; my_off = GOFF + B4 + (lane >> 3); }
    if (my_sel > 0 && my_off - GOFF >= 3 + p.S) my_sel = -1;    // zero padding channel
    // GEOM = false: the opacity and depth cotangents have no appearance gradient and are not read
    const float dpix_d = GEOM && inside ? p.dL_dpix_d[vpix] : 0.0f;
    const float dpix_o = GEOM && inside ? p.dL_dpix_o[vpix] : 0.0f;
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
    // feature channels enter dL_dalpha only when backward_geometry is set (backward.cu:563-566)
    float dsel[NC];
#pragma unroll
    for (int c = 0; c < NC; ++c) dsel[c] = (c < 3 || geo) ? dpix[c] : 0.0f;

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
    float4 r[RG];
#pragma unroll
    for (int g = 0; g < RG; ++g) r[g] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (lane < qcount) {
        k_cur = q[(qhead + lane) & (R3DG_QCAP - 1)];
        id_cur = plist[k_cur];
#pragma unroll
        for (int g = 0; g < RG; ++g) r[g] = rec4[(size_t)id_cur * rec4n + g];
    }

    while (qcount > 0) {
        const int n = min(32, qcount);
        __syncwarp();
        // element offset of the Gaussian's gradient row (ABS: the row index itself, also that of its absgrad pair)
        sId[warp][lane] = ABS ? id_cur : id_cur * (uint32_t)(GEOM ? p.recf : NC);
        sK[warp][lane] = k_cur;                                        // 0-based list position == contributor index
#pragma unroll
        for (int g = 0; g < RG; ++g) sRec[warp][g][lane] = r[g];
        qhead = (qhead + n) & (R3DG_QCAP - 1);
        qcount -= n;
        while (qcount < 64 && w_next >= w_low) scan_step();
        __syncwarp();
        if (lane < qcount) {
            k_cur = q[(qhead + lane) & (R3DG_QCAP - 1)];
            id_cur = plist[k_cur];
#pragma unroll
            for (int g = 0; g < RG; ++g) r[g] = rec4[(size_t)id_cur * rec4n + g];
        }
        // Rounds of U entries.  The kernel is latency-bound, not issue-bound (fewer resident CTAs make it slower), and the
        // heaviest pixel blocks walk hundreds of contributors one after the other,
        // so the round is laid out for instruction-level parallelism inside the warp: (1) everything that depends only on
        // the entry — record fetch, exp(), alpha, 1/(1-alpha), the entry's own cotangent dot D — for all U entries; (2) the
        // two short recurrences T and A in list order; (3) gradient rows and butterflies of the U entries, advanced level
        // by level together.  A round with fewer than U entries left re-evaluates the last one with its gate closed.
#pragma unroll 1
        for (int j0 = 0; j0 < n; j0 += U) {
            int ju[U];
            bool valid[U];
            float dx[U], dy[U], G[U], alpha[U], inv[U], D[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {                                   // (1)
                ju[u] = min(j0 + u, n - 1);
                const int k = (int)sK[warp][ju[u]];
                const float4 a = sRec[warp][0][ju[u]];
                const float4 b = sRec[warp][1][ju[u]];
                dx[u] = sub_(a.x, pxf); dy[u] = sub_(a.y, pyf);
                const float qd = fma_(dx[u], mul_(dx[u], a.z), mul_(dy[u], mul_(dy[u], b.x)));
                const float power = fma_(qd, -0.5f, -mul_(dy[u], mul_(dx[u], a.w)));
                G[u] = expf(power);
                alpha[u] = fminf(0.99f, mul_(b.y, G[u]));
                // the same three tests as the forward pass (identical arithmetic) + "not behind this pixel's last contributor"
                valid[u] = j0 + u < n && k < last_contributor && !(power > 0.0f) && !(alpha[u] < 1.0f / 255.0f);
                // a skipped entry of a non-positive-definite conic can have power > 88: expf = inf, and the gated
                // products below (0 * inf) would be NaN.  Composited entries have power <= 0, so G <= 1 is unchanged.
                G[u] = valid[u] ? G[u] : 0.0f;
                asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(inv[u]) : "f"(1.0f - alpha[u]));   // 1 - alpha in [0.01, 1]: one MUFU
                float d = 0.0f;
                if constexpr (GEOM) {
                    d = fmaf(b.z, dpix_d, dpix_o);                          // depth * dL_ddepth + 1 * dL_dopacity
#pragma unroll
                    for (int g = 0; g < NG; ++g) {
                        const float4 c4 = sRec[warp][2 + g][ju[u]];
                        d = fmaf(c4.x, dsel[4 * g + 0], d);
                        d = fmaf(c4.y, dsel[4 * g + 1], d);
                        d = fmaf(c4.z, dsel[4 * g + 2], d);
                        d = fmaf(c4.w, dsel[4 * g + 3], d);
                    }
                }
                D[u] = d;
            }
            float dcc[U], dL_dalpha[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {                                   // (2) branch-free: lanes that did not composite
                const float gate = valid[u] ? 1.0f : 0.0f;                  // the entry contribute zeros and keep their state
                const float Tn = T * inv[u];                                // T before this entry (backward.cu:533)
                dcc[u] = gate * alpha[u] * Tn;
                if constexpr (GEOM) {
                    dL_dalpha[u] = gate * fmaf(D[u] - A, Tn, -(T_final * inv[u]) * bg_dot);
                    if (valid[u]) { A = fmaf(alpha[u], D[u] - A, A); T = Tn; } // A <- alpha D + (1 - alpha) A
                } else if (valid[u]) {
                    T = Tn;
                }
            }
            float v0[U][8], mine[U];
            if constexpr (!GEOM) {
#pragma unroll
                for (int u = 0; u < U; ++u) mine[u] = 0.0f;
            }
#pragma unroll
            for (int u = 0; u < U && GEOM; ++u) {                           // (3)
                const float4 a = sRec[warp][0][ju[u]];
                const float4 b = sRec[warp][1][ju[u]];
                const float dL_dG = b.y * dL_dalpha[u];
                const float gdx = G[u] * dx[u], gdy = G[u] * dy[u];
                const float dG_ddelx = -gdx * a.z - gdy * a.w;
                const float dG_ddely = -gdy * b.x - gdx * a.w;
                v0[u][0] = dL_dG * dG_ddelx * ddelx_dx;
                v0[u][1] = dL_dG * dG_ddely * ddely_dy;
                v0[u][2] = dpix_d * dcc[u];
                v0[u][3] = G[u] * dL_dalpha[u];
                v0[u][4] = -0.5f * gdx * dx[u] * dL_dG;
                v0[u][5] = -0.5f * gdx * dy[u] * dL_dG;
                v0[u][6] = -0.5f * gdy * dy[u] * dL_dG;
                v0[u][7] = 0.0f;
            }
            float av[U][2], asum[U];
            if constexpr (ABS) {                                            // before the butterfly below overwrites v0
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    av[u][0] = valid[u] ? fabsf(v0[u][0]) : 0.0f;
                    av[u][1] = valid[u] ? fabsf(v0[u][1]) : 0.0f;
                }
                reduce_scatter_multi<U, 2>(av, lane, asum);                 // |x| total on lanes 0-15, |y| on 16-31
            }
            if constexpr (GEOM) reduce_scatter_multi<U, 8>(v0, lane, mine); // geometry slots: lanes 0 mod 4
            if constexpr (C16 > 0) {
                float x[U][16], t[U];
#pragma unroll
                for (int u = 0; u < U; ++u)
#pragma unroll
                    for (int i = 0; i < 16; ++i) x[u][i] = dcc[u] * cst16[i];
                reduce_scatter_permuted_multi<U, 16>(x, t);
#pragma unroll
                for (int u = 0; u < U; ++u) if (my_sel == 1) mine[u] = t[u];
            }
            if constexpr (C8 > 0) {
                float x[U][8], t[U];
#pragma unroll
                for (int u = 0; u < U; ++u)
#pragma unroll
                    for (int i = 0; i < 8; ++i) x[u][i] = dcc[u] * cst8[i];
                reduce_scatter_permuted_multi<U, 8>(x, t);
#pragma unroll
                for (int u = 0; u < U; ++u) if (my_sel == 2) mine[u] = t[u];
            }
            float t4[U];
            if constexpr (C4 > 0) {
                float x[U][4];
#pragma unroll
                for (int u = 0; u < U; ++u)
#pragma unroll
                    for (int i = 0; i < 4; ++i) x[u][i] = dcc[u] * cst4[i];
                reduce_scatter_permuted_multi<U, 4>(x, t4);
                if constexpr (!C4_SECOND) {
#pragma unroll
                    for (int u = 0; u < U; ++u) if (my_sel == 3) mine[u] = t4[u];
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (j0 + u < n) {                                           // (warp-uniform)
                    if constexpr (ABS) {
                        const size_t a = 2 * (size_t)sId[warp][ju[u]] + (lane >> 4);
                        if ((lane & 15) == 0) {
                            if constexpr (DET) det_add(p.det_abs, a, asum[u], e_geo);
                            else atomicAdd(p.abs_grad + a, asum[u]);
                        }
                    }
                    if constexpr (DET) {
                        size_t row;
                        if constexpr (ABS) row = (size_t)sId[warp][ju[u]] * p.recf;
                        else row = sId[warp][ju[u]];
                        if constexpr (C4_SECOND) {
                            if ((lane & 7) == 0 && B4 + (lane >> 3) < 3 + p.S) det_add(p.det, row + 8 + B4 + (lane >> 3), t4[u], e_app);
                        }
                        if (my_sel >= 0) det_add(p.det, row + my_off, mine[u], my_sel == 0 ? e_geo : e_app);
                    } else {
                        float* grow;
                        if constexpr (ABS) grow = p.grad + (size_t)sId[warp][ju[u]] * p.recf;
                        else grow = p.grad + sId[warp][ju[u]];
                        if constexpr (C4_SECOND) {
                            if ((lane & 7) == 0 && B4 + (lane >> 3) < 3 + p.S) atomicAdd(grow + 8 + B4 + (lane >> 3), t4[u]);
                        }
                        if (my_sel >= 0) atomicAdd(grow + my_off, mine[u]);
                    }
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
__device__ void det_scale_reduce(const CompositeBwdParams& p, int V, bool geometry, int nblocks, uint32_t* __restrict__ scale) {
    __shared__ uint32_t s_max[2][8];
    const size_t HW = (size_t)p.H * p.W, n_app = (size_t)(3 + p.S) * HW, n = n_app + (geometry ? 2 * HW : 0);
    const size_t stride = (size_t)nblocks * blockDim.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int v = 0; v < V; ++v) {
        const float* col = p.dL_dpix + (size_t)v * 3 * HW;
        const float* feat = p.dL_dpix_f + (size_t)v * p.S * HW;
        uint32_t m_app = 0u, m_geo = 0u;
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
            if (i < 3 * HW) m_app = max(m_app, det_abs_bits(col[i]));
            else if (i < n_app) m_app = max(m_app, det_abs_bits(feat[i - 3 * HW]));
            else if (i < n_app + HW) m_geo = max(m_geo, det_abs_bits(p.dL_dpix_o[(size_t)v * HW + (i - n_app)]));
            else m_geo = max(m_geo, det_abs_bits(p.dL_dpix_d[(size_t)v * HW + (i - n_app - HW)]));
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

DetAcc raster_det_abs(const r3dg_raster_bwd_args& a, size_t rows) {
    return det_acc((char*)a.det_work + det_bytes(rows * rec_floats(a.S)), 2 * rows);   // behind r3dg_raster_bwd_det_bytes
}

uint32_t* raster_det_scale(const RasterBuffers& b) {
    return reinterpret_cast<uint32_t*>(b.grad - (size_t)b.row_base * b.recf);     // the whole call's grad region
}

// resident CTAs per SM the register allocation is pinned to, by channel groups NG (the occupancy sweep in DESIGN.md §4.2)
template <int NG> struct BwdOcc { static constexpr int v = NG <= 3 ? 5 : (NG <= 5 ? 4 : 3); };
// the pin of an absgrad instantiation: BwdOcc's, except in deterministic mode at NG = 5, where the absgrad sums' fixed-
// point adds do not fit the 128 registers of 4 CTAs per SM (ptxas spills) and 3 CTAs are resident instead
template <int NG, bool DET> struct BwdOccAbs { static constexpr int v = DET && NG == 5 ? 3 : BwdOcc<NG>::v; };
int g_bwd_ctas = 0;             // r3dg_tune("composite_bwd_ctas"): resident CTAs per SM (0 = whatever fits)
int composite_bwd_tune(const char* key, int value, int* previous) {
    if (strcmp(key, "composite_bwd_ctas") != 0) return R3DG_ERR_UNSUPPORTED;
    if (previous) *previous = g_bwd_ctas;
    if (value < 0 || value > 32) return R3DG_ERR_BAD_ARG;
    g_bwd_ctas = value;
    return 0;
}
template <int NG, bool DET, bool GEOM, bool ABS = false>
static void launch_bwd_kernel(const CompositeBwdParams& p, int tiles, cudaStream_t stream) {
    constexpr auto kernel = composite_bwd_kernel<NG, 4, ABS ? BwdOccAbs<NG, DET>::v : BwdOcc<NG>::v, DET, GEOM, ABS>;
    kernel<<<tiles * 2, 128, residency_pad<kernel>(g_bwd_ctas), stream>>>(p);    // two 4-warp CTAs per tile
}
template <int NG>
static void launch_bwd_ng(const CompositeBwdParams& p, int tiles, bool det, bool geometry, bool absgrad, cudaStream_t stream) {
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
    p.grad = b.grad;
    p.n_contrib = b.n_contrib;
    const bool det = a.deterministic != 0;
    const size_t rows = (size_t)V * a.P;
    const int gradf = composite_bwd_row_floats(a.S, geometry);     // the gradient row: b.recf, or NC without geometry
    p.det = det_acc(a.det_work, rows * gradf);
    p.det_scale = det ? raster_det_scale(b) : nullptr;
    // absgrad (geometry only; the appearance-only backward ignores dL_dmeans2D_abs): the default mode adds into the
    // output itself, DET mode into its own accumulators behind the gradient rows' in det_work
    const bool absgrad = geometry && a.dL_dmeans2D_abs != nullptr;
    p.abs_grad = absgrad && !det ? a.dL_dmeans2D_abs : nullptr;
    p.det_abs = absgrad && det ? raster_det_abs(a, rows) : det_acc(nullptr, 0);
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
    switch (num_groups(a.S)) {
        case 1: launch_bwd_ng<1>(p, tiles, det, geometry, absgrad, stream); break;
        case 2: launch_bwd_ng<2>(p, tiles, det, geometry, absgrad, stream); break;
        case 3: launch_bwd_ng<3>(p, tiles, det, geometry, absgrad, stream); break;
        case 4: launch_bwd_ng<4>(p, tiles, det, geometry, absgrad, stream); break;
        case 5: launch_bwd_ng<5>(p, tiles, det, geometry, absgrad, stream); break;
        case 6: launch_bwd_ng<6>(p, tiles, det, geometry, absgrad, stream); break;
        case 7: launch_bwd_ng<7>(p, tiles, det, geometry, absgrad, stream); break;
        default: return R3DG_ERR_UNSUPPORTED;   // S > 24: reference backward limit (backward.cu:449)
    }
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace r3dg
