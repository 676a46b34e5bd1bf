// Stage 2 forward: per-tile front-to-back alpha compositing (reference K7, forward.cu:263-395)
// and the surface-xyz / pseudo-normal pass (K8+K9, forward.cu:398-491, fused into one kernel).
//
// Design notes
//  * each warp owns a compact 8x4 pixel block of a 16x16 tile and walks the tile's sorted list
//    AUTONOMOUSLY: no CTA barrier, per-warp early termination (the reference's CTA-wide
//    fetch/compute lock-step spent ~half of its stall samples at the barrier);
//  * stream compaction instead of per-warp culling: the binning scatter leaves one pre-filter byte
//    per (tile, Gaussian) instance; a warp streams the bytes 128 instances per step, compacts the
//    positions whose bit for ITS block is set into a circular queue and composites batches of 32
//    queued entries (id -> packed record prefetched one batch ahead, staged in a warp-private
//    shared-memory slab, exact ellipse / block test once per entry by the lane that staged it);
//  * the kernel is bound by per-warp latency and by its heaviest warps, not by issue slots
//    (tools/warp_timing.py): entries are composited in rounds of U whose alpha evaluations
//    are in flight together, the sequential part is branch-free (predicated FMAs);
//  * accumulators live in registers (template on the number of float4 channel groups) — the
//    reference's runtime-indexed F[33] spills to local memory;
//  * out_weights: one atomic instruction per (warp, batch) after one integer REDUX per entry
//    instead of one atomic per (pixel, Gaussian);
//  * for the backward pass the warp leaves one contributor bit per (instance, block) and, per
//    half-tile CTA, the number of entries its busiest warp composited (the backward launch order);
//  * per-pixel arithmetic keeps the association of the reference binary, so n_contrib and the
//    images are bit-identical to it for identical lists.
#include <cstdlib>
#include <cstring>
#include "common.cuh"
#include "detacc.cuh"
#include "kernels.h"

#ifndef R3DG_FWD_CTAS          // default resident CTAs per SM of the forward compositor (0 = whatever fits)
#define R3DG_FWD_CTAS 0
#endif
#ifndef R3DG_FWD_ILP           // staged entries whose alpha evaluation is in flight together (composite_fwd_kernel), S <= 5
#define R3DG_FWD_ILP 4
#endif
#ifndef R3DG_FWD_ILP_WIDE      // the same for S > 5 (more accumulators per pixel: registers)
#define R3DG_FWD_ILP_WIDE 2
#endif
namespace r3dg {

struct CompositeFwdParams {
    int W, H, gx, S, recf;
    const uint2* ranges;
    const uint32_t* point_list;  // per-tile depth-sorted Gaussian ids (binning.cu)
    const uint32_t* bmask32;     // per-instance block-touch masks (bin_scatter), viewed as words of 4 instances
    uint32_t* cmask32;           // per-instance contributor masks (zeroed by bin_scatter, set here)
    const GeomHeader* header;
    const uint32_t* tile_order;  // CTA -> tile, heaviest tiles first
    uint32_t* bwd_work;          // [2 tiles] entries composited by the busiest warp of each half-tile CTA (backward launch order)
    const float* rec;
    const float* bg;
    float* final_T;
    int* n_contrib;
    float *out_color, *out_opacity, *out_depth, *out_feature, *out_weights;
    uint64_t* det_weights;             // DET: [P] out_weights in exact 2^-24 units (zeroed), converted by det_weights_kernel
};

#ifdef R3DG_WARP_TIMING
__device__ WarpTiming g_wt_fwd[R3DG_WT_MAX];
extern "C" int r3dg_debug_wt_fwd(void* dst, size_t bytes) { return (int)cudaMemcpyFromSymbol(dst, g_wt_fwd, bytes); }
#endif

// NW = warps per CTA (4: two CTAs per tile).  Warps are autonomous: no
// CTA-wide barrier anywhere; the CTA only exists so that the warps of a tile share L1 lines.
//
// Per warp (one 8x4 pixel block): the tile's block pre-filter mask bytes are streamed 128 instances at a time and the
// positions whose bit for THIS block is set are compacted into a circular queue (warp scan); batches of 32 queued
// entries are then fetched (id -> packed record, registers, one batch ahead), staged in the warp's shared-memory slab
// and composited after a second, exact per-lane filter (see below).
//
// BULK = false: the next batch's records are prefetched into registers (r[RG]) and stored to a SoA slab.
// BULK = true : the TMA-unit experiment north_star asks for — every lane issues ONE 1-D bulk copy (cp.async.bulk, SASS
//   UBLKCP) of its entry's record (recf * 4 bytes, 16-byte aligned) straight into a double-buffered AoS slab; the
//   warp's mbarrier counts the transaction bytes.  No prefetch registers (12-28 fewer live registers), no staging
//   stores.  Selected with r3dg_tune("composite_bulk", 1); the register prefetch is the default.
// DET (deterministic mode): the per-warp integer weight sums go to a u64 per Gaussian instead of a float atomic, so
//   out_weights does not depend on the order in which warps finish.  Everything else is the same code.
template <int NG, int NW, int MINB, bool BULK, bool DET = false>
__global__ void __launch_bounds__(32 * NW, MINB) composite_fwd_kernel(const CompositeFwdParams p) {
    constexpr int RG = 2 + NG;                       // float4 groups per record
    __shared__ __align__(16) float4 sRec[BULK ? 1 : NW][BULK ? 1 : RG][BULK ? 1 : 32];   // this warp's current 32-entry batch, SoA
    __shared__ __align__(16) float4 sRecB[BULK ? NW : 1][BULK ? 2 : 1][BULK ? 32 : 1][BULK ? RG : 1];   // BULK: [stage][entry][group]
    __shared__ __align__(8) uint64_t sBar[NW][2];
    __shared__ uint32_t sId[NW][32];
    __shared__ uint32_t sQ[NW][R3DG_QCAP];           // queued list positions (relative to the tile's range)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int PARTS = 8 / NW;
    const int tile = (int)p.tile_order[blockIdx.x / PARTS];
    const int wb = (blockIdx.x % PARTS) * NW + warp;          // pixel block 0..7 inside the tile
    const int tx = tile % p.gx, ty = tile / p.gx;
    const int bx0 = tx * R3DG_TILE + (wb & 1) * 8, by0 = ty * R3DG_TILE + (wb >> 1) * 4;
    const int px = bx0 + (lane & 7), py = by0 + (lane >> 3);
    const bool inside = px < p.W && py < p.H;
    const float pxf = (float)px, pyf = (float)py;
    const uint2 range = p.ranges[tile];
    const uint32_t lo = range.x, hi = range.y;
    const float4* __restrict__ rec4 = reinterpret_cast<const float4*>(p.rec);
    const int rec4n = p.recf >> 2;
    const uint32_t* __restrict__ plist = p.point_list + lo;
    uint32_t* q = sQ[warp];

#ifdef R3DG_WARP_TIMING
    const unsigned long long wt_t0 = wt_now();
    unsigned wt_iters = 0;
#endif
    float T = 1.0f, Dp = 0.0f, Op = 0.0f;
    float C[4 * NG];
#pragma unroll
    for (int i = 0; i < 4 * NG; ++i) C[i] = 0.0f;
    uint32_t last_contributor = 0;
    bool done = !inside;

    // ---- mask stream: word w holds instances [4w, 4w+4); lane takes word w_next + lane --------------------
    const uint32_t w_end = (hi + 3) >> 2;
    uint32_t w_next = lo >> 2;
    uint32_t m_nxt = (w_next + lane < w_end) ? p.bmask32[w_next + lane] : 0u;       // prefetched one step ahead
    int qhead = 0, qcount = 0;
    auto scan_step = [&]() {
        const uint32_t w = w_next + lane;
        uint32_t flags = 0u;
        if (w < w_end) {
            flags = (m_nxt >> wb) & 0x01010101u;
            const uint32_t e0 = w << 2;
            if (e0 < lo) flags &= 0xffffffffu << (8 * (lo - e0));                   // instances of the previous tile
            if (e0 + 4 > hi) flags &= 0xffffffffu >> (8 * (e0 + 4 - hi));           // instances of the next tile
        }
        w_next += 32;
        m_nxt = (w_next + lane < w_end) ? p.bmask32[w_next + lane] : 0u;
        uint32_t total;
        uint32_t slot = (uint32_t)(qhead + qcount) + warp_excl_scan(__popc(flags), lane, total);
        const uint32_t rel = (w << 2) - lo;                                          // may wrap for the first word: only flagged bytes are used
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (flags & (1u << (8 * k))) { q[slot & (R3DG_QCAP - 1)] = rel + k; ++slot; }
        qcount += (int)total;
    };
    while (qcount < 64 && w_next < w_end) scan_step();
    __syncwarp();

    // software pipeline: records of the next batch are in flight (registers, or bulk copies into the other slab stage)
    // while the current one is composited
    uint32_t id_cur = 0u;
    float4 r[BULK ? 1 : RG];
    int stage = 0;
    unsigned phase0 = 0u, phase1 = 0u;
    const unsigned rec_bytes = (unsigned)p.recf * 4u;
    auto issue_bulk = [&](int s_, int nb, uint32_t id) {        // lanes < nb: one bulk copy each into stage s_
        fence_proxy_async_smem();                               // earlier generic reads of that stage are done (WAR)
        __syncwarp();
        if (lane == 0) mbar_arrive_expect_tx(&sBar[warp][s_], (unsigned)nb * rec_bytes);
        __syncwarp();
        if (lane < nb) bulk_copy_g2s(&sRecB[warp][s_][lane][0], p.rec + (size_t)id * p.recf, rec_bytes, &sBar[warp][s_]);
    };
    if (BULK) {
        if (lane == 0) { mbar_init(&sBar[warp][0], 1); mbar_init(&sBar[warp][1], 1); fence_proxy_async_smem(); }
        __syncwarp();
        if (lane < qcount) id_cur = plist[q[(qhead + lane) & (R3DG_QCAP - 1)]];
        if (qcount > 0) issue_bulk(0, min(32, qcount), id_cur);
    } else {
#pragma unroll
        for (int g = 0; g < RG; ++g) r[g] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (lane < qcount) {
            id_cur = plist[q[(qhead + lane) & (R3DG_QCAP - 1)]];
#pragma unroll
            for (int g = 0; g < RG; ++g) r[g] = rec4[(size_t)id_cur * rec4n + g];
        }
    }

    uint32_t composited = 0u;                                           // entries this warp composited = its backward twin's iterations
    bool all_done = __all_sync(0xffffffffu, done);
    while (qcount > 0 && !all_done) {
        const int n = min(32, qcount);
        const uint32_t mypos = q[(qhead + lane) & (R3DG_QCAP - 1)];     // valid for lane < n
        __syncwarp();
        sId[warp][lane] = id_cur;
        if (!BULK) {
#pragma unroll
            for (int g = 0; g < RG; ++g) sRec[warp][g][lane] = r[g];
        }
        // second, exact filter — each lane applies round 1's exact-conservative ellipse / rectangle test to ITS OWN staged
        // entry (one evaluation per entry): the block rectangle is conservative, the exact test drops the (warp, entry)
        // pairs whose ellipse misses the block, and every pair dropped here saves the alpha evaluation of the loop below
        uint32_t word;
        if (BULK) word = n == 32 ? 0xffffffffu : ((1u << n) - 1u);       // (records are not in registers in this variant)
        else word = __ballot_sync(0xffffffffu, lane < n && touch_block(r[0], r[1], (float)bx0, (float)by0));
        const int h0 = qhead;
        qhead = (qhead + n) & (R3DG_QCAP - 1);
        qcount -= n;
        while (qcount < 64 && w_next < w_end) scan_step();
        __syncwarp();
        // prefetch: id -> record of the next batch
        if (lane < qcount) id_cur = plist[q[(qhead + lane) & (R3DG_QCAP - 1)]];
        if (BULK) {
            if (qcount > 0) issue_bulk(stage ^ 1, min(32, qcount), id_cur);
            mbar_wait(&sBar[warp][stage], stage ? phase1 : phase0);      // the current batch has landed
            if (stage) phase1 ^= 1u; else phase0 ^= 1u;
        } else if (lane < qcount) {
#pragma unroll
            for (int g = 0; g < RG; ++g) r[g] = rec4[(size_t)id_cur * rec4n + g];
        }
        uint32_t cw = 0u;                                               // bit j: entry j was composited by some pixel
        int last_j = -1;                                                // this pixel's last accepted entry of the batch
        int my_wsum = 0;                                                // lane j keeps the warp's weight sum of entry j
        // U staged entries per round.  The alpha evaluations (record fetch, quadratic form, exp — two thirds of the
        // work) depend neither on one another nor on the pixel's state, so all U are issued back to back: U dependency
        // chains in flight per warp instead of one.  Only the short transmittance recurrence that follows is sequential,
        // in list order, with exactly the reference's arithmetic.  This is what bounds the kernel: the heaviest pixel
        // blocks composite many entries one after the other, and while the light tiles drain the machine those few
        // warps decide the makespan (tools/warp_timing.py).  A round with fewer than U
        // entries left re-evaluates the last one, masked out.
        constexpr int U = NG <= 2 ? R3DG_FWD_ILP : R3DG_FWD_ILP_WIDE;
        while (word) {
            int jj[U];
            bool pv[U];
            float al[U], om[U], dep[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {                                // (1) independent: alpha of U entries
                const bool have = word != 0u;
                jj[u] = have ? __ffs(word) - 1 : jj[u ? u - 1 : 0];
                word &= word - 1u;
#ifdef R3DG_WARP_TIMING
                wt_iters += have ? 1u : 0u;
#endif
                const float4 a = BULK ? sRecB[warp][stage][jj[u]][0] : sRec[warp][0][jj[u]];
                const float4 b = BULK ? sRecB[warp][stage][jj[u]][1] : sRec[warp][1][jj[u]];
                const float dx = sub_(a.x, pxf), dy = sub_(a.y, pyf);
                // power = -0.5f*(ca*dx*dx + cc*dy*dy) - cb*dx*dy  (forward.cu:344) as compiled
                const float qd = fma_(dx, mul_(dx, a.z), mul_(dy, mul_(dy, b.x)));
                const float power = fma_(qd, -0.5f, -mul_(dy, mul_(dx, a.w)));
                al[u] = fminf(0.99f, mul_(b.y, expf(power)));
                om[u] = sub_(1.0f, al[u]);
                dep[u] = b.z;
                pv[u] = have && !(power > 0.0f) && !(al[u] < 1.0f / 255.0f);
            }
            int wq[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {                                // (2) sequential, branch-free: T, accumulators
                const float test_T = mul_(T, om[u]);
                bool valid = !done && pv[u];
                const bool stop = valid && test_T < 0.0001f;             // forward.cu:352-356: this pixel is finished
                done = done || stop;
                valid = valid && !stop;
                const float w = mul_(T, al[u]);
#pragma unroll
                for (int g = 0; g < NG; ++g) {
                    const float4 c = BULK ? sRecB[warp][stage][jj[u]][2 + g] : sRec[warp][2 + g][jj[u]];
                    fma4_if(valid, w, c, C[4 * g + 0], C[4 * g + 1], C[4 * g + 2], C[4 * g + 3]);
                }
                fma_add_if(valid, w, dep[u], Dp, Op);
                T = valid ? test_T : T;
                last_j = valid ? jj[u] : last_j;
                // w in [0,1) in 2^-24 fixed point for the out_weights statistic (below); >= 6 whenever the entry was accepted
                wq[u] = valid ? __float2int_rn(w * 16777216.0f) : 0;
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {                                // (3) independent again: per-entry warp sums
                // sum over the warp's pixels of w for out_weights: one integer REDUX instead of a 5-step float shuffle tree
                // (error <= 1e-6 per warp, far below the reference's own atomic-order noise on this statistic); non-zero
                // exactly when some pixel accepted the entry.  Lane j keeps entry j's sum: ONE atomic instruction per batch.
                const int wsum = __reduce_add_sync(0xffffffffu, wq[u]);
                if (wsum != 0) {
                    cw |= 1u << jj[u];
                    if (lane == jj[u]) my_wsum = wsum;
                }
            }
            if (__all_sync(0xffffffffu, done)) { all_done = true; break; }      // once per round: entries after the last
        }                                                                        // pixel finished change nothing (valid needs !done)
        if (last_j >= 0) last_contributor = q[(h0 + last_j) & (R3DG_QCAP - 1)] + 1u;     // 1-based position in the tile list
        if constexpr (DET) {
            if (my_wsum != 0) det_red_u64(p.det_weights + sId[warp][lane], (uint64_t)(uint32_t)my_wsum);   // my_wsum > 0
        } else {
            if (my_wsum != 0) atomicAdd(&p.out_weights[sId[warp][lane]], (float)my_wsum * (1.0f / 16777216.0f));
        }
        stage ^= 1;
        composited += (uint32_t)__popc(cw);
        // contributor bits for the backward pass: one fire-and-forget atomic per composited entry
        if ((cw >> lane) & 1u) {
            const uint32_t e = lo + mypos;
            atomicOr(&p.cmask32[e >> 2], 1u << (8 * (e & 3u) + wb));
        }
    }
    if (lane == 0 && composited) atomicMax(&p.bwd_work[blockIdx.x % PARTS + PARTS * tile], composited);
    if (inside) {
        const size_t HW = (size_t)p.H * p.W, pix = (size_t)p.W * py + px;
        p.final_T[pix] = T;
        p.n_contrib[pix] = (int)last_contributor;
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) p.out_color[ch * HW + pix] = fma_(p.bg[ch], T, C[ch]);
#pragma unroll
        for (int ch = 3; ch < 4 * NG; ++ch)
            if (ch - 3 < p.S) p.out_feature[(size_t)(ch - 3) * HW + pix] = C[ch];
        p.out_depth[pix] = Dp;
        p.out_opacity[pix] = Op;
    }
#ifdef R3DG_WARP_TIMING
    if (lane == 0 && blockIdx.x * NW + warp < R3DG_WT_MAX) g_wt_fwd[blockIdx.x * NW + warp] = WarpTiming{wt_t0, wt_now(), wt_iters, wt_smid()};
#endif
}

// Deterministic mode: out_weights = the exact integer total in 2^-24 units, rounded to fp32 once.
__global__ void __launch_bounds__(256) det_weights_kernel(int P, const uint64_t* __restrict__ acc, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < P) out[i] = __fmul_rn(__ull2float_rn(acc[i]), 1.0f / 16777216.0f);
}

// renderSurfaceXYZCUDA + renderPseudoNormalCUDA fused: neighbours' surface points are recomputed
// from (opacity, depth) with the identical formula, so no second pass over surface_xyz is needed.
__global__ void __launch_bounds__(256) surface_normal_kernel(int W, int H, const float* __restrict__ viewmatrix,
                                                             float focal_x, float focal_y, float cx, float cy,
                                                             const float* __restrict__ opacity,
                                                             const float* __restrict__ depth,
                                                             float* __restrict__ out_normal,
                                                             float* __restrict__ out_xyz) {
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= W || y >= H) return;
    const size_t HW = (size_t)H * W;
    auto point = [&](int xx, int yy, float* o) {
        const size_t q = (size_t)W * yy + xx;
        const float d = div_(depth[q], fmaxf(opacity[q], 0.0000001f));
        o[0] = mul_(div_(sub_((float)xx, cx), focal_x), d);
        o[1] = mul_(div_(sub_((float)yy, cy), focal_y), d);
        o[2] = d;
    };
    const size_t pix = (size_t)W * y + x;
    float c[3];
    point(x, y, c);
    out_xyz[pix] = c[0]; out_xyz[HW + pix] = c[1]; out_xyz[2 * HW + pix] = c[2];
    const int xm = x == 0 ? 0 : x - 1, xp = x == W - 1 ? W - 1 : x + 1;
    const int ym = y == 0 ? 0 : y - 1, yp = y == H - 1 ? H - 1 : y + 1;
    float p00[3], p01[3], p02[3], p10[3], p12[3], p20[3], p21[3], p22[3];
    point(xm, ym, p00); point(x, ym, p01); point(xp, ym, p02);
    point(xm, y, p10);                     point(xp, y, p12);
    point(xm, yp, p20); point(x, yp, p21); point(xp, yp, p22);
    float ga[3], gb[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const float h = mul_(p00[i], -0.125f);
        ga[i] = fma_(p22[i], 0.125f, fma_(p20[i], -0.125f, fma_(p12[i], 0.25f, fma_(p10[i], -0.25f, fma_(p02[i], 0.125f, h)))));
        gb[i] = fma_(p22[i], 0.125f, fma_(p21[i], 0.25f, fma_(p20[i], 0.125f, fma_(p02[i], -0.125f, fma_(p01[i], -0.25f, h)))));
    }
    const float n0 = fma_(ga[1], gb[2], -mul_(ga[2], gb[1]));
    const float n1 = fma_(ga[2], gb[0], -mul_(ga[0], gb[2]));
    const float n2 = fma_(ga[0], gb[1], -mul_(ga[1], gb[0]));
    const float norm = sqrt_(fma_(n2, n2, fma_(n0, n0, mul_(n1, n1))));
    float o0 = 0.0f, o1 = 0.0f, o2 = 0.0f;
    if (!(norm <= 0.0f)) {
        const float N0 = div_(-n0, norm), N1 = div_(-n1, norm), N2 = div_(-n2, norm);
        const float* V = viewmatrix;
        o0 = dot3_(V[0], N0, V[1], N1, V[2], N2);
        o1 = dot3_(V[4], N0, V[5], N1, V[6], N2);
        o2 = dot3_(V[8], N0, V[9], N1, V[10], N2);
    }
    out_normal[pix] = o0; out_normal[HW + pix] = o1; out_normal[2 * HW + pix] = o2;
}

// resident CTAs per SM the register allocation is pinned to (ptxas otherwise drifts a few registers above the
// count that fits one more CTA): by channel groups NG, for the 4-warp CTA (the 8-warp variant is left to ptxas)
#ifndef R3DG_FWD_OCC2          // resident CTAs per SM the kernels are compiled for, by channel groups (tools/occ_sweep.sh)
#define R3DG_FWD_OCC2 7
#endif
#ifndef R3DG_FWD_OCC5
#define R3DG_FWD_OCC5 5
#endif
template <int NG> struct FwdOcc { static constexpr int v = NG <= 2 ? R3DG_FWD_OCC2 : (NG <= 3 ? 6 : (NG <= 5 ? R3DG_FWD_OCC5 : (NG <= 6 ? 4 : 3))); };

int g_composite_bulk = -1;      // r3dg_tune("composite_bulk"): 1 = TMA bulk-copy record staging in the forward compositor
int g_fwd_ctas = -1;            // r3dg_tune("composite_fwd_ctas"): resident CTAs per SM (0 = whatever fits)
static void composite_env() {
    if (g_composite_bulk < 0) { const char* e = getenv("R3DG_COMPOSITE_BULK"); g_composite_bulk = (e && atoi(e) == 1) ? 1 : 0; }
    if (g_fwd_ctas < 0) { const char* e = getenv("R3DG_FWD_CTAS"); g_fwd_ctas = e ? atoi(e) : R3DG_FWD_CTAS; if (g_fwd_ctas < 0) g_fwd_ctas = 0; }
}
int composite_tune(const char* key, int value, int* previous) {
    composite_env();
    if (strcmp(key, "composite_bulk") == 0) {
        if (previous) *previous = g_composite_bulk;
        if (value != 0 && value != 1) return R3DG_ERR_BAD_ARG;
        g_composite_bulk = value;
        return 0;
    }
    if (strcmp(key, "composite_fwd_ctas") == 0) {
        if (previous) *previous = g_fwd_ctas;
        if (value < 0 || value > 32) return R3DG_ERR_BAD_ARG;
        g_fwd_ctas = value;
        return 0;
    }
    return R3DG_ERR_UNSUPPORTED;
}
template <typename K>
static void launch_fwd_kernel(K kernel, const CompositeFwdParams& p, int tiles, cudaStream_t stream) {
    static int pad_for = -1, pad_dev = -1;
    static size_t pad = 0;
    int dev = 0;
    cudaGetDevice(&dev);
    if (pad_for != g_fwd_ctas || pad_dev != dev) { pad = residency_pad(kernel, g_fwd_ctas); pad_for = g_fwd_ctas; pad_dev = dev; }
    kernel<<<tiles * 2, 128, pad, stream>>>(p);                          // two 4-warp CTAs per tile
}
template <int NG>
static void launch_fwd_ng(const CompositeFwdParams& p, int tiles, cudaStream_t stream) {
    composite_env();
    if (p.det_weights) {
        if (g_composite_bulk == 1 && NG <= 6) launch_fwd_kernel(composite_fwd_kernel<NG <= 6 ? NG : 1, 4, FwdOcc<NG>::v, true, true>, p, tiles, stream);
        else launch_fwd_kernel(composite_fwd_kernel<NG, 4, FwdOcc<NG>::v, false, true>, p, tiles, stream);
        return;
    }
    if (g_composite_bulk == 1 && NG <= 6) launch_fwd_kernel(composite_fwd_kernel<NG <= 6 ? NG : 1, 4, FwdOcc<NG>::v, true>, p, tiles, stream);
    else launch_fwd_kernel(composite_fwd_kernel<NG, 4, FwdOcc<NG>::v, false>, p, tiles, stream);
}

int launch_composite_forward(const r3dg_raster_fwd_args& a, const GeomLayout& gl, const ImgLayout& il,
                             char* bin, const BinLayout& bl, cudaStream_t stream, stage_mark_fn mark) {
    char* geom = (char*)a.geom;
    char* img = (char*)a.img;
    CompositeFwdParams p;
    p.W = a.W; p.H = a.H; p.gx = (a.W + R3DG_TILE - 1) / R3DG_TILE; p.S = a.S; p.recf = gl.recf;
    const int gy = (a.H + R3DG_TILE - 1) / R3DG_TILE;
    p.ranges = (const uint2*)(img + il.ranges);
    p.point_list = (const uint32_t*)(bin + bl.point_list);
    p.bmask32 = (const uint32_t*)(bin + bl.bmask); p.cmask32 = (uint32_t*)(bin + bl.cmask);
    p.header = (const GeomHeader*)(geom + gl.header);
    p.tile_order = (const uint32_t*)(img + il.tile_order);
    p.bwd_work = (uint32_t*)(img + il.bwd_work);
    p.rec = (const float*)(geom + gl.rec);
    p.bg = a.background;
    p.final_T = (float*)(img + il.final_T);
    p.n_contrib = (int*)(img + il.n_contrib);
    p.out_color = a.out_color; p.out_opacity = a.out_opacity; p.out_depth = a.out_depth;
    p.out_feature = a.out_feature; p.out_weights = a.out_weights;
    p.det_weights = a.deterministic ? (uint64_t*)a.det_work : nullptr;
    if (p.det_weights) R3DG_CUDA_TRY(cudaMemsetAsync(p.det_weights, 0, (size_t)a.P * 8, stream));
    const int tiles = p.gx * gy;
    switch (num_groups(a.S)) {
        case 1: launch_fwd_ng<1>(p, tiles, stream); break;
        case 2: launch_fwd_ng<2>(p, tiles, stream); break;
        case 3: launch_fwd_ng<3>(p, tiles, stream); break;
        case 4: launch_fwd_ng<4>(p, tiles, stream); break;
        case 5: launch_fwd_ng<5>(p, tiles, stream); break;
        case 6: launch_fwd_ng<6>(p, tiles, stream); break;
        case 7: launch_fwd_ng<7>(p, tiles, stream); break;
        case 8: launch_fwd_ng<8>(p, tiles, stream); break;
        case 9: launch_fwd_ng<9>(p, tiles, stream); break;
        default: return R3DG_ERR_UNSUPPORTED;
    }
    if (p.det_weights && a.P > 0) det_weights_kernel<<<(a.P + 255) / 256, 256, 0, stream>>>(a.P, p.det_weights, a.out_weights);
    const size_t HW = (size_t)a.H * a.W;
    mark(6, stream);
    if (a.computer_pseudo_normal) {
        const float focal_y = a.H / (2.0f * a.tan_fovy), focal_x = a.W / (2.0f * a.tan_fovx);
        dim3 grid((a.W + 31) / 32, (a.H + 7) / 8);
        surface_normal_kernel<<<grid, 256, 0, stream>>>(a.W, a.H, a.viewmatrix, focal_x, focal_y, a.cx, a.cy,
                                                        a.out_opacity, a.out_depth, a.out_normal, a.out_surface_xyz);
    } else {
        R3DG_CUDA_TRY(cudaMemsetAsync(a.out_normal, 0, 3 * HW * 4, stream));
        R3DG_CUDA_TRY(cudaMemsetAsync(a.out_surface_xyz, 0, 3 * HW * 4, stream));
    }
    if (a.n_contrib)   // the reference returns n_contrib as a view of imgBuffer (rasterize_points.cu:136-139)
        R3DG_CUDA_TRY(cudaMemcpyAsync(a.n_contrib, img + il.n_contrib, HW * 4, cudaMemcpyDeviceToDevice, stream));
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace r3dg
