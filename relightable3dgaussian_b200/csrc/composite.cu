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
//    queued entries (id -> packed record prefetched one batch ahead, exact ellipse / block test once
//    per entry by the lane that holds it, the accepted entries compacted in list order into a
//    warp-private shared-memory slab);
//  * the kernel is bound by per-warp latency and by its heaviest warps, not by issue slots
//    (DESIGN.md §4.2): entries are composited in rounds of U whose alpha evaluations
//    are in flight together, the sequential part is branch-free (predicated FMAs);
//  * accumulators live in registers (template on the number of float4 channel groups) — the
//    reference's runtime-indexed F[33] spills to local memory;
//  * out_weights: one atomic instruction per (warp, batch) after one integer REDUX per entry
//    instead of one atomic per (pixel, Gaussian);
//  * for the backward pass the warp leaves one contributor bit per (instance, block) and, per
//    half-tile CTA, the number of entries its busiest warp composited (the backward launch order);
//  * per-pixel arithmetic keeps the association of the reference binary, so n_contrib and the
//    images are bit-identical to it for identical lists.
#include <cstring>
#include "common.cuh"
#include "detacc.cuh"
#include "kernels.h"

namespace r3dg {

struct CompositeFwdParams {
    int W, H, gx, gy, S, recf;   // gy: tile rows of one view; view v of a several-view call owns rows [v gy, (v+1) gy)
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
    uint32_t* clamped32;               // the rows' clamped bytes as words: kComposited is set for every composited row
    float *out_depth2, *out_median;    // DS: sum w d^2 and the median depth per pixel
    int* median_pos;                   // DS: the median entry's 1-based position in the tile list (0: none)
    uint32_t* depth_bound;             // DS: per view, the largest |d| of an accepted entry as float bits (zeroed)
};

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
// RD (ray-depth mode, register prefetch only): the record's appended group, the depth plane p, is staged with the
//   others, and an entry adds  tz - p.x dx - p.y dy  (dx, dy its mean minus the pixel) to the depth instead of tz.
// DS (depth statistics, register prefetch only): the entry's depth d (the one added to the depth) also goes into
//   sum w d^2 (as w * (d * d), the rounding of a d^2 feature channel), and the running median: while T before an
//   accepted entry is > 0.5 the entry's d and 1-based list position replace the previous ones (2DGS's rule).  The
//   warp's largest |d| of an accepted entry goes to its view's bound word (the deterministic backward's scale).
template <int NG, int NW, int MINB, bool BULK, bool DET = false, bool RD = false, bool DS = false>
__global__ void __launch_bounds__(32 * NW, MINB) composite_fwd_kernel(const CompositeFwdParams p) {
    static_assert(!(BULK && RD), "the bulk-copy slab holds records without the depth plane");
    static_assert(!(BULK && DS), "the depth statistics are instantiated with the register prefetch only");
    constexpr int RG = 2 + NG;                       // float4 groups per record
    constexpr int RGX = RG + (RD ? 1 : 0);           // staged groups: RD adds the depth plane (group RG)
    __shared__ __align__(16) float4 sRec[BULK ? 1 : NW][BULK ? 1 : RGX][BULK ? 1 : 32];   // this warp's current 32-entry batch, SoA
    __shared__ __align__(16) float4 sRecB[BULK ? NW : 1][BULK ? 2 : 1][BULK ? 32 : 1][BULK ? RG : 1];   // BULK: [stage][entry][group]
    __shared__ __align__(8) uint64_t sBar[NW][2];
    __shared__ uint32_t sId[NW][32];                 // slab slot -> Gaussian id
    __shared__ uint32_t sPos[NW][32];                // slab slot -> list position (relative to the tile's range)
    __shared__ uint32_t sQ[NW][R3DG_QCAP];           // queued list positions (relative to the tile's range)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int PARTS = 8 / NW;
    const int tile = (int)p.tile_order[blockIdx.x / PARTS];
    const int wb = (blockIdx.x % PARTS) * NW + warp;          // pixel block 0..7 inside the tile
    const int tx = tile % p.gx, tyv = tile / p.gx;
    const int view = tyv / p.gy, ty = tyv - view * p.gy;          // the view's image and its view-local tile row
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

    float T = 1.0f, Dp = 0.0f, Op = 0.0f;
    float C[4 * NG];
#pragma unroll
    for (int i = 0; i < 4 * NG; ++i) C[i] = 0.0f;
    uint32_t last_contributor = 0;
    float D2 = 0.0f, med = 0.0f, dmax = 0.0f;                           // DS only
    uint32_t med_pos = 0u;
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
    float4 r[BULK ? 1 : RGX];
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
        for (int g = 0; g < RGX; ++g) r[g] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (lane < qcount) {
            id_cur = plist[q[(qhead + lane) & (R3DG_QCAP - 1)]];
#pragma unroll
            for (int g = 0; g < RGX; ++g) r[g] = rec4[(size_t)id_cur * rec4n + g];
        }
    }

    uint32_t composited = 0u;                                           // entries this warp composited = its backward twin's iterations
    bool all_done = __all_sync(0xffffffffu, done);
    constexpr int U = NG <= 2 ? 4 : 2;                                  // entries per round of the loop below
    while (qcount > 0 && !all_done) {
        const int n = min(32, qcount);
        const uint32_t mypos = q[(qhead + lane) & (R3DG_QCAP - 1)];     // valid for lane < n
        // second, exact filter — each lane applies round 1's exact-conservative ellipse / rectangle test to ITS OWN staged
        // entry (one evaluation per entry): the block rectangle is conservative, the exact test drops the (warp, entry)
        // pairs whose ellipse misses the block, and every pair dropped here saves the alpha evaluation of the loop below
        uint32_t word;
        if (BULK) word = n == 32 ? 0xffffffffu : ((1u << n) - 1u);       // (records are not in registers in this variant)
        else word = __ballot_sync(0xffffffffu, lane < n && touch_block(r[0], r[1], (float)bx0, (float)by0));
        // the accepted entries are compacted in list order: entry k of the loop below is slab slot k (BULK: every entry
        // is accepted and its bulk copy already sits at slot k = lane).  sId / sPos map a slot back to its Gaussian and
        // its list position.  Slots [n_acc, n_acc + U) get a zero record: opacity 0 gives alpha 0 < 1/255, so a round
        // running past n_acc fails the per-pixel test with finite values and no extra predicate.
        const int n_acc = __popc(word);
        const int k = __popc(word & ((1u << lane) - 1u));
        __syncwarp();
        if ((word >> lane) & 1u) {
            sId[warp][k] = id_cur;
            sPos[warp][k] = mypos;
            if (!BULK) {
#pragma unroll
                for (int g = 0; g < RGX; ++g) sRec[warp][g][k] = r[g];
            }
        }
        if (!BULK && lane >= n_acc && lane < n_acc + U) {
#pragma unroll
            for (int g = 0; g < RGX; ++g) sRec[warp][g][lane] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
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
            for (int g = 0; g < RGX; ++g) r[g] = rec4[(size_t)id_cur * rec4n + g];
        }
        int last_k = -1;                                                // this pixel's last accepted entry of the batch
        int med_k = -1;                                                 // DS: its median entry of the batch, if any
        int my_wsum = 0;                                                // lane k keeps the warp's weight sum of entry k
        // U staged entries per round.  The alpha evaluations (record fetch, quadratic form, exp — two thirds of the
        // work) depend neither on one another nor on the pixel's state, so all U are issued back to back: U dependency
        // chains in flight per warp instead of one.  Only the short transmittance recurrence that follows is sequential,
        // in list order, with exactly the reference's arithmetic.  This is what bounds the kernel: the heaviest pixel
        // blocks composite many entries one after the other, and while the light tiles drain the machine those few
        // warps decide the makespan (DESIGN.md §4.2).  U = 4 for S <= 5, 2 for S > 5 (more accumulators per pixel:
        // registers).
        for (int k0 = 0; k0 < n_acc; k0 += U) {
            bool pv[U];
            float al[U], om[U], dep[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {                                // (1) independent: alpha of U entries
                const float4 a = BULK ? sRecB[warp][stage][k0 + u][0] : sRec[warp][0][k0 + u];
                const float4 b = BULK ? sRecB[warp][stage][k0 + u][1] : sRec[warp][1][k0 + u];
                const float dx = sub_(a.x, pxf), dy = sub_(a.y, pyf);
                // power = -0.5f*(ca*dx*dx + cc*dy*dy) - cb*dx*dy  (forward.cu:344) as compiled
                const float qd = fma_(dx, mul_(dx, a.z), mul_(dy, mul_(dy, b.x)));
                const float power = fma_(qd, -0.5f, -mul_(dy, mul_(dx, a.w)));
                al[u] = fminf(0.99f, mul_(b.y, expf(power)));
                om[u] = sub_(1.0f, al[u]);
                if constexpr (RD) {
                    const float4 pl = sRec[warp][RG][k0 + u];
                    dep[u] = fmaf(-pl.y, dy, fmaf(-pl.x, dx, b.z));     // tz + p . (pixel - mean)
                } else {
                    dep[u] = b.z;
                }
                // BULK has no zero-record padding: its slots past n_acc hold whatever the last copy left there
                pv[u] = (!BULK || k0 + u < n_acc) && !(power > 0.0f) && !(al[u] < 1.0f / 255.0f);
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
                    const float4 c = BULK ? sRecB[warp][stage][k0 + u][2 + g] : sRec[warp][2 + g][k0 + u];
                    fma4_if(valid, w, c, C[4 * g + 0], C[4 * g + 1], C[4 * g + 2], C[4 * g + 3]);
                }
                fma_add_if(valid, w, dep[u], Dp, Op);
                if constexpr (DS) {
                    const float d2 = mul_(dep[u], dep[u]);
                    D2 = valid ? fma_(w, d2, D2) : D2;
                    const bool m = valid && T > 0.5f;                    // T before the entry (2DGS's median rule)
                    med = m ? dep[u] : med;
                    med_k = m ? k0 + u : med_k;
                    dmax = valid ? fmaxf(dmax, fabsf(dep[u])) : dmax;
                }
                T = valid ? test_T : T;
                last_k = valid ? k0 + u : last_k;
                // w in [0,1) in 2^-24 fixed point for the out_weights statistic (below); >= 6 whenever the entry was accepted
                wq[u] = valid ? __float2int_rn(w * 16777216.0f) : 0;
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {                                // (3) independent again: per-entry warp sums
                // sum over the warp's pixels of w for out_weights: one integer REDUX instead of a 5-step float shuffle tree
                // (error <= 1e-6 per warp, far below the reference's own atomic-order noise on this statistic); non-zero
                // exactly when some pixel accepted the entry.  Lane k keeps entry k's sum: ONE atomic instruction per batch.
                const int wsum = __reduce_add_sync(0xffffffffu, wq[u]);
                if (lane == k0 + u) my_wsum = wsum;
            }
            if (__all_sync(0xffffffffu, done)) { all_done = true; break; }      // once per round: entries after the last
        }                                                                        // pixel finished change nothing (valid needs !done)
        if (last_k >= 0) last_contributor = sPos[warp][last_k] + 1u;    // 1-based position in the tile list
        if (DS && med_k >= 0) med_pos = sPos[warp][med_k] + 1u;
        const uint32_t cw = __ballot_sync(0xffffffffu, my_wsum != 0);   // bit k: entry k was composited by some pixel
        if (my_wsum != 0) {
            const uint32_t id = sId[warp][lane];
            if constexpr (DET) det_red_u64(p.det_weights + id, (uint64_t)(uint32_t)my_wsum);   // my_wsum > 0
            else atomicAdd(&p.out_weights[id], (float)my_wsum * (1.0f / 16777216.0f));
            // the row was composited: its gradient row is zeroed and read in the backward (no byte atomics: OR the word)
            atomicOr(&p.clamped32[id >> 2], kComposited << (8 * (id & 3u)));
            // contributor bit for the backward pass: one fire-and-forget atomic per composited entry
            const uint32_t e = lo + sPos[warp][lane];
            atomicOr(&p.cmask32[e >> 2], 1u << (8 * (e & 3u) + wb));
        }
        stage ^= 1;
        composited += (uint32_t)__popc(cw);
    }
    if (lane == 0 && composited) atomicMax(&p.bwd_work[blockIdx.x % PARTS + PARTS * tile], composited);
    if constexpr (DS) {                                 // |d| as float bits: integer order is float order
        const uint32_t b = __reduce_max_sync(0xffffffffu, __float_as_uint(dmax));
        if (lane == 0 && b) atomicMax(p.depth_bound + view, b);
    }
    if (inside) {
        const size_t HW = (size_t)p.H * p.W, pix = (size_t)p.W * py + px, vpix = (size_t)view * HW + pix;
        p.final_T[vpix] = T;
        p.n_contrib[vpix] = (int)last_contributor;
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) p.out_color[(size_t)(3 * view + ch) * HW + pix] = fma_(p.bg[3 * view + ch], T, C[ch]);
#pragma unroll
        for (int ch = 3; ch < 4 * NG; ++ch)
            if (ch - 3 < p.S) p.out_feature[((size_t)view * p.S + (ch - 3)) * HW + pix] = C[ch];
        p.out_depth[vpix] = Dp;
        p.out_opacity[vpix] = Op;
        if constexpr (DS) {
            p.out_depth2[vpix] = D2;
            p.out_median[vpix] = med;
            p.median_pos[vpix] = (int)med_pos;
        }
    }
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
// count that fits one more CTA): by channel groups NG, for the 4-warp CTA (the 8-warp variant is left to ptxas).
// The values are those of the occupancy sweep in DESIGN.md §4.2.
template <int NG> struct FwdOcc { static constexpr int v = NG <= 2 ? 7 : (NG <= 3 ? 6 : (NG <= 5 ? 5 : (NG <= 6 ? 4 : 3))); };
// ray-depth mode (the depth plane's 4 more prefetch registers): fewer CTAs where the count above spills (-Xptxas -v)
template <int NG> struct FwdOccRD { static constexpr int v = FwdOcc<NG>::v - (NG == 2 ? 2 : (NG == 5 ? 1 : 0)); };
// depth statistics (five more per-pixel registers), without and with the ray-depth mode: fewer CTAs where the counts
// above spill (-Xptxas -v)
template <int NG, bool RD> struct FwdOccDS {
    static constexpr int v = RD ? FwdOccRD<NG>::v - (NG <= 3 ? 1 : 0) : FwdOcc<NG>::v - (NG == 2 ? 2 : (NG == 3 || NG == 5 ? 1 : 0));
};

int g_composite_bulk = 0;       // r3dg_tune("composite_bulk"): 1 = TMA bulk-copy record staging in the forward compositor
int g_fwd_ctas = 0;             // r3dg_tune("composite_fwd_ctas"): resident CTAs per SM (0 = whatever fits)
int composite_tune(const char* key, int value, int* previous) {
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
template <auto K>
static void launch_fwd_kernel(const CompositeFwdParams& p, int tiles, cudaStream_t stream) {
    K<<<tiles * 2, 128, residency_pad<K>(g_fwd_ctas), stream>>>(p);    // two 4-warp CTAs per tile
}
template <int NG>
static void launch_fwd_ng(const CompositeFwdParams& p, int tiles, bool ray_depth, bool ds, cudaStream_t stream) {
    if (ds) {                                         // (register prefetch, as the ray-depth mode)
        if (ray_depth) {
            if (p.det_weights) launch_fwd_kernel<composite_fwd_kernel<NG, 4, FwdOccDS<NG, true>::v, false, true, true, true>>(p, tiles, stream);
            else launch_fwd_kernel<composite_fwd_kernel<NG, 4, FwdOccDS<NG, true>::v, false, false, true, true>>(p, tiles, stream);
        } else {
            if (p.det_weights) launch_fwd_kernel<composite_fwd_kernel<NG, 4, FwdOccDS<NG, false>::v, false, true, false, true>>(p, tiles, stream);
            else launch_fwd_kernel<composite_fwd_kernel<NG, 4, FwdOccDS<NG, false>::v, false, false, false, true>>(p, tiles, stream);
        }
        return;
    }
    if (ray_depth) {                                  // (register prefetch: r3dg_tune("composite_bulk") does not apply)
        if (p.det_weights) launch_fwd_kernel<composite_fwd_kernel<NG, 4, FwdOccRD<NG>::v, false, true, true>>(p, tiles, stream);
        else launch_fwd_kernel<composite_fwd_kernel<NG, 4, FwdOccRD<NG>::v, false, false, true>>(p, tiles, stream);
        return;
    }
    if (p.det_weights) {
        if (g_composite_bulk == 1 && NG <= 6) launch_fwd_kernel<composite_fwd_kernel<NG <= 6 ? NG : 1, 4, FwdOcc<NG>::v, true, true>>(p, tiles, stream);
        else launch_fwd_kernel<composite_fwd_kernel<NG, 4, FwdOcc<NG>::v, false, true>>(p, tiles, stream);
        return;
    }
    if (g_composite_bulk == 1 && NG <= 6) launch_fwd_kernel<composite_fwd_kernel<NG <= 6 ? NG : 1, 4, FwdOcc<NG>::v, true>>(p, tiles, stream);
    else launch_fwd_kernel<composite_fwd_kernel<NG, 4, FwdOcc<NG>::v, false>>(p, tiles, stream);
}

int launch_composite_forward(const r3dg_raster_fwd_args& a, const RasterBuffers& b, cudaStream_t stream,
                             stage_mark_fn mark) {
    CompositeFwdParams p;
    const int V = b.V;
    p.W = a.W; p.H = a.H; p.gx = b.gx; p.gy = b.gy; p.S = a.S; p.recf = b.recf;
    p.ranges = b.ranges;
    p.point_list = b.point_list;
    p.bmask32 = (const uint32_t*)b.bmask; p.cmask32 = (uint32_t*)b.cmask;
    p.header = b.header;
    p.tile_order = b.tile_order;
    p.bwd_work = b.bwd_work;
    p.rec = b.rec;
    p.bg = a.background;
    p.final_T = b.final_T;
    p.n_contrib = b.n_contrib;
    p.out_color = a.out_color; p.out_opacity = a.out_opacity; p.out_depth = a.out_depth;
    p.out_feature = a.out_feature; p.out_weights = a.out_weights;
    p.det_weights = a.deterministic ? (uint64_t*)a.det_work : nullptr;
    p.clamped32 = (uint32_t*)b.clamped;               // 256-byte aligned, padded to whole words (api.cu GeomLayout)
    const bool ds = a.depth_stats != 0;
    p.out_depth2 = a.out_depth2; p.out_median = a.out_median_depth;
    p.median_pos = b.median_pos; p.depth_bound = b.depth_bound;
    if (ds) R3DG_CUDA_TRY(cudaMemsetAsync(b.depth_bound, 0, V * sizeof(uint32_t), stream));
    const size_t rows = (size_t)V * a.P;
    if (p.det_weights) R3DG_CUDA_TRY(cudaMemsetAsync(p.det_weights, 0, rows * 8, stream));
    const int tiles = V * b.tiles;                    // the tall grid of all views
    const bool rd = a.ray_depth != 0;
    switch (num_groups(a.S)) {
        case 1: launch_fwd_ng<1>(p, tiles, rd, ds, stream); break;
        case 2: launch_fwd_ng<2>(p, tiles, rd, ds, stream); break;
        case 3: launch_fwd_ng<3>(p, tiles, rd, ds, stream); break;
        case 4: launch_fwd_ng<4>(p, tiles, rd, ds, stream); break;
        case 5: launch_fwd_ng<5>(p, tiles, rd, ds, stream); break;
        case 6: launch_fwd_ng<6>(p, tiles, rd, ds, stream); break;
        case 7: launch_fwd_ng<7>(p, tiles, rd, ds, stream); break;
        case 8: launch_fwd_ng<8>(p, tiles, rd, ds, stream); break;
        case 9: launch_fwd_ng<9>(p, tiles, rd, ds, stream); break;
        default: return R3DG_ERR_UNSUPPORTED;
    }
    if (p.det_weights && a.P > 0) det_weights_kernel<<<(int)((rows + 255) / 256), 256, 0, stream>>>((int)rows, p.det_weights, a.out_weights);
    const size_t HW = (size_t)a.H * a.W;
    mark(6, stream);
    if (a.computer_pseudo_normal) {
        for (int v = 0; v < V; ++v) {                 // each view with its own intrinsics
            float tan_fovx = a.tan_fovx, tan_fovy = a.tan_fovy, cx = a.cx, cy = a.cy;
            view_cam(V, a.view_cams, v, tan_fovx, tan_fovy, cx, cy);
            const float focal_y = a.H / (2.0f * tan_fovy), focal_x = a.W / (2.0f * tan_fovx);
            dim3 grid((a.W + 31) / 32, (a.H + 7) / 8);
            surface_normal_kernel<<<grid, 256, 0, stream>>>(a.W, a.H, a.viewmatrix + 16 * v, focal_x, focal_y, cx, cy,
                                                            a.out_opacity + v * HW, a.out_depth + v * HW,
                                                            a.out_normal + 3 * v * HW, a.out_surface_xyz + 3 * v * HW);
        }
    } else {
        R3DG_CUDA_TRY(cudaMemsetAsync(a.out_normal, 0, 3 * V * HW * 4, stream));
        R3DG_CUDA_TRY(cudaMemsetAsync(a.out_surface_xyz, 0, 3 * V * HW * 4, stream));
    }
    if (a.n_contrib)   // the reference returns n_contrib as a view of imgBuffer (rasterize_points.cu:136-139)
        R3DG_CUDA_TRY(cudaMemcpyAsync(a.n_contrib, b.n_contrib, V * HW * 4, cudaMemcpyDeviceToDevice, stream));
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace r3dg
