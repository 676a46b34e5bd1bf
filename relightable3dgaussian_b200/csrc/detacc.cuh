// Order-independent fp32 accumulation for the deterministic mode (torch.use_deterministic_algorithms(True)).
//
// A float atomicAdd makes a sum depend on the order in which warps arrive.  Here every fp32 term is converted to a
// signed fixed-point integer with R3DG_DET_FRAC fraction bits, and integer addition, which is associative, adds it
// to an accumulator.  The total is converted back to fp32 once, when it is read.  So a total depends only on the set
// of its terms, never on their order.
//
// Scale.  Every accumulator class has a binary exponent e (det_scale_exp): a term x is accumulated as x * 2^-e and
// the total read back times 2^e.  Both are exact (shifts of the fixed point), so results are bitwise equivariant under
// power-of-two scaling of the inputs.  The callers take e from the largest |cotangent| that class's terms are linear in,
// reduced on the device per call (det_max_bits): scaled, that maximum lies in [1, 2), so resolution and range below
// are relative to the call's cotangent scale rather than absolute.  A training loss averaged over 3 H W pixels has
// cotangents near 2^-21; with a fixed 2^-48 unit a faint term (alpha T cot ~ 1e-12) would lose ~1e-3 of itself.
//
// Format (in units of the scaled term x * 2^-e).  A term is rounded to the nearest multiple of 2^-48 (ties to even)
// and held as a 96-bit two's complement integer q, split into three 32-bit chunks: lo and mid unsigned, hi signed.
// An accumulator is three 64-bit words, each the sum of one chunk over the terms, added with `red.global.add.u64`
// (no return value):
//     total = hi_sum * 2^64 + mid_sum * 2^32 + lo_sum          (in units of 2^(e-48))
// The lo and mid words add 32-bit chunks, so they cannot overflow before 2^32 terms; hi_sum is a signed 64-bit word.
//   * resolution 2^(e-48): each term is off by at most 2^(e-49), i.e. 2^-48 of the largest cotangent, rounded the
//     same way every time.  That is ~1e-8 of a 1e-7 term at unit scale, below fp32's own rounding of it; the
//     reference's float atomics already differ run to run by ~1e-6 relative on the parity cases' gradients
//     (tests/golden/live_raster*.npz noise_*).
//   * term range |x * 2^-e| < 2^47 = 1.4e14, eleven decades above the largest gradient-row entries of the parity
//     goldens at unit cotangents (dL_dmeans2D, below 1e3 in tests/golden/raster_*.npz).  A finite term outside the
//     range saturates to +-Inf, as an fp32 overflow would: it never wraps.
//   * e is clamped to [-R3DG_DET_SCALE_MAX, R3DG_DET_SCALE_MAX], and is 0 for an all-zero, NaN or Inf maximum (the
//     flags below carry NaN and Inf).
//   * at most 2^31 terms per accumulator, so |total| < 2^126 units: reading never overflows fp32 before the 2^e.
//   * NaN and +-Inf set sticky flag bits (2 per accumulator, 16 accumulators per 32-bit word, atomicOr): bit 0 = a
//     +Inf (or an out-of-range positive term), bit 1 = a -Inf (or out-of-range negative term), both = NaN.  So NaN
//     wins and +Inf with -Inf gives NaN, as IEEE addition does.
//   * the read rounds the exact integer total to nearest fp32 once, then multiplies by 2^e (exact unless the result
//     is subnormal); an exact zero total reads as +0.
// Memory: 24 B + 2 bits per accumulator, laid out as three planes of n words ([lo][mid][hi]) and the flag words; the
// callers add one 32-bit maximum word per class.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <cuda_runtime.h>

#define R3DG_DET_FRAC 48
#define R3DG_DET_RANGE_LOG2 47       // |term * 2^-e| < 2^47
#define R3DG_DET_SCALE_MAX 100       // |e| <= 100

namespace r3dg {

struct DetTerm { uint64_t lo, mid, hi; uint32_t flag; };

__host__ __device__ inline uint32_t det_f32_bits(float x) {
#ifdef __CUDA_ARCH__
    return __float_as_uint(x);
#else
    uint32_t u;
    memcpy(&u, &x, 4);
    return u;
#endif
}
__host__ __device__ inline float det_f32_from_bits(uint32_t u) {
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float x;
    memcpy(&x, &u, 4);
    return x;
#endif
}

// The exponent e of a class whose largest |input| has the float bits `max_bits` (sign cleared): floor(log2 max),
// clamped; 0 for a zero, subnormal, Inf or NaN maximum
__host__ __device__ inline int det_scale_exp(uint32_t max_bits) {
    const int b = (int)(max_bits >> 23);
    if (b == 0 || b >= 255) return 0;
    const int e = b - 127;
    return e < -R3DG_DET_SCALE_MAX ? -R3DG_DET_SCALE_MAX : (e > R3DG_DET_SCALE_MAX ? R3DG_DET_SCALE_MAX : e);
}

// fp32 term x -> three chunk words of x * 2^-e (or a flag for NaN / +-Inf / out of range)
__host__ __device__ inline DetTerm det_term(float x, int sc) {
    const uint32_t u = det_f32_bits(x);
    const uint32_t e = (u >> 23) & 0xffu, neg = u >> 31;
    uint32_t m = u & 0x7fffffu;
    DetTerm t = {0u, 0u, 0u, 0u};
    if (e == 255u) { t.flag = m ? 3u : (neg ? 2u : 1u); return t; }
    if ((int)e >= 127 + R3DG_DET_RANGE_LOG2 + sc) { t.flag = neg ? 2u : 1u; return t; }
    if (e) m |= 0x800000u;
    const int s = (e ? (int)e : 1) - 150 + R3DG_DET_FRAC - sc;   // x * 2^-sc = m * 2^(s - FRAC)
    unsigned __int128 q;
    if (s >= 0) {
        q = (unsigned __int128)m << s;                       // s <= 71: q < 2^95
    } else if (s <= -25) {
        q = 0;                                               // m < 2^24 <= half a unit
    } else {
        const int r = -s;
        uint32_t k = m >> r;
        const uint32_t rem = m & ((1u << r) - 1u), half = 1u << (r - 1);
        if (rem > half || (rem == half && (k & 1u))) ++k;    // round to nearest, ties to even
        q = k;
    }
    if (neg) q = (unsigned __int128)0 - q;
    t.lo = (uint32_t)q;
    t.mid = (uint32_t)(q >> 32);
    t.hi = (uint64_t)(int64_t)(int32_t)(uint32_t)(q >> 64);
    return t;
}

// The fp32 value of an accumulator of class exponent e (words summed modulo 2^64, flag = its 2 flag bits), rounded once.
__host__ __device__ inline float det_value(uint64_t lo, uint64_t mid, uint64_t hi, uint32_t flag, int e) {
    if (flag == 3u) return det_f32_from_bits(0x7fc00000u);
    if (flag == 1u) return det_f32_from_bits(0x7f800000u);
    if (flag == 2u) return det_f32_from_bits(0xff800000u);
    const unsigned __int128 T = ((unsigned __int128)hi << 64) + ((unsigned __int128)mid << 32) + lo;
    const bool neg = (T >> 127) != 0;
    const unsigned __int128 mag = neg ? (unsigned __int128)0 - T : T;
    const uint64_t top = (uint64_t)(mag >> 64);
    int k = 0;                                               // shift that leaves at most 64 significant bits
    if (top) {
#ifdef __CUDA_ARCH__
        k = 64 - __clzll((long long)top);
#else
        k = 64 - __builtin_clzll(top);
#endif
    }
    uint64_t v = (uint64_t)(mag >> k);
    if (k && (uint64_t)(mag & ((((unsigned __int128)1) << k) - 1))) v |= 1u;   // sticky bit: one correct rounding below
#ifdef __CUDA_ARCH__
    const float f = __ull2float_rn(v);
#else
    const float f = (float)v;
#endif
    const float scale = det_f32_from_bits((uint32_t)(127 + k - R3DG_DET_FRAC) << 23);   // exact power of two
    const float r = f * scale * det_f32_from_bits((uint32_t)(127 + e) << 23);   // |e| <= 100: both exact powers of two
    return neg ? -r : r;
}

// n accumulators in a caller-provided, zero-initialised workspace
struct DetAcc {
    uint64_t* words;     // [3][n]
    uint32_t* flags;     // [(n + 15) / 16]
    size_t n;
};
__host__ __device__ inline size_t det_flags_offset(size_t n) { return (3 * n * 8 + 255) / 256 * 256; }
__host__ __device__ inline size_t det_bytes(size_t n) { return det_flags_offset(n) + ((n + 15) / 16 * 4 + 255) / 256 * 256; }
inline DetAcc det_acc(void* base, size_t n) {
    DetAcc a;
    a.words = (uint64_t*)base;
    a.flags = base ? (uint32_t*)((char*)base + det_flags_offset(n)) : nullptr;
    a.n = n;
    return a;
}

#ifdef __CUDACC__
__device__ __forceinline__ void det_red_u64(uint64_t* p, uint64_t v) {
    asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// words / flags may be global or shared (n = plane stride)
__device__ __forceinline__ void det_add(uint64_t* words, uint32_t* flags, size_t n, size_t i, float x, int e, bool shared) {
    const DetTerm t = det_term(x, e);
    if (t.flag) { atomicOr(flags + (i >> 4), t.flag << (2 * (i & 15))); return; }
    if (shared) {
        if (t.lo) atomicAdd((unsigned long long*)(words + i), (unsigned long long)t.lo);
        if (t.mid) atomicAdd((unsigned long long*)(words + n + i), (unsigned long long)t.mid);
        if (t.hi) atomicAdd((unsigned long long*)(words + 2 * n + i), (unsigned long long)t.hi);
    } else {
        if (t.lo) det_red_u64(words + i, t.lo);
        if (t.mid) det_red_u64(words + n + i, t.mid);
        if (t.hi) det_red_u64(words + 2 * n + i, t.hi);
    }
}
__device__ __forceinline__ void det_add(const DetAcc& a, size_t i, float x, int e) { det_add(a.words, a.flags, a.n, i, x, e, false); }
__device__ __forceinline__ float det_load(const DetAcc& a, size_t i, int e) {
    return det_value(a.words[i], a.words[a.n + i], a.words[2 * a.n + i], (a.flags[i >> 4] >> (2 * (i & 15))) & 3u, e);
}
// |x| as float bits (sign cleared): unsigned order is the order of |x|, with +Inf above every finite value and NaN
// above +Inf.  The per-class maximum is combined with atomicMax on these bits, which is exact and order-independent.
__device__ __forceinline__ uint32_t det_abs_bits(float x) { return __float_as_uint(x) & 0x7fffffffu; }
// the warp's maximum of v, added to *max_bits by lane 0 (every lane of the warp calls it)
__device__ __forceinline__ void det_max_bits(uint32_t* max_bits, uint32_t v) {
    v = __reduce_max_sync(0xffffffffu, v);
    if ((threadIdx.x & 31) == 0 && v) atomicMax(max_bits, v);
}
#endif

}  // namespace r3dg
