// Order-independent fp32 accumulation for the deterministic mode (torch.use_deterministic_algorithms(True)).
//
// A float atomicAdd makes a sum depend on the order in which warps arrive.  Here every fp32 term is converted to a
// signed fixed-point integer with R3DG_DET_FRAC fraction bits, and integer addition, which is associative, adds it
// to an accumulator.  The total is converted back to fp32 once, when it is read.  So a total depends only on the set
// of its terms, never on their order.
//
// Format.  A term x is rounded to the nearest multiple of 2^-48 (ties to even) and held as a 96-bit two's complement
// integer q, split into three 32-bit chunks: lo and mid unsigned, hi signed.  An accumulator is three 64-bit words,
// each the sum of one chunk over the terms, added with `red.global.add.u64` (no return value):
//     total = hi_sum * 2^64 + mid_sum * 2^32 + lo_sum          (in units of 2^-48)
// The lo and mid words add 32-bit chunks, so they cannot overflow before 2^32 terms; hi_sum is a signed 64-bit word.
//   * resolution 2^-48 = 3.6e-15: each term is off by at most 2^-49, rounded the same way every time.  That is ~1e-8
//     of a 1e-7 term, below fp32's own rounding of it; the reference's float atomics already differ run to run by
//     ~1e-6 relative on the parity cases' gradients (tests/golden/live_raster*.npz noise_*).
//   * term range |x| < 2^47 = 1.4e14, eleven decades above the largest gradient-row entries of the parity goldens
//     (dL_dmeans2D, below 1e3 in tests/golden/raster_*.npz).  A finite term outside the range saturates to +-Inf, as an fp32
//     overflow would: it never wraps.
//   * at most 2^31 terms per accumulator, so |total| < 2^126 units: reading never overflows fp32 (< 2^78).
//   * NaN and +-Inf set sticky flag bits (2 per accumulator, 16 accumulators per 32-bit word, atomicOr): bit 0 = a
//     +Inf (or an out-of-range positive term), bit 1 = a -Inf (or out-of-range negative term), both = NaN.  So NaN
//     wins and +Inf with -Inf gives NaN, as IEEE addition does.
//   * the read rounds the exact integer total to nearest fp32 once; an exact zero total reads as +0.
// Memory: 24 B + 2 bits per accumulator, laid out as three planes of n words ([lo][mid][hi]) and the flag words.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <cuda_runtime.h>

#define R3DG_DET_FRAC 48
#define R3DG_DET_RANGE_LOG2 47       // |term| < 2^47

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

// fp32 term -> three chunk words (or a flag for NaN / +-Inf / out of range)
__host__ __device__ inline DetTerm det_term(float x) {
    const uint32_t u = det_f32_bits(x);
    const uint32_t e = (u >> 23) & 0xffu, neg = u >> 31;
    uint32_t m = u & 0x7fffffu;
    DetTerm t = {0u, 0u, 0u, 0u};
    if (e == 255u) { t.flag = m ? 3u : (neg ? 2u : 1u); return t; }
    if (e >= 127u + R3DG_DET_RANGE_LOG2) { t.flag = neg ? 2u : 1u; return t; }
    if (e) m |= 0x800000u;
    const int s = (e ? (int)e : 1) - 150 + R3DG_DET_FRAC;    // x = m * 2^(s - FRAC)
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

// The fp32 value of an accumulator (words summed modulo 2^64, flag = its 2 flag bits), rounded once.
__host__ __device__ inline float det_value(uint64_t lo, uint64_t mid, uint64_t hi, uint32_t flag) {
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
    const float r = f * scale;
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
__device__ __forceinline__ void det_add(uint64_t* words, uint32_t* flags, size_t n, size_t i, float x, bool shared) {
    const DetTerm t = det_term(x);
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
__device__ __forceinline__ void det_add(const DetAcc& a, size_t i, float x) { det_add(a.words, a.flags, a.n, i, x, false); }
__device__ __forceinline__ float det_load(const DetAcc& a, size_t i) {
    return det_value(a.words[i], a.words[a.n + i], a.words[2 * a.n + i], (a.flags[i >> 4] >> (2 * (i & 15))) & 3u);
}
#endif

}  // namespace r3dg
