// sample.cuh -- seeded randomizer draws: the element Field.sample(os.urandom(17)) gives (code/algebra.py:118-120)
// when os.urandom returns the counter-mode expansion of a 32-byte seed (DESIGN section 3.13):
//   draw(s, j)    = blake2b(s || j as 8 little-endian bytes).digest()[:17]
//   element(s, j) = int.from_bytes(draw(s, j), "big") mod p
// and the index map of sa_sample_seeded.  __host__ __device__ so tests/emu can run the same code on the CPU.
#pragma once
#include "../../include/sa_b200.h"
#include "hash.cuh"

namespace sa {

SA_HD uint64_t sample_bswap64(uint64_t x) {
#if defined(__CUDA_ARCH__)
    return ((uint64_t)__byte_perm((uint32_t)x, 0, 0x0123) << 32) | __byte_perm((uint32_t)(x >> 32), 0, 0x0123);
#else
    return __builtin_bswap64(x);
#endif
}

// x = top * 2^128 + hi * 2^64 + lo (x < 2^136, so top < 2^8) -> x mod p, canonical.
// Write x = h * 2^119 + l with l < 2^119 and h = x >> 119 < 2^17, and h = 407 q + m with m < 407.  Since
// 407 * 2^119 = p - 1, x = q (p - 1) + m 2^119 + l = q p + (r0 - q) with r0 = m 2^119 + l <= 406 2^119 + 2^119 - 1
// = p - 2 and q <= (2^17 - 1) / 407 = 322.  So r0 - q lies in [-322, p - 2]: r0 - q, plus p when it borrows.
SA_HD fe sample_reduce(uint32_t top, uint64_t hi, uint64_t lo) {
    const uint32_t h = (top << 9) | (uint32_t)(hi >> 55);
    const uint32_t q = h / 407u, m = h - 407u * q;
    const uint64_t r_hi = ((uint64_t)m << 55) | (hi & ((1ULL << 55) - 1));
    // (r_hi, lo) - q, then + p = (1, 407 << 55) on a borrow
    const uint64_t d_lo = lo - q;
    const uint64_t br = lo < q;
    uint64_t d_hi = r_hi - br;
    const uint64_t neg = r_hi < br;  // only with r0 < q: r_hi = 0 and lo < q
    const uint64_t a_lo = d_lo + neg;
    d_hi += (neg ? (407ULL << 55) : 0) + (a_lo < d_lo);
    return fe_make((uint32_t)a_lo, (uint32_t)(a_lo >> 32), (uint32_t)d_hi, (uint32_t)(d_hi >> 32));
}

// the digest's first 17 bytes, big-endian, reduced: digest byte i is byte i % 8 of word i / 8 (little-endian)
SA_HD fe sample_from_digest(uint64_t w0, uint64_t w1, uint64_t w2) {
    const uint64_t b0 = sample_bswap64(w0), b1 = sample_bswap64(w1);  // bytes 0..7 and 8..15 as big-endian ints
    // x = b0 2^72 + b1 2^8 + byte16
    const uint64_t lo = (b1 << 8) | (w2 & 0xFF);
    const uint64_t hi = (b0 << 8) | (b1 >> 56);
    return sample_reduce((uint32_t)(b0 >> 56), hi, lo);
}

// element(seed, j): one compression of the 40-byte block seed || j (seed as four little-endian words)
SA_HD fe seeded_element(uint64_t s0, uint64_t s1, uint64_t s2, uint64_t s3, uint64_t j) {
    uint64_t m[16], d[8];
    m[0] = s0;
    m[1] = s1;
    m[2] = s2;
    m[3] = s3;
    m[4] = j;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int i = 5; i < 16; i++) m[i] = 0;
    blake2b_single_block(d, m, 40u);
    return sample_from_digest(d[0], d[1], d[2]);
}

// word w of a 32-byte seed read byte by byte (the seeds need no alignment)
SA_HD uint64_t sample_seed_word(const uint8_t *seed, int w) {
    uint64_t x = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int i = 7; i >= 0; i--) x = (x << 8) | seed[8 * w + i];
    return x;
}

// item i < nseeds * count of sa_sample_seeded: seed b = i / count, draw first + j with j = i % count, written at
// element offset b * seed_stride + (j % width) * lane_stride + j / width of out
SA_HD void sample_seeded_elem(fe *out, const uint8_t *seeds, uint64_t first, long long count, long long width,
                              long long lane_stride, long long seed_stride, long long i) {
    const long long b = i / count, j = i - b * count;
    const uint8_t *s = seeds + 32 * b;
    const fe x = seeded_element(sample_seed_word(s, 0), sample_seed_word(s, 1), sample_seed_word(s, 2),
                                sample_seed_word(s, 3), first + (uint64_t)j);
    const long long lane = j / width;
    out[b * seed_stride + (j - lane * width) * lane_stride + lane] = x;
}

// the arguments sa_sample_seeded refuses with SA_ESIZE, and its item count nseeds * count (0: nothing to do): width 0,
// a draw index first + count - 1 above 2^64 - 1, and an item count or largest element offset at or above 2^59 (so
// that its byte offset fits a signed 64-bit integer).  The largest offset is bounded by (nseeds - 1) seed_stride +
// (min(count, width) - 1) lane_stride + (count - 1) / width.
inline int sample_check(size_t nseeds, size_t seed_stride, uint64_t first, size_t count, size_t width,
                        size_t lane_stride, long long *total) {
    *total = 0;
    if (width == 0) return SA_ESIZE;
    if (nseeds == 0 || count == 0) return SA_OK;
    const unsigned long long lim = 1ULL << 59;
    if (count - 1 > ~first) return SA_ESIZE;
    unsigned long long items, a, c;
    if (__builtin_mul_overflow((unsigned long long)nseeds, (unsigned long long)count, &items) || items >= lim)
        return SA_ESIZE;
    const unsigned long long lanes = (count < width ? count : width) - 1;
    if (__builtin_mul_overflow((unsigned long long)(nseeds - 1), (unsigned long long)seed_stride, &a) || a >= lim ||
        __builtin_mul_overflow(lanes, (unsigned long long)lane_stride, &c) || c >= lim)
        return SA_ESIZE;
    if (a + c + (count - 1) / width >= lim) return SA_ESIZE;  // three terms below 2^59: no wrap
    *total = (long long)items;
    return SA_OK;
}

}  // namespace sa
