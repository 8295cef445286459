// rescue.cuh -- the Rescue-Prime permutation of state width m = 2 over many inputs (code/rescue_prime.py hash and
// trace, DESIGN section 3.14): absorb [x, 0]; N rounds of a forward half-round (S-box x^alpha, MDS, constants
// 4r + i) and a backward half-round (S-box x^alphainv, MDS, constants 4r + 2 + i); squeeze state[0].  Trace row 0 is
// the absorbed state and row r + 1 the state after round r.
//
// The MDS matrix, the round constants and both exponents are the caller's: nothing here is a Rescue constant.  The
// constants are converted to Montgomery form once per block (rescue_load), the state stays in Montgomery form in
// registers, and each S-box is one uniform left-to-right square-and-multiply over the exponent's bits with the two
// registers' chains interleaved.  __host__ __device__ so that tests/emu runs the same code on the CPU.
#pragma once
#include "../../include/sa_b200.h"
#include "field.cuh"

namespace sa {

// an exponent e < 2^128 and its bit length (0 for e = 0)
struct RescueExp {
    uint64_t lo, hi;
    int bits;
};

inline RescueExp rescue_exp(const uint64_t e[2]) {
    RescueExp x;
    x.lo = e[0];
    x.hi = e[1];
    x.bits = e[1] ? 128 - __builtin_clzll(e[1]) : (e[0] ? 64 - __builtin_clzll(e[0]) : 0);
    return x;
}

// the number of elements of the constant block: the MDS matrix (4) and 4 constants per round
SA_HD long long rescue_nconst(long long rounds) { return 4 + 4 * rounds; }

// constant i of the caller's canonical block, in Montgomery form
SA_HD fe rescue_load(const fe *constants, long long i) { return fe_to_mont(constants[i]); }

// (x0^e, x1^e), Montgomery form in and out: left to right over e's bits, the first set bit taking x itself, and
// the two chains interleaved so that each thread has two independent products in flight.  The branch on a bit is
// the same in every thread.  x^0 = 1 for every x, 0 included, as FieldElement.__xor__ gives.
SA_HD void rescue_pow2(fe &x0, fe &x1, const RescueExp &e) {
    if (e.bits == 0) {
        x0 = x1 = fe_mont_one();
        return;
    }
    fe a0 = x0, a1 = x1;
    for (int i = e.bits - 2; i >= 0; i--) {
        a0 = fe_montmul(a0, a0);
        a1 = fe_montmul(a1, a1);
        const uint64_t bit = i >= 64 ? (e.hi >> (i - 64)) & 1 : (e.lo >> i) & 1;
        if (bit) {
            a0 = fe_montmul(a0, x0);
            a1 = fe_montmul(a1, x1);
        }
    }
    x0 = a0;
    x1 = a1;
}

// one half-round on the Montgomery state: S-box, MDS (mds row-major), then add rc[0], rc[1]
SA_HD void rescue_half_round(fe &s0, fe &s1, const fe *mds, const fe *rc, const RescueExp &e) {
    rescue_pow2(s0, s1, e);
    const fe t0 = fe_add(fe_add(fe_montmul(mds[0], s0), fe_montmul(mds[1], s1)), rc[0]);
    const fe t1 = fe_add(fe_add(fe_montmul(mds[2], s0), fe_montmul(mds[3], s1)), rc[1]);
    s0 = t0;
    s1 = t1;
}

// input b < count: its hash into hashes[b] (when hashes is not NULL) and its trace (when trace is not NULL),
// register s of row r at b * inst_stride + s * lane_stride + r.  kc is the constant block in Montgomery form.
SA_HD void rescue_elem(fe *hashes, fe *trace, const fe *inputs, const fe *kc, long long rounds, const RescueExp &ea,
                       const RescueExp &eb, long long inst_stride, long long lane_stride, long long b) {
    const fe x = inputs[b];
    fe s0 = fe_to_mont(x), s1 = fe_zero();
    fe *row = trace ? trace + b * inst_stride : nullptr;
    if (row) {
        row[0] = x;
        row[lane_stride] = fe_zero();
    }
    for (long long r = 0; r < rounds; r++) {
        rescue_half_round(s0, s1, kc, kc + 4 + 4 * r, ea);
        rescue_half_round(s0, s1, kc, kc + 6 + 4 * r, eb);
        if (row) {
            row[r + 1] = fe_from_mont(s0);
            row[lane_stride + r + 1] = fe_from_mont(s1);
        }
    }
    if (hashes) hashes[b] = fe_from_mont(s0);
}

// the arguments sa_rescue refuses with SA_ESIZE: both outputs NULL, rounds outside 1..SA_RESCUE_MAX_ROUNDS, and a
// count or largest element offset at or above 2^59 (so that its byte offset fits a signed 64-bit integer).  The
// largest trace offset is (count - 1) inst_stride + lane_stride + rounds.
inline int rescue_check(const void *hashes, const void *trace, size_t count, size_t rounds, size_t inst_stride,
                        size_t lane_stride) {
    if (!hashes && !trace) return SA_ESIZE;
    if (rounds == 0 || rounds > SA_RESCUE_MAX_ROUNDS) return SA_ESIZE;
    if (count == 0) return SA_OK;
    const unsigned long long lim = 1ULL << 59;
    if (count >= lim) return SA_ESIZE;
    if (trace) {
        unsigned long long a;
        if (__builtin_mul_overflow((unsigned long long)(count - 1), (unsigned long long)inst_stride, &a) ||
            a >= lim || lane_stride >= lim || a + lane_stride + rounds >= lim)  // three terms below 2^59: no wrap
            return SA_ESIZE;
    }
    return SA_OK;
}

}  // namespace sa
