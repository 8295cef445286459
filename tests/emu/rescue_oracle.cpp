// tests/emu/rescue_oracle.cpp -- TEST INFRASTRUCTURE: an independent restatement of the Rescue-Prime permutation
// (code/rescue_prime.py hash and trace, state width 2) for checking the kernel at sizes Python cannot afford.  It
// shares no code with csrc/: two 64-bit limbs, a generic CIOS Montgomery product with -p^-1 computed at start-up, and
// right-to-left exponentiation.  tests/test_rescue_cpu.py pins it to tests/golden/rescue.json.
//
// Constants and exponents are arguments, in sa_rescue's order: the MDS matrix row-major, then 4 * rounds round
// constants.  Outputs are dense: hashes[b], and trace[(b * 2 + s) * (rounds + 1) + r].
#include <stddef.h>
#include <stdint.h>

typedef unsigned __int128 u128;

static const u128 kP = ((u128)407 << 119) + 1;

static uint64_t neg_pinv() {  // -p^-1 mod 2^64 by Newton's iteration on the low word
    const uint64_t p0 = (uint64_t)kP;
    uint64_t x = 1;
    for (int i = 0; i < 6; i++) x *= 2 - p0 * x;
    return 0 - x;
}

static u128 add_mod(u128 a, u128 b) { return a >= kP - b ? a - (kP - b) : a + b; }

// a * b * 2^-128 mod p, CIOS over two words
static u128 mont(u128 a, u128 b, uint64_t np) {
    const uint64_t A[2] = {(uint64_t)a, (uint64_t)(a >> 64)}, B[2] = {(uint64_t)b, (uint64_t)(b >> 64)};
    const uint64_t M[2] = {(uint64_t)kP, (uint64_t)(kP >> 64)};
    uint64_t t[4] = {0, 0, 0, 0};
    for (int i = 0; i < 2; i++) {
        u128 c = 0;
        for (int j = 0; j < 2; j++) {
            c += (u128)t[j] + (u128)A[j] * B[i];
            t[j] = (uint64_t)c;
            c >>= 64;
        }
        c += t[2];
        t[2] = (uint64_t)c;
        t[3] = (uint64_t)(c >> 64);
        const uint64_t m = t[0] * np;
        c = (u128)t[0] + (u128)m * M[0];
        c >>= 64;
        c += (u128)t[1] + (u128)m * M[1];
        t[0] = (uint64_t)c;
        c >>= 64;
        c += t[2];
        t[1] = (uint64_t)c;
        t[2] = t[3] + (uint64_t)(c >> 64);
    }
    u128 r = ((u128)t[1] << 64) | t[0];
    if (t[2] || r >= kP) r -= kP;
    return r;
}

struct Ctx {
    uint64_t np;
    u128 one, r2;  // 2^128 and 2^256 mod p
};

static Ctx ctx() {
    Ctx c;
    c.np = neg_pinv();
    c.one = (u128)0 - kP;  // 2^128 - p < p
    c.r2 = c.one;
    for (int i = 0; i < 128; i++) c.r2 = add_mod(c.r2, c.r2);
    return c;
}

static u128 pow_mont(u128 x, u128 e, const Ctx &c) {
    u128 acc = c.one;
    while (e) {
        if (e & 1) acc = mont(acc, x, c.np);
        x = mont(x, x, c.np);
        e >>= 1;
    }
    return acc;
}

static u128 load(const uint64_t *v) { return ((u128)v[1] << 64) | v[0]; }
static void store(uint64_t *out, u128 x) {
    out[0] = (uint64_t)x;
    out[1] = (uint64_t)(x >> 64);
}

extern "C" {

// x^e mod p for canonical x and any 128-bit e (x^0 = 1)
void rescue_oracle_pow(uint64_t *out, const uint64_t *x, const uint64_t *e) {
    const Ctx c = ctx();
    store(out, mont(pow_mont(mont(load(x), c.r2, c.np), load(e), c), 1, c.np));
}

void rescue_oracle(uint64_t *hashes, uint64_t *trace, const uint64_t *inputs, size_t count, const uint64_t *constants,
                   size_t rounds, const uint64_t *alpha, const uint64_t *alphainv) {
    const Ctx c = ctx();
    const u128 ea = load(alpha), eb = load(alphainv);
    u128 mds[4];
    for (int i = 0; i < 4; i++) mds[i] = mont(load(constants + 2 * i), c.r2, c.np);
    const size_t rows = rounds + 1;
    for (size_t b = 0; b < count; b++) {
        u128 st[2] = {mont(load(inputs + 2 * b), c.r2, c.np), 0};
        uint64_t *tr = trace ? trace + 2 * (2 * b * rows) : nullptr;
        for (size_t r = 0; r <= rounds; r++) {
            if (r > 0) {
                for (int half = 0; half < 2; half++) {
                    const u128 e = half ? eb : ea;
                    const u128 x0 = pow_mont(st[0], e, c), x1 = pow_mont(st[1], e, c);
                    const uint64_t *k = constants + 2 * (4 + 4 * (r - 1) + 2 * half);
                    for (int i = 0; i < 2; i++)
                        st[i] = add_mod(add_mod(mont(mds[2 * i], x0, c.np), mont(mds[2 * i + 1], x1, c.np)),
                                        mont(load(k + 2 * i), c.r2, c.np));
                }
            }
            if (tr) {
                store(tr + 2 * r, mont(st[0], 1, c.np));
                store(tr + 2 * (rows + r), mont(st[1], 1, c.np));
            }
        }
        if (hashes) store(hashes + 2 * b, mont(st[0], 1, c.np));
    }
}

}  // extern "C"
