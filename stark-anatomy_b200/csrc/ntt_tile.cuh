// ntt_tile.cuh -- the NTT building block: L-point transforms (L = 2^LOGL <= 1024)
// on a tile of C columns, natural order in, natural order out.
// Reproduces code/ntt.py:3-18 (out[i] = sum_j v[j] * w^(i*j)); bit-exact because
// every operation is exact arithmetic on canonical residues (field.cuh).
//
// Algorithm (GPU-first, not the reference's recursion): mixed-radix
// decimation with register blocks of E = 2^ELOG elements (E = 16 or 8).  A thread
// owns E elements of one column, runs a complete E-point transform in registers,
// applies the inter-stage twiddle, and exchanges through shared memory only
// between register blocks.  All stages work in place on tile row
// p = K*M' + d*M + m (d = the digit being transformed), so the first block loads
// straight from global memory into registers and the last one stores straight
// from registers, digit-reversed, to the natural output index.
//
// The full-radix stages share ONE copy of the E-point transform code (a rolled
// loop with run-time strides), which keeps the kernel inside the instruction
// cache; only the first (global loads) and last (output twiddle + global stores)
// differ.
//
// A tile row is C columns x 16 bytes.  With C = 8 a row is one 128-byte line:
// lanes 0-7 of every quarter warp cover a full row, every shared-memory access
// is conflict free and every global access is a full line.  C = 4 / 2 give 64 /
// 32-byte segments (still whole sectors) with smaller tiles, i.e. more
// independent CTAs per SM.
//
// The functions are __host__ __device__: tests/emu runs exactly this code on the
// CPU, thread by thread and phase by phase.
#pragma once
#include "field.cuh"

namespace sa {

constexpr int TILE_MAX_PEERS = 7;  // 8 GPUs per NVSwitch domain: self + 7

struct TileArgs {
    const fe *in;
    fe *out;
    const fe *tw;   // tw[e] = w_L^e (Montgomery form), e < L
    const fe *twb;  // optional output twiddle matrix [k * twb_stride + col]; nullptr = none
    long long in_sr, in_sc, in_sb;     // element strides of (row, column, batch) on input
    long long out_sr, out_sc, out_sb;  // ... and on output
    long long twb_stride;
    // batch item bb splits as (bb / inner, bb % inner): offset = (bb / inner) * sb + (bb % inner) * sb2
    long long in_sb2, out_sb2;
    int inner;   // 1 = plain batch
    int ncols;   // valid columns per batch item
    int nbatch;  // batch items
    int has_scale;
    fe scale;   // Montgomery-form scalar applied to every output when has_scale
    fe cst[8];  // cst[k] = w_16^k (Montgomery form) when L >= 16, else w_L^k; k < 8
    // multi-GPU assembly (sa_ntt_multi): the last stage also stores every output to the same element
    // offset of these peer buffers (device memory of other GPUs mapped over NVLink), so the result lands
    // on every rank while it is being computed and no gather pass follows
    fe *peer_out[TILE_MAX_PEERS];
    int npeer;
    // ... or ONE multicast address (NVLink SHARP / NVLS: a multicast object with every rank's buffer bound to it):
    // a single multimem.st leaves the GPU and the switch delivers it to every rank's buffer, the own one included
    fe *mc_out;
    // factored output twiddle (TF_TWB2 kernels only): the ncols = n2 * n3 columns split as col = j2 * n3 + j3
    // with n2 = twb_stride, and the factor of row k is twb[k * n2 + j2] * twb_b[k * n3 + j3].  (One pointer
    // fills the struct's tail padding, so the kernel parameters after it keep their offsets.)
    const fe *twb_b;
};
static_assert(sizeof(TileArgs) == 352, "TileArgs outgrew its tail padding: every tile kernel's parameters move");

// kernel variants: with TF_DYNAMIC everything is decided at run time (partial tiles, optional
// output twiddle / scale); the static variants drop the predication and branches.  TF_TWB2 applies the
// factored output twiddle (twb and twb_b), in full-tile or dynamic kernels; it is never decided at run time.
enum { TF_FULL = 1, TF_TWB = 2, TF_SCALE = 4, TF_DYNAMIC = 8, TF_PEERS = 16, TF_TWB2 = 32 };

template <int LOGL, int ELOG, int C>
struct TilePlan {
    static constexpr int L = 1 << LOGL;
    static constexpr int EL = LOGL >= ELOG ? ELOG : LOGL;  // log2 elements per thread
    static constexpr int E = 1 << EL;
    static constexpr int NFULL = LOGL / EL;        // stages of radix E
    static constexpr int REM = LOGL % EL;          // log2 radix of the trailing stage (0 = none)
    static constexpr int NST = NFULL + (REM ? 1 : 0);
    static constexpr int NLOOP = NST - 1;          // full-radix stages that are not the last stage
    static constexpr int LASTLOG = REM ? REM : EL;  // log2 radix of the last stage
    static constexpr int TPT = (L / E) * C;        // threads per tile
    // tiles per CTA: small tiles are packed into 128-thread CTAs.  (Single-column CTAs of 64 threads for lone
    // 2^20 transforms were tried and lost: the 16-byte-per-row accesses cost more than the balance gains.)
    static constexpr int TPC = TPT >= 128 ? 1 : 128 / TPT;
    static constexpr int THREADS = TPT * TPC;
    // dynamic shared memory: the tile rows, then the stage-twiddle table (L elements, staged by one
    // bulk-async copy, see tile_stage_twiddles), then the 8-byte mbarrier it completes on
    static constexpr size_t TILE_BYTES = (size_t)TPC * L * C * sizeof(fe);
    static constexpr size_t TW_BYTES = (size_t)L * sizeof(fe);
    SA_HDC size_t smem_bytes() { return NST > 1 ? TILE_BYTES + TW_BYTES + 16 : 0; }
};

// slot of w^e in the stage-twiddle table: the low three bits are XORed with the next three, so the
// strided look-ups of the middle stages ((k*m) << 3: all multiples of 8) spread over the eight
// 16-byte bank groups of shared memory instead of piling onto one
SA_HDC int tile_tw_slot(int e) { return e ^ ((e >> 3) & 7); }

// log2 of a power of two
SA_HD int tile_log2(unsigned x) {
#if defined(__CUDA_ARCH__)
    return __ffs(x) - 1;
#else
    return __builtin_ctz(x);
#endif
}

SA_HDC int tile_bitrev(int i, int r) {
    int j = 0;
    for (int b = 1, bb = r >> 1; b < r; b <<= 1, bb >>= 1)
        if (i & b) j |= bb;
    return j;
}

// ---- the tile's own field product and butterfly.  Same canonical residues as fe_montmul / fe_add /
// fe_sub; the device bodies are written for the tile kernels' instruction mix (field.cuh stays what every
// other kernel compiles), the host and SA_PORTABLE_FIELD bodies are the portable field.
#if defined(__CUDA_ARCH__) && !defined(SA_PORTABLE_FIELD)
// Montgomery product x * w * 2^-128 mod p, the reduction of fe_montmul (field.cuh).  Every multiply-add
// is one IMAD.WIDE whose 64-bit accumulator is an aligned register pair from start to end:
//  * the schoolbook sums the products with i+j even into pairs (0,1) (2,3) (4,5) (6,7) and the odd ones
//    into (1,2) (3,4) (5,6).  A chain either ends in a pair it initialises (a*b + carry, no addend) or
//    leaves its carry in a register; the three such carries (word 5, 6, 7) are the addend of pair (5,6)
//    and the word-7 term of the final merge t = even + odd, so no pair is built from a copy or a zero.
//  * the reduction's four products t0 P3, t1 P3, t2 P3, m3 P3 are plain 64-bit products (no addend), merged
//    by one add chain into u = m P3 >> 32.  The borrow w of m3 = t3 - x is taken again as the borrow-in of
//    r = t_hi - u - w: a carry chain never consumes a borrow (that mix computed wrong results on the device).
//  Rows of the product as 32-bit halves (mul.lo + mul.hi) become IMAD + IMAD.HI, and IMAD.HI costs as much
//  as IMAD.WIDE (tools/pipebench.cu), so the first row and the reduction use mul.wide.  The add-back of p
//  keeps its mask words on the multiplier pipe: the ALU pipe is the busier one once the copies are gone.
__device__ __forceinline__ fe tile_mul(const fe &x, const fe &w) {
    uint32_t t0, t1, t2, t3, t4, t5, t6, t7;
    asm("{\n\t"
        ".reg .u32 e1, e2, e3, e4, e5, e6, e7, o1, o2, o3, o4, o5, o6, k5, k6, k7;\n\t"
        ".reg .u64 E0, E2, O1, O3;\n\t"
        "mul.wide.u32 E0, %8, %12;\n\t"  // (0,0)@0 -> (t0, e1)
        "mul.wide.u32 E2, %8, %14;\n\t"  // (0,2)@2
        "mul.wide.u32 O1, %8, %13;\n\t"  // (0,1)@1
        "mul.wide.u32 O3, %8, %15;\n\t"  // (0,3)@3
        "mov.b64 {%0, e1}, E0;\n\t"
        "mov.b64 {e2, e3}, E2;\n\t"
        "mov.b64 {o1, o2}, O1;\n\t"
        "mov.b64 {o3, o4}, O3;\n\t"
        "mad.lo.cc.u32 e2, %9, %13, e2;\n\t"  // (1,1)@2, then (1,3) initialises (4,5)
        "madc.hi.cc.u32 e3, %9, %13, e3;\n\t"
        "madc.lo.cc.u32 e4, %9, %15, 0;\n\t"
        "madc.hi.u32 e5, %9, %15, 0;\n\t"
        "mad.lo.cc.u32 e4, %11, %13, e4;\n\t"  // (3,1)@4 -> carry k6
        "madc.hi.cc.u32 e5, %11, %13, e5;\n\t"
        "addc.u32 k6, 0, 0;\n\t"
        "mad.lo.cc.u32 o3, %10, %13, o3;\n\t"  // (2,1)@3 -> carry k5
        "madc.hi.cc.u32 o4, %10, %13, o4;\n\t"
        "addc.u32 k5, 0, 0;\n\t"
        "mad.lo.cc.u32 o1, %9, %12, o1;\n\t"  // (1,0)@1 (1,2)@3, then (2,3) + (k5, k6) initialises (5,6)
        "madc.hi.cc.u32 o2, %9, %12, o2;\n\t"
        "madc.lo.cc.u32 o3, %9, %14, o3;\n\t"
        "madc.hi.cc.u32 o4, %9, %14, o4;\n\t"
        "madc.lo.cc.u32 o5, %10, %15, k5;\n\t"
        "madc.hi.u32 o6, %10, %15, k6;\n\t"
        "mad.lo.cc.u32 o3, %11, %12, o3;\n\t"  // (3,0)@3 (3,2)@5 -> carry k7
        "madc.hi.cc.u32 o4, %11, %12, o4;\n\t"
        "madc.lo.cc.u32 o5, %11, %14, o5;\n\t"
        "madc.hi.cc.u32 o6, %11, %14, o6;\n\t"
        "addc.u32 k7, 0, 0;\n\t"
        "mad.lo.cc.u32 e2, %10, %12, e2;\n\t"  // (2,0)@2 (2,2)@4, then (3,3) initialises (6,7)
        "madc.hi.cc.u32 e3, %10, %12, e3;\n\t"
        "madc.lo.cc.u32 e4, %10, %14, e4;\n\t"
        "madc.hi.cc.u32 e5, %10, %14, e5;\n\t"
        "madc.lo.cc.u32 e6, %11, %15, 0;\n\t"
        "madc.hi.u32 e7, %11, %15, 0;\n\t"
        "add.cc.u32 %1, e1, o1;\n\t"  // t = even + (odd << 32) + (k7 << 224)
        "addc.cc.u32 %2, e2, o2;\n\t"
        "addc.cc.u32 %3, e3, o3;\n\t"
        "addc.cc.u32 %4, e4, o4;\n\t"
        "addc.cc.u32 %5, e5, o5;\n\t"
        "addc.cc.u32 %6, e6, o6;\n\t"
        "addc.u32 %7, e7, k7;\n\t"
        "}"
        : "=r"(t0), "=r"(t1), "=r"(t2), "=r"(t3), "=r"(t4), "=r"(t5), "=r"(t6), "=r"(t7)
        : "r"(x.v[0]), "r"(x.v[1]), "r"(x.v[2]), "r"(x.v[3]), "r"(w.v[0]), "r"(w.v[1]), "r"(w.v[2]), "r"(w.v[3]));
    uint32_t r0, r1, r2, r3, top;
    asm("{\n\t"
        ".reg .u32 x, m3, h0, q1, q2, g2, g3, v3, v4, u1, u2, u3, u4;\n\t"
        ".reg .u64 T, Q, G, V;\n\t"
        "mul.wide.u32 T, %5, 0xCB800000;\n\t"  // (x, h0) = t0 P3: x = t0 P3 mod 2^32
        "mul.wide.u32 Q, %6, 0xCB800000;\n\t"
        "mul.wide.u32 G, %7, 0xCB800000;\n\t"
        "mov.b64 {x, h0}, T;\n\t"
        "mov.b64 {q1, q2}, Q;\n\t"
        "mov.b64 {g2, g3}, G;\n\t"
        "sub.u32 m3, %8, x;\n\t"  // m3 = t3 - x mod 2^32
        "mul.wide.u32 V, m3, 0xCB800000;\n\t"
        "mov.b64 {v3, v4}, V;\n\t"
        "add.cc.u32 u1, h0, q1;\n\t"  // u = m P3 >> 32
        "addc.cc.u32 u2, q2, g2;\n\t"
        "addc.cc.u32 u3, g3, v3;\n\t"
        "addc.u32 u4, v4, 0;\n\t"
        "sub.cc.u32 x, %8, x;\n\t"  // the borrow w of t3 - x starts r = t_hi - u - w, in (-p, p)
        "subc.cc.u32 %0, %9, u1;\n\t"
        "subc.cc.u32 %1, %10, u2;\n\t"
        "subc.cc.u32 %2, %11, u3;\n\t"
        "subc.cc.u32 %3, %12, u4;\n\t"
        "subc.u32 %4, 0, 0;\n\t"
        "}"
        : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3), "=r"(top)
        : "r"(t0), "r"(t1), "r"(t2), "r"(t3), "r"(t4), "r"(t5), "r"(t6), "r"(t7));
    return fe_cond_add_p<false>(r0, r1, r2, r3, top);
}
// (e, x) -> (e + x w, e - x w)
__device__ __forceinline__ void tile_bfly(fe &e, fe &x, const fe &w) {
    const fe t = tile_mul(x, w);
    x = fe_sub(e, t);
    e = fe_add(e, t);
}
#else
SA_HD fe tile_mul(const fe &x, const fe &w) { return fe_montmul_portable(x, w); }
SA_HD void tile_bfly(fe &e, fe &x, const fe &w) {
    const fe t = fe_montmul_portable(x, w);
    x = fe_sub_portable(e, t);
    e = fe_add_portable(e, t);
}
#endif

// one radix-2 decimation-in-time level (span LEN) of an R-point transform held in registers
template <int R, int LEN>
SA_HD void dft_level(fe *x, const fe *cst, int cstep) {
    constexpr int HALF = LEN / 2, STEP = R / LEN;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int g = 0; g < R; g += LEN) {
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (int k = 0; k < HALF; k++) {
            if (k == 0) {
                const fe e = x[g], t = x[g + HALF];
                x[g] = fe_add(e, t);
                x[g + HALF] = fe_sub(e, t);
            } else {
                tile_bfly(x[g + k], x[g + k + HALF], cst[k * STEP * cstep]);
            }
        }
    }
    if constexpr (LEN < R) dft_level<R, LEN * 2>(x, cst, cstep);
}

// natural-order R-point transform of x[0..R) in registers; w_R^j = cst[j * cstep]
template <int R>
SA_HD void dft_regs(fe *x, const fe *cst, int cstep) {
    // bit-reversal permutation (register renaming once unrolled)
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int i = 0; i < R; i++) {
        const int j = tile_bitrev(i, R);
        if (i < j) {
            const fe tmp = x[i];
            x[i] = x[j];
            x[j] = tmp;
        }
    }
    if constexpr (R >= 2) dft_level<R, 2>(x, cst, cstep);
}

// position p = (k_0, k_1, ..., k_last), k_0 most significant -> output index
// k_0 + R_0 k_1 + R_0 R_1 k_2 + ...   (digit reversal of the mixed radix)
template <int LOGL, int ELOG, int C>
SA_HD int tile_digit_reverse(int p) {
    using P = TilePlan<LOGL, ELOG, C>;
    int o = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int i = 0; i < P::NST; i++) {
        const int rl = (i < P::NFULL) ? P::EL : P::REM;
        const int ml = (i < P::NFULL) ? LOGL - (i + 1) * P::EL : 0;  // log2 M_i
        const int k = (p >> ml) & ((1 << rl) - 1);
        o |= k << (i * P::EL);  // product of the earlier radices = E^i
    }
    return o;
}

SA_HD fe tile_ld(const fe *p) {
#if defined(__CUDA_ARCH__)
    const uint4 v = *reinterpret_cast<const uint4 *>(p);
    return fe_make(v.x, v.y, v.z, v.w);
#else
    return *p;
#endif
}
SA_HD fe tile_ldg(const fe *p) {
#if defined(__CUDA_ARCH__)
    const uint4 v = __ldg(reinterpret_cast<const uint4 *>(p));
    return fe_make(v.x, v.y, v.z, v.w);
#else
    return *p;
#endif
}
SA_HD void tile_st(fe *p, const fe &x) {
#if defined(__CUDA_ARCH__)
    *reinterpret_cast<uint4 *>(p) = make_uint4(x.v[0], x.v[1], x.v[2], x.v[3]);
#else
    *p = x;
#endif
}

// 16-byte store through a multicast address (sm_90+: multimem.st; the f32 type only names the vector shape)
SA_HD void tile_st_multicast(fe *p, const fe &x) {
#if defined(__CUDA_ARCH__)
    asm volatile("multimem.st.weak.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(__uint_as_float(x.v[0])),
                 "f"(__uint_as_float(x.v[1])), "f"(__uint_as_float(x.v[2])), "f"(__uint_as_float(x.v[3]))
                 : "memory");
#else
    *p = x;
#endif
}

SA_HD long long tile_batch_offset(long long b, int inner, long long sb, long long sb2) {
    return inner <= 1 ? b * sb : (b / inner) * sb + (b % inner) * sb2;
}

// A full-radix (E-point) stage that is NOT the last stage: one unit per thread.
//   ml = log2 M of this stage (run-time, so all such stages share one copy of the code)
#if defined(__CUDA_ARCH__)
// TMA-style staging of the per-stage twiddle table: one thread arms an mbarrier with the byte count
// and issues a single bulk-async copy global -> shared (SASS: UBLKCP); everybody waits on the
// barrier's phase right before the first twiddle is needed, so the copy overlaps the first block's
// global loads and register transform.
__device__ __forceinline__ void tile_stage_twiddles(fe *dst, const fe *src, uint32_t bytes, uint64_t *bar) {
    const uint32_t bar_a = (uint32_t)__cvta_generic_to_shared(bar);
    const uint32_t dst_a = (uint32_t)__cvta_generic_to_shared(dst);
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_a),
                 "l"(src), "r"(bytes), "r"(bar_a)
                 : "memory");
}
__device__ __forceinline__ void tile_wait_twiddles(uint64_t *bar) {
    const uint32_t bar_a = (uint32_t)__cvta_generic_to_shared(bar);
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "TW_WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n\t"
        "@p bra TW_DONE_%=;\n\t"
        "bra TW_WAIT_%=;\n\t"
        "TW_DONE_%=:\n\t"
        "}" ::"r"(bar_a)
        : "memory");
}
#endif

//   tw  = the stage-twiddle table (shared memory on the device, see tile_stage_twiddles)
//   bar = its mbarrier (device) / nullptr (host emulation)
template <int LOGL, int ELOG, int C, int FLAGS>
SA_HD void ntt_tile_full_stage(int t, fe *sm, const TileArgs &a, long long b, int col0, bool valid, bool first,
                               int ml, const fe *tw, uint64_t *bar) {
    using P = TilePlan<LOGL, ELOG, C>;
    constexpr int R = P::E;
    constexpr int CSTEP = 16 / R;  // a non-last stage exists only when L > E >= 8, so cst = w_16^k
    const int c = t % C, q = t / C;
    const int col = col0 + c;
    const bool active = (FLAGS & TF_FULL) ? true : (valid && col < a.ncols);
    const int M = 1 << ml, wlog = LOGL - ml - P::EL;
    const int K = q >> ml, m = q & (M - 1);
    const int row0 = (K << (ml + P::EL)) + m;
    fe x[R];
    if (first) {
        const fe *src = a.in + tile_batch_offset(b, a.inner, a.in_sb, a.in_sb2) + (long long)col * a.in_sc;
        // row offsets fit 32 bits (row < 1024, stride <= 2^20): one IMAD.WIDE per address
        const unsigned sr = (unsigned)a.in_sr, step = (unsigned)M * sr, off0 = (unsigned)row0 * sr;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (int d = 0; d < R; d++) x[d] = active ? tile_ld(src + (off0 + (unsigned)d * step)) : fe_zero();
    } else {
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (int d = 0; d < R; d++) x[d] = tile_ld(sm + (row0 + d * M) * C + c);
    }
    dft_regs<R>(x, a.cst, CSTEP);
#if defined(__CUDA_ARCH__)
    // table and barrier sit at fixed offsets of the dynamic shared memory window: address them from
    // the window base (immediate offsets) instead of keeping two more pointers live across the loop
    extern __shared__ uint4 sa_smem_u4[];
    tw = reinterpret_cast<const fe *>(sa_smem_u4) + P::TILE_BYTES / sizeof(fe);
    if (first) tile_wait_twiddles(reinterpret_cast<uint64_t *>(const_cast<fe *>(tw) + P::L));
    (void)bar;
#else
    (void)bar;
#endif
    // multiply output k by w_{M*R}^(k*m) = w_L^((k*m) << wlog), then park it in row row0 + k*M.  The stage
    // before the last one (M = 2^LASTLOG) parks its outputs as they are and the last stage multiplies them as it
    // loads them (ntt_tile_last_stage).  Here the factors of one (m = 0) belong to whole units, a quarter of the
    // threads at M = 4; there they are the unrolled row d = 0 of every unit, so every thread and every warp skips
    // the same share (a skip confined to some warps leaves the SM sub-partitions of the others just as busy)
    tile_st(sm + row0 * C + c, x[0]);
    if (ml == P::LASTLOG) {
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (int k = 1; k < R; k++) tile_st(sm + (row0 + k * M) * C + c, x[k]);
    } else {
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (int k = 1; k < R; k++) {
            const fe w = tile_ld(tw + tile_tw_slot((k * m) << wlog));
            tile_st(sm + (row0 + k * M) * C + c, tile_mul(x[k], w));
        }
    }
}

// The last stage (radix 2^LASTLOG, M = 1): E / R units per thread, output twiddle, global stores.
template <int LOGL, int ELOG, int C, int FLAGS>
SA_HD void ntt_tile_last_stage(int t, fe *sm, const TileArgs &a, long long b, int col0, bool valid) {
    using P = TilePlan<LOGL, ELOG, C>;
    constexpr int R = 1 << P::LASTLOG, U = P::E / R;
    constexpr bool FIRST = P::NST == 1;
    constexpr int CSTEP = LOGL >= 4 ? 16 / R : (1 << LOGL) / R;
    const int c = t % C, q = t / C;
    const int col = col0 + c;
    const bool active = (FLAGS & TF_FULL) ? true : (valid && col < a.ncols);
    constexpr bool TWB2 = (FLAGS & TF_TWB2) != 0;
    const bool use_twb = (FLAGS & TF_DYNAMIC) ? (a.twb != nullptr) : ((FLAGS & TF_TWB) != 0);
    const bool use_scale = (FLAGS & TF_DYNAMIC) ? (a.has_scale != 0) : ((FLAGS & TF_SCALE) != 0);
    const fe *twb = use_twb ? a.twb + col : nullptr;
    const unsigned out_sr = (unsigned)a.out_sr, twb_sr = (unsigned)a.twb_stride;
    // factored twiddle: the row-k factor is twb_a[k * twb_sr] * twb_b[k * twb_b_sr]
    const fe *twb_a = nullptr, *twb_b = nullptr;
    unsigned twb_b_sr = 0;
    if constexpr (TWB2) {
        twb_b_sr = (unsigned)a.ncols / twb_sr;  // n3, a power of two
        twb_a = a.twb + ((unsigned)col >> tile_log2(twb_b_sr));
        twb_b = a.twb_b + ((unsigned)col & (twb_b_sr - 1));
    }
    fe *dst = a.out + tile_batch_offset(b, a.inner, a.out_sb, a.out_sb2) + (long long)col * a.out_sc;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int s = 0; s < U; s++) {
        const int row0 = (q * U + s) * R;
        fe x[R];
        if constexpr (FIRST) {
            const fe *src = a.in + tile_batch_offset(b, a.inner, a.in_sb, a.in_sb2) + (long long)col * a.in_sc;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
            for (int d = 0; d < R; d++) x[d] = active ? tile_ld(src + (unsigned)(row0 + d) * (unsigned)a.in_sr) : fe_zero();
        } else {
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
            for (int d = 0; d < R; d++) x[d] = tile_ld(sm + (row0 + d) * C + c);
            // the inter-stage twiddles of the stage before, which parked its outputs unmultiplied: row row0 + d
            // is its output k = (row0 / R) mod E of unit m = d (that stage has M = R), so the factor is
            // w_L^((k*d) << wlog) and row d = 0 has none
            const fe *tw = a.tw;
#if defined(__CUDA_ARCH__)
            extern __shared__ uint4 sa_smem_u4[];
            tw = reinterpret_cast<const fe *>(sa_smem_u4) + P::TILE_BYTES / sizeof(fe);
#endif
            constexpr int WLOG = LOGL - P::LASTLOG - P::EL;
            const int k = (row0 >> P::LASTLOG) & (P::E - 1);
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
            for (int d = 1; d < R; d++) x[d] = tile_mul(x[d], tile_ld(tw + tile_tw_slot((k * d) << WLOG)));
        }
        dft_regs<R>(x, a.cst, CSTEP);
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (int k = 0; k < R; k++) {
            const unsigned o = (unsigned)tile_digit_reverse<LOGL, ELOG, C>(row0 + k);
            fe v = x[k];
            if constexpr (TWB2) {
                if (active) v = tile_mul(tile_mul(v, tile_ldg(twb_a + o * twb_sr)), tile_ldg(twb_b + o * twb_b_sr));
            } else if (use_twb && active) {
                v = tile_mul(v, tile_ldg(twb + o * twb_sr));
            }
            if (use_scale) v = tile_mul(v, a.scale);
            if (active) {
                if constexpr ((FLAGS & TF_PEERS) != 0) {
                    const long long rel = (dst - a.out) + (long long)(o * out_sr);
                    if (a.mc_out != nullptr) {
                        tile_st_multicast(a.mc_out + rel, v);
                    } else {
                        tile_st(dst + o * out_sr, v);
                        for (int pi = 0; pi < a.npeer; pi++) tile_st(a.peer_out[pi] + rel, v);
                    }
                } else {
                    tile_st(dst + o * out_sr, v);
                }
            }
        }
    }
}

// the whole tile for thread t; `sync` is __syncthreads on the device and a no-op marker on
// the host (the emulator calls the stages phase by phase instead)
template <int LOGL, int ELOG, int C, int FLAGS = TF_DYNAMIC>
struct TileStages {
    using P = TilePlan<LOGL, ELOG, C>;
    // stage index st < NLOOP -> full stage with ml = LOGL - (st + 1) * EL
    SA_HD static void full(int st, int t, fe *sm, const TileArgs &a, long long b, int col0, bool valid,
                           const fe *tw, uint64_t *bar) {
        ntt_tile_full_stage<LOGL, ELOG, C, FLAGS>(t, sm, a, b, col0, valid, st == 0, LOGL - (st + 1) * P::EL, tw,
                                                   bar);
    }
    SA_HD static void last(int t, fe *sm, const TileArgs &a, long long b, int col0, bool valid) {
        ntt_tile_last_stage<LOGL, ELOG, C, FLAGS>(t, sm, a, b, col0, valid);
    }
};

// which static variant (if any) fits these arguments; TF_DYNAMIC otherwise
template <int LOGL, int ELOG, int C>
SA_HD int tile_variant(const TileArgs &a) {
    using P = TilePlan<LOGL, ELOG, C>;
    const long long tiles = (long long)((a.ncols + C - 1) / C) * a.nbatch;
    const int peers = (a.npeer > 0 || a.mc_out != nullptr) ? TF_PEERS : 0;
    if (a.twb_b != nullptr) {  // factored output twiddle: pass 1 of a three-pass plan, so no peers
        const bool full = LOGL >= 5 && a.ncols % C == 0 && tiles % P::TPC == 0 && !a.has_scale;
        return TF_TWB2 | (full ? TF_FULL : TF_DYNAMIC);
    }
    if (LOGL < 5 || a.ncols % C != 0 || tiles % P::TPC != 0 || a.has_scale) return TF_DYNAMIC | peers;
    if (peers) return a.twb == nullptr ? (TF_FULL | TF_PEERS) : (TF_DYNAMIC | TF_PEERS);
    return TF_FULL | (a.twb != nullptr ? TF_TWB : 0);
}

}  // namespace sa
