// tests/emu/emu_large.cpp -- TEST INFRASTRUCTURE: the CPU emulation of emu.cpp (included whole, so the tile
// shapes, table builders and every emu_* entry point are the same code) plus the plans above 2^26, whose
// pass 1 applies factored twiddles A (n1 x n2) and B (n1 x n3) with the TF_TWB2 tile variant (ntt_plan.cuh).
// It is NOT a fallback: nothing in the product loads this library.
//
// Build: g++ -O2 -std=c++17 -shared -fPIC -o libsa_emu_large.so emu_large.cpp
#include "emu.cpp"

// the variant choice of launch_tile (ntt.cu), TF_TWB2 included.  The library has the TF_TWB2 kernels for 2^9-
// and 2^10-point tiles only; here every tile length and shape runs them, so forced small plans cover the code.
template <int LOGL, int ELOG, int C>
static void run_tiles_large(const TileArgs &a) {
    const int variant = tile_variant<LOGL, ELOG, C>(a);
    if (!(variant & TF_TWB2)) return run_tiles<LOGL, ELOG, C>(a);
    if (variant & TF_FULL) return run_tiles_variant<LOGL, ELOG, C, TF_FULL | TF_TWB2>(a);
    return run_tiles_variant<LOGL, ELOG, C, TF_DYNAMIC | TF_TWB2>(a);
}
template <int LOGL>
static void run_tiles_shape_large(const TileArgs &a) {  // the shapes of emu_set_shape, as in run_tiles_shape
    if (g_elog == 3 && g_c == 8) return run_tiles_large<LOGL, 3, 8>(a);
    if (g_elog == 3 && g_c == 4) return run_tiles_large<LOGL, 3, 4>(a);
    if (g_elog == 3 && g_c == 2) return run_tiles_large<LOGL, 3, 2>(a);
    if (g_elog == 4 && g_c == 4) return run_tiles_large<LOGL, 4, 4>(a);
    if (g_elog == 4 && g_c == 2) return run_tiles_large<LOGL, 4, 2>(a);
    if (g_elog == 4 && g_c == 3) return run_tiles_large<LOGL, 4, 3>(a);
    if (g_elog == 4 && g_c == 7) return run_tiles_large<LOGL, 4, 7>(a);
    return run_tiles_large<LOGL, 4, 8>(a);
}
static void run_tiles_dyn_large(int logl, const TileArgs &a) {
    switch (logl) {
        case 1: run_tiles_shape_large<1>(a); break;
        case 2: run_tiles_shape_large<2>(a); break;
        case 3: run_tiles_shape_large<3>(a); break;
        case 4: run_tiles_shape_large<4>(a); break;
        case 5: run_tiles_shape_large<5>(a); break;
        case 6: run_tiles_shape_large<6>(a); break;
        case 7: run_tiles_shape_large<7>(a); break;
        case 8: run_tiles_shape_large<8>(a); break;
        case 9: run_tiles_shape_large<9>(a); break;
        case 10: run_tiles_shape_large<10>(a); break;
    }
}

// the library's tables of shape s (ntt_build_tables with the k_pow_table / k_twb_table thread bodies), kept in
// `store`
static void build_tables(NttTables &t, std::vector<std::vector<fe>> &store, const NttShape &s, const fe &root_m,
                         int inverse) {
    auto keep = [&](fe **table, std::vector<fe> v) {
        store.push_back(std::move(v));
        *table = store.back().data();
        return SA_OK;
    };
    ntt_build_tables(
        t, s, root_m, inverse, [&](fe **table, const fe &base_m, long long cnt) { return keep(table, pow_table(base_m, cnt, 1)); },
        [&](fe **table, const fe &w_m, const fe &scale_m, int rows, long long cols) {
            return keep(table, twb_table(w_m, scale_m, rows, cols));
        });
}

extern "C" {

// sa_ntt through the library's plan and pass sequence over the emulated tile passes, every variant included.
// force3: 0 = the plan of the size, 1 = three passes (normally only above 2^20), 2 = three passes with factored
// pass-1 twiddles (normally only above 2^26), so that both three-pass plans can be exercised at small sizes.
int emu_ntt_plan(uint64_t *out, const uint64_t *in, int log_n, const uint64_t *root, int inverse, size_t batch,
                 int force3) {
    const size_t n = size_t(1) << log_n;
    if (log_n == 0) {
        memcpy(out, in, 16 * batch);
        return 0;
    }
    const fe root_m = fe_to_mont(fe_from_limbs(root));
    int rc = ntt_check_root(root_m, log_n);
    if (rc != SA_OK) return rc;
    const NttShape s = ntt_shape(log_n, force3);
    std::vector<std::vector<fe>> store;
    NttTables t;
    build_tables(t, store, s, root_m, inverse);
    // a single pass in place would overwrite input that later emulated threads still read: it reads a copy
    std::vector<fe> tmp(n * batch);
    const fe *src = (const fe *)in;
    if (s.l2 == 0) src = (const fe *)memcpy(tmp.data(), in, 16 * n * batch);
    return ntt_run_passes(s, t, src, (fe *)out, tmp.data(), batch, [](int logl, TileArgs &a, bool) {
        run_tiles_dyn_large(logl, a);
        return SA_OK;
    });
}

// The library's plan of size 2^log_n and the pass-1 twiddle factors it applies to row k1[i], column m[i]:
// a_out[i] * b_out[i] (plain form).  Factored plans give A[k1][m >> l3] and B[k1][m & (n3 - 1)], the others the
// matrix entry and 1.  shape_out = l1, l2, l3, twb_split.  Only the three-pass plans have a pass-1 matrix.
int emu_ntt_pass1_twiddles(int *shape_out, uint64_t *a_out, uint64_t *b_out, int log_n, const uint64_t *root,
                           int inverse, const long long *k1, const long long *m, size_t count) {
    const fe root_m = fe_to_mont(fe_from_limbs(root));
    int rc = ntt_check_root(root_m, log_n);
    if (rc != SA_OK) return rc;
    const NttShape s = ntt_shape(log_n);
    shape_out[0] = s.l1, shape_out[1] = s.l2, shape_out[2] = s.l3, shape_out[3] = s.twb_split;
    if (s.l3 == 0) return SA_ESIZE;
    std::vector<std::vector<fe>> store;
    NttTables t;
    build_tables(t, store, s, root_m, inverse);
    const long long n2 = 1ll << s.l2, n3 = 1ll << s.l3;
    for (size_t i = 0; i < count; i++) {
        const fe a = fe_from_mont(s.twb_split ? t.twb[k1[i] * n2 + (m[i] >> s.l3)] : t.twb[k1[i] * (n2 * n3) + m[i]]);
        const fe b = fe_from_mont(s.twb_split ? t.twb_b[k1[i] * n3 + (m[i] & (n3 - 1))] : fe_mont_one());
        memcpy(a_out + 2 * i, &a, 16);
        memcpy(b_out + 2 * i, &b, 16);
    }
    return SA_OK;
}

}  // extern "C"
