// tests/emu/emu_tile_count.cpp -- TEST INFRASTRUCTURE: the CPU emulation of emu.cpp (included whole) with every
// field product of the NTT tile counted.  The host bodies of tile_mul and tile_bfly (ntt_tile.cuh) call
// fe_montmul_portable; while the tile header is compiled here that name is bound to a counting wrapper, so the
// counts are exactly the products the tile's stage code issues.  field.cuh is compiled first and keeps its own
// product, so nothing else is counted.
// It is NOT a fallback: nothing in the product loads this library.
//
// Build: g++ -O2 -std=c++17 -shared -fPIC -o libsa_emu_tile_count.so emu_tile_count.cpp
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../stark-anatomy_b200/csrc/field.cuh"

namespace sa {
static long long g_tile_products = 0;
inline fe tile_counted_montmul(const fe &a, const fe &b) {
    g_tile_products++;
    return fe_montmul_portable(a, b);
}
}  // namespace sa

#define fe_montmul_portable tile_counted_montmul
#include "../../stark-anatomy_b200/csrc/ntt_tile.cuh"
#undef fe_montmul_portable

#include "emu.cpp"

// One full tile of C forward 2^LOGL-point transforms (16-element blocks, the static TF_FULL variant) through the
// library's single-pass tables, phase by phase as the kernel runs it.  counts[phase * TPT + t] = the products
// thread t issued in that phase (phases: the NLOOP full stages, then the last stage).
template <int LOGL, int C>
static int tile_count(uint64_t *out, const uint64_t *in, const uint64_t *root, long long *counts) {
    using P = TilePlan<LOGL, 4, C>;
    using S = TileStages<LOGL, 4, C, TF_FULL>;
    const fe root_m = fe_to_mont(fe_from_limbs(root));
    int rc = ntt_check_root(root_m, LOGL);
    if (rc != SA_OK) return rc;
    const NttShape s = ntt_shape(LOGL);
    if (s.l2 != 0) return SA_ESIZE;
    std::vector<std::vector<fe>> tables;
    NttTables t;
    rc = ntt_build_tables(
        t, s, root_m, 0,
        [&](fe **table, const fe &base_m, long long count) {
            tables.push_back(pow_table(base_m, count, 1));
            *table = tables.back().data();
            return SA_OK;
        },
        [&](fe **, const fe &, const fe &, int, long long) { return SA_ESIZE; });
    if (rc != SA_OK) return rc;
    TileArgs a;
    memset(&a, 0, sizeof(a));
    ntt_fill_single(a, (const fe *)in, (fe *)out, LOGL, C, t.tw1, t.cst1, 0, fe_mont_one());
    if (tile_variant<LOGL, 4, C>(a) != TF_FULL) return SA_ESIZE;
    std::vector<fe> sm((size_t)P::L * C);
    for (int st = 0; st <= P::NLOOP; st++)
        for (int th = 0; th < P::TPT; th++) {
            g_tile_products = 0;
            if (st < P::NLOOP)
                S::full(st, th, sm.data(), a, 0, 0, true, a.tw, nullptr);
            else
                S::last(th, sm.data(), a, 0, 0, true);
            counts[(size_t)st * P::TPT + th] = g_tile_products;
        }
    return SA_OK;
}

extern "C" {

// in / out: c transforms of 2^logl points, transform j at [j << logl]; the launched tile shapes with a middle
// stage: logl 9 or 10, c = 4 (every such pass) or 8 (the pass that also stores to peers)
int emu_tile_products(uint64_t *out, const uint64_t *in, int logl, int c, const uint64_t *root, long long *counts) {
    if (logl == 10 && c == 4) return tile_count<10, 4>(out, in, root, counts);
    if (logl == 9 && c == 4) return tile_count<9, 4>(out, in, root, counts);
    if (logl == 10 && c == 8) return tile_count<10, 8>(out, in, root, counts);
    if (logl == 9 && c == 8) return tile_count<9, 8>(out, in, root, counts);
    return SA_ESIZE;
}

}  // extern "C"
