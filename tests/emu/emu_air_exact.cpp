// tests/emu/emu_air_exact.cpp -- TEST INFRASTRUCTURE: the CPU emulation of emu_air.cpp (included whole, so the AIR
// plan and the unchecked apply are the same emulated code) plus the exact apply (air.cuh: air_exact_check,
// air_quotients_exact) over a backend whose k_air_store_exact runs warps of 32 indices: each lane's
// air_store_exact_elem, the warp's ballot, then boundary_flag_leader's lanes raise their row's flag.
// It is NOT a fallback: nothing in the product loads this library.
//
// Build: g++ -O2 -std=c++17 -shared -fPIC -o libsa_emu_air_exact.so emu_air_exact.cpp
#include "emu_air.cpp"

// EmuAir plus the flags' memset and k_air_store_exact, counting its atomicOr calls
struct EmuAirExact : EmuAir {
    int clear_flags(uint32_t *flags, size_t n) {
        memset(flags, 0, sizeof(uint32_t) * n);
        return SA_OK;
    }
    int air_store_exact(fe *out, uint32_t *flags, const fe *ws, const fe *ipw_m, long long qlen, long long tail,
                        int log_n, long long batch) {
        for (long long w = 0; w < batch << log_n; w += 32) {
            uint32_t ballot = 0;
            for (int lane = 0; lane < 32; lane++)
                if (air_store_exact_elem(out, ws, ipw_m, qlen, tail, log_n, batch, w + lane)) ballot |= 1u << lane;
            for (int lane = 0; lane < 32; lane++)
                if ((ballot >> lane & 1u) && boundary_flag_leader(ballot, lane, log_n)) {
                    flags[(w + lane) >> log_n] |= 1u;
                    store_atomics++;
                }
        }
        return SA_OK;
    }
    long long store_atomics = 0;
};

// the atomicOr count of the last emulated exact apply's stores (one per flagged row a warp touches)
static long long g_store_atomics = 0;

extern "C" {

// sa_air_quotients_exact with host rows: the workspace, out and flags start from a stale pattern once the checks
// pass, so an element the schedule fails to write, or a flag it fails to clear, shows up
int emu_air_quotients_exact(uint64_t *out, uint32_t *flags, const uint64_t *plan, const uint64_t *trace, size_t nregs,
                            size_t ncoef, size_t qlen, size_t ncons, size_t tail, int log_n, const uint64_t *root) {
    SA_TRY(air_exact_check(log_n, nregs, ncoef, qlen, ncons, tail, root));
    std::vector<fe> ws = stale_workspace(air_ws_elems(nregs, ncons, log_n));
    const std::vector<fe> stale = stale_workspace(ncons * qlen);
    memcpy(out, stale.data(), sizeof(fe) * stale.size());
    for (size_t c = 0; c < ncons; c++) flags[c] = 0x5a5a5a5au;
    EmuAirExact b;
    const int rc = air_quotients_exact(b, (fe *)out, flags, (const fe *)plan, (const fe *)trace, nregs, ncoef, qlen,
                                       ncons, tail, log_n, root, ws.data());
    g_store_atomics = b.store_atomics;
    return rc;
}
long long emu_air_store_atomics() { return g_store_atomics; }

}  // extern "C"
