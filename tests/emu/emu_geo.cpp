// tests/emu/emu_geo.cpp -- TEST INFRASTRUCTURE: the CPU emulation of emu_coset.cpp (included whole, so sa_ntt's
// emulation, the batch inversion and the coset product are the same code) plus geometric interpolation plans, their
// batched apply, geometric zerofiers and the prefix-product scan: the library's own checks and schedules (geo.cuh)
// over a backend whose kernels are loops over their element functions.
// It is NOT a fallback: nothing in the product loads this library.
//
// Build: g++ -O2 -std=c++17 -shared -fPIC -o libsa_emu_geo.so emu_geo.cpp
#include "emu_coset.cpp"

#include "../../stark-anatomy_b200/csrc/geo.cuh"

// EmuCoset plus the kernels of the geometric schedules
struct EmuGeo : EmuCoset {
    int geo_scan_runs(fe *x, long long n, fe *tot) {
        return each((n + GEO_SCAN_RUN - 1) / GEO_SCAN_RUN, [&](long long r) { geo_scan_run_elem(x, n, tot, r); });
    }
    int geo_scan_add(fe *x, long long n, const fe *tot) {
        return each(n - GEO_SCAN_RUN, [&](long long i) { geo_scan_add_elem(x, tot, i); });
    }
    int geo_factor(fe *P, const fe *pw_m, long long count) {
        return each(count, [&](long long m) { geo_factor_elem(P, pw_m, m); });
    }
    int geo_seed(fe *out, const fe *pw_m, long long n, long long len) {
        return each(len, [&](long long t) { geo_seed_elem(out, pw_m, n, t); });
    }
    int geo_zerofier(fe *z, const fe *chirp_m, const fe *P_m, const fe *iP, long long k, int canon, long long len) {
        return each(len, [&](long long i) { geo_zerofier_elem(z, chirp_m, P_m, iP, k, canon, i); });
    }
    int geo_weight(fe *c, const fe *iP, long long k) {
        return each(k, [&](long long i) { geo_weight_elem(c, iP, k, i); });
    }
    int geo_load(fe *ws, const fe *values, const fe *c_m, long long k, int logK, long long batch) {
        return each(batch << logK, [&](long long i) { geo_load_elem(ws, values, c_m, k, logK, i); });
    }
    int geo_mid(fe *dst, const fe *src, const fe *ic_m, long long k, int logK, long long batch) {
        return each(batch << logK, [&](long long i) { geo_mid_elem(dst, src, ic_m, k, logK, i); });
    }
};

extern "C" {

size_t emu_geo_plan_bytes(size_t k) { return sizeof(fe) * geo_plan_layout(k).elems; }
size_t emu_geo_batch_max(size_t k) { return geo_batch_max(k); }
// sa_geo_plan with a host plan; the workspace starts from the stale pattern
int emu_geo_plan(uint64_t *plan, const uint64_t *step, size_t k) {
    SA_TRY(geo_check(k, step));
    std::vector<fe> ws = stale_workspace(geo_work_layout(k, geo_chirp_len(k, true)).elems);
    int flag = 0;
    EmuGeo b;
    SA_TRY(geo_plan_build(b, (fe *)plan, step, k, ws.data(), &flag));
    return flag ? SA_EDIVZERO : SA_OK;
}
// sa_geo_interp_batch with host rows, in chunks of `chunk` vectors (0: the library's)
int emu_geo_interp_batch(uint64_t *out, const uint64_t *plan, const uint64_t *values, size_t k, size_t batch,
                         size_t chunk) {
    const GeoPlan L = geo_plan_layout(k);
    if (L.elems == 0) return SA_ESIZE;
    if (batch == 0) return SA_OK;
    if (chunk == 0) chunk = geo_batch_max(k);
    std::vector<fe> ws = stale_workspace(2 * (size_t)L.K * std::min(batch, chunk));
    EmuGeo b;
    return geo_apply(b, (fe *)out, (const fe *)plan, (const fe *)values, k, batch, ws.data(), chunk);
}
int emu_geo_zerofier(uint64_t *out, const uint64_t *step, size_t k) {
    SA_TRY(geo_check(k, step));
    std::vector<fe> ws = stale_workspace(geo_work_layout(k, geo_chirp_len(k, false)).elems + k + 1);
    int flag = 0;
    EmuGeo b;
    return geo_zerofier(b, (fe *)out, step, k, ws.data(), &flag,
                        [](int *f) { return *f ? SA_EDIVZERO : SA_OK; });
}
// the scan alone: x[0..n) (canonical) <- its prefix products
void emu_geo_scan(uint64_t *x, size_t n) {
    std::vector<fe> v(n), tmp = stale_workspace(geo_scan_elems((long long)n));
    for (size_t i = 0; i < n; i++) v[i] = fe_to_mont(fe_from_limbs(x + 2 * i));
    EmuGeo b;
    geo_scan(b, v.data(), (long long)n, tmp.data());
    for (size_t i = 0; i < n; i++) {
        const fe c = fe_from_mont(v[i]);
        memcpy(x + 2 * i, &c, 16);
    }
}
size_t emu_geo_scan_elems(size_t n) { return geo_scan_elems((long long)n); }

}  // extern "C"
