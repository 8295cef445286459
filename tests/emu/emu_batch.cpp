// tests/emu/emu_batch.cpp -- TEST INFRASTRUCTURE: the CPU emulation of emu_air_exact.cpp (included whole, so the AIR
// plan, the element functions and the exact store are the same emulated code) plus what proving many statements of
// one AIR at once adds: the batched applies of air.cuh (air_quotients and air_quotients_exact over a batch of traces,
// with chunk sizes the caller may make small enough to cross at emulated sizes), coset.cuh's combination into many
// rows, and fri_merkle.cuh's gathers and Merkle paths with an index set per group of rows.
// It is NOT a fallback: nothing in the product loads this library.
//
// Build: g++ -O2 -std=c++17 -shared -fPIC -o libsa_emu_batch.so emu_batch.cpp
#include "emu_air_exact.cpp"

// EmuAirExact with k_air_eval over a chunk of traces, plus k_coset_combine over many rows
struct EmuBatch : EmuAirExact {
    int air_eval(fe *V, const fe *prog, const fe *x_m, const fe *iz_m, const fe *ext, long long r0, long long nb,
                 long long ncons, long long bp, int nregs, int log_n) {
        return each(1ll << log_n, [&](long long i) {
            air_eval_rows_elem(V, prog, x_m, iz_m, ext, r0, nb, ncons, bp, nregs, log_n, i);
        });
    }
    int coset_combine(fe *out, const CombineGroup &g, const fe *pw_m, long long ncomb, int log_n, long long nrows,
                      int first) {
        return each(nrows << log_n, [&](long long i) { coset_combine_elem(out, g, pw_m, ncomb, first, log_n, i); });
    }
};

// the library's chunks (air_chunks) unless the caller asks for traces > 0 traces and rows > 0 rows per chunk
static AirChunks emu_chunks(size_t nregs, size_t ncons, size_t batch, int log_n, size_t traces, size_t rows) {
    AirChunks k = air_chunks(nregs, ncons, batch, log_n);
    if (traces) k.traces = traces;
    if (rows) k.rows = rows;
    return k;
}

extern "C" {

size_t emu_air_batch_max(size_t nregs, size_t ncons, int log_n) { return air_batch_max(nregs, ncons, log_n); }

// sa_air_quotients_batch with host rows; out and the workspace start from the stale pattern once the checks pass
int emu_air_quotients_batch(uint64_t *out, const uint64_t *plan, const uint64_t *trace, size_t nregs, size_t ncoef,
                            size_t qlen, size_t ncons, size_t batch, int log_n, const uint64_t *root, size_t traces,
                            size_t rows) {
    SA_TRY(air_apply_check(log_n, nregs, ncoef, qlen, ncons, root));
    if (batch == 0) return SA_OK;
    const AirChunks k = emu_chunks(nregs, ncons, batch, log_n, traces, rows);
    std::vector<fe> ws = stale_workspace(air_ws_elems(nregs, k, log_n));
    const std::vector<fe> stale = stale_workspace(batch * ncons * qlen);
    memcpy(out, stale.data(), sizeof(fe) * stale.size());
    EmuBatch b;
    return air_quotients(b, (fe *)out, (const fe *)plan, (const fe *)trace, nregs, ncoef, qlen, ncons, batch, log_n,
                         root, ws.data(), k);
}
// sa_air_quotients_exact_batch with host rows; out, flags and the workspace start from a stale pattern
int emu_air_quotients_exact_batch(uint64_t *out, uint32_t *flags, const uint64_t *plan, const uint64_t *trace,
                                  size_t nregs, size_t ncoef, size_t qlen, size_t ncons, size_t batch, size_t tail,
                                  int log_n, const uint64_t *root, size_t traces, size_t rows) {
    SA_TRY(air_exact_check(log_n, nregs, ncoef, qlen, ncons, tail, root));
    if (batch == 0) return SA_OK;
    const AirChunks k = emu_chunks(nregs, ncons, batch, log_n, traces, rows);
    std::vector<fe> ws = stale_workspace(air_ws_elems(nregs, k, log_n));
    const std::vector<fe> stale = stale_workspace(batch * ncons * qlen);
    memcpy(out, stale.data(), sizeof(fe) * stale.size());
    for (size_t c = 0; c < batch * ncons; c++) flags[c] = 0x5a5a5a5au;
    EmuBatch b;
    return air_quotients_exact(b, (fe *)out, flags, (const fe *)plan, (const fe *)trace, nregs, ncoef, qlen, ncons,
                               batch, tail, log_n, root, ws.data(), k);
}
// sa_coset_combine_evaluate_batch with host source rows; out starts from the stale pattern once the checks pass
int emu_coset_combine_evaluate_batch(uint64_t *out, size_t nrows, int log_n, const uint64_t *root,
                                     const uint64_t *offset, const void *const *srcs, const size_t *lens,
                                     const size_t *shifts, const size_t *rows, const uint64_t *weights, size_t nterms) {
    SA_TRY(coset_combine_check(log_n, lens, shifts, rows, nrows, nterms, root));
    if (nrows == 0) return SA_OK;
    std::vector<fe> pw = stale_workspace(coset_combine_len(lens, shifts, nterms));
    const std::vector<fe> stale = stale_workspace(nrows << log_n);
    memcpy(out, stale.data(), sizeof(fe) * stale.size());
    EmuBatch b;
    return coset_combine_evaluate(b, (fe *)out, nrows, log_n, root, offset, (const fe *const *)srcs, lens, shifts,
                                  rows, weights, nterms, pw.data());
}
// sa_gather_batch_sets with host rows: index_sets_check, then gather_sets_elem over every output
int emu_gather_batch_sets(uint64_t *out, const uint64_t *values, size_t n, size_t batch, size_t group,
                          const uint64_t *indices, size_t k) {
    size_t count = 0;
    SA_TRY(index_sets_check(indices, batch, group, k, n, &count));
    for (long long t = 0; t < (long long)(batch * k); t++)
        gather_sets_elem((fe *)out, (const fe *)values, (long long)n, indices, (long long)k, (long long)group, t);
    return SA_OK;
}
// sa_merkle_open_batch_sets with host trees: the same checks, then merkle_path_sets_elem over every output word
int emu_merkle_open_batch_sets(uint8_t *paths, const uint8_t *trees, size_t n, size_t batch, size_t group,
                               const uint64_t *indices, size_t k) {
    if (!host_is_pow2(n)) return SA_ENOTPOW2;
    const int depth = host_log2(n);
    size_t count = 0;
    SA_TRY(index_sets_check(indices, batch, group, k, n, &count));
    for (long long t = 0; t < (long long)(batch * k * depth * 8); t++)
        merkle_path_sets_elem((uint64_t *)paths, (const uint64_t *)trees, (long long)n, depth, indices, (long long)k,
                              (long long)group, t);
    return SA_OK;
}

}  // extern "C"
