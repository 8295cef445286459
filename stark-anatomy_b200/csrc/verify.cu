// verify.cu -- the verifier's data-parallel checks (verify.cuh): Merkle paths, FRI colinearity, the combination at
// the opened indices, the degree of many codewords' coefficient rows and the AIR program the combination walks.
//
// One thread per item in every kernel.  A Merkle path is a chain of dependent compressions, so a warp per path would
// leave 31 lanes idle at every level; a thread per path keeps every lane on its own path, and a batch has tens of
// thousands of them.  The colinearity and combination items are one independent field computation each.
#include <vector>

#include "runtime.cuh"
#include "verify.cuh"

using namespace sa;

constexpr int VERIFY_BLOCK = 128;

__global__ void __launch_bounds__(VERIFY_BLOCK) k_merkle_verify(uint32_t *flags, const uint64_t *roots, const fe *leaves,
                                                               const uint64_t *leaf_index, const uint32_t *depth,
                                                               const uint64_t *paths, const uint64_t *path_offset,
                                                               long long count) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride)
        flags[i] = merkle_verify_elem(roots, leaves, leaf_index, depth, paths, path_offset, i);
}

__global__ void __launch_bounds__(VERIFY_BLOCK) k_fri_colinear(uint32_t *flags, const fe *ay, const fe *by, const fe *cy,
                                                              const uint64_t *a_index, const fe *alpha,
                                                              const uint32_t *round, fe offset_m, fe omega_m,
                                                              long long count) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride)
        flags[i] = fri_colinear_elem(ay, by, cy, a_index, alpha, round, offset_m, omega_m, i);
}

__global__ void __launch_bounds__(VERIFY_BLOCK) k_verify_combination(uint32_t *flags, const fe *items, const fe *proofs,
                                                                    long long k, long long count, const fe *prog,
                                                                    long long ncons, int nregs, long long blen,
                                                                    const fe *zcoef, long long zlen, fe offset_m,
                                                                    fe omega_m, int log_n, long long ef) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < count; j += stride)
        flags[j] = verify_combination_elem(items, proofs, k, prog, ncons, nregs, blen, zcoef, zlen, offset_m, omega_m,
                                           log_n, ef, j);
}

__global__ void __launch_bounds__(256) k_poly_degree(long long *degrees, const fe *coeffs, int log_n, long long total) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += stride) {
        const long long d = degree_elem(coeffs, log_n, idx);
        if (d >= 0) atomicMax(degrees + (idx >> log_n), d);
    }
}

extern "C" {

int sa_merkle_verify_batch(uint32_t *flags, const void *roots, const void *leaves, const uint64_t *leaf_index,
                           const uint32_t *depth, const void *paths, const uint64_t *path_offset, size_t count,
                           void *stream) {
    SA_TRY(verify_count_check(count));
    if (count == 0) return SA_OK;
    if (!flags || !roots || !leaves || !leaf_index || !depth || !paths || !path_offset) return SA_ESIZE;
    k_merkle_verify<<<grid_for((long long)count, VERIFY_BLOCK), VERIFY_BLOCK, 0, (cudaStream_t)stream>>>(
        flags, (const uint64_t *)roots, (const fe *)leaves, leaf_index, depth, (const uint64_t *)paths, path_offset,
        (long long)count);
    SA_LAUNCH_CHECK();
    return SA_OK;
}

int sa_fri_colinear_batch(uint32_t *flags, const void *ay, const void *by, const void *cy, const uint64_t *a_index,
                          const void *alpha, const uint32_t *round, const uint64_t offset[2], const uint64_t omega[2],
                          size_t count, void *stream) {
    SA_TRY(verify_count_check(count));
    if (count == 0) return SA_OK;
    if (!flags || !ay || !by || !cy || !a_index || !alpha || !round) return SA_ESIZE;
    k_fri_colinear<<<grid_for((long long)count, VERIFY_BLOCK), VERIFY_BLOCK, 0, (cudaStream_t)stream>>>(
        flags, (const fe *)ay, (const fe *)by, (const fe *)cy, a_index, (const fe *)alpha, round,
        fe_to_mont(fe_from_limbs(offset)), fe_to_mont(fe_from_limbs(omega)), (long long)count);
    SA_LAUNCH_CHECK();
    return SA_OK;
}

int sa_verify_combination(uint32_t *flags, const void *items, const void *proofs, size_t k, size_t nproofs,
                          const void *prog, size_t ncons, size_t nregs, size_t blen, const void *zcoef, size_t zlen,
                          const uint64_t offset[2], const uint64_t omega[2], int log_n, size_t ef, void *stream) {
    SA_TRY(verify_combination_check(k, nproofs, ncons, nregs, blen, zlen, zcoef != nullptr, log_n, ef));
    const long long count = (long long)(k * nproofs);
    if (count == 0) return SA_OK;
    if (!flags || !items || !proofs || !prog) return SA_ESIZE;
    k_verify_combination<<<grid_for(count, VERIFY_BLOCK), VERIFY_BLOCK, 0, (cudaStream_t)stream>>>(
        flags, (const fe *)items, (const fe *)proofs, (long long)k, count, (const fe *)prog, (long long)ncons,
        (int)nregs, (long long)blen, (const fe *)zcoef, (long long)zlen, fe_to_mont(fe_from_limbs(offset)),
        fe_to_mont(fe_from_limbs(omega)), log_n, (long long)ef);
    SA_LAUNCH_CHECK();
    return SA_OK;
}

int sa_poly_degree_batch(long long *degrees, const void *coeffs, size_t n, size_t batch, void *stream) {
    if (n == 0 || (n & (n - 1)) || n > ((size_t)1 << 30)) return SA_ESIZE;
    SA_TRY(verify_count_check(batch));
    if (batch >= VERIFY_LIMIT / n) return SA_ESIZE;
    if (batch == 0) return SA_OK;
    if (!degrees || !coeffs) return SA_ESIZE;
    int log_n = 0;
    while (((size_t)1 << log_n) < n) log_n++;
    cudaStream_t st = (cudaStream_t)stream;
    SA_CUDA(cudaMemsetAsync(degrees, 0xFF, sizeof(long long) * batch, st));  // -1: the zero row
    const long long total = (long long)(batch * n);
    k_poly_degree<<<grid_for(total, 256), 256, 0, st>>>(degrees, (const fe *)coeffs, log_n, total);
    SA_LAUNCH_CHECK();
    return SA_OK;
}

size_t sa_air_program_bytes(size_t nterms, size_t nregs) {
    if (nregs == 0 || nregs > AIR_MAX_TERMS || nterms >= AIR_MAX_TERMS) return 0;
    return sizeof(fe) * (1 + nterms * air_rec(nregs));
}

int sa_air_program(void *prog, const uint64_t *coeffs, const uint32_t *exps, const size_t *term_start, size_t ncons,
                   size_t nregs, void *stream) {
    if (ncons == 0 || nregs == 0 || !prog || !term_start) return SA_ESIZE;
    for (size_t c = 0; c < ncons; c++)
        if (term_start[c + 1] < term_start[c]) return SA_ESIZE;
    if (sa_air_program_bytes(term_start[ncons] - term_start[0], nregs) == 0) return SA_ESIZE;
    const std::vector<fe> host = air_compile(coeffs, exps, term_start, ncons, nregs);
    cudaStream_t st = (cudaStream_t)stream;
    SA_CUDA(cudaMemcpyAsync(prog, host.data(), sizeof(fe) * host.size(), cudaMemcpyHostToDevice, st));
    SA_CUDA(cudaStreamSynchronize(st));  // `host` goes out of scope here
    return SA_OK;
}

}  // extern "C"
