// transcript.cu -- proofs read from their pickled bytes (transcript.cuh): parse, Fiat-Shamir, draws and the sections
// of the verifier's chunk, for a batch of proofs of one plan's shape.
//
// The parse is sequential within a proof, so one thread parses one proof; a batch gives one thread per proof.  The
// hashes run one thread per Fiat-Shamir message, the draws one thread per proof, and the section writers one thread
// per path, per path digest and per proof.
#include "runtime.cuh"
#include "transcript.cuh"

using namespace sa;

constexpr int TRANSCRIPT_BLOCK = 128;
constexpr unsigned long long TRANSCRIPT_LIMIT = 1ULL << 59;

// the section offsets, passed by value
struct SectionAt {
    uint64_t at[SA_TRANSCRIPT_SECTIONS];
};

__global__ void __launch_bounds__(TRANSCRIPT_BLOCK, 1) k_transcript_parse(uint8_t *ws, const uint8_t *proofs,
                                                                      const uint64_t *proof_at,
                                                                      const uint8_t *prefixes, TShape s, TLayout l,
                                                                      long long nproofs) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x; b < nproofs; b += stride) {
        uint8_t *w = ws + b * l.total;
        const bool fits = *(const uint64_t *)(prefixes + b * SA_TRANSCRIPT_PREFIX) <= 128;
        *(uint32_t *)(w + l.status) = fits && transcript_parse(proofs + proof_at[2 * b], proof_at[2 * b + 1], s, w, l);
    }
}

__global__ void __launch_bounds__(TRANSCRIPT_BLOCK) k_transcript_fs(uint8_t *ws, const uint8_t *proofs,
                                                                   const uint64_t *proof_at, const uint8_t *prefixes,
                                                                   TShape s, TLayout l, long long count) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) {
        const long long b = i / s.nfs();
        const uint32_t m = (uint32_t)(i - b * s.nfs());
        uint8_t *w = ws + b * l.total;
        if (!*(const uint32_t *)(w + l.status)) continue;
        const uint64_t *span = (const uint64_t *)(w + l.span);
        const uint8_t *pre = prefixes + b * SA_TRANSCRIPT_PREFIX;
        transcript_fs_digest((uint64_t *)(w + l.fsd) + 4 * m, pre + 16, (uint32_t) * (const uint64_t *)pre, s.proto,
                             proofs + proof_at[2 * b] + span[0], span[1 + m] - span[0], s.fs_objects(m));
    }
}

__global__ void __launch_bounds__(TRANSCRIPT_BLOCK) k_transcript_draws(uint8_t *ws, TShape s, TLayout l,
                                                                      long long nproofs) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x; b < nproofs; b += stride) {
        uint8_t *w = ws + b * l.total;
        uint32_t *status = (uint32_t *)(w + l.status);
        if (*status && !transcript_draws(s, w, l)) *status = 0;
    }
}

__global__ void __launch_bounds__(TRANSCRIPT_BLOCK) k_transcript_paths(uint8_t *sec, SectionAt at,
                                                                      uint8_t *ws, const uint8_t *proofs,
                                                                      const uint64_t *proof_at, const uint8_t *zroot,
                                                                      TShape s, TLayout l, long long count) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    const long long np = (long long)s.npaths();
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) {
        const long long b = i / np;
        transcript_path_elem(sec, at.at, s, proofs + proof_at[2 * b], ws + b * l.total, l, zroot, b, i - b * np);
    }
}

__global__ void __launch_bounds__(TRANSCRIPT_BLOCK) k_transcript_digests(uint8_t *sec, SectionAt at,
                                                                        const uint8_t *ws, const uint8_t *proofs,
                                                                        const uint64_t *proof_at, TShape s, TLayout l,
                                                                        long long count) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    const long long nd = (long long)s.path_digests();
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) {
        const long long b = i / nd;
        transcript_digest_elem(sec, at.at, s, proofs + proof_at[2 * b], ws + b * l.total, l, b, i - b * nd);
    }
}

__global__ void __launch_bounds__(TRANSCRIPT_BLOCK, 1) k_transcript_proofs(uint8_t *sec, SectionAt at,
                                                                       uint8_t *ws, const uint8_t *proofs,
                                                                       const uint64_t *proof_at, const fe *statement,
                                                                       long long nstat, uint8_t *out, TShape s,
                                                                       TLayout l, long long nproofs) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x; b < nproofs; b += stride)
        transcript_proof_elem(sec, at.at, s, proofs + proof_at[2 * b], ws + b * l.total, l, statement, nstat,
                              out + b * SA_TRANSCRIPT_OUT, b);
}


extern "C" {

size_t sa_transcript_bytes(const uint64_t shape[SA_TRANSCRIPT_SHAPE]) {
    if (!shape || !transcript_shape_ok(shape)) return 0;
    const TLayout l = transcript_layout(transcript_shape(shape));
    return l.total >= TRANSCRIPT_LIMIT ? 0 : (size_t)l.total;
}

int sa_transcript_sections(void *sections, const uint64_t section_at[SA_TRANSCRIPT_SECTIONS], void *out,
                           void *workspace, const void *proofs, const uint64_t *proof_at, const void *prefixes,
                           const void *statement, size_t nstat, const void *zroot, size_t nproofs,
                           const uint64_t shape[SA_TRANSCRIPT_SHAPE], void *stream) {
    if (sa_transcript_bytes(shape) == 0 || !section_at) return SA_ESIZE;
    const TShape s = transcript_shape(shape);
    const TLayout l = transcript_layout(s);
    if (nproofs >= TRANSCRIPT_LIMIT || nstat >= ((size_t)1 << 32) || (zroot != nullptr) != (s.nopen == s.nregs + 2))
        return SA_ESIZE;
    const unsigned long long per = l.total > s.path_digests() * 64 ? l.total : s.path_digests() * 64;
    unsigned long long total;
    if (__builtin_mul_overflow((unsigned long long)nproofs, per, &total) || total >= TRANSCRIPT_LIMIT) return SA_ESIZE;
    if (nproofs == 0) return SA_OK;
    if (!sections || !out || !workspace || !proofs || !proof_at || !prefixes || (nstat && !statement))
        return SA_ESIZE;
    cudaStream_t st = (cudaStream_t)stream;
    SectionAt a;
    for (int i = 0; i < SA_TRANSCRIPT_SECTIONS; i++) a.at[i] = section_at[i];
    uint8_t *sec = (uint8_t *)sections, *ws = (uint8_t *)workspace;
    const uint8_t *pr = (const uint8_t *)proofs;
    const long long B = (long long)nproofs;
    k_transcript_parse<<<grid_for(B, TRANSCRIPT_BLOCK), TRANSCRIPT_BLOCK, 0, st>>>(ws, pr, proof_at,
                                                                                    (const uint8_t *)prefixes, s, l, B);
    SA_LAUNCH_CHECK();
    const long long nfs = B * s.nfs();
    k_transcript_fs<<<grid_for(nfs, TRANSCRIPT_BLOCK), TRANSCRIPT_BLOCK, 0, st>>>(
        ws, pr, proof_at, (const uint8_t *)prefixes, s, l, nfs);
    SA_LAUNCH_CHECK();
    k_transcript_draws<<<grid_for(B, TRANSCRIPT_BLOCK), TRANSCRIPT_BLOCK, 0, st>>>(ws, s, l, B);
    SA_LAUNCH_CHECK();
    const long long np = B * (long long)s.npaths(), nd = B * (long long)s.path_digests();
    k_transcript_paths<<<grid_for(np, TRANSCRIPT_BLOCK), TRANSCRIPT_BLOCK, 0, st>>>(
        sec, a, ws, pr, proof_at, (const uint8_t *)zroot, s, l, np);
    SA_LAUNCH_CHECK();
    k_transcript_digests<<<grid_for(nd, TRANSCRIPT_BLOCK), TRANSCRIPT_BLOCK, 0, st>>>(sec, a, ws, pr, proof_at,
                                                                                      s, l, nd);
    SA_LAUNCH_CHECK();
    k_transcript_proofs<<<grid_for(B, TRANSCRIPT_BLOCK), TRANSCRIPT_BLOCK, 0, st>>>(
        sec, a, ws, pr, proof_at, (const fe *)statement, (long long)nstat, (uint8_t *)out, s, l, B);
    SA_LAUNCH_CHECK();
    return SA_OK;
}

}  // extern "C"
