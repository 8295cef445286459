// tests/emu/emu_transcript.cpp -- TEST INFRASTRUCTURE: the CPU emulation of the transcript reader
// (csrc/transcript.cuh): sa_transcript_sections run proof by proof and item by item in the kernels' order, and the
// hashes and reductions on their own.
// It is NOT a fallback: nothing in the product loads this library.
//
// Build: g++ -O2 -std=c++17 -shared -fPIC -o libsa_emu_transcript.so emu_transcript.cpp
#include <cstring>

#include "../../stark-anatomy_b200/csrc/transcript.cuh"

using namespace sa;

extern "C" {

size_t emu_transcript_bytes(const uint64_t *shape) {
    if (!transcript_shape_ok(shape)) return 0;
    return (size_t)transcript_layout(transcript_shape(shape)).total;
}

// sa_transcript_sections on host buffers (the caller checked the sizes as the C ABI does)
int emu_transcript_sections(void *sections, const uint64_t *section_at, void *out, void *workspace,
                            const void *proofs, const uint64_t *proof_at, const void *prefixes, const void *statement,
                            size_t nstat, const void *zroot, size_t nproofs, const uint64_t *shape) {
    if (!transcript_shape_ok(shape)) return SA_ESIZE;
    const TShape s = transcript_shape(shape);
    const TLayout l = transcript_layout(s);
    uint8_t *sec = (uint8_t *)sections, *ws = (uint8_t *)workspace, *o = (uint8_t *)out;
    const uint8_t *pr = (const uint8_t *)proofs, *pre = (const uint8_t *)prefixes;
    for (size_t b = 0; b < nproofs; b++) {
        uint8_t *w = ws + b * l.total;
        const bool fits = *(const uint64_t *)(pre + b * SA_TRANSCRIPT_PREFIX) <= 128;
        *(uint32_t *)(w + l.status) = fits && transcript_parse(pr + proof_at[2 * b], proof_at[2 * b + 1], s, w, l);
    }
    for (size_t b = 0; b < nproofs; b++) {
        uint8_t *w = ws + b * l.total;
        if (!*(uint32_t *)(w + l.status)) continue;
        const uint64_t *span = (const uint64_t *)(w + l.span);
        const uint8_t *p = pre + b * SA_TRANSCRIPT_PREFIX;
        for (uint32_t m = 0; m < s.nfs(); m++)
            transcript_fs_digest((uint64_t *)(w + l.fsd) + 4 * m, p + 16, (uint32_t) * (const uint64_t *)p, s.proto,
                                 pr + proof_at[2 * b] + span[0], span[1 + m] - span[0], s.fs_objects(m));
    }
    for (size_t b = 0; b < nproofs; b++) {
        uint8_t *w = ws + b * l.total;
        uint32_t *status = (uint32_t *)(w + l.status);
        if (*status && !transcript_draws(s, w, l)) *status = 0;
    }
    for (size_t b = 0; b < nproofs; b++)
        for (uint64_t q = 0; q < s.npaths(); q++)
            transcript_path_elem(sec, section_at, s, pr + proof_at[2 * b], ws + b * l.total, l,
                                 (const uint8_t *)zroot, b, q);
    for (size_t b = 0; b < nproofs; b++)
        for (uint64_t t = 0; t < s.path_digests(); t++)
            transcript_digest_elem(sec, section_at, s, pr + proof_at[2 * b], ws + b * l.total, l, b, t);
    for (size_t b = 0; b < nproofs; b++)
        transcript_proof_elem(sec, section_at, s, pr + proof_at[2 * b], ws + b * l.total, l, (const fe *)statement,
                              nstat, o + b * SA_TRANSCRIPT_OUT, b);
    return SA_OK;
}

// the Fiat-Shamir digests of proof b after emu_transcript_sections (32 bytes per message), and its draws
void emu_transcript_draws(void *fsd, void *weights, void *alphas, uint64_t *top, const void *workspace, size_t b,
                          const uint64_t *shape) {
    const TShape s = transcript_shape(shape);
    const TLayout l = transcript_layout(s);
    const uint8_t *w = (const uint8_t *)workspace + b * l.total;
    memcpy(fsd, w + l.fsd, 32 * s.nfs());
    memcpy(weights, w + l.weights, 16 * (size_t)s.nweights);
    memcpy(alphas, w + l.alphas, 16 * (size_t)s.rounds);
    memcpy(top, w + l.top, 8 * (size_t)s.k);
}

// shake_256(msg).digest(32)
void emu_shake256(uint8_t *out, const uint8_t *msg, size_t n) {
    Shake256 h;
    h.init();
    h.bytes(msg, n);
    uint64_t d[4];
    h.final32(d);
    memcpy(out, d, 32);
}

// blake2b(seed + bytes(zeros)).digest()
void emu_blake2b_zeros(uint8_t *out, const uint8_t *seed, uint64_t zeros) {
    uint64_t s[4], d[8];
    memcpy(s, seed, 32);
    blake2b_seed_zeros(d, s, zeros);
    memcpy(out, d, 64);
}

// int.from_bytes(data[:nbytes], "big") % p for nbytes 32 or 64, as 16 little-endian bytes
void emu_reduce_be(uint8_t *out, const uint8_t *data, int nbytes) {
    uint64_t w[8];
    memcpy(w, data, nbytes);
    const fe v = transcript_reduce_be(w, nbytes);
    memcpy(out, &v, 16);
}

}  // extern "C"
