// tests/emu/emu_sample.cpp -- TEST INFRASTRUCTURE: the CPU emulation of seeded randomizer draws (csrc/sample.cuh):
// the element functions the kernel runs, and sa_sample_seeded's checks and grid-stride index map run thread by thread
// over a grid of `threads` threads.
// It is NOT a fallback: nothing in the product loads this library.
//
// Build: g++ -O2 -std=c++17 -shared -fPIC -o libsa_emu_sample.so emu_sample.cpp
#include <cstring>

#include "../../stark-anatomy_b200/csrc/sample.cuh"

using namespace sa;

extern "C" {

// (top, hi, lo) = x < 2^136 -> x mod p as two little-endian words
void emu_sample_reduce(uint64_t *out, uint32_t top, uint64_t hi, uint64_t lo) {
    const fe r = sample_reduce(top, hi, lo);
    memcpy(out, &r, 16);
}

// element(seed, j) as two little-endian words
void emu_seeded_element(uint64_t *out, const uint8_t *seed, uint64_t j) {
    const fe r = seeded_element(sample_seed_word(seed, 0), sample_seed_word(seed, 1), sample_seed_word(seed, 2),
                                sample_seed_word(seed, 3), j);
    memcpy(out, &r, 16);
}

// sa_sample_seeded with host buffers: its checks, then thread t of `threads` takes items t, t + threads, ...
int emu_sample_seeded(uint64_t *out, const uint8_t *seeds, size_t nseeds, size_t seed_stride, uint64_t first,
                      size_t count, size_t width, size_t lane_stride, long long threads) {
    long long total = 0;
    const int rc = sample_check(nseeds, seed_stride, first, count, width, lane_stride, &total);
    if (rc != SA_OK || total == 0) return rc;
    for (long long t = 0; t < threads; t++)
        for (long long i = t; i < total; i += threads)
            sample_seeded_elem((fe *)out, seeds, first, (long long)count, (long long)width, (long long)lane_stride,
                               (long long)seed_stride, i);
    return SA_OK;
}

}  // extern "C"
