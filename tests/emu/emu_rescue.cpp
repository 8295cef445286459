// tests/emu/emu_rescue.cpp -- TEST INFRASTRUCTURE: the CPU emulation of the Rescue-Prime kernel (csrc/rescue.cuh):
// sa_rescue's checks, the per-block constant conversion and the grid-stride loop run thread by thread over a grid of
// `threads` threads.  The same library carries rescue_oracle.cpp, an independent restatement used as the oracle.
// It is NOT a fallback: nothing in the product loads this library.
//
// Build: g++ -O2 -std=c++17 -shared -fPIC -o libsa_emu_rescue.so emu_rescue.cpp rescue_oracle.cpp
#include <vector>

#include "../../stark-anatomy_b200/csrc/rescue.cuh"

using namespace sa;

extern "C" {

// sa_rescue with host buffers (hashes and trace may be NULL)
int emu_rescue(uint64_t *hashes, uint64_t *trace, const uint64_t *inputs, size_t count, const uint64_t *constants,
               size_t rounds, const uint64_t *alpha, const uint64_t *alphainv, size_t inst_stride, size_t lane_stride,
               long long threads) {
    const int rc = rescue_check(hashes, trace, count, rounds, inst_stride, lane_stride);
    if (rc != SA_OK || count == 0) return rc;
    const long long nconst = rescue_nconst((long long)rounds);
    std::vector<fe> kc(nconst);
    for (long long i = 0; i < nconst; i++) kc[i] = rescue_load((const fe *)constants, i);
    const RescueExp ea = rescue_exp(alpha), eb = rescue_exp(alphainv);
    for (long long t = 0; t < threads; t++)
        for (long long b = t; b < (long long)count; b += threads)
            rescue_elem((fe *)hashes, (fe *)trace, (const fe *)inputs, kc.data(), (long long)rounds, ea, eb,
                        (long long)inst_stride, (long long)lane_stride, b);
    return SA_OK;
}

}  // extern "C"
