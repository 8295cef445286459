// host.cuh -- host-side helpers of the library and of the headers the CPU emulation (tests/emu) compiles too.
#pragma once
#include <stddef.h>

#include "../../include/sa_b200.h"

static inline bool host_is_pow2(size_t n) { return n && !(n & (n - 1)); }
// ceil(log2 n): the exponent of the smallest power of two >= n
static inline int host_log2(size_t n) {
    int l = 0;
    while ((size_t(1) << l) < n) l++;
    return l;
}

// returns the error code of a call that fails
#define SA_TRY(expr) do { const int _rc = (expr); if (_rc != SA_OK) return _rc; } while (0)
