// rescue.cu -- the Rescue-Prime permutation over many inputs (rescue.cuh): sa_rescue, one thread per input.
#include "runtime.cuh"
#include "rescue.cuh"

using namespace sa;

constexpr int RESCUE_BLOCK = 128;

// each block converts the caller's constants into shared memory once; every thread then reads the same constant at
// the same time (a broadcast)
__global__ void __launch_bounds__(RESCUE_BLOCK) k_rescue(fe *hashes, fe *trace, const fe *inputs, long long count,
                                                         const fe *constants, long long rounds, RescueExp ea,
                                                         RescueExp eb, long long inst_stride, long long lane_stride) {
    extern __shared__ fe kc[];
    const long long nconst = rescue_nconst(rounds);
    for (long long i = threadIdx.x; i < nconst; i += blockDim.x) kc[i] = rescue_load(constants, i);
    __syncthreads();
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x; b < count; b += stride)
        rescue_elem(hashes, trace, inputs, kc, rounds, ea, eb, inst_stride, lane_stride, b);
}

extern "C" {

int sa_rescue(void *hashes, void *trace, const void *inputs, size_t count, const void *constants, size_t rounds,
              const uint64_t alpha[2], const uint64_t alphainv[2], size_t inst_stride, size_t lane_stride,
              void *stream) {
    const int rc = rescue_check(hashes, trace, count, rounds, inst_stride, lane_stride);
    if (rc != SA_OK || count == 0) return rc;
    const size_t smem = sizeof(fe) * (size_t)rescue_nconst((long long)rounds);
    k_rescue<<<grid_for((long long)count, RESCUE_BLOCK), RESCUE_BLOCK, smem, (cudaStream_t)stream>>>(
        (fe *)hashes, (fe *)trace, (const fe *)inputs, (long long)count, (const fe *)constants, (long long)rounds,
        rescue_exp(alpha), rescue_exp(alphainv), (long long)inst_stride, (long long)lane_stride);
    SA_LAUNCH_CHECK();
    return SA_OK;
}

}  // extern "C"
