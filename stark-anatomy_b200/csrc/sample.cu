// sample.cu -- seeded randomizer draws (sample.cuh): sa_sample_seeded, one draw per thread.
#include "runtime.cuh"
#include "sample.cuh"

using namespace sa;

__global__ void __launch_bounds__(256) k_sample_seeded(fe *out, const uint8_t *seeds, uint64_t first, long long count,
                                                       long long width, long long lane_stride, long long seed_stride,
                                                       long long total) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride)
        sample_seeded_elem(out, seeds, first, count, width, lane_stride, seed_stride, i);
}

extern "C" {

int sa_sample_seeded(void *out, const void *seeds, size_t nseeds, size_t seed_stride, uint64_t first, size_t count,
                     size_t width, size_t lane_stride, void *stream) {
    long long total = 0;
    const int rc = sample_check(nseeds, seed_stride, first, count, width, lane_stride, &total);
    if (rc != SA_OK || total == 0) return rc;
    k_sample_seeded<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
        (fe *)out, (const uint8_t *)seeds, first, (long long)count, (long long)width, (long long)lane_stride,
        (long long)seed_stride, total);
    SA_LAUNCH_CHECK();
    return SA_OK;
}

}  // extern "C"
