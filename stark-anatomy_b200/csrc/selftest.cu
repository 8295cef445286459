// selftest.cu -- the field self tests (PTX carry chains of field.cuh and of the NTT tile's butterfly against
// the portable C++ arithmetic) and the microbenchmarks of the field product and the blake2b compression.
#include "fri_merkle.cuh"
#include "ntt_tile.cuh"
#include "runtime.cuh"

using namespace sa;

// --- self test: PTX carry-chain field ops vs the portable C++ ones -------------------------
__device__ __forceinline__ uint64_t sa_splitmix(uint64_t &s) {
    uint64_t z = (s += 0x9E3779B97F4A7C15ULL);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}
__device__ __forceinline__ fe sa_rand_fe(uint64_t &s, int kind) {
    const uint64_t a = sa_splitmix(s), b = sa_splitmix(s);
    fe r = fe_make((uint32_t)a, (uint32_t)(a >> 32), (uint32_t)b, (uint32_t)(b >> 32));
    switch (kind & 15) {  // edge cases
        case 0: r = fe_zero(); break;
        case 1: r = fe_one(); break;
        case 2: r = fe_make(0, 0, 0, P3); break;                                  // p - 1
        case 3: r = fe_make(0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, P3 - 1); break;  // p - 2
        case 4: r.v[3] = P3; r.v[2] = 0; r.v[1] = 0; r.v[0] = 0; break;
        case 5: r.v[0] = 0; break;
        case 6: r.v[0] = 0; r.v[1] = 0; r.v[2] = 0; break;
        default: break;
    }
    // canonicalise: force below p
    if (r.v[3] > P3 || (r.v[3] == P3 && (r.v[2] | r.v[1] | r.v[0]) != 0)) r.v[3] -= P3;
    return r;
}
__global__ void k_selftest_field(unsigned long long *mismatches, long long count, uint64_t seed) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    uint64_t s = seed + 0x1234567ULL * (uint64_t)i;
    const fe a = sa_rand_fe(s, (int)(i % 37)), b = sa_rand_fe(s, (int)((i / 37) % 41));
    int bad = 0;
    bad += !fe_eq(fe_add(a, b), fe_add_portable(a, b));
    bad += !fe_eq(fe_sub(a, b), fe_sub_portable(a, b));
    bad += !fe_eq(fe_montmul(a, b), fe_montmul_portable(a, b));
    if (bad) atomicAdd(mismatches, (unsigned long long)bad);
}

// tile_mul / tile_bfly (ntt_tile.cuh) against the portable field: item i < npairs takes (x, w) from the
// caller's list, the others draw random and edge operands; the butterfly's e is always drawn
__global__ void k_selftest_tile(unsigned long long *mismatches, long long count, uint64_t seed, const fe *pairs,
                                long long npairs) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count + npairs) return;
    uint64_t s = seed + 0x9E3779B1ULL * (uint64_t)i;
    const fe e = sa_rand_fe(s, (int)(i % 43));
    fe x, w;
    if (i < npairs) {
        x = pairs[2 * i];
        w = pairs[2 * i + 1];
    } else {
        x = sa_rand_fe(s, (int)(i % 37));
        w = sa_rand_fe(s, (int)((i / 37) % 41));
    }
    const fe t = fe_montmul_portable(x, w);
    fe lo = e, hi = x;
    tile_bfly(lo, hi, w);
    int bad = 0;
    bad += !fe_eq(tile_mul(x, w), t);
    bad += !fe_eq(lo, fe_add_portable(e, t));
    bad += !fe_eq(hi, fe_sub_portable(e, t));
    if (bad) atomicAdd(mismatches, (unsigned long long)bad);
}

template <int OP, int ILP>
__global__ void k_microbench(fe *sink, int iters) {
    fe x[ILP], y[ILP];
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
#pragma unroll
    for (int i = 0; i < ILP; i++) {
        x[i] = fe_make(t + i, t * 3 + 1, i + 7, 0x12345678u + i);
        y[i] = fe_make(t * 5 + i, t + 11, i + 3, 0x0ABCDEF0u + i);
    }
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < ILP; i++) {
            if (OP == 0) x[i] = fe_montmul(x[i], y[i]);
            if (OP == 1) x[i] = fe_add(x[i], y[i]);
            if (OP == 2) x[i] = fe_sub(x[i], y[i]);
            if (OP == 3) {
                const fe tt = fe_montmul(y[i], x[(i + 1) % ILP]);
                const fe e = x[i];
                x[i] = fe_add(e, tt);
                y[i] = fe_sub(e, tt);
            }
            if (OP == 5) {  // op 3 through the NTT tile's butterfly
                const fe w = x[(i + 1) % ILP];
                tile_bfly(x[i], y[i], w);
            }
        }
    }
    fe acc = x[0];
#pragma unroll
    for (int i = 1; i < ILP; i++) acc = fe_add(acc, fe_add(x[i], y[i]));
    if (acc.v[0] == 0xDEADBEEFu && acc.v[1] == 0x1u) tile_st(sink + t, acc);
}

extern "C" {

long long sa_selftest_field(size_t count, uint64_t seed) {
    unsigned long long *d = nullptr, h = 0;
    SA_CUDA(cudaMalloc(&d, 8));
    SA_CUDA(cudaMemset(d, 0, 8));
    k_selftest_field<<<(unsigned)((count + 255) / 256), 256>>>(d, (long long)count, seed);
    SA_LAUNCH_CHECK();
    SA_CUDA(cudaMemcpy(&h, d, 8, cudaMemcpyDeviceToHost));
    cudaFree(d);
    return (long long)h;
}

long long sa_selftest_tile(size_t count, uint64_t seed, const uint64_t *pairs, size_t npairs) {
    if (npairs > 0 && pairs == nullptr) return SA_ESIZE;
    for (size_t k = 0; k < 2 * npairs; k++) {  // the pairs are field elements: canonical, below p
        const uint64_t hi = pairs[2 * k + 1];
        if (hi > ((uint64_t)P3 << 32) || (hi == ((uint64_t)P3 << 32) && pairs[2 * k] != 0)) return SA_ESIZE;
    }
    // one allocation: the mismatch counter, then the pairs as 16-byte elements
    char *d = nullptr;
    unsigned long long h = 0;
    SA_CUDA(cudaMalloc(&d, sizeof(fe) * (1 + 2 * npairs)));
    const fe *dp = reinterpret_cast<const fe *>(d) + 1;
    cudaError_t e = cudaMemset(d, 0, 8);
    if (e == cudaSuccess && npairs > 0)
        e = cudaMemcpy((void *)dp, pairs, sizeof(fe) * 2 * npairs, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        cudaFree(d);
        SA_CUDA(e);
    }
    const long long total = (long long)(count + npairs);
    if (total > 0)
        k_selftest_tile<<<(unsigned)((total + 255) / 256), 256>>>(reinterpret_cast<unsigned long long *>(d),
                                                                  (long long)count, seed, dp, (long long)npairs);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpy(&h, d, 8, cudaMemcpyDeviceToHost);
    cudaFree(d);
    SA_CUDA(e);
    if (total > 0) g_launches.fetch_add(1, std::memory_order_relaxed);
    return (long long)h;
}

}  // extern "C"
template <int OP>
static double microbench_op(int ilp, int iters, int blocks, int threads, fe *sink) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    auto run = [&](int it) {
        switch (ilp) {
            case 1: k_microbench<OP, 1><<<blocks, threads>>>(sink, it); break;
            case 2: k_microbench<OP, 2><<<blocks, threads>>>(sink, it); break;
            case 4: k_microbench<OP, 4><<<blocks, threads>>>(sink, it); break;
            default: k_microbench<OP, 8><<<blocks, threads>>>(sink, it); break;
        }
    };
    run(iters / 8 + 1);  // warm up
    cudaEventRecord(e0);
    run(iters);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    return (double)ms;
}
extern "C" {
double sa_microbench(int op, int ilp, int iters, int blocks, int threads) {
    fe *sink = nullptr;
    if (cudaMalloc(&sink, sizeof(fe) * (size_t)blocks * (threads > MK_THREADS ? threads : MK_THREADS)) != cudaSuccess)
        return -1.0;
    double ms = -1.0;
    switch (op) {
        case 0: ms = microbench_op<0>(ilp, iters, blocks, threads, sink); break;
        case 1: ms = microbench_op<1>(ilp, iters, blocks, threads, sink); break;
        case 2: ms = microbench_op<2>(ilp, iters, blocks, threads, sink); break;
        case 3: ms = microbench_op<3>(ilp, iters, blocks, threads, sink); break;
        case 4: ms = microbench_b2_ms(ilp, iters, blocks, (uint64_t *)sink); break;  // (merkle_fri.cu)
        case 5: ms = microbench_op<5>(ilp, iters, blocks, threads, sink); break;
    }
    g_launches.fetch_add(2);
    if (cudaGetLastError() != cudaSuccess) ms = -1.0;
    cudaFree(sink);
    return ms;
}

}  // extern "C"
