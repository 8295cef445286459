// poly.cu -- polynomial kernels: element-wise products, batch inversion, Horner evaluation, the
// direct zerofier and Lagrange kernels, the kernels of the subproduct tree (poly_tree.cuh) behind
// sa_zerofier, sa_interpolate and sa_poly_eval, and those of coset division plans, batched coset
// evaluation and coset combinations (coset.cuh), of transition quotients (air.cuh) and of boundary quotients
// (boundary.cuh) and of geometric interpolation plans and zerofiers (geo.cuh), with the backend that launches them for
// the headers' schedules.
//
// Reference behaviour reproduced (bit-exact): code/ntt.py:61-176, code/algebra.py:53-57,75-94.
#include <algorithm>

#include "air.cuh"
#include "boundary.cuh"
#include "coset.cuh"
#include "geo.cuh"
#include "ntt_tile.cuh"
#include "poly_tree.cuh"
#include "runtime.cuh"

using namespace sa;

// f(i) for every i < n, i = this thread's index, + the grid's thread count, ...
template <class F>
__device__ __forceinline__ void grid_stride(long long n, F f) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) f(i);
}
__device__ __forceinline__ long long thread_index() { return (long long)blockIdx.x * blockDim.x + threadIdx.x; }

__global__ void k_pointwise_mul(fe *out, const fe *a, const fe *b, long long n) {
    grid_stride(n, [&](long long i) { pointwise_mul_elem(out, a, b, i); });
}
// inv_m[i] = Montgomery form of 1/b[i] (the interpolation plan's 1/M'(d_i), the coset plan's 1/R_i): each thread
// runs batch_inverse_group on groups of 8 elements `stride` apart
__global__ void k_batch_inverse(fe *inv_m, const fe *b, long long n, int *zero_flag) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long base = thread_index(); base < n; base += stride * 8)
        batch_inverse_group(b, n, base, stride, zero_flag, [&](long long i, const fe &binv) { tile_st(inv_m + i, binv); });
}
// Horner, one thread per point
__global__ void k_poly_eval(fe *out, const fe *coeffs, long long ncoef, const fe *points, long long npts) {
    const long long j = thread_index();
    if (j >= npts) return;
    tile_st(out + j, poly_horner(coeffs, ncoef, tile_ld(points + j)));
}
// prod (X - d_i): one CTA, coefficients in shared memory, one sweep per domain point
constexpr int ZF_THREADS = 1024, ZF_MAXK = 4096, ZF_PER = (ZF_MAXK + 1 + ZF_THREADS - 1) / ZF_THREADS;
__global__ void __launch_bounds__(ZF_THREADS) k_zerofier(fe *out, const fe *domain, int k) {
    extern __shared__ uint4 sa_smem_u4[];
    fe *c = reinterpret_cast<fe *>(sa_smem_u4);
    fe *dm = c + (k + 1);
    const int tid = threadIdx.x;
    for (int j = tid; j <= k; j += ZF_THREADS) c[j] = (j == 0) ? fe_one() : fe_zero();
    for (int j = tid; j < k; j += ZF_THREADS) dm[j] = fe_to_mont(tile_ld(domain + j));
    __syncthreads();
    for (int i = 0; i < k; i++) {
        const fe d = dm[i];
        fe val[ZF_PER];
#pragma unroll
        for (int s = 0; s < ZF_PER; s++) {
            const int j = tid + s * ZF_THREADS;
            if (j <= i + 1) {  // new[j] = old[j-1] - d * old[j]
                const fe lower = j ? c[j - 1] : fe_zero();
                const fe cur = (j <= i) ? c[j] : fe_zero();
                val[s] = fe_sub(lower, fe_montmul(cur, d));
            }
        }
        __syncthreads();
#pragma unroll
        for (int s = 0; s < ZF_PER; s++) {
            const int j = tid + s * ZF_THREADS;
            if (j <= i + 1) c[j] = val[s];
        }
        __syncthreads();
    }
    for (int j = tid; j <= k; j += ZF_THREADS) tile_st(out + j, c[j]);
}
// Lagrange interpolation pieces.  q_i = z / (X - d_i) by synthetic division (descending m):
//   q_i[m-1] = z[m] + d_i * q_i[m];  D_i = q_i(d_i) = z'(d_i);  weight w_i = v_i / D_i
// dinv_m[i] = Montgomery form of 1/D_i (the plan's part: it depends on the domain only)
__global__ void k_interp_weights(fe *dinv_m, const fe *domain, const fe *z, int k, int *zero_flag) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= k) return;
    const fe d = fe_to_mont(tile_ld(domain + i));
    fe carry = fe_zero(), denom = fe_zero();
    for (int m = k; m > 0; m--) {
        carry = fe_add(tile_ldg(z + m), fe_montmul(carry, d));
        denom = fe_add(fe_montmul(denom, d), carry);
    }
    if (fe_is_zero(denom)) {
        *zero_flag = 1;
        denom = fe_one();
    }
    tile_st(dinv_m + i, fe_mont_inv(fe_to_mont(denom)));
}
// QT[m][i] = q_i[m] / D_i, the Lagrange basis polynomials' coefficients, in Montgomery form like the twiddles
// (coalesced over i; domain only)
__global__ void k_interp_rows(fe *QT, const fe *domain, const fe *dinv_m, const fe *z, int k) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= k) return;
    const fe d = fe_to_mont(tile_ld(domain + i)), w = fe_to_mont(tile_ld(dinv_m + i));
    fe carry = fe_zero();
    for (int m = k; m > 0; m--) {
        carry = fe_add(tile_ldg(z + m), fe_montmul(carry, d));
        tile_st(QT + (size_t)(m - 1) * k + i, fe_montmul(carry, w));
    }
}
__device__ __forceinline__ fe fe_shfl_down(const fe &x, int off) {
    fe y;
#pragma unroll
    for (int j = 0; j < 4; j++) y.v[j] = __shfl_down_sync(0xffffffffu, x.v[j], off);
    return y;
}
// out[b][m] = sum_i V[b][i] * QT[m][i], b < B, m < k: the Lagrange sums of B value vectors as one field matrix
// product.  A CTA owns IM_TB vectors x IM_TM coefficients and all its threads split the sum over i, so a single
// vector still spreads over k / IM_TM CTAs: each thread keeps IM_TB x IM_TM partial sums in registers (every V
// element it loads serves IM_TM products, every QT element IM_TB; QT is in Montgomery form, so a product is one
// fe_montmul), then the warps add theirs by shuffles and the CTA through shared memory.
constexpr int IM_TM = 2, IM_TB = 4, IM_THREADS = 256;
__global__ void __launch_bounds__(IM_THREADS) k_interp_matmul(fe *out, const fe *V, const fe *QT, int k, long long B) {
    __shared__ uint4 red_u4[IM_THREADS / 32][IM_TB * IM_TM];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long long b0 = (long long)blockIdx.x * IM_TB;
    const int m0 = blockIdx.y * IM_TM, nb = (int)(B - b0 < IM_TB ? B - b0 : IM_TB);
    fe acc[IM_TB][IM_TM];
#pragma unroll
    for (int r = 0; r < IM_TB; r++)
#pragma unroll
        for (int c = 0; c < IM_TM; c++) acc[r][c] = fe_zero();
    for (int i = tid; i < k; i += IM_THREADS) {
        fe q[IM_TM];
#pragma unroll
        for (int c = 0; c < IM_TM; c++) q[c] = (m0 + c < k) ? tile_ld(QT + (size_t)(m0 + c) * k + i) : fe_zero();
#pragma unroll
        for (int r = 0; r < IM_TB; r++) {
            if (r >= nb) break;
            const fe v = tile_ld(V + (b0 + r) * k + i);
#pragma unroll
            for (int c = 0; c < IM_TM; c++) acc[r][c] = fe_add(acc[r][c], fe_montmul(v, q[c]));
        }
    }
    fe *red = reinterpret_cast<fe *>(red_u4);
#pragma unroll
    for (int r = 0; r < IM_TB; r++) {
        if (r >= nb) break;
#pragma unroll
        for (int c = 0; c < IM_TM; c++) {
            fe s = acc[r][c];
#pragma unroll
            for (int off = 16; off >= 1; off >>= 1) s = fe_add(s, fe_shfl_down(s, off));
            if (lane == 0) red[warp * IM_TB * IM_TM + r * IM_TM + c] = s;
        }
    }
    __syncthreads();
    const int r = tid / IM_TM, m = m0 + tid % IM_TM;
    if (tid < IM_TB * IM_TM && r < nb && m < k) {
        fe s = red[tid];
        for (int w = 1; w < IM_THREADS / 32; w++) s = fe_add(s, red[w * IM_TB * IM_TM + tid]);
        tile_st(out + (b0 + r) * k + m, s);
    }
}

// ---- subproduct tree kernels: each runs its element function of poly_tree.cuh over its index range ----
__global__ void k_tree_leaves(fe *v0, const fe *domain, long long k, long long K) {
    if (const long long i = thread_index(); i < K) tree_leaves_elem(v0, domain, k, i);
}
__global__ void k_tree_pad(fe *dst, const fe *src, long long K, int mlog) {
    grid_stride(2 * K, [&](long long idx) { tree_pad_elem(dst, src, mlog, idx); });
}
__global__ void k_tree_pairmul(fe *out, const fe *in, long long K, int mlog) {
    grid_stride(K, [&](long long idx) { tree_pairmul_elem(out, in, mlog, idx); });
}
__global__ void k_tree_cross(fe *out, const fe *Pt, const fe *Vt, long long K, long long batch, int mlog) {
    grid_stride(batch * K, [&](long long idx) { tree_cross_elem(out, Pt, Vt, K, mlog, idx); });
}
__global__ void k_tree_fix(fe *parent, const fe *add, long long K, long long batch, int mlog, long long k) {
    grid_stride(batch * K / 2, [&](long long idx) { tree_fix_elem(parent, add, K, mlog, k, idx); });
}
__global__ void k_derivative(fe *out, const fe *z, long long k) {
    if (const long long i = thread_index(); i < k) derivative_elem(out, z, i);
}
__global__ void k_tree_qleaves(fe *P0, const fe *values, const fe *inv_m, long long k, int logK, long long batch) {
    if (const long long idx = thread_index(); idx < batch << logK) tree_qleaves_elem(P0, values, inv_m, k, logK, idx);
}
__global__ void k_tree_root(fe *out, const fe *root, long long k, long long K) {
    if (const long long i = thread_index(); i <= k) tree_root_elem(out, root, K, i);
}
__global__ void k_series_pad(fe *W, const fe *z, long long k, const fe *alpha, long long s) {
    grid_stride(8 * s, [&](long long idx) { series_pad_elem(W, z, k, alpha, s, idx); });
}
__global__ void k_series_step(fe *W, long long n4) {
    grid_stride(n4, [&](long long t) { series_step_elem(W, n4, t); });
}
__global__ void k_eval_top_pad(fe *W, const fe *f, long long nf, const fe *alpha, long long n, long long n2) {
    grid_stride(2 * n2, [&](long long idx) { eval_top_pad_elem(W, f, nf, alpha, n, n2, idx); });
}
__global__ void k_eval_root(fe *c, const fe *s, long long n, long long k, long long K) {
    if (const long long i = thread_index(); i < K) eval_root_elem(c, s, n, k, i);
}
__global__ void k_tree_down(fe *O, const fe *chat, const fe *VT, long long K, int mlog) {
    grid_stride(2 * K, [&](long long idx) { tree_down_elem(O, chat, VT, mlog, idx); });
}
__global__ void k_tree_down_fix(fe *next, const fe *O, const fe *cur, long long K, int mlog, long long k) {
    grid_stride(K, [&](long long idx) { tree_down_fix_elem(next, O, cur, mlog, k, idx); });
}

// ---- coset division and evaluation kernels: each runs its element function of coset.cuh over batch rows of n ----
__global__ void k_coset_load(fe *ws, const fe *lhs, const fe *pw_m, long long ncoef, int log_n, long long batch) {
    grid_stride(batch << log_n, [&](long long idx) { coset_load_elem(ws, lhs, pw_m, ncoef, log_n, idx); });
}
__global__ void k_coset_quot(fe *ws, const fe *inv_m, int log_n, long long batch) {
    grid_stride(batch << log_n, [&](long long idx) { coset_quot_elem(ws, inv_m, log_n, idx); });
}
__global__ void k_coset_store(fe *out, const fe *ws, const fe *ipw_m, long long qlen, int log_n, long long batch) {
    grid_stride(batch << log_n, [&](long long idx) { coset_store_elem(out, ws, ipw_m, qlen, log_n, idx); });
}
// one group of a combination's terms over all nrows * n outputs; the group is a kernel parameter, so the call uploads
// nothing
__global__ void k_coset_combine(fe *out, const __grid_constant__ CombineGroup g, const fe *pw_m, long long ncomb,
                                int log_n, long long nrows, int first) {
    grid_stride(nrows << log_n, [&](long long idx) { coset_combine_elem(out, g, pw_m, ncomb, first, log_n, idx); });
}
// the quotient values of nb constraint rows of a chunk of bp traces, one thread per point
__global__ void k_air_eval(fe *V, const fe *prog, const fe *x_m, const fe *iz_m, const fe *ext, long long r0,
                           long long nb, long long ncons, long long bp, int nregs, int log_n) {
    grid_stride(1ll << log_n,
                [&](long long i) { air_eval_rows_elem(V, prog, x_m, iz_m, ext, r0, nb, ncons, bp, nregs, log_n, i); });
}
// the boundary quotient codewords of batch registers in place, one thread per point
__global__ void k_boundary_point(fe *cw, const fe *ival, const fe *izinv_m, long long stride, int log_n,
                                 long long batch) {
    grid_stride(batch << log_n, [&](long long idx) { boundary_point_elem(cw, ival, izinv_m, stride, log_n, idx); });
}
// the quotient rows of batch registers and their remainder flags: every lane of a warp runs the same iterations (the
// range is rounded up to whole warps), so the ballot is over the full warp and each row a warp touches costs one
// atomicOr at most
__global__ void k_boundary_store(fe *quot, uint32_t *flags, const fe *ws, const fe *ipw_m, const fe *deg,
                                 long long ncoef, int log_n, long long batch) {
    grid_stride(((batch << log_n) + 31) & ~31ll, [&](long long idx) {
        const bool bad = boundary_store_elem(quot, ws, ipw_m, deg, ncoef, log_n, batch, idx);
        const uint32_t ballot = __ballot_sync(0xFFFFFFFFu, bad);
        if (bad && boundary_flag_leader(ballot, threadIdx.x & 31, log_n)) atomicOr(flags + (idx >> log_n), 1u);
    });
}
// the exact apply's store: k_coset_store's rows and their remainder flags, with k_boundary_store's warp ballot (the
// range rounded up to whole warps) and one atomicOr per row a warp touches at most
__global__ void k_air_store_exact(fe *out, uint32_t *flags, const fe *ws, const fe *ipw_m, long long qlen,
                                  long long tail, int log_n, long long batch) {
    grid_stride(((batch << log_n) + 31) & ~31ll, [&](long long idx) {
        const bool bad = air_store_exact_elem(out, ws, ipw_m, qlen, tail, log_n, batch, idx);
        const uint32_t ballot = __ballot_sync(0xFFFFFFFFu, bad);
        if (bad && boundary_flag_leader(ballot, threadIdx.x & 31, log_n)) atomicOr(flags + (idx >> log_n), 1u);
    });
}
// ---- geometric plans and zerofiers: each runs its element function of geo.cuh over its index range ----
__global__ void k_geo_scan_runs(fe *x, long long n, fe *tot) {
    grid_stride((n + GEO_SCAN_RUN - 1) / GEO_SCAN_RUN, [&](long long r) { geo_scan_run_elem(x, n, tot, r); });
}
__global__ void k_geo_scan_add(fe *x, long long n, const fe *tot) {
    grid_stride(n - GEO_SCAN_RUN, [&](long long idx) { geo_scan_add_elem(x, tot, idx); });
}
__global__ void k_geo_factor(fe *P, const fe *pw_m, long long count) {
    grid_stride(count, [&](long long m) { geo_factor_elem(P, pw_m, m); });
}
__global__ void k_geo_seed(fe *out, const fe *pw_m, long long n, long long len) {
    grid_stride(len, [&](long long t) { geo_seed_elem(out, pw_m, n, t); });
}
__global__ void k_geo_zerofier(fe *z, const fe *chirp_m, const fe *P_m, const fe *iP, long long k, int canon,
                               long long len) {
    grid_stride(len, [&](long long i) { geo_zerofier_elem(z, chirp_m, P_m, iP, k, canon, i); });
}
__global__ void k_geo_weight(fe *c, const fe *iP, long long k) {
    grid_stride(k, [&](long long i) { geo_weight_elem(c, iP, k, i); });
}
__global__ void k_geo_load(fe *ws, const fe *values, const fe *c_m, long long k, int logK, long long batch) {
    grid_stride(batch << logK, [&](long long idx) { geo_load_elem(ws, values, c_m, k, logK, idx); });
}
__global__ void k_geo_mid(fe *dst, const fe *src, const fe *ic_m, long long k, int logK, long long batch) {
    grid_stride(batch << logK, [&](long long idx) { geo_mid_elem(dst, src, ic_m, k, logK, idx); });
}

extern "C" {

int sa_pointwise_mul(void *out, const void *a, const void *b, size_t n, void *stream) {
    if (n == 0) return SA_OK;
    k_pointwise_mul<<<grid_for((long long)n, 256), 256, 0, (cudaStream_t)stream>>>((fe *)out, (const fe *)a,
                                                                                   (const fe *)b, (long long)n);
    SA_LAUNCH_CHECK();
    return SA_OK;
}

static int poly_eval_horner(void *out, const void *coeffs, size_t ncoef, const void *points, size_t npoints,
                            void *stream) {
    if (npoints == 0) return SA_OK;
    const int bs = 64;
    k_poly_eval<<<(unsigned)((npoints + bs - 1) / bs), bs, 0, (cudaStream_t)stream>>>(
        (fe *)out, (const fe *)coeffs, (long long)ncoef, (const fe *)points, (long long)npoints);
    SA_LAUNCH_CHECK();
    return SA_OK;
}

}  // extern "C"

// ---- the backend of the tree's and the coset schedules (poly_tree.cuh, coset.cuh): their kernels, sa_ntt and the
// copies, on one stream ----
static inline unsigned tree_grid(long long n) { return grid_for(n, 256, 8); }
static inline unsigned blocks256(long long n) { return (unsigned)((n + 255) / 256); }
// one method per kernel, launching it with its grid; the arguments are the kernel's
struct DeviceTree {
    using ll = long long;
    cudaStream_t st;
    template <int BS = 256, class... P, class... A>
    int go(void (*kernel)(P...), unsigned grid, A... args) {
        kernel<<<grid, BS, 0, st>>>(args...);
        SA_LAUNCH_CHECK();
        return SA_OK;
    }
    int leaves(fe *v, const fe *d, ll k, ll K) { return go(k_tree_leaves, blocks256(K), v, d, k, K); }
    int pad(fe *d, const fe *s, ll K, int j) { return go(k_tree_pad, tree_grid(2 * K), d, s, K, j); }
    int pairmul(fe *o, const fe *in, ll K, int j) { return go(k_tree_pairmul, tree_grid(K), o, in, K, j); }
    int cross(fe *o, const fe *P, const fe *V, ll K, ll nb, int j) {
        return go(k_tree_cross, tree_grid(nb * K), o, P, V, K, nb, j);
    }
    int fix(fe *p, const fe *a, ll K, ll nb, int j, ll k) {
        return go(k_tree_fix, tree_grid(nb * K / 2), p, a, K, nb, j, k);
    }
    int derivative(fe *o, const fe *z, ll k) { return go(k_derivative, blocks256(k), o, z, k); }
    int qleaves(fe *P, const fe *v, const fe *im, ll k, int lK, ll nb) {
        return go(k_tree_qleaves, blocks256(nb << lK), P, v, im, k, lK, nb);
    }
    int root(fe *o, const fe *r, ll k, ll K) { return go(k_tree_root, blocks256(k + 1), o, r, k, K); }
    int series_pad(fe *W, const fe *z, ll k, const fe *al, ll s) {
        return go(k_series_pad, tree_grid(8 * s), W, z, k, al, s);
    }
    int series_step(fe *W, ll n4) { return go(k_series_step, tree_grid(n4), W, n4); }
    int eval_top_pad(fe *W, const fe *f, ll nf, const fe *al, ll n, ll n2) {
        return go(k_eval_top_pad, tree_grid(2 * n2), W, f, nf, al, n, n2);
    }
    int pointwise_mul(fe *o, const fe *a, const fe *b, ll n) { return go(k_pointwise_mul, tree_grid(n), o, a, b, n); }
    int eval_root(fe *c, const fe *s, ll n, ll k, ll K) { return go(k_eval_root, blocks256(K), c, s, n, k, K); }
    int down(fe *O, const fe *ch, const fe *VT, ll K, int j) {
        return go(k_tree_down, tree_grid(2 * K), O, ch, VT, K, j);
    }
    int down_fix(fe *nx, const fe *O, const fe *cur, ll K, int j, ll k) {
        return go(k_tree_down_fix, tree_grid(K), nx, O, cur, K, j, k);
    }
    int batch_inverse(fe *im, const fe *b, ll n, int *flag) {
        return go<128>(k_batch_inverse, grid_for((n + 7) / 8, 128), im, b, n, flag);
    }
    int horner(fe *o, const fe *c, ll nc, const fe *x, ll nx) { return poly_eval_horner(o, c, nc, x, nx, st); }
    int pow_table(fe *o, const fe &base_m, ll count) { return launch_pow_table(o, base_m, fe_mont_one(), count, st); }
    int coset_load(fe *ws, const fe *l, const fe *pw, ll nc, int lg, ll nb) {
        return go(k_coset_load, tree_grid(nb << lg), ws, l, pw, nc, lg, nb);
    }
    int coset_quot(fe *ws, const fe *inv, int lg, ll nb) { return go(k_coset_quot, tree_grid(nb << lg), ws, inv, lg, nb); }
    int coset_store(fe *o, const fe *ws, const fe *ipw, ll q, int lg, ll nb) {
        return go(k_coset_store, tree_grid(nb << lg), o, ws, ipw, q, lg, nb);
    }
    int coset_combine(fe *o, const CombineGroup &g, const fe *pw, ll nc, int lg, ll nrows, int first) {
        return go(k_coset_combine, tree_grid(nrows << lg), o, g, pw, nc, lg, nrows, first);
    }
    int ntt(fe *o, const fe *i, int lg, const uint64_t *r, int inv, size_t nb) { return sa_ntt(o, i, lg, r, inv, nb, st); }
    int copy(fe *dst, const fe *src, size_t n) {
        SA_CUDA(cudaMemcpyAsync(dst, src, sizeof(fe) * n, cudaMemcpyDeviceToDevice, st));
        return SA_OK;
    }
    int copy2d(fe *dst, size_t dpitch, const fe *src, size_t spitch, size_t width, size_t rows) {
        SA_CUDA(cudaMemcpy2DAsync(dst, sizeof(fe) * dpitch, src, sizeof(fe) * spitch, sizeof(fe) * width, rows,
                                  cudaMemcpyDeviceToDevice, st));
        return SA_OK;
    }
    int store(fe *dst, const fe &v) {
        SA_CUDA(cudaMemcpyAsync(dst, &v, sizeof(fe), cudaMemcpyHostToDevice, st));
        return SA_OK;
    }
};
// DeviceTree plus the launches only the AIR schedules make (air.cuh)
struct DeviceAir : DeviceTree {
    int pow_table_lead(fe *o, const fe &base_m, const fe &lead_m, ll count) {
        return launch_pow_table(o, base_m, lead_m, count, st);
    }
    int upload(fe *dst, const fe *src, size_t n) {
        SA_CUDA(cudaMemcpyAsync(dst, src, sizeof(fe) * n, cudaMemcpyHostToDevice, st));
        return SA_OK;
    }
    int air_eval(fe *V, const fe *prog, const fe *x, const fe *iz, const fe *ext, ll r0, ll nb, ll ncons, ll bp,
                 int nregs, int lg) {
        return go(k_air_eval, tree_grid(1ll << lg), V, prog, x, iz, ext, r0, nb, ncons, bp, nregs, lg);
    }
};
// DeviceAir (its upload) plus the copies and launches only the boundary schedules make (boundary.cuh)
struct DeviceBoundary : DeviceAir {
    int download(fe *dst, const fe *src, size_t n) {
        SA_CUDA(cudaMemcpyAsync(dst, src, sizeof(fe) * n, cudaMemcpyDeviceToHost, st));
        return SA_OK;
    }
    int clear_flags(uint32_t *flags, size_t n) {
        SA_CUDA(cudaMemsetAsync(flags, 0, sizeof(uint32_t) * n, st));
        return SA_OK;
    }
    int boundary_point(fe *cw, const fe *iv, const fe *iz, ll stride, int lg, ll nb) {
        return go(k_boundary_point, tree_grid(nb << lg), cw, iv, iz, stride, lg, nb);
    }
    int boundary_store(fe *q, uint32_t *flags, const fe *ws, const fe *ipw, const fe *deg, ll nc, int lg, ll nb) {
        return go(k_boundary_store, tree_grid(nb << lg), q, flags, ws, ipw, deg, nc, lg, nb);
    }
};
// DeviceBoundary (its flags' memset) plus the store of the AIR's exact apply (air.cuh)
struct DeviceAirExact : DeviceBoundary {
    int air_store_exact(fe *o, uint32_t *flags, const fe *ws, const fe *ipw, ll q, ll tail, int lg, ll nb) {
        return go(k_air_store_exact, tree_grid(nb << lg), o, flags, ws, ipw, q, tail, lg, nb);
    }
};
// DeviceTree plus the launches of the geometric schedules (geo.cuh)
struct DeviceGeo : DeviceTree {
    int geo_scan_runs(fe *x, ll n, fe *tot) {
        return go(k_geo_scan_runs, tree_grid((n + GEO_SCAN_RUN - 1) / GEO_SCAN_RUN), x, n, tot);
    }
    int geo_scan_add(fe *x, ll n, const fe *tot) { return go(k_geo_scan_add, tree_grid(n - GEO_SCAN_RUN), x, n, tot); }
    int geo_factor(fe *P, const fe *pw, ll count) { return go(k_geo_factor, tree_grid(count), P, pw, count); }
    int geo_seed(fe *o, const fe *pw, ll n, ll len) { return go(k_geo_seed, tree_grid(len), o, pw, n, len); }
    int geo_zerofier(fe *z, const fe *ch, const fe *P, const fe *iP, ll k, int canon, ll len) {
        return go(k_geo_zerofier, tree_grid(len), z, ch, P, iP, k, canon, len);
    }
    int geo_weight(fe *c, const fe *iP, ll k) { return go(k_geo_weight, tree_grid(k), c, iP, k); }
    int geo_load(fe *ws, const fe *v, const fe *c, ll k, int lK, ll nb) {
        return go(k_geo_load, tree_grid(nb << lK), ws, v, c, k, lK, nb);
    }
    int geo_mid(fe *d, const fe *s, const fe *ic, ll k, int lK, ll nb) {
        return go(k_geo_mid, tree_grid(nb << lK), d, s, ic, k, lK, nb);
    }
};
static int tree_workspace(Tree &t, cudaStream_t st) {
    return get_workspace((void **)&t.ws, sizeof(fe) * t.elems, st, WS_TREE);
}

// Up to ZF_DIRECT_MAX points the one-CTA sweep kernel builds a zerofier, up to INTERP_DIRECT_MAX the k x k Lagrange
// kernels interpolate.  Horner (one thread per point, ncoef * npoints products) evaluates up to EVAL_TREE_MIN
// products, the transposed tree walk above: Horner's time grows with the product count, the walk's with k log^2 k
// plus a fixed launch ladder; tools/poly_sweep.py times both sides of the switch.
constexpr size_t ZF_DIRECT_MAX = 512;
constexpr double EVAL_TREE_MIN = 189812531.0;  // 2^27.5
static_assert(ZF_DIRECT_MAX <= ZF_MAXK && INTERP_DIRECT_MAX <= ZF_MAXK, "direct paths beyond the sweep kernel");

extern "C" {

int sa_zerofier(void *out, const void *domain, size_t k, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (k == 0) {  // the empty product (the drop-in answers Polynomial([]) before it gets here, ntt.py:70-71)
        const fe one = fe_one();
        SA_CUDA(cudaMemcpyAsync(out, &one, sizeof(fe), cudaMemcpyHostToDevice, st));
        SA_CUDA(cudaStreamSynchronize(st));
        return SA_OK;
    }
    if (k <= ZF_DIRECT_MAX) {
        const size_t smem = sizeof(fe) * (2 * k + 1);
        static std::atomic<bool> attr_done[SA_MAX_DEVICES];
        const int rc = optin_smem(k_zerofier, attr_done, sizeof(fe) * (2 * ZF_MAXK + 1));
        if (rc != SA_OK) return rc;
        k_zerofier<<<1, ZF_THREADS, smem, st>>>((fe *)out, (const fe *)domain, (int)k);
        SA_LAUNCH_CHECK();
        return SA_OK;
    }
    Tree t = tree_layout(k, TREE_ZEROFIER, 0);
    if (t.elems == 0) return SA_ESIZE;
    SA_TRY(tree_workspace(t, st));
    DeviceTree b{st};
    return tree_zerofier(b, t, (fe *)out, (const fe *)domain);
}

// the plan of the Lagrange kernels: domain, z and 1/z'(d_i)
static int interp_plan_direct(fe *plan, const InterpPlan &L, const fe *domain, size_t k, int *flag, cudaStream_t st) {
    fe *z = plan + L.sec[1];
    SA_CUDA(cudaMemcpyAsync(plan, domain, sizeof(fe) * k, cudaMemcpyDeviceToDevice, st));
    int rc = sa_zerofier(z, domain, k, (void *)st);
    if (rc != SA_OK) return rc;
    const int bs = 128, grid = (int)((k + bs - 1) / bs);
    k_interp_weights<<<grid, bs, 0, st>>>(plan + L.sec[2], domain, z, (int)k, flag);
    SA_LAUNCH_CHECK();
    return SA_OK;
}
// the tree's plan; M'(d_i) by the walk from 2^13.75 points (Horner is k^2 products)
static int interp_plan_device_tree(fe *plan, const InterpPlan &L, const fe *domain, size_t k, int *flag,
                                   cudaStream_t st) {
    const bool walk = (double)k * (double)k >= EVAL_TREE_MIN;
    Tree t = tree_layout(k, TREE_PLAN, walk ? k : 0);
    SA_TRY(tree_workspace(t, st));
    DeviceTree b{st};
    return interp_plan_tree(b, t, plan, L, domain, walk, flag);
}

size_t sa_interp_plan_bytes(size_t k) { return sizeof(fe) * interp_plan_layout(k).elems; }

int sa_interp_plan(void *plan, const void *domain, size_t k, void *stream) {
    const InterpPlan L = interp_plan_layout(k);
    if (L.elems == 0) return SA_ESIZE;
    cudaStream_t st = (cudaStream_t)stream;
    int *flag = nullptr;
    int rc = get_workspace((void **)&flag, 16, st, WS_PLAN_FLAG);
    if (rc != SA_OK) return rc;
    SA_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), st));
    rc = L.direct ? interp_plan_direct((fe *)plan, L, (const fe *)domain, k, flag, st)
                  : interp_plan_device_tree((fe *)plan, L, (const fe *)domain, k, flag, st);
    if (rc != SA_OK) return rc;
    int h = 0;
    SA_CUDA(cudaMemcpyAsync(&h, flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    SA_CUDA(cudaStreamSynchronize(st));
    return h ? SA_EDIVZERO : SA_OK;
}

size_t sa_interp_batch_max(size_t k) { return interp_batch_max(interp_plan_layout(k)); }

// Reads the plan only; its scratch is the stream's workspace (WS_INTERP_APPLY): Q' (k * k) for the Lagrange
// kernels, 4K per vector of a chunk above them (see interp_sweep).
int sa_interp_apply_batch(void *out, const void *plan, const void *values, size_t k, size_t batch, void *stream) {
    const InterpPlan L = interp_plan_layout(k);
    if (L.elems == 0) return SA_ESIZE;
    if (batch == 0) return SA_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const fe *p = (const fe *)plan, *v = (const fe *)values;
    fe *o = (fe *)out, *ws = nullptr;
    const size_t tree_ws = 4 * (size_t)L.K * std::min(batch, interp_batch_max(L));
    SA_TRY(get_workspace((void **)&ws, sizeof(fe) * (L.direct ? k * k : tree_ws), st, WS_INTERP_APPLY));
    if (L.direct) {  // Q'[m][i] = q_i[m] / z'(d_i) from the plan, then out = V Q'^T
        const int bs = 128, grid = (int)((k + bs - 1) / bs);
        k_interp_rows<<<grid, bs, 0, st>>>(ws, p, p + L.sec[2], p + L.sec[1], (int)k);
        SA_LAUNCH_CHECK();
        const dim3 mgrid((unsigned)((batch + IM_TB - 1) / IM_TB), (unsigned)((k + IM_TM - 1) / IM_TM));
        k_interp_matmul<<<mgrid, IM_THREADS, 0, st>>>(o, v, ws, (int)k, (long long)batch);
        SA_LAUNCH_CHECK();
        return SA_OK;
    }
    DeviceTree b{st};
    return interp_apply_tree(b, o, p, L, v, k, batch, ws);
}

int sa_interp_apply(void *out, const void *plan, const void *values, size_t k, void *stream) {
    return sa_interp_apply_batch(out, plan, values, k, 1, stream);
}

// plan (per-stream workspace WS_INTERP_PLAN) + apply: one implementation for the one-shot call and for plans
int sa_interpolate(void *out, const void *domain, const void *values, size_t k, void *stream) {
    if (k == 0) return SA_OK;
    const size_t bytes = sa_interp_plan_bytes(k);
    if (bytes == 0) return SA_ESIZE;
    void *plan = nullptr;
    int rc = get_workspace(&plan, bytes, (cudaStream_t)stream, WS_INTERP_PLAN);
    if (rc != SA_OK) return rc;
    if ((rc = sa_interp_plan(plan, domain, k, stream)) != SA_OK) return rc;
    return sa_interp_apply(out, plan, values, k, stream);
}

// fast_evaluate (ntt.py:82-100): Horner for small jobs, the transposed tree walk (tree_multipoint) for big ones
int sa_poly_eval_mode(void *out, const void *coeffs, size_t ncoef, const void *points, size_t npoints, int mode,
                      void *stream) {
    if (npoints == 0) return SA_OK;
    if (mode < 0 || mode > 2) return SA_ESIZE;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t nmax = ncoef > npoints ? ncoef : npoints;
    if (mode == 0)
        mode = (ncoef < 2 || npoints < 2 || (double)ncoef * (double)npoints < EVAL_TREE_MIN ||
                nmax > ((size_t)1 << TREE_MAX_LOG)) ? 1 : 2;
    if (mode == 1) return poly_eval_horner(out, coeffs, ncoef, points, npoints, stream);
    if (nmax > ((size_t)1 << TREE_MAX_LOG)) return SA_ESIZE;
    if (ncoef == 0) {  // the zero polynomial
        SA_CUDA(cudaMemsetAsync(out, 0, sizeof(fe) * npoints, st));
        return SA_OK;
    }
    Tree t = tree_layout(npoints, TREE_EVAL, ncoef);
    SA_TRY(tree_workspace(t, st));
    DeviceTree b{st};
    return tree_poly_eval(b, t, (fe *)out, (const fe *)coeffs, ncoef, (const fe *)points);
}
int sa_poly_eval(void *out, const void *coeffs, size_t ncoef, const void *points, size_t npoints, void *stream) {
    return sa_poly_eval_mode(out, coeffs, ncoef, points, npoints, 0, stream);
}

// ---- coset division plans and batched coset evaluation (coset.cuh) ----
size_t sa_coset_div_plan_bytes(int log_n) { return sizeof(fe) * coset_div_plan_layout(log_n).elems; }

size_t sa_coset_batch_max(int log_n) { return coset_batch_max(log_n); }

// scratch: the divisor's codeword (n elements, WS_COSET) and the zero flag (WS_PLAN_FLAG)
int sa_coset_div_plan(void *plan, const void *divisor, size_t dlen, int log_n, const uint64_t root[2],
                      const uint64_t offset[2], void *stream) {
    SA_TRY(coset_div_plan_check(log_n, dlen, root, offset));
    cudaStream_t st = (cudaStream_t)stream;
    int *flag = nullptr;
    fe *ws = nullptr;
    SA_TRY(get_workspace((void **)&flag, 16, st, WS_PLAN_FLAG));
    SA_TRY(get_workspace((void **)&ws, sizeof(fe) << log_n, st, WS_COSET));
    SA_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), st));
    DeviceTree b{st};
    SA_TRY(coset_div_plan_build(b, (fe *)plan, (const fe *)divisor, dlen, log_n, root, offset, ws, flag));
    int h = 0;
    SA_CUDA(cudaMemcpyAsync(&h, flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    SA_CUDA(cudaStreamSynchronize(st));
    return h ? SA_EDIVZERO : SA_OK;
}

// Reads the plan only; its scratch is the stream's workspace (WS_COSET): n elements per row of a chunk.
int sa_coset_div_apply_batch(void *out, const void *plan, const void *lhs, size_t ncoef, size_t qlen, int log_n,
                             const uint64_t root[2], size_t batch, void *stream) {
    SA_TRY(coset_check(log_n, ncoef, qlen, root));
    if (batch == 0) return SA_OK;
    cudaStream_t st = (cudaStream_t)stream;
    fe *ws = nullptr;
    const size_t chunk = std::min(batch, coset_batch_max(log_n));
    SA_TRY(get_workspace((void **)&ws, (sizeof(fe) << log_n) * chunk, st, WS_COSET));
    DeviceTree b{st};
    return coset_div_apply(b, (fe *)out, (const fe *)plan, (const fe *)lhs, ncoef, qlen, log_n, root, batch, ws);
}

// scratch: offset^i for i < ncoef (WS_COSET); the rows are transformed in out
int sa_coset_evaluate_batch(void *out, const void *coeffs, size_t ncoef, int log_n, const uint64_t root[2],
                            const uint64_t offset[2], size_t batch, void *stream) {
    SA_TRY(coset_check(log_n, ncoef, 1, root));
    if (batch == 0) return SA_OK;
    cudaStream_t st = (cudaStream_t)stream;
    fe *pw = nullptr;
    SA_TRY(get_workspace((void **)&pw, sizeof(fe) * ncoef, st, WS_COSET));
    DeviceTree b{st};
    return coset_evaluate(b, (fe *)out, (const fe *)coeffs, ncoef, log_n, root, offset, batch, pw);
}

// scratch: offset^i for i < ncomb (WS_COSET); the terms travel as kernel parameters and out is transformed in place
int sa_coset_combine_evaluate_batch(void *out, size_t nrows, int log_n, const uint64_t root[2],
                                    const uint64_t offset[2], const void *const *srcs, const size_t *lens,
                                    const size_t *shifts, const size_t *rows, const uint64_t *weights, size_t nterms,
                                    void *stream) {
    SA_TRY(coset_combine_check(log_n, lens, shifts, rows, nrows, nterms, root));
    if (nrows == 0) return SA_OK;
    cudaStream_t st = (cudaStream_t)stream;
    fe *pw = nullptr;
    const size_t ncomb = coset_combine_len(lens, shifts, nterms);
    if (ncomb) SA_TRY(get_workspace((void **)&pw, sizeof(fe) * ncomb, st, WS_COSET));
    DeviceTree b{st};
    return coset_combine_evaluate(b, (fe *)out, nrows, log_n, root, offset, (const fe *const *)srcs, lens, shifts,
                                  rows, weights, nterms, pw);
}

int sa_coset_combine_evaluate(void *out, int log_n, const uint64_t root[2], const uint64_t offset[2],
                              const void *const *srcs, const size_t *lens, const size_t *shifts,
                              const uint64_t *weights, size_t nterms, void *stream) {
    return sa_coset_combine_evaluate_batch(out, 1, log_n, root, offset, srcs, lens, shifts, nullptr, weights, nterms,
                                           stream);
}

// ---- transition quotients (air.cuh) ----
size_t sa_air_plan_bytes(int log_n, size_t max_ncoef, size_t nregs, size_t nterms) {
    return sizeof(fe) * air_plan_layout(log_n, max_ncoef, nregs, nterms).elems;
}

// scratch: the zerofier's codeword (n elements, WS_AIR) and the zero flag (WS_PLAN_FLAG); the compiled program is
// uploaded from host memory that outlives the closing synchronisation
int sa_air_plan(void *plan, const uint64_t *coeffs, const uint32_t *exps, const size_t *term_start, size_t ncons,
                size_t nregs, size_t max_ncoef, const void *zerofier, size_t zlen, int log_n, const uint64_t root[2],
                const uint64_t offset[2], const uint64_t step[2], void *stream) {
    SA_TRY(air_plan_check(log_n, exps, term_start, ncons, nregs, max_ncoef, zlen, root));
    const std::vector<fe> prog = air_compile(coeffs, exps, term_start, ncons, nregs);
    cudaStream_t st = (cudaStream_t)stream;
    int *flag = nullptr;
    fe *ws = nullptr;
    SA_TRY(get_workspace((void **)&flag, 16, st, WS_PLAN_FLAG));
    SA_TRY(get_workspace((void **)&ws, sizeof(fe) << log_n, st, WS_AIR));
    SA_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), st));
    DeviceAir b{{st}};
    SA_TRY(air_plan_build(b, (fe *)plan, prog, (const fe *)zerofier, zlen, log_n, root, offset, step, ws, flag));
    int h = 0;
    SA_CUDA(cudaMemcpyAsync(&h, flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    SA_CUDA(cudaStreamSynchronize(st));
    return h ? SA_EDIVZERO : SA_OK;
}

size_t sa_air_batch_max(size_t nregs, size_t ncons, int log_n) { return air_batch_max(nregs, ncons, log_n); }

// Reads the plan only; its scratch is the stream's workspace (WS_AIR): 2 nregs rows of n per trace of a chunk, and n
// per constraint row of a row chunk (air_chunks)
int sa_air_quotients_batch(void *out, const void *plan, const void *trace, size_t nregs, size_t ncoef, size_t qlen,
                           size_t ncons, size_t batch, int log_n, const uint64_t root[2], void *stream) {
    SA_TRY(air_apply_check(log_n, nregs, ncoef, qlen, ncons, root));
    if (batch == 0) return SA_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const AirChunks k = air_chunks(nregs, ncons, batch, log_n);
    fe *ws = nullptr;
    SA_TRY(get_workspace((void **)&ws, sizeof(fe) * air_ws_elems(nregs, k, log_n), st, WS_AIR));
    DeviceAir b{{st}};
    return air_quotients(b, (fe *)out, (const fe *)plan, (const fe *)trace, nregs, ncoef, qlen, ncons, batch, log_n,
                         root, ws, k);
}

int sa_air_quotients(void *out, const void *plan, const void *trace, size_t nregs, size_t ncoef, size_t qlen,
                     size_t ncons, int log_n, const uint64_t root[2], void *stream) {
    return sa_air_quotients_batch(out, plan, trace, nregs, ncoef, qlen, ncons, 1, log_n, root, stream);
}

// sa_air_quotients_batch plus the flags: the same workspace, one memset and the exact store in place of
// k_coset_store
int sa_air_quotients_exact_batch(void *out, uint32_t *flags, const void *plan, const void *trace, size_t nregs,
                                 size_t ncoef, size_t qlen, size_t ncons, size_t batch, size_t tail, int log_n,
                                 const uint64_t root[2], void *stream) {
    SA_TRY(air_exact_check(log_n, nregs, ncoef, qlen, ncons, tail, root));
    if (batch == 0) return SA_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const AirChunks k = air_chunks(nregs, ncons, batch, log_n);
    fe *ws = nullptr;
    SA_TRY(get_workspace((void **)&ws, sizeof(fe) * air_ws_elems(nregs, k, log_n), st, WS_AIR));
    DeviceAirExact b{{{{st}}}};
    return air_quotients_exact(b, (fe *)out, flags, (const fe *)plan, (const fe *)trace, nregs, ncoef, qlen, ncons,
                               batch, tail, log_n, root, ws, k);
}

int sa_air_quotients_exact(void *out, uint32_t *flags, const void *plan, const void *trace, size_t nregs,
                           size_t ncoef, size_t qlen, size_t ncons, size_t tail, int log_n, const uint64_t root[2],
                           void *stream) {
    return sa_air_quotients_exact_batch(out, flags, plan, trace, nregs, ncoef, qlen, ncons, 1, tail, log_n, root,
                                        stream);
}

// ---- boundary quotients (boundary.cuh) ----
size_t sa_boundary_plan_bytes(int log_n, size_t nregs) {
    return sizeof(fe) * boundary_plan_layout(log_n, nregs).elems;
}

// scratch: one register's zerofier codeword at a time (n elements, WS_COSET) and the zero flag (WS_PLAN_FLAG); the
// top coefficients and the degrees go through host memory that outlives the closing synchronisation
int sa_boundary_plan(void *plan, const void *const *zerofiers, const size_t *zlens, const void *const *interpolants,
                     const size_t *ilens, size_t nregs, int log_n, const uint64_t root[2], const uint64_t offset[2],
                     void *stream) {
    SA_TRY(boundary_plan_check(log_n, zlens, ilens, nregs, root, offset));
    cudaStream_t st = (cudaStream_t)stream;
    int *flag = nullptr;
    fe *ws = nullptr;
    SA_TRY(get_workspace((void **)&flag, 16, st, WS_PLAN_FLAG));
    SA_TRY(get_workspace((void **)&ws, sizeof(fe) << log_n, st, WS_COSET));
    SA_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), st));
    std::vector<fe> tops(nregs), degs(nregs);
    DeviceBoundary b{{{st}}};
    SA_TRY(boundary_plan_build(b, (fe *)plan, (const fe *const *)zerofiers, zlens, (const fe *const *)interpolants,
                               ilens, nregs, log_n, root, offset, ws, flag, tops.data(), degs.data()));
    int h = 0;
    SA_CUDA(cudaMemcpyAsync(&h, flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    SA_CUDA(cudaStreamSynchronize(st));
    return boundary_plan_verdict(tops.data(), nregs, h);
}

// Reads the plan only; its scratch is the stream's workspace (WS_COSET): n elements per register of a chunk
int sa_boundary_quotients(void *quot, void *codewords, uint32_t *flags, const void *plan, const void *trace,
                          size_t nregs, size_t ncoef, int log_n, const uint64_t root[2], void *stream) {
    SA_TRY(boundary_apply_check(log_n, nregs, ncoef, root));
    cudaStream_t st = (cudaStream_t)stream;
    fe *ws = nullptr;
    const size_t chunk = std::min(nregs, coset_batch_max(log_n));
    SA_TRY(get_workspace((void **)&ws, (sizeof(fe) << log_n) * chunk, st, WS_COSET));
    DeviceBoundary b{{{st}}};
    return boundary_quotients(b, (fe *)quot, (fe *)codewords, flags, (const fe *)plan, (const fe *)trace, nregs, ncoef,
                              log_n, root, ws);
}

// ---- geometric interpolation plans and zerofiers (geo.cuh) ----
size_t sa_geo_plan_bytes(size_t k) { return sizeof(fe) * geo_plan_layout(k).elems; }

size_t sa_geo_batch_max(size_t k) { return geo_batch_max(k); }

// scratch: the build's workspace (WS_GEO) and the zero flag (WS_PLAN_FLAG)
int sa_geo_plan(void *plan, const uint64_t step[2], size_t k, void *stream) {
    SA_TRY(geo_check(k, step));
    cudaStream_t st = (cudaStream_t)stream;
    int *flag = nullptr;
    fe *ws = nullptr;
    SA_TRY(get_workspace((void **)&flag, 16, st, WS_PLAN_FLAG));
    SA_TRY(get_workspace((void **)&ws, sizeof(fe) * geo_work_layout(k, geo_chirp_len(k, true)).elems, st, WS_GEO));
    SA_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), st));
    DeviceGeo b{{st}};
    SA_TRY(geo_plan_build(b, (fe *)plan, step, k, ws, flag));
    int h = 0;
    SA_CUDA(cudaMemcpyAsync(&h, flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    SA_CUDA(cudaStreamSynchronize(st));
    return h ? SA_EDIVZERO : SA_OK;
}

// Reads the plan only; its scratch is the stream's workspace (WS_INTERP_APPLY): 2K elements per vector of a chunk
int sa_geo_interp_batch(void *out, const void *plan, const void *values, size_t k, size_t batch, void *stream) {
    if (geo_plan_layout(k).elems == 0) return SA_ESIZE;
    if (batch == 0) return SA_OK;
    cudaStream_t st = (cudaStream_t)stream;
    fe *ws = nullptr;
    const size_t K = (size_t)geo_plan_layout(k).K, chunk = geo_batch_max(k);
    SA_TRY(get_workspace((void **)&ws, sizeof(fe) * 2 * K * std::min(batch, chunk), st, WS_INTERP_APPLY));
    DeviceGeo b{{st}};
    return geo_apply(b, (fe *)out, (const fe *)plan, (const fe *)values, k, batch, ws, chunk);
}

// scratch: the build's workspace and the chirp (WS_GEO) and the zero flag (WS_PLAN_FLAG); the flag is read before the
// coefficients are written, so an error leaves out untouched
int sa_geo_zerofier(void *out, const uint64_t step[2], size_t k, void *stream) {
    SA_TRY(geo_check(k, step));
    cudaStream_t st = (cudaStream_t)stream;
    int *flag = nullptr;
    fe *ws = nullptr;
    SA_TRY(get_workspace((void **)&flag, 16, st, WS_PLAN_FLAG));
    SA_TRY(get_workspace((void **)&ws, sizeof(fe) * (geo_work_layout(k, geo_chirp_len(k, false)).elems + k + 1), st,
                         WS_GEO));
    SA_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), st));
    DeviceGeo b{{st}};
    return geo_zerofier(b, (fe *)out, step, k, ws, flag, [&](int *f) -> int {
        int h = 0;
        SA_CUDA(cudaMemcpyAsync(&h, f, sizeof(int), cudaMemcpyDeviceToHost, st));
        SA_CUDA(cudaStreamSynchronize(st));
        return h ? SA_EDIVZERO : SA_OK;
    });
}

}  // extern "C"
