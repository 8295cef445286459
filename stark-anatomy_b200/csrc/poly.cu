// poly.cu -- polynomial kernels: element-wise products and quotients, scaling, Horner evaluation, the
// direct zerofier and Lagrange kernels, and the kernels of the subproduct tree (poly_tree.cuh) behind
// sa_zerofier, sa_interpolate and sa_poly_eval, with the backend that launches them for the tree's schedule.
//
// Reference behaviour reproduced (bit-exact): code/ntt.py:61-172, code/algebra.py:53-57,75-94.
#include <algorithm>

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
// batch_inverse_group over the grid: each thread takes groups of 8 elements `stride` apart
template <class Emit>
__device__ __forceinline__ void batch_inverse(const fe *b, long long n, int *zero_flag, Emit emit) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long base = thread_index(); base < n; base += stride * 8)
        batch_inverse_group(b, n, base, stride, zero_flag, emit);
}
// out = a / b
__global__ void k_pointwise_div(fe *out, const fe *a, const fe *b, long long n, int *zero_flag) {
    batch_inverse(b, n, zero_flag, [&](long long i, const fe &binv) { tile_st(out + i, fe_montmul(tile_ld(a + i), binv)); });
}
// inv_m[i] = Montgomery form of 1/b[i]: the interpolation plan's 1/M'(d_i)
__global__ void k_batch_inverse(fe *inv_m, const fe *b, long long n, int *zero_flag) {
    batch_inverse(b, n, zero_flag, [&](long long i, const fe &binv) { tile_st(inv_m + i, binv); });
}
// out[i] = in[i] * factor^i; thread handles i, i + T, i + 2T, ... with running factor^T
__global__ void k_scale(fe *out, const fe *in, long long n, fe factor_m, fe factor_T_m) {
    const long long T = (long long)gridDim.x * blockDim.x;
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fe f = fe_mont_pow_u64(factor_m, (uint64_t)i);
    for (; i < n; i += T) {
        tile_st(out + i, fe_montmul(tile_ld(in + i), f));
        f = fe_montmul(f, factor_T_m);
    }
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

extern "C" {

int sa_pointwise_mul(void *out, const void *a, const void *b, size_t n, void *stream) {
    if (n == 0) return SA_OK;
    k_pointwise_mul<<<grid_for((long long)n, 256), 256, 0, (cudaStream_t)stream>>>((fe *)out, (const fe *)a,
                                                                                   (const fe *)b, (long long)n);
    SA_LAUNCH_CHECK();
    return SA_OK;
}

int sa_pointwise_div(void *out, const void *a, const void *b, size_t n, void *stream) {
    if (n == 0) return SA_OK;
    cudaStream_t st = (cudaStream_t)stream;
    int *flag = nullptr;
    keep_pool_memory();
    SA_CUDA(cudaMallocAsync((void **)&flag, sizeof(int), st));
    SA_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), st));
    k_pointwise_div<<<grid_for(((long long)n + 7) / 8, 128), 128, 0, st>>>((fe *)out, (const fe *)a,
                                                                          (const fe *)b, (long long)n, flag);
    SA_LAUNCH_CHECK();
    int h = 0;
    SA_CUDA(cudaMemcpyAsync(&h, flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    SA_CUDA(cudaStreamSynchronize(st));
    cudaFreeAsync(flag, st);
    return h ? SA_EDIVZERO : SA_OK;
}

int sa_scale(void *out, const void *in, size_t n, const uint64_t factor[2], void *stream) {
    if (n == 0) return SA_OK;
    const int bs = 256;
    const unsigned grid = grid_for((long long)n, bs, 4);
    const fe f_m = fe_to_mont(fe_from_limbs(factor));
    const fe fT_m = fe_mont_pow_u64(f_m, (uint64_t)grid * bs);
    k_scale<<<grid, bs, 0, (cudaStream_t)stream>>>((fe *)out, (const fe *)in, (long long)n, f_m, fT_m);
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

// ---- the tree schedule's backend (poly_tree.cuh): its kernels, sa_ntt and the copies, on one stream ----
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

}  // extern "C"
