// poly.cu -- polynomial kernels: element-wise products and quotients, scaling, Horner evaluation, the
// direct zerofier and Lagrange kernels, and the subproduct tree behind sa_zerofier, sa_interpolate and
// sa_poly_eval.
//
// Reference behaviour reproduced (bit-exact): code/ntt.py:61-172, code/algebra.py:53-57,75-94.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <mutex>

#include "ntt_tile.cuh"
#include "runtime.cuh"

using namespace sa;

__global__ void k_pointwise_mul(fe *out, const fe *a, const fe *b, long long n) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        tile_st(out + i, fe_montmul(fe_to_mont(tile_ld(a + i)), tile_ld(b + i)));
}
// Montgomery's batch-inversion trick over 8 strided elements per thread (one Fermat inverse per 8 elements):
// emit(i, Montgomery form of 1/b[i]) for every i < n; a zero b[i] raises *zero_flag and is inverted as 1
template <class Emit>
__device__ __forceinline__ void batch_inverse(const fe *b, long long n, int *zero_flag, Emit emit) {
    constexpr int G = 8;
    const long long stride = (long long)gridDim.x * blockDim.x;
    const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (long long base = i0; base < n; base += stride * G) {
        fe bm[G], pre[G];
        fe acc = fe_mont_one();
#pragma unroll
        for (int g = 0; g < G; g++) {
            const long long i = base + g * stride;
            fe v = (i < n) ? tile_ld(b + i) : fe_one();
            if (fe_is_zero(v)) {
                *zero_flag = 1;
                v = fe_one();
            }
            bm[g] = fe_to_mont(v);
            pre[g] = acc;
            acc = fe_montmul(acc, bm[g]);
        }
        fe inv = fe_mont_inv(acc);
#pragma unroll
        for (int g = G - 1; g >= 0; g--) {
            const long long i = base + g * stride;
            const fe binv = fe_montmul(inv, pre[g]);
            inv = fe_montmul(inv, bm[g]);
            if (i < n) emit(i, binv);
        }
    }
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
// Horner, one thread per point (coefficients are read through the read-only path, broadcast)
__global__ void k_poly_eval(fe *out, const fe *coeffs, long long ncoef, const fe *points, long long npts) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= npts) return;
    const fe x_m = fe_to_mont(tile_ld(points + j));
    fe acc = fe_zero();
    for (long long i = ncoef - 1; i >= 0; i--) acc = fe_add(fe_montmul(acc, x_m), tile_ldg(coeffs + i));
    tile_st(out + j, acc);
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

// ---- subproduct tree over a domain of k points (fast_zerofier / fast_interpolate, ntt.py:66-130) ----
// The k points sit in the first k of K = 2^ceil(log2 k) leaf slots.  Level j has K >> j nodes of
// m = 2^j coefficients each, stored back to back.  A node whose leaf range lies completely inside the
// domain is FULL: its zerofier is monic of degree exactly m and only the low m coefficients are stored
// (the leading 1 is implied).  Any other node is stored EXPLICITLY (degree < m, all coefficients); a node
// without points is the constant 1.  With child vectors vL, vR a parent is
//     cyclic_product_2m(vL, vR) + x^m * ([L full] vR + [R full] vL)
// (the cyclic product of size 2m never wraps: both factors have degree < m), FULL iff both children are.
__device__ __forceinline__ bool tree_full(long long node, int mlog, long long k) { return ((node + 1) << mlog) <= k; }
__global__ void k_tree_leaves(fe *v0, const fe *domain, long long k, long long K) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < K) tile_st(v0 + i, i < k ? fe_neg(tile_ld(domain + i)) : fe_one());
}
// dst node (2m slots) = [src node (m coefficients), m zeros]
__global__ void k_tree_pad(fe *dst, const fe *src, long long K, int mlog) {
    const long long stride = (long long)gridDim.x * blockDim.x, m = 1ll << mlog;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < 2 * K; idx += stride) {
        const long long node = idx >> (mlog + 1), t = idx & (2 * m - 1);
        tile_st(dst + idx, t < m ? tile_ld(src + node * m + t) : fe_zero());
    }
}
// transformed children (blocks of 2m) -> transformed parents: out[p][t] = in[2p][t] * in[2p+1][t]
__global__ void k_tree_pairmul(fe *out, const fe *in, long long K, int mlog) {
    const long long stride = (long long)gridDim.x * blockDim.x, two_m = 2ll << mlog;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < K; idx += stride) {
        const long long p = idx >> (mlog + 1), t = idx & (two_m - 1);
        const fe a = tile_ld(in + (2 * p) * two_m + t), b = tile_ld(in + (2 * p + 1) * two_m + t);
        tile_st(out + idx, fe_montmul(fe_to_mont(a), b));
    }
}
// interpolation up-sweep of `batch` trees of K slots, back to back, over one tree's node transforms Vt (2K):
// out[p][t] = P[2p][t] * V[2p+1][t] + P[2p+1][t] * V[2p][t]
__global__ void k_tree_cross(fe *out, const fe *Pt, const fe *Vt, long long K, long long batch, int mlog) {
    const long long stride = (long long)gridDim.x * blockDim.x, two_m = 2ll << mlog;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < batch * K; idx += stride) {
        const long long p = idx >> (mlog + 1), t = idx & (two_m - 1);
        const long long l = (2 * p) * two_m + t, r = (2 * p + 1) * two_m + t;
        const fe a = fe_montmul(fe_to_mont(tile_ld(Pt + l)), tile_ld(Vt + (r & (2 * K - 1))));
        const fe b = fe_montmul(fe_to_mont(tile_ld(Pt + r)), tile_ld(Vt + (l & (2 * K - 1))));
        tile_st(out + idx, fe_add(a, b));
    }
}
// parent[p][m + t] += [L full] right[t] + [R full] left[t]; (left, right) = the child vectors of `add`
// (the zerofier tree adds the children's own vectors, the interpolation sweep the OTHER tree's: P_L * M_R
// picks up x^m * P_L when M_R is full, so `swap` exchanges the roles).  `batch` trees of K slots, back to back:
// a node is full by its index within its own tree.
__global__ void k_tree_fix(fe *parent, const fe *add, long long K, long long batch, int mlog, long long k, int swap) {
    const long long stride = (long long)gridDim.x * blockDim.x, m = 1ll << mlog;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < batch * K / 2; idx += stride) {
        const long long p = idx >> mlog, t = idx & (m - 1), left_node = (2 * p) & ((K >> mlog) - 1);
        const bool lfull = tree_full(left_node, mlog, k), rfull = tree_full(left_node + 1, mlog, k);
        if (!lfull && !rfull) continue;
        const fe left = tile_ld(add + (2 * p) * m + t), right = tile_ld(add + (2 * p + 1) * m + t);
        fe acc = tile_ld(parent + p * 2 * m + m + t);
        if (swap) {
            if (rfull) acc = fe_add(acc, left);
            if (lfull) acc = fe_add(acc, right);
        } else {
            if (lfull) acc = fe_add(acc, right);
            if (rfull) acc = fe_add(acc, left);
        }
        tile_st(parent + p * 2 * m + m + t, acc);
    }
}
// out[i] = (i + 1) * z[i + 1], i < k  (formal derivative of a polynomial with k + 1 coefficients)
__global__ void k_derivative(fe *out, const fe *z, long long k) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < k) tile_st(out + i, fe_montmul(fe_to_mont(fe_from_u64((uint64_t)(i + 1))), tile_ld(z + i + 1)));
}
// leaves of the interpolation sweep: q_i = v_i / M'(d_i) for i < k (inv_m = the plan's Montgomery 1/M'(d_i)),
// 0 for the empty slots; vector b (values + b * k) fills the K = 2^logK slots at P0 + b * K
__global__ void k_tree_qleaves(fe *P0, const fe *values, const fe *inv_m, long long k, int logK, long long batch) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= batch << logK) return;
    const long long b = idx >> logK, i = idx & ((1ll << logK) - 1);
    tile_st(P0 + idx, i < k ? fe_montmul(tile_ld(values + b * k + i), tile_ld(inv_m + i)) : fe_zero());
}
// zerofier coefficients from the tree's root vector: k == K -> implied leading 1
__global__ void k_tree_root(fe *out, const fe *root, long long k, long long K) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= k) tile_st(out + i, (i == K) ? fe_one() : tile_ld(root + i));
}

// ---- multi-point evaluation over the same tree (fast_evaluate, ntt.py:82-100, and M'(d_i) of fast_interpolate) ----
// The reference walks DOWN a remainder tree (f mod left zerofier, f mod right zerofier, ...).  Here the walk down is
// the TRANSPOSE of the interpolation up-sweep (Bostan-Lecerf-Schost): the up-sweep q -> P = sum q_i M / (X - d_i) is
// linear, rev(P) / rev(M) = sum q_i / (1 - d_i x) has the power sums sum_i q_i d_i^j as coefficients, i.e.
// (transposed Vandermonde) = (multiply by alpha = 1 / rev(M) mod x^n) o (reverse) o (up-sweep), so
//   f(d_i) = (up-sweep)^T [ (rev(f) * alpha mod x^n) shifted ],
// and the transposed up-sweep turns every product P_L * M_R into a CORRELATION with M_R: with the node transforms
// kept from the build, c_L = IDFT(DFT(c_node)[t] * DFT(M_R)[-t])[0..m) (+ c_node[m..2m) for the implied leading 1 of
// a full M_R), c_R likewise with M_L.  No division anywhere: one power-series inverse (Newton) at the top, then per
// level one batched forward transform, one pointwise kernel, one batched inverse transform, one fix-up.
// W (two blocks of 4s): [0] = rev_k(z) mod x^2s, zero padded; [1] = alpha mod x^s, zero padded.  z has k + 1 coefficients.
__global__ void k_series_pad(fe *W, const fe *z, long long k, const fe *alpha, long long s) {
    const long long stride = (long long)gridDim.x * blockDim.x, n4 = 4 * s;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < 2 * n4; idx += stride) {
        const long long t = idx & (n4 - 1);
        fe v = fe_zero();
        if (idx < n4) {
            if (t < 2 * s && t <= k) v = tile_ld(z + (k - t));
        } else if (t < s) {
            v = tile_ld(alpha + t);
        }
        tile_st(W + idx, v);
    }
}
// Newton step in the transform domain: W[0][t] = a * (2 - r * a), r = W[0][t], a = W[1][t]  (degree < 4s: no wrap)
__global__ void k_series_step(fe *W, long long n4) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    const fe two = fe_make(2, 0, 0, 0);
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n4; t += stride) {
        const fe r = tile_ld(W + t), a_m = fe_to_mont(tile_ld(W + n4 + t));
        const fe ra = fe_montmul(a_m, r);  // canonical r * a
        tile_st(W + t, fe_montmul(a_m, fe_sub(two, ra)));
    }
}
// W (two blocks of n2): [0] = rev_{n-1}(f) (f has nf <= n coefficients), [1] = alpha mod x^n, both zero padded
__global__ void k_eval_top_pad(fe *W, const fe *f, long long nf, const fe *alpha, long long n, long long n2) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < 2 * n2; idx += stride) {
        const long long t = idx & (n2 - 1);
        fe v = fe_zero();
        if (idx < n2) {
            if (t < n && n - 1 - t < nf) v = tile_ld(f + (n - 1 - t));
        } else if (t < n) {
            v = tile_ld(alpha + t);
        }
        tile_st(W + idx, v);
    }
}
// root vector of the walk down: c[i] = s[n - k + i] for i < k (s = rev(f) * alpha), 0 for the empty slots
__global__ void k_eval_root(fe *c, const fe *s, long long n, long long k, long long K) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < K) tile_st(c + i, i < k ? tile_ld(s + (n - k + i)) : fe_zero());
}
// O[child][t] = chat[parent][t] * VT[sibling][(2m - t) mod 2m]   (child blocks of 2m; VT = level-mlog transforms)
__global__ void k_tree_down(fe *O, const fe *chat, const fe *VT, long long K, int mlog) {
    const long long stride = (long long)gridDim.x * blockDim.x, two_m = 2ll << mlog;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < 2 * K; idx += stride) {
        const long long child = idx >> (mlog + 1), t = idx & (two_m - 1);
        const fe a = tile_ld(chat + (child >> 1) * two_m + t);
        const fe b = tile_ld(VT + (child ^ 1) * two_m + ((two_m - t) & (two_m - 1)));
        tile_st(O + idx, fe_montmul(fe_to_mont(a), b));
    }
}
// next[child][j] = O[child][j] + [sibling full] * cur[parent][m + j],  j < m
__global__ void k_tree_down_fix(fe *next, const fe *O, const fe *cur, long long K, int mlog, long long k) {
    const long long stride = (long long)gridDim.x * blockDim.x, m = 1ll << mlog;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < K; idx += stride) {
        const long long child = idx >> mlog, j = idx & (m - 1);
        fe v = tile_ld(O + child * 2 * m + j);
        if (tree_full(child ^ 1, mlog, k)) v = fe_add(v, tile_ld(cur + (child >> 1) * 2 * m + m + j));
        tile_st(next + idx, v);
    }
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

// ---- subproduct tree on the device (see the kernels above) ----
constexpr int TREE_MAX_LOG = 20;  // 2^20 points: ~1 GiB of tree, transforms and scratch
static int g_zf_direct_max = 512;       // up to here the one-CTA sweep kernel (SA_ZF_DIRECT_MAX with -DSA_TUNE)
static int g_interp_direct_max = 1024;  // up to here the k x k Lagrange kernels (SA_INTERP_DIRECT_MAX)
// Horner (one thread per point, ncoef * npoints products) up to this many products, the transposed tree walk above
// (SA_EVAL_TREE_MIN_LOG = log2 of the product count with -DSA_TUNE).  Horner's time grows with the product count,
// the walk's with k log^2 k plus a fixed launch ladder; tools/poly_sweep.py times both sides of the switch.
static double g_eval_tree_min = 189812531.0;  // 2^27.5
static void tree_config() {
#ifdef SA_TUNE
    static std::once_flag once;
    std::call_once(once, [] {
        if (const char *e = getenv("SA_ZF_DIRECT_MAX")) g_zf_direct_max = atoi(e);
        if (const char *e = getenv("SA_INTERP_DIRECT_MAX")) g_interp_direct_max = atoi(e);
        if (const char *e = getenv("SA_EVAL_TREE_MIN_LOG")) g_eval_tree_min = ldexp(1.0, atoi(e));
    });
#endif
}
// primitive 2^log-th root of unity: generator^(2^119 / 2^log), algebra.py:100-114
static void tree_root_of_unity(uint64_t out[2], int log) {
    // algebra.py:100-102: generator 85408008396924667383611388730472331217 has order 2^119; the table is built
    // once (a tree of 2^16 points asks ~60 times per call, each a chain of up to 118 host-side squarings)
    static uint64_t table[120][2];
    static std::once_flag once;
    std::call_once(once, [] {
        const uint64_t g[2] = {0xb5038f9c18f6f7d1ull, 0x4040fbed12ee470full};
        fe w = fe_to_mont(fe_from_limbs(g));
        for (int i = 119; i >= 0; i--) {
            const fe c = fe_from_mont(w);
            table[i][0] = (uint64_t)c.v[0] | ((uint64_t)c.v[1] << 32);
            table[i][1] = (uint64_t)c.v[2] | ((uint64_t)c.v[3] << 32);
            w = fe_montmul(w, w);
        }
    });
    out[0] = table[log][0];
    out[1] = table[log][1];
}
struct PolyTree {
    int logK = 0;
    long long k = 0, K = 0;
    fe *levels = nullptr;      // (logK + 1) * K: level j at levels + j * K
    fe *transforms = nullptr;  // logK * 2K: level j's node vectors zero-padded to 2m and transformed (or nullptr)
    fe *scratch = nullptr;     // 2K
};
static inline unsigned tree_grid(long long n) { return grid_for(n, 256, 8); }
// builds every level of the zerofier tree of domain[0..k) in `t` (buffers already assigned)
static int tree_build(PolyTree &t, const fe *domain, cudaStream_t st) {
    const long long K = t.K;
    int rc;
    k_tree_leaves<<<(unsigned)((K + 255) / 256), 256, 0, st>>>(t.levels, domain, t.k, K);
    SA_LAUNCH_CHECK();
    for (int j = 0; j < t.logK; j++) {
        uint64_t root[2];
        tree_root_of_unity(root, j + 1);
        fe *T = t.transforms ? t.transforms + (size_t)j * 2 * K : t.scratch;
        fe *child = t.levels + (size_t)j * K, *parent = t.levels + (size_t)(j + 1) * K;
        k_tree_pad<<<tree_grid(2 * K), 256, 0, st>>>(T, child, K, j);
        SA_LAUNCH_CHECK();
        if ((rc = sa_ntt(T, T, j + 1, root, 0, (size_t)(K >> j), st)) != SA_OK) return rc;
        k_tree_pairmul<<<tree_grid(K), 256, 0, st>>>(parent, T, K, j);
        SA_LAUNCH_CHECK();
        if ((rc = sa_ntt(parent, parent, j + 1, root, 1, (size_t)(K >> (j + 1)), st)) != SA_OK) return rc;
        k_tree_fix<<<tree_grid(K / 2), 256, 0, st>>>(parent, child, K, 1, j, t.k, 0);
        SA_LAUNCH_CHECK();
    }
    return SA_OK;
}
// keep_transforms: every level's node transforms stay (logK * 2K elements, read by the walk down and the up-sweep),
// in `transforms` when the caller gives a buffer (an interpolation plan), else in the workspace
static int tree_alloc(PolyTree &t, size_t k, bool keep_transforms, size_t extra_elems, fe **extra, cudaStream_t st,
                      fe *transforms = nullptr) {
    t.k = (long long)k;
    t.logK = 0;
    while ((size_t(1) << t.logK) < k) t.logK++;
    if (t.logK > TREE_MAX_LOG) return SA_ESIZE;
    t.K = 1ll << t.logK;
    const size_t K = (size_t)t.K;
    const bool in_ws = keep_transforms && !transforms;
    const size_t lv = (size_t)(t.logK + 1) * K, tr = in_ws ? (size_t)t.logK * 2 * K : 0, sc = 2 * K;
    fe *ws = nullptr;
    int rc = get_workspace((void **)&ws, sizeof(fe) * (lv + tr + sc + extra_elems), st, 8);
    if (rc != SA_OK) return rc;
    t.levels = ws;
    t.transforms = in_ws ? ws + lv : keep_transforms ? transforms : nullptr;
    t.scratch = ws + lv + tr;
    if (extra) *extra = ws + lv + tr + sc;
    return SA_OK;
}

static inline size_t pow2_ceil(size_t x) {
    size_t p = 1;
    while (p < x) p <<= 1;
    return p;
}
// elements of extra workspace tree_multipoint needs for nf coefficients at the tree's k points
static size_t multipoint_extra(size_t nf, size_t k) {
    const size_t N = pow2_ceil(nf > k ? nf : k), K = pow2_ceil(k);
    return 4 * N + N + 2 * K + 16;
}
// vals[i] = f(d_i), i < k, for the tree `t` (built with transforms kept) whose root polynomial is z (k + 1
// coefficients); f has nf >= 1 coefficients.  `ws` = multipoint_extra(nf, k) elements.  See the kernels' comment.
static int tree_multipoint(const PolyTree &t, const fe *z, const fe *f, size_t nf, fe *vals, fe *ws, cudaStream_t st) {
    const long long k = t.k, K = t.K;
    const long long n = (long long)(nf > (size_t)k ? nf : (size_t)k), N = (long long)pow2_ceil((size_t)n);
    fe *W = ws, *alpha = W + 4 * N, *c0 = alpha + N, *c1 = c0 + K;
    int rc;
    uint64_t root[2];
    // alpha = 1 / rev_k(z) mod x^N by Newton: alpha_2s = alpha_s (2 - r alpha_s) mod x^2s in transforms of size 4s
    const fe one = fe_one();
    SA_CUDA(cudaMemcpyAsync(alpha, &one, sizeof(fe), cudaMemcpyHostToDevice, st));
    for (long long s = 1; s < N; s <<= 1) {
        const int lg = host_log2((size_t)(4 * s));
        tree_root_of_unity(root, lg);
        k_series_pad<<<tree_grid(8 * s), 256, 0, st>>>(W, z, k, alpha, s);
        SA_LAUNCH_CHECK();
        if ((rc = sa_ntt(W, W, lg, root, 0, 2, st)) != SA_OK) return rc;
        k_series_step<<<tree_grid(4 * s), 256, 0, st>>>(W, 4 * s);
        SA_LAUNCH_CHECK();
        if ((rc = sa_ntt(W, W, lg, root, 1, 1, st)) != SA_OK) return rc;
        SA_CUDA(cudaMemcpyAsync(alpha, W, sizeof(fe) * 2 * s, cudaMemcpyDeviceToDevice, st));
    }
    // s = rev_{n-1}(f) * alpha mod x^n; the walk starts from c_root[i] = s[n - k + i]
    {
        const long long n2 = 2 * N;
        const int lg = host_log2((size_t)n2);
        tree_root_of_unity(root, lg);
        k_eval_top_pad<<<tree_grid(2 * n2), 256, 0, st>>>(W, f, (long long)nf, alpha, n, n2);
        SA_LAUNCH_CHECK();
        if ((rc = sa_ntt(W, W, lg, root, 0, 2, st)) != SA_OK) return rc;
        k_pointwise_mul<<<tree_grid(n2), 256, 0, st>>>(W, W, W + n2, n2);
        SA_LAUNCH_CHECK();
        if ((rc = sa_ntt(W, W, lg, root, 1, 1, st)) != SA_OK) return rc;
        k_eval_root<<<(unsigned)((K + 255) / 256), 256, 0, st>>>(c0, W, n, k, K);
        SA_LAUNCH_CHECK();
    }
    // walk down: level j + 1 (nodes of 2m) -> level j (nodes of m); W is free again: chat = W[0, K), O = W[K, 3K)
    fe *cur = c0, *nxt = c1, *chat = W, *O = W + K;
    for (int j = t.logK - 1; j >= 0; j--) {
        tree_root_of_unity(root, j + 1);
        const fe *VT = t.transforms + (size_t)j * 2 * K;
        if ((rc = sa_ntt(chat, cur, j + 1, root, 0, (size_t)(K >> (j + 1)), st)) != SA_OK) return rc;
        k_tree_down<<<tree_grid(2 * K), 256, 0, st>>>(O, chat, VT, K, j);
        SA_LAUNCH_CHECK();
        if ((rc = sa_ntt(O, O, j + 1, root, 1, (size_t)(K >> j), st)) != SA_OK) return rc;
        k_tree_down_fix<<<tree_grid(K), 256, 0, st>>>(nxt, O, cur, K, j, k);
        SA_LAUNCH_CHECK();
        fe *tmp = cur;
        cur = nxt;
        nxt = tmp;
    }
    SA_CUDA(cudaMemcpyAsync(vals, cur, sizeof(fe) * (size_t)k, cudaMemcpyDeviceToDevice, st));
    return SA_OK;
}

extern "C" {

int sa_zerofier(void *out, const void *domain, size_t k, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    tree_config();
    if (k == 0) {  // the empty product (the drop-in answers Polynomial([]) before it gets here, ntt.py:70-71)
        const fe one = fe_one();
        SA_CUDA(cudaMemcpyAsync(out, &one, sizeof(fe), cudaMemcpyHostToDevice, st));
        SA_CUDA(cudaStreamSynchronize(st));
        return SA_OK;
    }
    if (k <= (size_t)g_zf_direct_max && k <= (size_t)ZF_MAXK) {
        const size_t smem = sizeof(fe) * (2 * k + 1);
        static std::atomic<bool> attr_done[SA_MAX_DEVICES];
        const int rc = optin_smem(k_zerofier, attr_done, sizeof(fe) * (2 * ZF_MAXK + 1));
        if (rc != SA_OK) return rc;
        k_zerofier<<<1, ZF_THREADS, smem, st>>>((fe *)out, (const fe *)domain, (int)k);
        SA_LAUNCH_CHECK();
        return SA_OK;
    }
    PolyTree t;
    int rc = tree_alloc(t, k, false, 0, nullptr, st);
    if (rc != SA_OK) return rc;
    if ((rc = tree_build(t, (const fe *)domain, st)) != SA_OK) return rc;
    k_tree_root<<<(unsigned)((k + 1 + 255) / 256), 256, 0, st>>>((fe *)out, t.levels + (size_t)t.logK * t.K, t.k, t.K);
    SA_LAUNCH_CHECK();
    return SA_OK;
}

// ---- interpolation plans: the half of fast_interpolate (ntt.py:102-130) that depends on the domain alone ----
// A plan is a device buffer of sa_interp_plan_bytes(k) bytes, laid out by k alone.  Every section starts on a
// 256-byte (16-element) boundary, i.e. each section's length is rounded up to a multiple of 16 elements:
//   k <= g_interp_direct_max (the k x k Lagrange kernels):  domain (k) | z = prod (X - d_i) (k + 1) | 1/z'(d_i) (k)
//   above (the subproduct tree):  node transforms of levels 0 .. log K - 1, as tree_build keeps them (log K * 2K)
//                                 | 1/M'(d_i) (K; the first k are written)
// The inverses are in Montgomery form, so one product per point gives v_i / M'(d_i).  The tree's levels and z stay
// in the build's workspace: the up-sweep reads the node transforms only.  2^20 points: 41 * 2^20 elements, 656 MiB.
struct InterpPlan {
    bool direct = false;
    int logK = 0;
    long long K = 0;
    size_t sec[3] = {0, 0, 0};  // element offsets: domain, z, 1/z'  |  transforms, 1/M'
    size_t elems = 0;           // 0: no plan for this k
};
static inline size_t plan_section(size_t elems) { return (elems + 15) & ~(size_t)15; }
static InterpPlan interp_plan_layout(size_t k) {
    InterpPlan L;
    tree_config();
    if (k == 0 || k > ((size_t)1 << TREE_MAX_LOG)) return L;
    L.direct = k <= (size_t)g_interp_direct_max && k <= (size_t)ZF_MAXK;
    if (L.direct) {
        L.sec[1] = plan_section(k);
        L.sec[2] = L.sec[1] + plan_section(k + 1);
        L.elems = L.sec[2] + plan_section(k);
    } else {
        L.logK = host_log2(k);
        L.K = 1ll << L.logK;
        L.sec[1] = plan_section((size_t)L.logK * 2 * (size_t)L.K);
        L.elems = L.sec[1] + plan_section((size_t)L.K);
    }
    return L;
}
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
// M = prod (X - d_i) by the tree (its node transforms go into the plan), M'(d_i) from one Horner kernel (k^2 / 2
// multiply-adds, all points in parallel) or, from 2^13.75 points, the walk down the tree, then one batch inversion;
// coinciding points give M'(d_i) = 0 -> the zero flag (SA_EDIVZERO like the division at ntt.py:124-125)
static int interp_plan_tree(fe *plan, const InterpPlan &L, const fe *domain, size_t k, int *flag, cudaStream_t st) {
    PolyTree t;
    fe *extra = nullptr;
    const size_t K = (size_t)L.K;
    const bool walk = (double)k * (double)k >= g_eval_tree_min;  // M'(d_i): Horner is k^2 products
    // extra: z (K + 1) | dz (K) | ev (K) | the walk's workspace
    int rc = tree_alloc(t, k, true, 3 * K + 1 + (walk ? multipoint_extra(k, k) : 0), &extra, st, plan + L.sec[0]);
    if (rc != SA_OK) return rc;
    fe *z = extra, *dz = z + K + 1, *ev = dz + K, *mp = ev + K;
    if ((rc = tree_build(t, domain, st)) != SA_OK) return rc;
    k_tree_root<<<(unsigned)((k + 1 + 255) / 256), 256, 0, st>>>(z, t.levels + (size_t)t.logK * K, t.k, t.K);
    SA_LAUNCH_CHECK();
    k_derivative<<<(unsigned)((k + 255) / 256), 256, 0, st>>>(dz, z, (long long)k);
    SA_LAUNCH_CHECK();
    if (walk)
        rc = tree_multipoint(t, z, dz, k, ev, mp, st);
    else
        rc = poly_eval_horner(ev, dz, k, domain, k, (void *)st);
    if (rc != SA_OK) return rc;
    k_batch_inverse<<<grid_for(((long long)k + 7) / 8, 128), 128, 0, st>>>(plan + L.sec[1], ev, (long long)k, flag);
    SA_LAUNCH_CHECK();
    return SA_OK;
}

size_t sa_interp_plan_bytes(size_t k) { return sizeof(fe) * interp_plan_layout(k).elems; }

int sa_interp_plan(void *plan, const void *domain, size_t k, void *stream) {
    const InterpPlan L = interp_plan_layout(k);
    if (L.elems == 0) return SA_ESIZE;
    cudaStream_t st = (cudaStream_t)stream;
    int *flag = nullptr;
    int rc = get_workspace((void **)&flag, 16, st, 7);
    if (rc != SA_OK) return rc;
    SA_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), st));
    rc = L.direct ? interp_plan_direct((fe *)plan, L, (const fe *)domain, k, flag, st)
                  : interp_plan_tree((fe *)plan, L, (const fe *)domain, k, flag, st);
    if (rc != SA_OK) return rc;
    int h = 0;
    SA_CUDA(cudaMemcpyAsync(&h, flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    SA_CUDA(cudaStreamSynchronize(st));
    return h ? SA_EDIVZERO : SA_OK;
}

// Above the Lagrange kernels a batched apply needs 4K elements of its own workspace (tag 10) and 2K of the NTT's
// inter-pass intermediate (tag 0) per vector: 96K bytes.  It runs in chunks that keep both at or below 1 GiB.
constexpr size_t INTERP_CHUNK_BYTES = (size_t)1 << 30;
size_t sa_interp_batch_max(size_t k) {
    const InterpPlan L = interp_plan_layout(k);
    if (L.elems == 0) return 0;
    if (L.direct) return SIZE_MAX;
    const size_t b = INTERP_CHUNK_BYTES / (sizeof(fe) * 6 * (size_t)L.K);
    return b ? b : 1;
}

// the interpolants sum_i q_i M / (X - d_i), q_i = v_i / M'(d_i), of nb value vectors, combined bottom-up over the
// plan's tree: P_node = P_L * M_R + P_R * M_L.  Every level is one batch over the nodes of all nb trees, so the
// launches do not depend on nb.  ws = 4K * nb elements: transform scratch [nb][2K], P ping-pong 2 x [nb][K].
static int interp_sweep(fe *out, const fe *p, const InterpPlan &L, const fe *v, size_t k, size_t nb, fe *ws,
                        cudaStream_t st) {
    const size_t K = (size_t)L.K;
    const long long n = (long long)(nb * K);
    fe *scratch = ws, *cur = ws + 2 * K * nb, *nxt = cur + K * nb;
    int rc;
    k_tree_qleaves<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(cur, v, p + L.sec[1], (long long)k, L.logK,
                                                                (long long)nb);
    SA_LAUNCH_CHECK();
    for (int j = 0; j < L.logK; j++) {
        uint64_t root[2];
        tree_root_of_unity(root, j + 1);
        const fe *VT = p + L.sec[0] + (size_t)j * 2 * K;
        k_tree_pad<<<tree_grid(2 * n), 256, 0, st>>>(scratch, cur, n, j);
        SA_LAUNCH_CHECK();
        if ((rc = sa_ntt(scratch, scratch, j + 1, root, 0, nb * (K >> j), (void *)st)) != SA_OK) return rc;
        k_tree_cross<<<tree_grid(n), 256, 0, st>>>(nxt, scratch, VT, L.K, (long long)nb, j);
        SA_LAUNCH_CHECK();
        if ((rc = sa_ntt(nxt, nxt, j + 1, root, 1, nb * (K >> (j + 1)), (void *)st)) != SA_OK) return rc;
        k_tree_fix<<<tree_grid(n / 2), 256, 0, st>>>(nxt, cur, L.K, (long long)nb, j, (long long)k, 1);
        SA_LAUNCH_CHECK();
        fe *tmp = cur;
        cur = nxt;
        nxt = tmp;
    }
    SA_CUDA(cudaMemcpy2DAsync(out, sizeof(fe) * k, cur, sizeof(fe) * K, sizeof(fe) * k, nb, cudaMemcpyDeviceToDevice,
                              st));
    return SA_OK;
}

// Reads the plan only; its scratch is the stream's workspace (tag 10): Q' (k * k) for the Lagrange kernels, 4K per
// vector of a chunk above them (see interp_sweep).
int sa_interp_apply_batch(void *out, const void *plan, const void *values, size_t k, size_t batch, void *stream) {
    const InterpPlan L = interp_plan_layout(k);
    if (L.elems == 0) return SA_ESIZE;
    if (batch == 0) return SA_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const fe *p = (const fe *)plan, *v = (const fe *)values;
    fe *o = (fe *)out, *ws = nullptr;
    const size_t chunk = L.direct ? batch : std::min(batch, sa_interp_batch_max(k));
    int rc = get_workspace((void **)&ws, sizeof(fe) * (L.direct ? k * k : 4 * (size_t)L.K * chunk), st, 10);
    if (rc != SA_OK) return rc;
    if (L.direct) {  // Q'[m][i] = q_i[m] / z'(d_i) from the plan, then out = V Q'^T
        const int bs = 128, grid = (int)((k + bs - 1) / bs);
        k_interp_rows<<<grid, bs, 0, st>>>(ws, p, p + L.sec[2], p + L.sec[1], (int)k);
        SA_LAUNCH_CHECK();
        const dim3 mgrid((unsigned)((batch + IM_TB - 1) / IM_TB), (unsigned)((k + IM_TM - 1) / IM_TM));
        k_interp_matmul<<<mgrid, IM_THREADS, 0, st>>>(o, v, ws, (int)k, (long long)batch);
        SA_LAUNCH_CHECK();
        return SA_OK;
    }
    for (size_t b0 = 0; b0 < batch; b0 += chunk)
        if ((rc = interp_sweep(o + b0 * k, p, L, v + b0 * k, k, std::min(chunk, batch - b0), ws, st)) != SA_OK)
            return rc;
    return SA_OK;
}

int sa_interp_apply(void *out, const void *plan, const void *values, size_t k, void *stream) {
    return sa_interp_apply_batch(out, plan, values, k, 1, stream);
}

// plan (per-stream workspace, tag 9) + apply: one implementation for the one-shot call and for plans
int sa_interpolate(void *out, const void *domain, const void *values, size_t k, void *stream) {
    if (k == 0) return SA_OK;
    const size_t bytes = sa_interp_plan_bytes(k);
    if (bytes == 0) return SA_ESIZE;
    void *plan = nullptr;
    int rc = get_workspace(&plan, bytes, (cudaStream_t)stream, 9);
    if (rc != SA_OK) return rc;
    if ((rc = sa_interp_plan(plan, domain, k, stream)) != SA_OK) return rc;
    return sa_interp_apply(out, plan, values, k, stream);
}

// fast_evaluate (ntt.py:82-100): Horner for small jobs, the transposed tree walk (tree_multipoint) for big ones
int sa_poly_eval_mode(void *out, const void *coeffs, size_t ncoef, const void *points, size_t npoints, int mode,
                      void *stream) {
    if (npoints == 0) return SA_OK;
    if (mode < 0 || mode > 2) return SA_ESIZE;
    tree_config();
    cudaStream_t st = (cudaStream_t)stream;
    const size_t nmax = ncoef > npoints ? ncoef : npoints;
    if (mode == 0)
        mode = (ncoef < 2 || npoints < 2 || (double)ncoef * (double)npoints < g_eval_tree_min ||
                nmax > ((size_t)1 << TREE_MAX_LOG)) ? 1 : 2;
    if (mode == 1) return poly_eval_horner(out, coeffs, ncoef, points, npoints, stream);
    if (nmax > ((size_t)1 << TREE_MAX_LOG)) return SA_ESIZE;
    if (ncoef == 0) {  // the zero polynomial
        SA_CUDA(cudaMemsetAsync(out, 0, sizeof(fe) * npoints, st));
        return SA_OK;
    }
    PolyTree t;
    fe *extra = nullptr;
    const size_t K = pow2_ceil(npoints);
    int rc = tree_alloc(t, npoints, true, K + 1 + 16 + multipoint_extra(ncoef, npoints), &extra, st);
    if (rc != SA_OK) return rc;
    fe *z = extra, *mp = z + K + 1 + 15;
    if ((rc = tree_build(t, (const fe *)points, st)) != SA_OK) return rc;
    k_tree_root<<<(unsigned)((npoints + 1 + 255) / 256), 256, 0, st>>>(z, t.levels + (size_t)t.logK * t.K, t.k, t.K);
    SA_LAUNCH_CHECK();
    return tree_multipoint(t, z, (const fe *)coeffs, ncoef, (fe *)out, mp, st);
}
int sa_poly_eval(void *out, const void *coeffs, size_t ncoef, const void *points, size_t npoints, void *stream) {
    return sa_poly_eval_mode(out, coeffs, ncoef, points, npoints, 0, stream);
}

}  // extern "C"
