/*
 * sa_b200.h -- C ABI of the H100 (sm_90a) NTT + FRI engine that stands in for the
 * hot path of aszepieniec/stark-anatomy (code/ntt.py, code/fri.py, code/merkle.py).
 *
 * The reference is pure Python and has no FFI: its boundary is the Python module
 * surface (SURVEY.md section 8b).  The entry points below are what a ctypes
 * binding for that path binds; stark-anatomy_b200/sa_engine.py is that binding
 * and INTEGRATION.md shows the stub a maintainer would add to the reference.
 *
 * Conventions
 *  - One field element = 16 bytes: two little-endian uint64 limbs (lo, hi) of the
 *    canonical residue in [0, p), p = 1 + 407 * 2^119 (code/algebra.py:96-98).
 *  - Scalars (roots, offsets, challenges) are passed as `const uint64_t x[2]`.
 *  - `void *` data pointers are DEVICE pointers unless the function name ends in
 *    `_host`; `stream` is a cudaStream_t (NULL = default stream).  Calls are
 *    asynchronous on `stream` unless stated otherwise.
 *  - Return value: 0 on success, otherwise one of the SA_E* codes; the Python
 *    binding turns SA_E* into the AssertionError (with the reference's message)
 *    the corresponding reference function raises.
 *  - No torch types, no C++ types: plain pointers and sizes.
 *  - Thread safety: entry points may be called from several host threads; the
 *    twiddle/plan caches are guarded by a mutex (tables are built outside of it).  Work submitted to different
 *    streams is independent (scratch buffers and the Merkle arrival counter are per
 *    device and stream); two threads must not be inside calls on the SAME stream at
 *    the same time.  sa_ntt_host calls on one device run one after the other
 *    (they share the copy streams - and the PCIe link).
 */
#ifndef SA_B200_H
#define SA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
    SA_OK = 0,
    SA_ENOTPOW2 = -1,   /* ntt.py:4   "cannot compute ntt of non-power-of-two sequence" */
    SA_EROOTORDER = -2, /* ntt.py:10  "primitive root must be nth root of unity, where n is len(values)" */
    SA_ENOTPRIM = -3,   /* ntt.py:11  "primitive root is not primitive nth root of unity, ..." */
    SA_EDIVZERO = -4,   /* algebra.py:92 "divide by zero" (element-wise division, ntt.py:172) */
    SA_EINDEX = -5,     /* merkle.py:18 "cannot open invalid index" */
    SA_ESIZE = -6,      /* unsupported size (log_n > 30, n == 0, ...) */
    SA_ECALLBACK = -7,  /* the challenge callback of sa_fri_commit returned non-zero */
    SA_ECUDA = -100     /* CUDA runtime error; sa_last_error() has the text */
};

/* Version / build info, e.g. "sa_b200 0.1 sm_90a". */
const char *sa_version(void);
/* Text of the last CUDA error seen by this thread's calls (empty string if none). */
const char *sa_last_error(void);
/* Number of kernel launches issued by this library since load (bench.py's gpu_launches). */
uint64_t sa_launch_count(void);

/* ---- code/ntt.py:3-18 ntt, code/ntt.py:20-30 intt -------------------------------------
 * out[b][i] = sum_j in[b][j] * root^(i*j), natural order in and out, for `batch`
 * contiguous transforms of n = 2^log_n elements.  inverse != 0 computes intt: the
 * transform with root^-1 followed by the multiplication with n^-1.
 * Validates root^n == 1 and root^(n/2) != 1 exactly like the reference's asserts.
 * in == out is allowed.  log_n in [0, 30]; a transform of n elements needs a workspace of n
 * elements besides its input and output (16 GiB each at 2^30).  The caller's buffers must hold
 * batch * n elements: the library cannot check their length.                              */
int sa_ntt(void *out, const void *in, int log_n, const uint64_t root[2], int inverse, size_t batch,
           void *stream);
/* Multi-GPU assembly (SURVEY 8e; no reference counterpart: the reference is one thread on one CPU).
 * The same transforms, but the results are written to element offset `out_offset` of EVERY buffer
 * outs[0 .. nouts), nouts <= 8: outs[0] is memory of the current device, the others are buffers of
 * other GPUs mapped into this process (CUDA IPC / peer access over NVLink - stark-anatomy_b200/sa_dist.py
 * does the mapping with torch).  The stores to the peers are issued by the last pass of the
 * transform itself, tile by tile, so when every rank has run its shard of a batch each rank holds the
 * whole batch and no gather pass follows.  Completion on the peers is the caller's to synchronise
 * (a barrier across the ranks after the stream has drained).                                  */
int sa_ntt_multi(void *const *outs, int nouts, size_t out_offset, const void *in, int log_n,
                 const uint64_t root[2], int inverse, size_t batch, void *stream);
/* The same through ONE multicast address (NVLS: a multicast object that every rank's buffer is bound to, e.g.
 * torch.distributed._symmetric_memory's multicast_ptr): the last pass issues multimem.st, one store leaves the
 * GPU and the NVSwitch delivers it to every rank's buffer, the own one included.  `local` is this rank's own
 * buffer (same layout; intermediates of the three-pass sizes go there), log_n >= 1.                          */
int sa_ntt_mcast(void *mc, void *local, size_t out_offset, const void *in, int log_n, const uint64_t root[2],
                 int inverse, size_t batch, void *stream);
/* Buffers shared between the processes of one box (one process per GPU): sa_peer_alloc = cudaMalloc (zeroed) +
 * CUDA IPC handle (64 bytes, to be sent to the other processes, e.g. with all_gather_object); sa_peer_open maps
 * another process's buffer into the address space of the CURRENT device and enables peer access to its owner
 * over NVLink, so that this device's kernels (sa_ntt_multi) and copy engines (sa_copy_async) can write it;
 * sa_peer_close / sa_peer_free undo them.  sa_copy_async = cudaMemcpyAsync(cudaMemcpyDefault) on `stream`.   */
int sa_peer_alloc(void **ptr, size_t bytes, uint8_t handle_out[64]);
int sa_peer_open(void **ptr, const uint8_t handle[64]);
int sa_peer_close(void *ptr);
int sa_peer_free(void *ptr);
int sa_copy_async(void *dst, const void *src, size_t bytes, void *stream);
/* One kernel that reads `bytes` (multiple of 16, 16-byte aligned) at src once and stores them to every dsts[i],
 * i < ndst <= 7 (peer-mapped buffers): fully coalesced stores, a warp writes 512 contiguous bytes per
 * destination.  The push half of sa_dist's "p2p-push" assembly: transform i is pushed on a side stream while
 * transform i + 1 computes.  SA_PUSH_CTAS = CTAs of the push kernel (default: one per SM).                          */
int sa_push(void *const *dsts, int ndst, const void *src, size_t bytes, void *stream);
/* The same through ONE multicast address (see sa_ntt_mcast): one multimem.st per 16 bytes, the NVSwitch replicates. */
int sa_push_mcast(void *mc_dst, const void *src, size_t bytes, void *stream);
/* Lets kernels of the CURRENT device store to memory of `peer_device` that is mapped into this process
 * (cudaDeviceEnablePeerAccess; fine if it already is enabled).  A buffer opened from an IPC handle belongs to
 * its owner's device ordinal in this process, and opening it under that ordinal does not enable access from
 * another device (sa_peer_open opens under the accessing device instead, which does).                        */
int sa_enable_peer_access(int peer_device);
/* Same through HOST buffers: H2D copy, transforms, D2H copy, synchronises before
 * returning (the end-to-end call bench.py times as `e2e`).                               */
int sa_ntt_host(void *out_host, const void *in_host, int log_n, const uint64_t root[2], int inverse,
                size_t batch, void *stream);
/* Host buffers for sa_ntt_host (no reference counterpart: the reference keeps Python lists).
 * Page-locked, and allocated on the NUMA node of the current CUDA device (the calling thread is
 * moved onto the CPUs listed in /sys/bus/pci/devices/<gpu>/local_cpulist for the allocation), so
 * that with one process per GPU the copies do not cross the socket interconnect (4 ranks:
 * 6.9e10 -> 9.6e10 butterflies/s end to end).  Any other host memory works too, pageable
 * memory at the speed of pageable copies.  NULL on failure (sa_last_error).               */
void *sa_host_alloc(size_t bytes);
int sa_host_free(void *p);

/* ---- the element-wise piece of fast_multiply ------------------------------------------ */
/* code/ntt.py:61  out[i] = a[i] * b[i]                                                   */
int sa_pointwise_mul(void *out, const void *a, const void *b, size_t n, void *stream);
/* code/univariate.py:130-136 at many points (fast_evaluate's values, ntt.py:82-100):
 * out[j] = sum_i coeffs[i] * points[j]^i                                                 */
int sa_poly_eval(void *out, const void *coeffs, size_t ncoef, const void *points, size_t npoints,
                 void *stream);
/* The same with the algorithm chosen by the caller: mode 0 = what sa_poly_eval does (Horner, one thread per
 * point, below 2^27.5 coefficient-point products; above that the walk down the subproduct tree of the points,
 * max(ncoef, npoints) <= 2^20), 1 = Horner, 2 = the tree walk (ncoef, npoints >= 1).  The reference walks down a
 * remainder tree (ntt.py:82-100); the device walks down the TRANSPOSED interpolation tree (no divisions): one
 * power-series inverse at the root, then one batched transform pair per level.  Same values.                 */
int sa_poly_eval_mode(void *out, const void *coeffs, size_t ncoef, const void *points, size_t npoints, int mode,
                      void *stream);

/* code/ntt.py:66-80 fast_zerofier: out[0..k] = coefficients of prod_i (X - domain[i]) (monic,
 * k + 1 coefficients), k <= 2^20.  Small domains: one kernel; larger ones: the subproduct tree of
 * the reference, built level by level on the device with batched transforms (all nodes of a level
 * in one sa_ntt call).                                                                       */
int sa_zerofier(void *out, const void *domain, size_t k, void *stream);
/* code/ntt.py:102-130 fast_interpolate: out[0..k) = coefficients of the polynomial of degree
 * < k with value values[i] at domain[i], k <= 2^20.  SA_EDIVZERO when two domain points coincide
 * (the reference's element-wise division asserts there).  Small k: Lagrange kernels; larger k:
 * zerofier tree, weights v_i / M'(d_i), and a bottom-up combination over the same tree - one call,
 * everything on the device.  Synchronises.  It is sa_interp_plan into a per-stream workspace
 * followed by sa_interp_apply.                                                                */
int sa_interpolate(void *out, const void *domain, const void *values, size_t k, void *stream);
/* Interpolation plans: the part of sa_interpolate that depends on the domain alone (the zerofier tree
 * and 1/M'(d_i)), built once and applied to any number of value vectors over the same domain.
 * The plan is a device buffer the caller owns, of sa_interp_plan_bytes(k) bytes; its layout is
 * internal and depends on k alone (656 MiB at k = 2^20).
 * sa_interp_plan_bytes: 0 when k == 0 or k > 2^20.  Host-only: no CUDA call.                  */
size_t sa_interp_plan_bytes(size_t k);
/* Builds the plan of domain[0..k).  SA_ESIZE for k == 0 or k > 2^20, SA_EDIVZERO when two domain
 * points coincide.  Synchronises (it reads the zero flag).                                    */
int sa_interp_plan(void *plan, const void *domain, size_t k, void *stream);
/* out[0..k) = the coefficients sa_interpolate gives for values[0..k) over the plan's domain; k must
 * be the plan's k.  Asynchronous: no host synchronisation, and no allocation once the stream's
 * workspace has grown to this size, so the call can be captured in a CUDA graph after one call on
 * the capturing stream (the graph keeps that stream's workspace: replay it where that stream's other
 * work cannot run concurrently, and make no larger call on that stream while the graph is in use).
 * Reads the plan only: one plan may be applied on several streams at once.  It is
 * sa_interp_apply_batch with batch 1.                                                         */
int sa_interp_apply(void *out, const void *plan, const void *values, size_t k, void *stream);
/* out[b*k .. b*k+k) = the coefficients sa_interp_apply gives for values[b*k .. b*k+k), b < batch:
 * many value vectors over one plan's domain in one call.  Rows are contiguous; out must not
 * overlap values.  batch == 0 returns SA_OK without a launch, a k outside 1..2^20 gives SA_ESIZE.
 * The same promises as sa_interp_apply: plan only read, no host synchronisation, and no
 * allocation once the stream's workspaces have grown for this k and chunk size.  Up to 1024
 * points the batch is one field matrix product (2 launches, k^2 elements of workspace whatever
 * the batch size); above, every level of the up-sweep is one batch over all vectors' nodes, in
 * chunks of sa_interp_batch_max(k) vectors, each chunk issuing the launches of one
 * sa_interp_apply.  A chunk takes 96 bytes per leaf slot (K = 2^ceil(log2 k) slots) per vector
 * of per-stream workspace.                                                                    */
int sa_interp_apply_batch(void *out, const void *plan, const void *values, size_t k, size_t batch, void *stream);
/* The most vectors one chunk of sa_interp_apply_batch takes for a k-point plan: SIZE_MAX up to
 * 1024 points (one pass whatever the batch), max(1, floor(2^30 / (96 K))) above (a chunk's
 * workspace stays at or below 1 GiB: 10 vectors at 2^20, 170 at 2^16), 0 when k == 0 or
 * k > 2^20.  Host-only: no CUDA call.                                                         */
size_t sa_interp_batch_max(size_t k);

/* ---- Geometric interpolation plans: interpolation over, and the zerofier of, the domain
 * 1, step, step^2, ..., step^(k-1), by the closed forms of the q-binomial theorem and two cyclic
 * convolutions of length K = 2^ceil(log2 2k) (DESIGN section 3.12).  No subproduct tree and no list
 * of points: k up to 2^26, where the tree stops at 2^20.  The coefficients are those sa_interp_apply
 * and sa_zerofier give over the explicit domain, bit for bit.
 * The method needs step^d != 1 for 1 <= d <= k and, from k = 2 on, step != 0.  d < k is "the points
 * are distinct"; d = k is one more condition: a step of order exactly k (the domain is a whole
 * subgroup, whose interpolation is an inverse NTT) is refused here although the tree interpolates it.
 * sa_geo_plan_bytes: the size of a plan, laid out by k alone: 16*(2*sec16(k) + 2K) bytes (96 MiB at
 * k = 2^20, where the tree's plan is 656 MiB); 0 when k == 0 or k > 2^26.  Host-only: no CUDA call. */
size_t sa_geo_plan_bytes(size_t k);
/* Builds the plan of (step, k) into a device buffer of sa_geo_plan_bytes(k) bytes the caller owns.
 * Before any launch: SA_ESIZE for k outside 1..2^26, SA_EDIVZERO for step == 0 with k >= 2.  After
 * the build's one synchronisation (it reads the zero flag): SA_EDIVZERO when step^d == 1 for some
 * 1 <= d <= k, k >= 2 (a single point is never refused); the plan's contents are then unspecified.  */
int sa_geo_plan(void *plan, const uint64_t step[2], size_t k, void *stream);
/* out[b*k .. b*k+k) = the coefficients of the polynomial of degree < k that takes values[b*k + i] at
 * step^i, b < batch, over a plan of (step, k); k must be the plan's.  Rows are contiguous; out must
 * not overlap values.  SA_ESIZE for k outside 1..2^26 before any launch; batch == 0 returns SA_OK
 * without a launch.  The promises of sa_interp_apply_batch: the plan is only read (one plan may serve
 * several streams at once), no host synchronisation, and no allocation once the stream's workspaces
 * have grown for this k and chunk size, so the call can be captured in a CUDA graph.  The batch runs
 * in chunks of sa_geo_batch_max(k) vectors, each issuing the launches of one vector: four kernels,
 * four batched transforms and one strided copy.  A chunk takes 32 bytes per slot (2K per vector) of
 * per-stream workspace and 16 of the transforms' intermediate.                                    */
int sa_geo_interp_batch(void *out, const void *plan, const void *values, size_t k, size_t batch, void *stream);
/* The most vectors one chunk of sa_geo_interp_batch takes: max(1, floor(2^30 / (48 K))) (10 at
 * k = 2^20), 0 when k == 0 or k > 2^26.  Host-only: no CUDA call.                                 */
size_t sa_geo_batch_max(size_t k);
/* out[0..k] = the coefficients of prod_{i<k} (X - step^i) (monic), with sa_geo_plan's limits and
 * refusals.  Synchronises once, to read the zero flag, before it writes out: an error leaves out
 * untouched.                                                                                     */
int sa_geo_zerofier(void *out, const uint64_t step[2], size_t k, void *stream);

/* ---- code/ntt.py:137-176 fast_coset_divide, many numerators over one divisor, and ntt.py:132-135
 * fast_coset_evaluate, many polynomials in one call ------------------------------------------------
 * n = 2^log_n, log_n in [1, 30]; `root` a primitive n-th root of unity (checked like sa_ntt's, before
 * any launch: SA_EROOTORDER / SA_ENOTPRIM).  With R_i = r(offset * root^i) and L_i = l(offset * root^i),
 * i < n, a row of an apply is out[j] = U[j] * offset^-j, j < qlen, U = intt(L_i / R_i): the reference's
 * fast_coset_divide at order n before its truncation.  So where n/2 <= max(deg l, deg r) < n (the
 * reference keeps order n) out[0 .. deg l - deg r] are its coefficients, bit for bit, and a clean
 * division with deg l < n gives the exact quotient followed by zeros.
 * A coset division plan holds what depends on (divisor, offset, root, log_n) alone: offset^i, 1/R_i and
 * offset^-i (i < n).  It is a device buffer the caller owns, of sa_coset_div_plan_bytes(log_n) bytes;
 * its layout is internal and depends on log_n alone (48 MiB at 2^20, 6 GiB at 2^27, 48 GiB at 2^30:
 * with the operands and workspaces, the largest sizes do not fit on one 80 GB device).
 * Offset 0 is allowed, as in the reference: its powers are 1, 0, 0, ... and its inverse is 0.
 * sa_coset_div_plan_bytes: 0 when log_n is outside 1..30.  Host-only: no CUDA call.                 */
size_t sa_coset_div_plan_bytes(int log_n);
/* Builds the plan of divisor[0..dlen) on the coset offset * <root>.  SA_ESIZE for dlen outside 1..n or
 * log_n outside 1..30 (before any launch), SA_EDIVZERO when some R_i == 0 (the zero divisor among
 * them: the reference's element-wise division raises there).  Synchronises (it reads the zero flag). */
int sa_coset_div_plan(void *plan, const void *divisor, size_t dlen, int log_n, const uint64_t root[2],
                      const uint64_t offset[2], void *stream);
/* out[b*qlen .. b*qlen+qlen) = row b of the division of lhs[b*ncoef .. b*ncoef+ncoef) by the plan's
 * divisor, b < batch; log_n and root must be the plan's.  Rows are contiguous; out must not overlap
 * lhs.  1 <= ncoef, qlen <= n, else SA_ESIZE before any launch; batch == 0 returns SA_OK without a
 * launch.  Asynchronous: no host synchronisation, and no allocation once the stream's workspaces
 * have grown for this log_n and chunk size, so the call can be captured in a CUDA graph after one
 * call on the capturing stream (the graph keeps that stream's workspace: replay it where that
 * stream's other work cannot run concurrently, and make no larger call on that stream while the
 * graph is in use).  Reads the plan only: one plan may be applied on several streams at once.
 * The batch runs in chunks of sa_coset_batch_max(log_n) rows; each chunk issues the same launches
 * whatever its size (load, one batched forward sa_ntt, quotient, one batched inverse sa_ntt, store)
 * and takes 32 bytes of per-stream workspace per element per row.                              */
int sa_coset_div_apply_batch(void *out, const void *plan, const void *lhs, size_t ncoef, size_t qlen, int log_n,
                             const uint64_t root[2], size_t batch, void *stream);
/* out[b*n .. b*n+n) = fast_coset_evaluate of coeffs[b*ncoef .. b*ncoef+ncoef) at order n:
 * ntt(coeffs[i] * offset^i, zero padded to n), b < batch.  Needs no plan.  The same checks (1 <=
 * ncoef <= n), chunks and asynchronous promises as sa_coset_div_apply_batch; out must not overlap
 * coeffs.                                                                                        */
int sa_coset_evaluate_batch(void *out, const void *coeffs, size_t ncoef, int log_n, const uint64_t root[2],
                            const uint64_t offset[2], size_t batch, void *stream);
/* code/fast_stark.py:125-148: the weighted, degree-shifted combination of many device polynomials and its
 * fast_coset_evaluate, in one call.  With n = 2^log_n, c[i] = sum_t w_t * srcs[t][i - shifts[t]] over the terms t
 * with shifts[t] <= i < shifts[t] + lens[t], and out[0..n) = ntt(c[i] * offset^i, zero padded to n): the
 * reference's combined_codeword for the same terms (x^s * q is q at shift s).  Term t is a DEVICE row of lens[t]
 * elements (rows may be slices of different buffers, and several terms may share one row), a shift and the weight
 * weights[2t], weights[2t+1] (the limbs of a canonical residue).  srcs, lens, shifts and weights are HOST arrays,
 * read before the call returns: the terms travel as kernel parameters, so the call uploads nothing.  A term with
 * lens[t] == 0 adds nothing; nterms == 0 writes n zeros (the empty combination).
 * Before any launch: SA_ESIZE for log_n outside 1..30 or any shifts[t] + lens[t] > n, and the root's
 * SA_EROOTORDER / SA_ENOTPRIM as for sa_coset_evaluate_batch.  Every offset is accepted, 0 included.
 * out must not overlap any source.  Launches: one offset^i table of ncomb = max_t(shifts[t] + lens[t]) elements
 * (per-stream workspace), one per group of 64 terms, one forward sa_ntt in place on out: 1 + ceil(nterms / 64)
 * plus the transform's (none but the group launches when ncomb == 0).  Asynchronous: no host synchronisation,
 * and no allocation once the stream's workspaces have grown for this ncomb and log_n, so the call can be
 * captured in a CUDA graph after one call on the capturing stream (the same conditions as
 * sa_coset_div_apply_batch); a replay uses the terms (rows, lengths, shifts, weights) it was captured with.   */
int sa_coset_combine_evaluate(void *out, int log_n, const uint64_t root[2], const uint64_t offset[2],
                              const void *const *srcs, const size_t *lens, const size_t *shifts,
                              const uint64_t *weights, size_t nterms, void *stream);
/* Many combinations in one call: term t is added into destination row rows[t] < nrows (a HOST array like the others),
 * and out[r*n .. r*n+n) is row r's combination evaluated as above -- the codeword sa_coset_combine_evaluate gives for
 * the terms of row r alone, zeros for a row without terms.  Rows are contiguous; out must not overlap any source.
 * Launches: one offset^i table of the longest row's ncomb elements, one per group of 64 terms over all rows, one
 * batched forward sa_ntt of the nrows rows in place: 1 + ceil(nterms / 64) plus the batched transform's, whatever
 * nrows -- no launch per row.  sa_coset_combine_evaluate is nrows = 1 of the same kernel.  Before any launch:
 * sa_coset_combine_evaluate's checks and SA_ESIZE for any rows[t] >= nrows; an error leaves out untouched.
 * nrows == 0 (and so no term) returns SA_OK without a launch.  The same asynchronous and graph-capture promises as
 * sa_coset_combine_evaluate.                                                                                       */
int sa_coset_combine_evaluate_batch(void *out, size_t nrows, int log_n, const uint64_t root[2],
                                    const uint64_t offset[2], const void *const *srcs, const size_t *lens,
                                    const size_t *shifts, const size_t *rows, const uint64_t *weights, size_t nterms,
                                    void *stream);
/* The most rows one chunk of sa_coset_div_apply_batch / sa_coset_evaluate_batch takes:
 * max(1, floor(2^30 / (32 n))) (32 at 2^20, 512 at 2^16), so a chunk's workspace stays at or below
 * 1 GiB; 0 when log_n is outside 1..30.  Host-only: no CUDA call.                                */
size_t sa_coset_batch_max(int log_n);

/* ---- code/fast_stark.py:108-113: the transition quotients of an AIR, without symbolic polynomials -------------
 * The constraints are polynomials in nvars = 1 + 2*nregs variables in FastStark's order: x, the trace rows T_s(x)
 * (variables 1..nregs) and the next rows T_s(step*x) (variables nregs+1..2*nregs).  Constraint c is the terms
 * term_start[c] .. term_start[c+1]; term t has the coefficient coeffs[2t], coeffs[2t+1] (the limbs of a canonical
 * residue) and the exponents exps[t*nvars .. t*nvars + nvars).  A constraint without terms is the zero polynomial.
 * With n = 2^log_n, x_i = offset * root^i and N_c(x) = C_c(x, T(x), T(step*x)), row c of an apply is
 *     out[c][j] = U_c[j] * offset^-j  (j < qlen),   U_c = intt(N_c(x_i) / Z(x_i)),
 * the numerator evaluated point by point on the coset and divided there.  Where every term's degree bound
 * e_0 + (e_1 + ... + e_2nregs) * (max_ncoef - 1) is below n (the build refuses anything else), N_c is the
 * polynomial MPolynomial.evaluate_symbolic gives, and out[c][0 .. deg N_c - deg Z] is fast_coset_divide's quotient
 * at order n, bit for bit, clean division or not.
 * A plan holds the zerofier's coset division plan, (offset*step)^j, the points x_i and the constraints compiled into
 * a program.  It is a device buffer the caller owns, of sa_air_plan_bytes(log_n, max_ncoef, nregs, nterms) bytes
 * with nterms = term_start[ncons]: 80*n + 16*sec16(1 + nterms*(2 + ceil(nregs/2))) from n = 16 on, sec16 rounding up
 * to a multiple of 16 (DESIGN section 2).  0 when log_n is outside 1..30, nregs == 0, max_ncoef is outside 1..n or
 * nterms >= 2^32.  Host-only: no CUDA call.                                                                     */
size_t sa_air_plan_bytes(int log_n, size_t max_ncoef, size_t nregs, size_t nterms);
/* Builds the plan.  coeffs, exps and term_start are HOST arrays, compiled into the plan; zerofier[0..zlen) is a
 * device row.  Before any launch: SA_ESIZE for log_n outside 1..30, nregs == 0, ncons == 0, max_ncoef or zlen outside
 * 1..n, a decreasing term_start, or a term whose degree bound (above) is >= n; the root's SA_EROOTORDER /
 * SA_ENOTPRIM.  SA_EDIVZERO when Z vanishes somewhere on the coset.  Every offset and step is accepted, 0 included.
 * Synchronises (it reads the zero flag).                                                                       */
int sa_air_plan(void *plan, const uint64_t *coeffs, const uint32_t *exps, const size_t *term_start, size_t ncons,
                size_t nregs, size_t max_ncoef, const void *zerofier, size_t zlen, int log_n, const uint64_t root[2],
                const uint64_t offset[2], const uint64_t step[2], void *stream);
/* out[c*qlen .. c*qlen+qlen) = row c (above) for c < ncons, from trace[nregs][ncoef], the trace polynomials'
 * coefficient rows (sa_interp_apply_batch's layout).  log_n, root, nregs and ncons must be the plan's and
 * ncoef <= the plan's max_ncoef.  SA_ESIZE before any launch for nregs or ncons == 0 or ncoef, qlen outside 1..n.
 * Rows are contiguous, so they feed sa_coset_combine_evaluate as they are.  Launches: two coset loads, one batched
 * forward sa_ntt of the 2*nregs rows, then per chunk of sa_coset_batch_max(log_n) constraints the evaluation kernel,
 * one batched inverse sa_ntt and the store -- the same count whatever nregs and the chunk's size.  Per-stream
 * workspace: 16*n*(2*nregs + chunk) bytes besides the transform's.  Asynchronous: no host synchronisation, and no
 * allocation once the stream's workspaces have grown, so the call can be captured in a CUDA graph (the same
 * conditions as sa_coset_div_apply_batch).  Reads the plan only: one plan may be applied on several streams at once. */
int sa_air_quotients(void *out, const void *plan, const void *trace, size_t nregs, size_t ncoef, size_t qlen,
                     size_t ncons, int log_n, const uint64_t root[2], void *stream);
/* code/stark.py:111: the same rows with an exact-division check.  out is exactly sa_air_quotients'; flags[c] = 0
 * exactly when U_c[j] = 0 for every tail <= j < n (U_c above, the row before the offset^-j store).  With
 * tail = n - deg Z it is the reference's remainder test of Polynomial.__truediv__ (univariate.py:50-53) for every
 * numerator, N_c = 0 and deg N_c < deg Z included:
 *   - the build guarantees deg N_c < n;
 *   - if U_c vanishes from n - deg Z on, U_c * Z has degree below n and agrees with N_c on the n points x_i, so Z
 *     divides N_c (and U_c is the quotient);
 *   - conversely an exact quotient has degree deg N_c - deg Z < n - deg Z.
 * SA_ESIZE before any launch for tail > n and for everything sa_air_quotients refuses; an error leaves out and flags
 * untouched.  Launches: sa_air_quotients' plus one memset that clears the flags (the store is a warp ballot over the
 * tail with one atomicOr per flagged row a warp touches, in place of the plain store).  Asynchronous: no host
 * synchronisation, and no allocation once the stream's workspaces have grown, so the call can be captured in a CUDA
 * graph; a replay clears the flags again.  Reads the plan only.                                                    */
int sa_air_quotients_exact(void *out, uint32_t *flags, const void *plan, const void *trace, size_t nregs,
                           size_t ncoef, size_t qlen, size_t ncons, size_t tail, int log_n, const uint64_t root[2],
                           void *stream);
/* The same applies for `batch` traces of one AIR in one call: trace[batch][nregs][ncoef] gives out[batch][ncons][qlen]
 * (and flags[batch][ncons]), trace b's rows (and flags) exactly what sa_air_quotients (sa_air_quotients_exact) gives
 * for trace b alone.  sa_air_quotients and sa_air_quotients_exact are batch 1, with the launches they always had.
 * The batch runs in chunks of whole traces, sa_air_batch_max(nregs, ncons, log_n) at most; a chunk issues the
 * launches of one trace's apply (two coset loads of all its traces' rows, one batched forward sa_ntt, then the
 * evaluation kernel, one batched inverse sa_ntt and the store per row chunk of at most sa_coset_batch_max(log_n)
 * constraint rows; the exact apply's flags memset once per call).  Per-stream workspace: 16*n*(2*nregs*traces +
 * rows) bytes for a chunk of `traces` traces and row chunks of `rows` rows, besides the transform's.  The same checks
 * before any launch as the single calls (an error leaves out and flags untouched); batch == 0 returns SA_OK without a
 * launch.  The same asynchronous and graph-capture promises; the plan is only read.                               */
int sa_air_quotients_batch(void *out, const void *plan, const void *trace, size_t nregs, size_t ncoef, size_t qlen,
                           size_t ncons, size_t batch, int log_n, const uint64_t root[2], void *stream);
int sa_air_quotients_exact_batch(void *out, uint32_t *flags, const void *plan, const void *trace, size_t nregs,
                                 size_t ncoef, size_t qlen, size_t ncons, size_t batch, size_t tail, int log_n,
                                 const uint64_t root[2], void *stream);
/* The most traces one chunk of a batched apply takes: max(1, floor(sa_coset_batch_max(log_n) / (2*nregs + ncons))),
 * so that a chunk of several traces keeps its 2*nregs transformed trace rows and ncons constraint rows per trace at
 * 32*n bytes per row with the transform's -- at most 1 GiB per stream -- and is one row chunk (64 traces of 2
 * registers and 4 constraints at 2^16, 4 at 2^20); 0 when log_n is outside 1..30.  Host-only: no CUDA call.        */
size_t sa_air_batch_max(size_t nregs, size_t ncons, int log_n);

/* ---- code/fast_stark.py:92-106: the boundary quotients, their coset codewords and a remainder check ------------
 * Register s has the trace polynomial T_s, the interpolant I_s of its boundary values and the zerofier Z_s of its
 * boundary points.  With n = 2^log_n and x_i = offset * root^i (FastStark's FRI domain: offset = the generator,
 * root = omega) an apply gives
 *     codewords[s][i] = (T_s(x_i) - I_s(x_i)) / Z_s(x_i),   quot[s][j] = U_s[j] * offset^-j (j < ncoef),
 * U_s = intt(codewords[s]), and flags[s] = 0 exactly when (T_s - I_s) / Z_s is a clean division: when U_s is zero at
 * every j >= max(0, ncoef - deg Z_s).  Then quot[s] is the reference's quotient followed by zeros and codewords[s] is
 * fast_coset_evaluate's of it, bit for bit; otherwise the reference raises "cannot perform polynomial division because
 * remainder is not zero" and the row is not a quotient.
 * A plan holds offset^i, offset^-i and per register 1/Z_s(x_i), I_s(x_i) and deg Z_s.  It is a device buffer the
 * caller owns, of sa_boundary_plan_bytes(log_n, nregs) bytes: 32*n*(1 + nregs) + 16*sec16(nregs) from n = 16 on,
 * sec16 rounding up to a multiple of 16 (DESIGN section 2).  0 when log_n is outside 1..30, nregs == 0 or the size
 * does not fit a size_t.  Host-only: no CUDA call.                                                                  */
size_t sa_boundary_plan_bytes(int log_n, size_t nregs);
/* Builds the plan from per-register device rows zerofiers[s][0..zlens[s]) and interpolants[s][0..ilens[s]); the
 * pointer and length arrays are HOST arrays.  Before any launch: SA_ESIZE for log_n outside 1..30, nregs == 0, a
 * zlens[s] or ilens[s] outside 1..n, and offset 0 (the check needs n distinct points); the root's SA_EROOTORDER /
 * SA_ENOTPRIM.  After the build's one synchronisation: SA_ESIZE when a zerofier row's top coefficient is zero (deg Z_s
 * is taken as zlens[s] - 1), else SA_EDIVZERO when some Z_s vanishes on the coset.                                  */
int sa_boundary_plan(void *plan, const void *const *zerofiers, const size_t *zlens, const void *const *interpolants,
                     const size_t *ilens, size_t nregs, int log_n, const uint64_t root[2], const uint64_t offset[2],
                     void *stream);
/* quot[nregs][ncoef], codewords[nregs][n] and flags[nregs] (above) from trace[nregs][ncoef], the trace polynomials'
 * coefficient rows (sa_interp_apply_batch's layout).  log_n, root and nregs must be the plan's.  SA_ESIZE before any
 * launch for nregs == 0 or ncoef outside 1..n.  Rows are contiguous, so they feed sa_coset_combine_evaluate and
 * sa_coset_evaluate_batch as they are.  Launches: a memset that clears the flags, then per chunk of
 * sa_coset_batch_max(log_n) registers the coset load, one batched forward sa_ntt in the codewords, the point kernel,
 * one batched inverse sa_ntt into the workspace and the store with the remainder check -- the same count whatever the
 * chunk's size.  Per-stream workspace: 16*n bytes per register of a chunk besides the transform's.  Asynchronous: no
 * host synchronisation, and no allocation once the stream's workspaces have grown, so the call can be captured in a
 * CUDA graph; a replay clears the flags again.  Reads the plan only: one plan may be applied on several streams.   */
int sa_boundary_quotients(void *quot, void *codewords, uint32_t *flags, const void *plan, const void *trace,
                          size_t nregs, size_t ncoef, int log_n, const uint64_t root[2], void *stream);

/* ---- code/merkle.py:6-14 Merkle.commit -------------------------------------------------
 * Builds the whole blake2b-512 tree over n = 2^k leaves, leaf = H(decimal ASCII of the
 * value), node = H(left || right).  `tree` receives 2n nodes of 64 bytes in heap order:
 * node 1 is the root, node i has children 2i and 2i+1, leaf j is node n + j, node 0 is
 * unused (set to zero).  It is sa_merkle_tree_batch with batch 1.                          */
int sa_merkle_tree(void *tree, const void *values, size_t n, void *stream);
/* The trees of `batch` codewords of n leaves each, in one launch ladder: tree b (2n nodes of
 * 64 bytes, sa_merkle_tree's layout) at trees + b*2n*64 bytes, built from values[b*n .. b*n+n).
 * A batch issues exactly the launches of one tree of n leaves, up to 65535 trees; larger
 * batches run in groups of 65535.  n not a power of two gives SA_ENOTPOW2 and batch == 0
 * returns SA_OK, both without a launch.  Asynchronous; a call with more trees than any
 * earlier call on the stream synchronises the stream once to grow its arrival counters.    */
int sa_merkle_tree_batch(void *trees, const void *values, size_t n, size_t batch, void *stream);
/* code/merkle.py:16-27 Merkle.open for k leaf indices (HOST array): paths_out receives
 * k * log2(n) digests of 64 bytes, siblings bottom-up per index (device memory).  It is
 * sa_merkle_open_batch with batch 1.                                                      */
int sa_merkle_open(void *paths_out, const void *tree, size_t n, const uint64_t *indices_host, size_t k,
                   void *stream);
/* The same k leaf indices opened in each of `batch` trees laid out as sa_merkle_tree_batch
 * lays them: paths_out[b][q][level] = the sibling at `level` (bottom-up) of leaf indices[q]
 * in tree b, 64 bytes each.  One index upload, one launch.  Before any launch: SA_ENOTPOW2
 * for n not a power of two, SA_EINDEX for any index >= n; batch == 0, k == 0 or n == 1
 * (no siblings) returns SA_OK without a launch.  Asynchronous.                            */
int sa_merkle_open_batch(void *paths_out, const void *trees, size_t n, size_t batch, const uint64_t *indices_host,
                         size_t k, void *stream);
/* out[i] = values[indices[i]] (the leaf triples of code/fri.py:104-105).  It is
 * sa_gather_batch with batch 1.                                                           */
int sa_gather(void *out, const void *values, size_t n, const uint64_t *indices_host, size_t k,
              void *stream);
/* out[b*k + q] = values[b*n + indices[q]]: the same k indices gathered from each of `batch`
 * rows of n elements (any n >= 1), one index upload, one launch.  SA_EINDEX for any index
 * >= n before any launch; batch == 0 or k == 0 returns SA_OK without a launch.
 * Asynchronous.                                                                           */
int sa_gather_batch(void *out, const void *values, size_t n, size_t batch, const uint64_t *indices_host, size_t k,
                    void *stream);
/* Openings with an index set per group of rows: rows (trees) are taken in groups of `group`, and group g reads its
 * own k indices from indices_host[g*k .. g*k+k), ceil(batch / group) sets (one when batch == 0).  So
 * out[b*k + q] = values[b*n + indices_host[(b / group)*k + q]] and paths_out[b][q][level] is the sibling at `level`
 * of leaf indices_host[(b / group)*k + q] in tree b.  With the committed rows of many proofs back to back, group =
 * rows per proof opens every proof's rows at that proof's own indices in one call.  sa_gather_batch and
 * sa_merkle_open_batch are group = batch of the same kernels.  Before any launch: SA_ESIZE for group == 0, and
 * everything the ungrouped calls refuse (SA_EINDEX for any index of any set >= n).  One index upload, one launch;
 * the same cases without a launch as the ungrouped calls.  Asynchronous.                                           */
int sa_gather_batch_sets(void *out, const void *values, size_t n, size_t batch, size_t group,
                         const uint64_t *indices_host, size_t k, void *stream);
int sa_merkle_open_batch_sets(void *paths_out, const void *trees, size_t n, size_t batch, size_t group,
                              const uint64_t *indices_host, size_t k, void *stream);

/* ---- code/fri.py:85 split-and-fold, and the fused round of Fri.commit (fri.py:64-88) ----
 * next[i] = 2^-1 * ((1 + alpha/(offset*omega^i)) * cw[i] + (1 - alpha/(offset*omega^i)) * cw[n/2+i])
 * for i < n/2.  sa_fri_round additionally builds the Merkle tree of `next` (n/2 leaves,
 * n nodes of 64 bytes) in the same kernel that folds; sa_fri_fold only folds.             */
int sa_fri_fold(void *next, const void *cw, size_t n, const uint64_t alpha[2], const uint64_t offset[2],
                const uint64_t omega[2], void *stream);
int sa_fri_round(void *next, void *next_tree, const void *cw, size_t n, const uint64_t alpha[2],
                 const uint64_t offset[2], const uint64_t omega[2], void *stream);

/* ---- code/fri.py:56-96 Fri.commit, the whole round loop in one call -----------------------
 * Round 0 builds the Merkle tree of `codeword` (n = 2^k elements); every later round is the
 * fused fold + tree kernel on the previous layer.  After each round the 64-byte root is copied
 * to the host and `challenge(user, round, root, alpha_out, want_alpha)` is called: the caller
 * pushes the root into its proof stream (fri.py:72) and, when want_alpha != 0, writes the
 * Fiat-Shamir challenge alpha = field.sample(proof_stream.prover_fiat_shamir()) (fri.py:79)
 * into alpha_out; a non-zero return aborts the commit (SA_ECALLBACK).  omega / offset are
 * squared per round (fri.py:87-88).
 *   layers : device buffer for layers 1 .. rounds-1, layer r (n >> r elements) at element
 *            offset n - (n >> (r-1)), i.e. back to back;  total n - (n >> (rounds-1)) elements
 *   trees  : device buffer for the trees of layers 0 .. rounds-1, back to back, tree r has
 *            2 * (n >> r) nodes of 64 bytes;  total 4n - (4n >> rounds) nodes               */
typedef int (*sa_fri_challenge_fn)(void *user, int round, const uint8_t root[64], uint64_t alpha_out[2],
                                   int want_alpha);
int sa_fri_commit(void *layers, void *trees, const void *codeword, size_t n, int rounds,
                  const uint64_t offset[2], const uint64_t omega[2], sa_fri_challenge_fn challenge, void *user,
                  void *stream);

/* ---- sa_fri_commit for `batch` codewords of one length n, one offset and one omega ----------
 * codewords[b*n .. b*n+n) is codeword b.  Round 0 is one tree ladder over the B codewords, every
 * later round one fused fold + tree ladder over all B rows, row b folding with its own alpha.
 * After each round the host waits once for the round's B roots, then calls
 * challenge(user, round, roots, alphas_out, want_alpha) once: roots holds B roots of 64 bytes
 * back to back, and when want_alpha != 0 the callback writes alpha b as two limbs at
 * alphas_out[2b], alphas_out[2b+1].  A non-zero return gives SA_ECALLBACK and nothing more is
 * launched.  The launches of a round are those of one codeword, per group of 65535 codewords.
 *   layers : rounds 1 .. rounds-1, round r as B back-to-back rows of n >> r elements, round after
 *            round;  total B * (n - (n >> (rounds-1))) elements (unused, may be NULL, for rounds 1)
 *   trees  : rounds 0 .. rounds-1, round r as B back-to-back trees of 2 (n >> r) nodes of 64 bytes
 *            (sa_merkle_tree_batch's layout), round after round;  total B * (4n - (4n >> rounds))
 *            nodes.  So sa_gather_batch_sets and sa_merkle_open_batch_sets with group = 1 open
 *            each row of a round at its own indices.
 * Before any launch: SA_ESIZE for n not a power of two, rounds < 1, rounds > log2(n) + 1, and a
 * NULL buffer, offset, omega or callback; batch == 0 returns SA_OK without work.              */
typedef int (*sa_fri_challenge_batch_fn)(void *user, int round, const uint8_t *roots, uint64_t *alphas_out,
                                         int want_alpha);
int sa_fri_commit_batch(void *layers, void *trees, const void *codewords, size_t n, size_t batch, int rounds,
                        const uint64_t offset[2], const uint64_t omega[2], sa_fri_challenge_batch_fn challenge,
                        void *user, void *stream);

/* ---- seeded randomizer draws (code/algebra.py:118-120 field.sample(os.urandom(17))) -------------
 * For a 32-byte seed s, draw j (a uint64) is the element field.sample gives when os.urandom(17) returns
 * blake2b(s || j as 8 little-endian bytes).digest()[:17] (64-byte digest, no key): that digest's first 17 bytes
 * read big-endian, mod p (DESIGN section 3.13).  For seed b (the 32 bytes at seeds + 32*b, device memory, no
 * alignment needed) and j < count, the element of draw first + j is written at element offset
 *     b*seed_stride + (j % width)*lane_stride + j / width
 * of out; no other element is touched.  With width = nregs and lane_stride = T this fills the randomizer rows of
 * register-major trace columns; with width = 1 it writes count consecutive elements per seed.  nseeds == 0 or
 * count == 0 returns SA_OK without a launch.  Before any launch: SA_ESIZE for width == 0, for first + count - 1
 * above 2^64 - 1, and for an item count nseeds*count or a largest offset at or above 2^59 elements.  One launch,
 * no allocation; asynchronous and graph-capturable.                                                       */
int sa_sample_seeded(void *out, const void *seeds, size_t nseeds, size_t seed_stride, uint64_t first, size_t count,
                     size_t width, size_t lane_stride, void *stream);

/* ---- Rescue-Prime over many inputs (code/rescue_prime.py:100-203 hash and trace, state width 2) -------------
 * For b < count, input x = inputs[b] (canonical, device memory): absorb [x, 0], then `rounds` rounds, round r a
 * forward half-round (S-box s^alpha, MDS, constants 4r + i) and a backward half-round (S-box s^alphainv, MDS,
 * constants 4r + 2 + i), i < 2.  `constants` (device memory, canonical) is the MDS matrix row-major (4 elements),
 * then the 4*rounds round constants in the reference's order; the exponents are 128-bit host values, lo word first.
 * The library holds no Rescue constant of its own.  hashes[b] receives state[0] after the last round (hashes may be
 * NULL); trace (may be NULL) receives register s of row r <= rounds at element offset
 *     b*inst_stride + s*lane_stride + r
 * where row 0 is the absorbed state and row r + 1 the state after round r; no other element is touched.  With
 * lane_stride = T and inst_stride = 2T this fills rows 0..rounds of register-major trace columns of length T.
 * count == 0 returns SA_OK without a launch.  Before any launch: SA_ESIZE for both outputs NULL, rounds of 0 or
 * above SA_RESCUE_MAX_ROUNDS (the constants live in shared memory), and a count or largest element offset at or
 * above 2^59.  One launch, no allocation; asynchronous and graph-capturable (DESIGN section 3.14).              */
#define SA_RESCUE_MAX_ROUNDS 512
int sa_rescue(void *hashes, void *trace, const void *inputs, size_t count, const void *constants, size_t rounds,
              const uint64_t alpha[2], const uint64_t alphainv[2], size_t inst_stride, size_t lane_stride,
              void *stream);

/* ---- device memory the library keeps between calls (no reference counterpart) ------------------
 * Twiddle tables (per device, log n, root, direction) and FRI x^-1 tables (per device, omega, n)
 * live in one least-recently-used cache bounded by bytes: default 4 GiB, SA_CACHE_LIMIT_MIB, or
 * sa_cache_limit(bytes), which also evicts down to the new limit right away and returns the bytes
 * still cached (sa_cache_limit(0) drops everything).  A table in use by an enqueued kernel is freed
 * only after that kernel has finished.  sa_cache_bytes() = bytes cached now.
 * sa_release_workspaces() synchronises the current device and frees its per-stream scratch buffers
 * (the n * batch intermediate of the multi-pass transforms, host-entry staging), which otherwise
 * only grow.                                                                                */
size_t sa_cache_limit(size_t bytes);
size_t sa_cache_bytes(void);
int sa_release_workspaces(void);

/* ---- batched verification (code/fast_stark.py:180-286, code/stark.py:172-275, code/fri.py:132-231) -----------
 * DESIGN section 3.15.  Every call writes one flag per item, 0 where the item's check passes; items are independent,
 * one thread each, in one grid-stride launch.  count == 0 returns SA_OK without a launch.  Before any launch: SA_ESIZE
 * for an item count (or a largest element offset the sizes imply) at or above 2^59 and for a NULL buffer.  No
 * allocation; asynchronous and graph-capturable.
 *
 * sa_merkle_verify_batch: Merkle.verify(root, index, path, leaf) for path i: blake2b of leaves[i]'s decimal ASCII,
 * then depth[i] levels bottom-up, level l hashing (cur || sibling) when bit l of leaf_index[i] is 0 and (sibling ||
 * cur) when it is 1, the last digest compared with the 64 bytes at roots + 64 i.  Sibling l of path i is the 64
 * bytes at paths + 64 (path_offset[i] + l): paths of different depths share one launch.  An index at or above
 * 2^depth[i] or a depth above 63 is a failed check.                                                              */
int sa_merkle_verify_batch(uint32_t *flags, const void *roots, const void *leaves, const uint64_t *leaf_index,
                           const uint32_t *depth, const void *paths, const uint64_t *path_offset, size_t count,
                           void *stream);
/* sa_fri_colinear_batch: FRI's colinearity test for item i of round r = round[i] at a-index a = a_index[i]:
 * test_colinearity([(ax, ay[i]), (-ax, by[i]), (alpha[i], cy[i])]) with ax = offset^(2^r) omega^(2^r a), computed
 * as the reference's Lagrange interpolant (inverse(0) = 0) having degree exactly 1.                            */
int sa_fri_colinear_batch(uint32_t *flags, const void *ay, const void *by, const void *cy, const uint64_t *a_index,
                          const void *alpha, const uint32_t *round, const uint64_t offset[2], const uint64_t omega[2],
                          size_t count, void *stream);
/* sa_verify_combination: the verifier's combination at k opened indices of each of nproofs proofs, items and
 * proofs laid out as csrc/verify.cuh states (verify_item, verify_proof): the trace values from each register's
 * boundary zerofier and interpolant (blen coefficients each) by Horner, the AIR at [x, cur, next] by walking the
 * program sa_air_program compiled (ncons constraints of nregs registers), the transition zerofier's value from the
 * item (zcoef NULL) or by Horner over zcoef[0..zlen), and the weighted sum with x^shift, compared with FRI's value.
 * x = offset omega^i on the domain of 2^log_n points, the next point at (i + ef) mod 2^log_n.  Flag 1 for a
 * mismatch, 2 for a zero zerofier value.  SA_ESIZE also for nregs outside 1..16, ncons or blen outside 1..2^32 - 1,
 * log_n outside 1..30, ef >= 2^log_n and zlen == 0 with zcoef.                                                  */
int sa_verify_combination(uint32_t *flags, const void *items, const void *proofs, size_t k, size_t nproofs,
                          const void *prog, size_t ncons, size_t nregs, size_t blen, const void *zcoef, size_t zlen,
                          const uint64_t offset[2], const uint64_t omega[2], int log_n, size_t ef, void *stream);
/* sa_poly_degree_batch: degrees[b] = the highest j < n with coeffs[b n + j] != 0, or -1 for a zero row (int64,
 * device memory), for batch rows of n elements.  SA_ESIZE for n not a power of two in 1..2^30.  One memset and one
 * launch.                                                                                                       */
int sa_poly_degree_batch(long long *degrees, const void *coeffs, size_t n, size_t batch, void *stream);
/* sa_air_program: the transition constraints (sa_air_plan's coeffs, exps, term_start, HOST arrays) compiled into
 * the program sa_air_plan keeps in its plan, written to prog (device memory of sa_air_program_bytes(nterms, nregs)
 * bytes, nterms = term_start[ncons] - term_start[0]; 0 for unsupported sizes).  Synchronises.  SA_ESIZE for ncons
 * or nregs == 0 or a decreasing term_start.                                                                     */
size_t sa_air_program_bytes(size_t nterms, size_t nregs);
int sa_air_program(void *prog, const uint64_t *coeffs, const uint32_t *exps, const size_t *term_start, size_t ncons,
                   size_t nregs, void *stream);

/* ---- proof transcripts from their pickled bytes (csrc/transcript.cuh, DESIGN section 3.17) ----------------------
 * A verifier plan's shape is SA_TRANSCRIPT_SHAPE words: nregs, FRI rounds, k, the last codeword's length, log2 of
 * the FRI domain, the opened codewords, the weights, the pickle protocol, the expansion factor and the memo capacity
 * (see transcript.cuh for the shapes taken).  sa_transcript_bytes: one proof's device workspace in bytes, 0 for a
 * shape refused.                                                                                                 */
#define SA_TRANSCRIPT_SHAPE 10
#define SA_TRANSCRIPT_SECTIONS 15
#define SA_TRANSCRIPT_PREFIX 144 /* per proof: the prefix length (uint64), then at 16 up to 128 prefix bytes */
#define SA_TRANSCRIPT_OUT 80     /* per proof: the accepted flag (uint32), then at 16 the last FRI root */
size_t sa_transcript_bytes(const uint64_t shape[SA_TRANSCRIPT_SHAPE]);
/* sa_transcript_sections: for nproofs proofs (proof b is proof_at[2b + 1] bytes at proofs + proof_at[2b]; device
 * memory), parse each as the canonical pickle of a stream of the shape, hash its Fiat-Shamir messages with the
 * prefix of prefixes + SA_TRANSCRIPT_PREFIX b, draw its weights, alphas and indices, and write the chunk sections
 * VerifierPlan._pack writes at the byte offsets section_at of `sections` (zeroed by the caller): proof_data holds
 * the weights, then nstat elements of `statement` per proof, and zroot (64 bytes, NULL without a zerofier codeword)
 * is the root of the last opened codeword.  out gets SA_TRANSCRIPT_OUT bytes per proof.  A refused proof has flag
 * 0 and zero values in its sections.  workspace: nproofs * sa_transcript_bytes(shape) bytes.  Six launches, no
 * synchronisation.  SA_ESIZE before any launch for a refused shape, NULL buffers, nproofs or its products with the
 * shape's sizes at or above 2^59, or a prefix longer than 128 bytes is read as a refusal of that proof.         */
int sa_transcript_sections(void *sections, const uint64_t section_at[SA_TRANSCRIPT_SECTIONS], void *out,
                           void *workspace, const void *proofs, const uint64_t *proof_at, const void *prefixes,
                           const void *statement, size_t nstat, const void *zroot, size_t nproofs,
                           const uint64_t shape[SA_TRANSCRIPT_SHAPE], void *stream);

/* ---- self checks (used by tests / smoke) ------------------------------------------------
 * Runs the device carry-chain field arithmetic against the portable C++ version on
 * `count` pseudo-random pairs (plus edge cases) on the device; returns the number of
 * mismatches (0 = pass) or a negative SA_E* code.                                         */
long long sa_selftest_field(size_t count, uint64_t seed);
/* The same for the NTT tile's own product and butterfly (tile_mul, tile_bfly): npairs operand
 * pairs (x, w) from the caller, each element two little-endian 64-bit words below p (pairs[4k..4k+1]
 * = x, pairs[4k+2..4k+3] = w), then `count` pseudo-random and edge pairs; the butterfly's other
 * operand is drawn.  Returns the number of mismatches, SA_ESIZE for a missing list or an element
 * not below p, or a negative SA_E* code.                                                  */
long long sa_selftest_tile(size_t count, uint64_t seed, const uint64_t *pairs, size_t npairs);
/* Micro-benchmark: n_threads threads each run `iters` dependent rounds of `ilp`
 * independent operations of kind op (0 montmul, 1 add, 2 sub, 3 butterfly; 4 = blake2b node
 * compressions, 256 threads per block whatever `threads` says, ilp 1 or 2; 5 = op 3 through
 * the NTT tile's butterfly tile_bfly).  Returns the kernel time in milliseconds (negative on
 * error).                                                                                  */
double sa_microbench(int op, int ilp, int iters, int blocks, int threads);

#ifdef __cplusplus
}
#endif
#endif /* SA_B200_H */
