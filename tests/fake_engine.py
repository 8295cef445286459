"""TEST DOUBLE for sa_engine.CudaEngine, backed by the CPU oracle.

It lets the ``not gpu`` tests drive the drop-in modules' HOST logic (marshalling,
list-length semantics, proof-stream pushes and object identity, assertion
messages) in this GPU-less container -- including running the reference's
unmodified code/fast_stark.py against the drop-in.  It lives in tests/ and is
installed with ``sa_engine.set_engine`` by tests only; the product's default
engine is the CUDA one and has no fallback.
"""
import numpy as np

import oracle as O
from coset_cases import formula
from sa_engine import SA_ERRORS, CosetDivPlan, SaError


class OracleEngine:
    name = "oracle-test-double"

    def __init__(self):
        self.calls = []

    def _log(self, name, *shape):
        self.calls.append((name,) + shape)

    # -------------------------------------------------------------- plumbing
    def empty(self, n):
        return np.zeros((n, 2), dtype=np.uint64)

    zeros = empty

    def length(self, vec):
        return vec.shape[0]

    def upload(self, buf):
        self._log("upload", len(buf) // 16 if not isinstance(buf, np.ndarray) else buf.size // 2)
        if isinstance(buf, np.ndarray):
            return buf.reshape(-1, 2).astype(np.uint64)
        return np.frombuffer(bytes(buf), dtype="<u8").reshape(-1, 2).copy()

    def download(self, vec):
        self._log("download", vec.shape[0])
        return np.ascontiguousarray(vec)

    def pad(self, vec, n):
        out = np.zeros((n, 2), dtype=np.uint64)
        out[:vec.shape[0]] = vec
        return out

    def slice(self, vec, lo, hi):
        return vec[lo:hi]

    def concat(self, vecs):
        return np.concatenate(vecs, axis=0)

    # ------------------------------------------------------------------- ops
    def ntt(self, vec, log_n, root, inverse=False, batch=1):
        self._log("ntt", log_n, inverse, batch)
        n = 1 << log_n
        assert vec.shape[0] == n * batch
        fn = O.intt_np if inverse else O.ntt_np
        try:
            return np.concatenate([fn(root, vec[b * n:(b + 1) * n]) for b in range(batch)], axis=0)
        except AssertionError as e:
            raise SaError(str(e))

    def ntt_into(self, out, vec, log_n, root, inverse=False, batch=1):
        out[:] = self.ntt(vec, log_n, root, inverse=inverse, batch=batch)
        return out

    def pointwise_mul(self, a, b):
        self._log("pointwise_mul", a.shape[0])
        return O.pointwise_mul_np(np.ascontiguousarray(a), np.ascontiguousarray(b))

    @staticmethod
    def _coset_rows(vecs, n):
        """CudaEngine._rows: the rows of a (ncoef, 2) or (B, ncoef, 2) array with 1 <= ncoef <= n"""
        if vecs.ndim not in (2, 3) or vecs.shape[-1] != 2 or not 1 <= vecs.shape[-2] <= n:
            raise SaError(SA_ERRORS[-6])
        return vecs.reshape(-1, vecs.shape[-2], 2)

    @staticmethod
    def _oracle_ntt_check(fn, *args):
        try:
            return fn(*args)
        except AssertionError as e:
            raise SaError(str(e))

    def coset_div_plan(self, divisor, log_n, root, offset):
        self._log("coset_div_plan", divisor.shape[0], log_n)
        if not 1 <= log_n <= 30 or divisor.ndim != 2:
            raise SaError(SA_ERRORS[-6])
        n = 1 << log_n
        self._coset_rows(divisor, n)
        scaled = np.zeros((n, 2), np.uint64)
        scaled[:divisor.shape[0]] = O.scale_np(divisor, offset)
        if not self._oracle_ntt_check(O.ntt_np, root, scaled).any(axis=1).all():
            raise SaError(SA_ERRORS[-4])
        return CosetDivPlan(O.from_np(divisor), log_n, root, offset)

    def coset_div_apply(self, plan, lhs, qlen):
        self._log("coset_div_apply", lhs.shape[-2], qlen)
        n = 1 << plan.log_n
        rows = self._coset_rows(lhs, n)
        if not 1 <= qlen <= n:
            raise SaError(SA_ERRORS[-6])
        out = np.zeros((rows.shape[0], qlen, 2), np.uint64)
        for b, row in enumerate(rows):
            out[b] = O.to_np(formula(O.from_np(row), plan.plan, plan.offset, plan.root, n, qlen))
        return out.reshape(lhs.shape[:-2] + (qlen, 2))

    def coset_evaluate(self, coeffs, log_n, root, offset):
        self._log("coset_evaluate", coeffs.shape[-2], log_n)
        if not 1 <= log_n <= 30:
            raise SaError(SA_ERRORS[-6])
        n = 1 << log_n
        rows = self._coset_rows(coeffs, n)
        out = np.zeros((rows.shape[0], n, 2), np.uint64)
        for b, row in enumerate(rows):
            out[b] = O.to_np(self._oracle_ntt_check(O.fast_coset_evaluate, O.from_np(row), offset, root, n))
        return out.reshape(coeffs.shape[:-2] + (n, 2))

    def poly_eval(self, coeffs, points):
        self._log("poly_eval", coeffs.shape[0], points.shape[0])
        return O.poly_eval_np(coeffs, points)

    MAX_DIRECT_POINTS = 1 << 20

    def zerofier(self, domain):
        self._log("zerofier", domain.shape[0])
        return O.zerofier_np(domain)

    def interpolate(self, domain, values):
        self._log("interpolate", domain.shape[0])
        try:
            return O.interpolate_np(domain, values)
        except AssertionError:
            raise SaError(SA_ERRORS[-4])

    def merkle_tree(self, vec):
        self._log("merkle_tree", vec.shape[0])
        return O.merkle_tree_np(vec)

    def tree_root(self, tree):
        return tree[1].tobytes()

    def download_tree(self, tree):
        self._log("download_tree", tree.shape[0] // 2)
        return np.ascontiguousarray(tree)

    def merkle_open(self, tree, indices):
        self._log("merkle_open", len(indices))
        n = tree.shape[0] // 2
        for i in indices:
            if not 0 <= i < n:
                raise SaError(SA_ERRORS[-5])
        return [O.merkle_open(tree, i) if n > 1 else [] for i in indices]

    def gather(self, vec, indices):
        self._log("gather", len(indices))
        return np.ascontiguousarray(vec[list(indices)]) if len(indices) else np.zeros((0, 2), np.uint64)

    def fri_fold(self, vec, alpha, offset, omega):
        self._log("fri_fold", vec.shape[0])
        return O.fri_fold_np(vec, alpha, offset, omega)

    def fri_round(self, vec, alpha, offset, omega):
        self._log("fri_round", vec.shape[0])
        nxt = O.fri_fold_np(vec, alpha, offset, omega)
        return nxt, O.merkle_tree_np(nxt)

    def fri_commit(self, vec, rounds, offset, omega, on_root):
        self._log("fri_commit", vec.shape[0], rounds)
        layers, trees = [vec], []
        cur = vec
        for r in range(rounds):
            tree = O.merkle_tree_np(cur)
            trees.append(tree)
            want = r != rounds - 1
            alpha = on_root(r, tree[1].tobytes(), want)
            if not want:
                break
            cur = O.fri_fold_np(cur, alpha, offset, omega)
            layers.append(cur)
            omega, offset = omega * omega % O.P, offset * offset % O.P
        return layers, trees

    def synchronize(self):
        pass

    def launch_count(self):
        return 0
