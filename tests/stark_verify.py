"""A test-side FastStark verifier, restated from the algorithm of the reference's FastStark.verify
(code/fast_stark.py:180-286), so that a device proof can be judged at sizes no test double reaches.

``verify`` gives the reference's accept/reject for a serialized proof.  ``combination_at`` is the verifier's
per-index equation (fast_stark.py:245-282): from the opened boundary-quotient values at i and i + expansion_factor,
the randomizer and zerofier values at i and the weights, it recomputes the combined codeword's value at i.  ``verify``
checks its FRI-opened indices with it, and the scale tests run the same function at every index they sweep, so a sweep
checks exactly what the verifier checks.

Everything besides FRI and the Merkle paths is Python ints: the boundary zerofiers and interpolants have a handful of
points, and a constraint is evaluated term by term.  The derived parameters and bounds are ``sa_stark.Params``'s,
FRI is the drop-in ``fri.Fri.verify``, and the stream and paths are the host types' ``ProofStream`` and
``Merkle.verify``."""
import sa_host
import sa_stark

P = sa_stark.P


def _eval(coeffs, x):
    acc = 0
    for c in reversed(coeffs):
        acc = (acc * x + c) % P
    return acc


def _mul_linear(coeffs, root):
    """coeffs * (X - root)"""
    out = [0] * (len(coeffs) + 1)
    for j, c in enumerate(coeffs):
        out[j + 1] = (out[j + 1] + c) % P
        out[j] = (out[j] - root * c) % P
    return out


def _interpolate(xs, ys):
    """Lagrange interpolant of the points, coefficients low to high"""
    acc = [0] * len(xs)
    for j, (xj, yj) in enumerate(zip(xs, ys)):
        basis, den = [1], 1
        for m, xm in enumerate(xs):
            if m != j:
                basis = _mul_linear(basis, xm)
                den = den * (xj - xm) % P
        f = yj * pow(den, P - 2, P) % P
        for k, b in enumerate(basis):
            acc[k] = (acc[k] + f * b) % P
    return acc


def _value(v):
    return int(getattr(v, "value", v))


class Statement:
    """What the verifier derives from the public input before it reads a proof: for every register the boundary
    zerofier and interpolant (fast_stark.py:53-67) as int coefficients, the transition quotients' and boundary
    quotients' shifts (fast_stark.py:272, 277), and the constraints as (exponent tuple, int) terms."""

    def __init__(self, stark, constraints, boundary):
        self.stark = stark
        nregs = stark.num_registers
        self.nregs = nregs
        self.omicron = stark.omicron.value
        self.generator = stark.generator.value
        self.omega = stark.omega.value
        self.n = stark.fri_domain_length
        self.expansion_factor = stark.expansion_factor
        # the trace length is inferred from the boundary (fast_stark.py:184-185)
        self.randomized_trace_length = 1 + max(int(c) for c, _, _ in boundary) + stark.num_randomizers
        self.zerofiers, self.interpolants = [], []
        for s in range(nregs):
            pts = [(pow(self.omicron, int(c), P), _value(v)) for c, r, v in boundary if int(r) == s]
            z = [1]
            for x, _ in pts:
                z = _mul_linear(z, x)
            self.zerofiers.append(z)
            self.interpolants.append(_interpolate([x for x, _ in pts], [y for _, y in pts]))
        self.terms = [sa_stark._terms(a) for a in constraints]
        max_degree = stark.max_degree(constraints)
        self.transition_shifts = [max_degree - b for b in stark.transition_quotient_degree_bounds(constraints)]
        self.boundary_shifts = [max_degree - b for b in
                                stark.boundary_quotient_degree_bounds(self.randomized_trace_length, boundary)]
        self.num_weights = 1 + 2 * len(self.terms) + 2 * nregs

    def point(self, i):
        """the FRI domain's i-th point, generator * omega^i (fast_stark.py:249)"""
        return self.generator * pow(self.omega, i % self.n, P) % P

    def trace_values(self, i, leaves):
        """the trace values at point i from the boundary-quotient values there (fast_stark.py:254-259)"""
        x = self.point(i)
        return [(_value(q) * _eval(z, x) + _eval(b, x)) % P
                for q, z, b in zip(leaves, self.zerofiers, self.interpolants)]

    def constraint_values(self, point):
        out = []
        for terms in self.terms:
            acc = 0
            for k, v in terms:
                t = v
                for x, e in zip(point, k):
                    if e:
                        t = t * pow(x, e, P) % P
                acc += t
            out.append(acc % P)
        return out


def combination_at(st, i, current, following, randomizer, zerofier, weights):
    """the verifier's combination value at FRI index i (fast_stark.py:245-279): `current` and `following` are the
    nregs boundary-quotient values at i and at (i + expansion_factor) % n, `randomizer` and `zerofier` the randomizer
    and transition zerofier codewords' values at i, `weights` the 1 + 2 * constraints + 2 * nregs weights"""
    x = st.point(i)
    point = [x] + st.trace_values(i, current) + st.trace_values(i + st.expansion_factor, following)
    zinv = pow(_value(zerofier), P - 2, P)
    terms = [_value(randomizer)]
    for tcv, shift in zip(st.constraint_values(point), st.transition_shifts):
        q = tcv * zinv % P
        terms += [q, q * pow(x, shift, P) % P]
    for bqv, shift in zip(current, st.boundary_shifts):
        bqv = _value(bqv)
        terms += [bqv, bqv * pow(x, shift, P) % P]
    assert len(terms) == len(weights), (len(terms), len(weights))
    return sum(t * _value(w) for t, w in zip(terms, weights)) % P


def weights(stark, proof, nconstraints):
    """the combination weights a verifier draws from the proof's first nregs + 1 roots (fast_stark.py:193-201)"""
    ps = sa_host.ip.ProofStream().deserialize(proof)
    for _ in range(stark.num_registers + 1):
        ps.pull()
    return [w.value for w in stark.sample_weights(1 + 2 * nconstraints + 2 * stark.num_registers,
                                                  ps.verifier_fiat_shamir())]


def verify(stark, proof, constraints, boundary, zerofier_root):
    """FastStark.verify's verdict (fast_stark.py:180-286) on a plain ProofStream's serialized proof"""
    merkle = sa_host.merkle.Merkle
    st = Statement(stark, constraints, boundary)
    n, ef = st.n, st.expansion_factor
    ps = sa_host.ip.ProofStream().deserialize(proof)

    # the boundary quotients' roots, the randomizer's root, then the weights (:192-201)
    roots = [ps.pull() for _ in range(st.nregs)]
    randomizer_root = ps.pull()
    w = [v.value for v in stark.sample_weights(st.num_weights, ps.verifier_fiat_shamir())]

    # FRI on the combined codeword, which also gives its values at the top-level indices (:203-211)
    opened = []
    if not stark.fri.verify(ps, opened):
        return False
    opened.sort(key=lambda iv: iv[0])

    # the leaves at each index and its neighbour, each with its path (:213-242); a repeated index is read again
    indices = sorted([i for i, _ in opened] + [(i + ef) % n for i, _ in opened])

    def read(root):
        leaves = {}
        for i in indices:
            leaves[i] = ps.pull()
            if not merkle.verify(root, i, ps.pull(), leaves[i]):
                return None
        return leaves
    opened_leaves = []
    for r in roots + [randomizer_root, zerofier_root]:
        leaves = read(r)
        if leaves is None:
            return False
        opened_leaves.append(leaves)
    boundary_leaves, randomizer, zerofier = opened_leaves[:-2], opened_leaves[-2], opened_leaves[-1]

    # the combination at every FRI-opened index (:244-284)
    for i, value in opened:
        j = (i + ef) % n
        got = combination_at(st, i, [b[i] for b in boundary_leaves], [b[j] for b in boundary_leaves],
                             randomizer[i], zerofier[i], w)
        if got != value.value:
            return False
    return True


# ---- the per-index equation over a whole codeword, for tests that hold the prover's buffers ----
def element(arr, i):
    """the residue at row i of a (n, 2) uint64 array of (lo, hi) limbs"""
    lo, hi = arr[i]
    return int(lo) | int(hi) << 64


def failures(st, indices, committed, combined, zerofier, w):
    """the indices among `indices` where combination_at, fed the prover's committed rows (nregs boundary codewords,
    then the randomizer codeword), the transition zerofier codeword and the weights w, differs from the combined
    codeword; every array is (n, 2) / (nregs + 1, n, 2) uint64 limbs on the host"""
    n, ef, nregs = st.n, st.expansion_factor, st.nregs
    bad = []
    for i in indices:
        j = (i + ef) % n
        got = combination_at(st, i, [element(committed[s], i) for s in range(nregs)],
                             [element(committed[s], j) for s in range(nregs)], element(committed[nregs], i),
                             element(zerofier, i), w)
        if got != element(combined, i):
            bad.append(i)
    return bad


class Recorder:
    """Wraps an engine's merkle_trees and coset_combine_evaluate for one prove (a context manager): `committed` is
    the one buffer committed with merkle_trees (the boundary codewords and the randomizer codeword), `terms` and
    `combined` the coset combination's terms and result.  `on_committed(vecs)` may change the buffer before it is
    committed and `on_terms(terms)` may return other terms to combine, so a test can perturb what the prover
    commits while the recorded terms stay the ones the prover asked for."""

    def __init__(self, eng, on_committed=None, on_terms=None):
        self.eng, self.on_committed, self.on_terms = eng, on_committed, on_terms
        self.trees_calls, self.committed, self.terms, self.combined = [], None, None, None

    def __enter__(self):
        eng = self.eng
        trees, combine = eng.merkle_trees, eng.coset_combine_evaluate

        def merkle_trees(vecs):
            self.trees_calls.append(tuple(vecs.shape))
            if self.on_committed is not None:
                self.on_committed(vecs)
            self.committed = vecs
            return trees(vecs)

        def coset_combine_evaluate(terms, log_n, root, offset):
            self.terms = list(terms)
            if self.on_terms is not None:
                terms = self.on_terms(list(terms))
            self.combined = combine(terms, log_n, root, offset)
            return self.combined
        eng.merkle_trees, eng.coset_combine_evaluate = merkle_trees, coset_combine_evaluate
        return self

    def __exit__(self, *exc):
        del self.eng.merkle_trees, self.eng.coset_combine_evaluate
        return False

    @property
    def weights(self):
        return [int(w) % P for _, _, w in self.terms]
