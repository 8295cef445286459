"""Cases of the device prover tests, shared by the CPU suite (tests/test_stark_cpu.py) and the GPU suite
(tests/test_gpu_stark.py): a test double that extends fake_engine.OracleEngine with the calls sa_stark makes, the
fixture tests/golden/stark.json and a way to run one of its cases, and seeded synthetic AIRs with valid traces.

The double computes each call's result from its definition with the CPU oracle: interpolation, the boundary
quotients and codewords (boundary_cases.expected, vectorised), the transition quotients on the coset
(air_cases.numerator divided at the plan's order), the coset combination (combine_cases' sum), batched trees, roots,
paths and gathers.  It is installed with sa_engine.set_engine by tests only."""
import hashlib
import json
import os
import pickle
import random
from hashlib import blake2s, shake_256

import numpy as np

import oracle as O
from air_cases import numerator
from boundary_cases import psub
from hostmirror_loader import load_host_types

T = load_host_types()  # puts the drop-in on sys.path

import sa_devlist  # noqa: E402
import sa_host  # noqa: E402
import sa_stark  # noqa: E402
from fake_engine import OracleEngine  # noqa: E402
from sa_engine import REMAINDER, SA_ERRORS, AirPlan, BoundaryPlan, InterpPlan, SaError  # noqa: E402

P = O.P
HERE = os.path.dirname(os.path.abspath(__file__))


def _row(coeffs, n):
    a = np.zeros((n, 2), np.uint64)
    if coeffs:
        a[:len(coeffs)] = O.to_np(coeffs)
    return a


def _coset_quotient(num, den, n, root, offset):
    """(cw, U) with cw = num(x_i) / den(x_i) on offset * <root> and U = intt(cw)"""
    ev = lambda c: O.ntt_np(root, O.scale_np(_row(c, n), offset))  # noqa: E731
    cw = O.pointwise_div_np(ev(num), ev(den))
    return cw, O.intt_np(root, cw)


class StarkEngine(OracleEngine):
    name = "oracle-test-double-stark"

    @staticmethod
    def _into(out, value):
        if out is None:
            return value
        if not isinstance(out, np.ndarray) or out.shape != value.shape:
            raise SaError(SA_ERRORS[-6])
        out[...] = value
        return out

    def interp_plan(self, domain):
        self._log("interp_plan", domain.shape[0])
        return InterpPlan(np.ascontiguousarray(domain), domain.shape[0])

    def interp_apply(self, plan, values):
        self._log("interp_apply", *values.shape[:-1])
        if values.ndim not in (2, 3) or tuple(values.shape[-2:]) != (plan.k, 2):
            raise SaError(SA_ERRORS[-6])
        rows = values.reshape(-1, plan.k, 2)
        return np.stack([O.interpolate_np(plan.plan, r) for r in rows]).reshape(values.shape)

    def coset_evaluate(self, coeffs, log_n, root, offset, out=None):
        return self._into(out, OracleEngine.coset_evaluate(self, coeffs, log_n, root, offset))

    def boundary_plan(self, boundary, nregs, omicron, log_n, root, offset):
        self._log("boundary_plan", nregs, log_n)
        if nregs < 1 or not 1 <= log_n <= 30 or int(offset) % P == 0:
            raise SaError(SA_ERRORS[-6])
        w = int(getattr(omicron, "value", omicron))
        points = [[] for _ in range(nregs)]
        for c, r, v in boundary:
            if not 0 <= int(r) < nregs:
                raise SaError(SA_ERRORS[-6])
            points[int(r)].append((pow(w, int(c), P), int(getattr(v, "value", v))))
        if any(not 1 <= len(pts) < 1 << log_n for pts in points):
            raise SaError(SA_ERRORS[-6])
        rows = []
        for pts in points:
            xs = O.to_np([x for x, _ in pts])
            try:
                i = O.from_np(O.interpolate_np(xs, O.to_np([v for _, v in pts])))
            except AssertionError:
                raise SaError(SA_ERRORS[-4])
            rows.append((O.from_np(O.zerofier_np(xs)), i))
        return BoundaryPlan(rows, log_n, int(root), int(offset) % P, nregs, [len(pts) for pts in points])

    def boundary_quotients(self, plan, trace, check=True, out=None):
        self._log("boundary_quotients", *trace.shape[:-1])
        n = 1 << plan.log_n
        if trace.ndim != 3 or trace.shape[0] != plan.nregs or not 1 <= trace.shape[1] <= n:
            raise SaError(SA_ERRORS[-6])
        ncoef = trace.shape[1]
        quot = np.zeros((plan.nregs, ncoef, 2), np.uint64)
        cws = np.zeros((plan.nregs, n, 2), np.uint64)
        flags = np.zeros(plan.nregs, np.int32)
        for s, (z, i) in enumerate(plan.plan):
            cw, u = _coset_quotient(psub(O.from_np(trace[s]), i), z, n, plan.root, plan.offset)
            cws[s] = cw
            quot[s] = O.scale_np(u[:ncoef], O.inverse(plan.offset))
            flags[s] = int(u[max(0, ncoef - (len(z) - 1)):].any())
        cws = self._into(out, cws)
        if check:
            bad = [s for s, f in enumerate(flags.tolist()) if f]
            if bad:
                raise SaError("%s (registers %s)" % (REMAINDER, bad))
        return quot, cws, flags

    def air_plan(self, constraints, nregs, zerofier, max_ncoef, log_n, root, offset, step):
        self._log("air_plan", len(constraints), log_n)
        n = 1 << log_n
        if nregs < 1 or not constraints or not 1 <= max_ncoef <= n:
            raise SaError(SA_ERRORS[-6])
        nvars = 1 + 2 * nregs
        air = []
        for a in constraints:
            d = {}
            for k, v in getattr(a, "dictionary", a).items():
                k = tuple(int(e) for e in k) + (0,) * (nvars - len(k))
                if k[0] + sum(k[1:]) * (max_ncoef - 1) >= n:
                    raise SaError(SA_ERRORS[-6])
                d[k] = (d.get(k, 0) + int(getattr(v, "value", v))) % P
            air.append(d)
        z = O.from_np(zerofier)
        if not O.ntt_np(root, O.scale_np(_row(z, n), offset)).any(axis=1).all():
            raise SaError(SA_ERRORS[-4])
        return AirPlan((air, z, int(step)), log_n, int(root), int(offset), nregs, len(air), max_ncoef)

    def air_quotients(self, plan, trace, qlen):
        self._log("air_quotients", *trace.shape[:-1], qlen)
        n = 1 << plan.log_n
        if trace.ndim != 3 or trace.shape[0] != plan.nregs or not 1 <= trace.shape[1] <= plan.max_ncoef \
                or not 1 <= qlen <= n:
            raise SaError(SA_ERRORS[-6])
        air, z, step = plan.plan
        rows = [O.from_np(r) for r in trace]
        out = np.zeros((len(air), qlen, 2), np.uint64)
        for c, d in enumerate(air):
            _, u = _coset_quotient(numerator(d, rows, step) or [0], z, n, plan.root, plan.offset)
            out[c] = O.scale_np(u[:qlen], O.inverse(plan.offset))
        return out

    def coset_combine_evaluate(self, terms, log_n, root, offset):
        self._log("coset_combine_evaluate", len(terms), log_n)
        n = 1 << log_n
        c = [0] * n
        for vec, shift, w in terms:
            if vec.ndim != 2 or vec.shape[1] != 2 or shift < 0 or shift + vec.shape[0] > n:
                raise SaError(SA_ERRORS[-6])
            w = int(w) % P
            for j, v in enumerate(O.from_np(vec)):
                c[shift + j] = (c[shift + j] + w * v) % P
        return O.to_np(O.fast_coset_evaluate(c, offset, root, n))

    def merkle_trees(self, vecs):
        self._log("merkle_trees", *vecs.shape[:-1])
        return np.stack([O.merkle_tree_np(v) for v in vecs])

    def tree_roots(self, trees):
        return [t[1].tobytes() for t in trees]

    def merkle_open_batch(self, trees, indices):
        self._log("merkle_open_batch", trees.shape[0], len(indices))
        n = trees.shape[1] // 2
        for i in indices:
            if not 0 <= i < n:
                raise SaError(SA_ERRORS[-5])
        return [[O.merkle_open(t, i) if n > 1 else [] for i in indices] for t in trees]

    def gather_batch(self, vecs, indices):
        self._log("gather_batch", vecs.shape[0], len(indices))
        return np.ascontiguousarray(vecs[:, list(indices)])


# ---- the proof streams ----
class SignatureProofStream(sa_host.ip.ProofStream):
    """FastRPSSS's signature stream: Fiat-Shamir over blake2s(document) followed by the serialized stream"""

    def __init__(self, document):
        sa_host.ip.ProofStream.__init__(self)
        self.document = document
        self.prefix = blake2s(bytes(document)).digest()

    def prover_fiat_shamir(self, num_bytes=32):
        return shake_256(self.prefix + self.serialize()).digest(num_bytes)


class Urandom:
    """os.urandom handing back recorded field values as 17 big-endian bytes, counting the draws"""

    def __init__(self, values):
        self.values, self.count = [int(v) for v in values], 0

    def __call__(self, n):
        assert n == 17
        v = self.values[self.count] if self.count < len(self.values) else 0
        self.count += 1
        return v.to_bytes(17, "big")


# ---- the fixture ----
def golden():
    with open(os.path.join(HERE, "golden", "stark.json")) as f:
        return json.load(f)


def params(rec):
    p = rec["params"]
    return sa_stark.Params(T.field, p["expansion_factor"], p["num_colinearity_checks"], p["security_level"],
                           p["num_registers"], p["num_cycles"], p["transition_constraints_degree"])


def air(rec):
    return [{tuple(t["e"]): T.fe(t["c"]) for t in cons} for cons in rec["air"]]


def zerofier(stark):
    """FastStark.preprocess: the zerofier of omicron^i, i < num_cycles - 1, and its codeword on the FRI domain"""
    w = stark.omicron.value
    z = O.from_np(O.zerofier_np(O.to_np([pow(w, i, P) for i in range(stark.original_trace_length - 1)])))
    cw = O.fast_coset_evaluate(z, stark.generator.value, stark.omega.value, stark.fri_domain_length)
    return T.Polynomial(T.elems(z)), cw


def zerofier_codeword(values, device_list):
    if device_list:
        return sa_devlist.DeviceCodeword(sa_devlist.to_device(T.elems(values)), None, T.field, len(values))
    return T.elems(values)


def run(stark, trace, constraints, boundary, zpoly, zcw, draws, stream=None, plan=None):
    """one prove with os.urandom replaced by `draws`: (proof bytes or the AssertionError, the stream)"""
    real = os.urandom
    os.urandom = draws
    try:
        if plan is not None:
            proof = plan.prove(trace, boundary, zcw, stream)
        else:
            proof = sa_stark.prove(stark, trace, constraints, boundary, zpoly, zcw, stream)
    except AssertionError as e:
        return e, stream
    finally:
        os.urandom = real
    return proof, stream


def inputs(rec):
    trace = [T.elems(row) for row in rec["trace"]]
    boundary = [(int(c), int(r), T.fe(v)) for c, r, v in rec["boundary"]]
    return trace, boundary


def stream(rec):
    if rec["stream"] == "signature":
        return SignatureProofStream(bytes.fromhex(rec["document"]))
    return sa_host.ip.ProofStream()


def prefix_digests(objects, nregs, nquad):
    block = 2 * nquad
    after_fri = len(objects) - (nregs + 2) * block
    cuts = [nregs, nregs + 1, after_fri] + [after_fri + block * (j + 1) for j in range(nregs + 2)]
    return [hashlib.sha256(pickle.dumps(objects[:k])).hexdigest() for k in cuts]


def check(rec, proof, ps, draws):
    """a prove's result against the recorded one"""
    assert draws.count == len(rec["draws"]), (draws.count, len(rec["draws"]))
    if "raises" in rec:
        assert isinstance(proof, AssertionError), "the reference raised %r" % rec["raises"]
        assert str(proof).startswith(rec["raises"]), (str(proof), rec["raises"])
        return
    assert not isinstance(proof, AssertionError), proof
    objects = pickle.loads(proof)
    nquad = 4 * rec["params"]["num_colinearity_checks"]
    assert prefix_digests(objects, rec["params"]["num_registers"], nquad) == rec["prefix_sha256"]
    assert (hashlib.sha256(proof).hexdigest(), len(proof)) == (rec["proof_sha256"], rec["proof_len"])
    if ps is not None:
        assert ps.serialize() == proof


def run_case(rec, device_list=True, plan=None, stark=None):
    """(proof or AssertionError, stream, draws) of a fixture case through the current engine"""
    stark = stark or params(rec)
    zpoly, zvals = zerofier(stark)
    trace, boundary = inputs(rec)
    draws = Urandom(rec["draws"])
    ps = stream(rec)
    proof, ps = run(stark, trace, air(rec), boundary, zpoly, zerofier_codeword(zvals, device_list), draws, ps, plan)
    return proof, ps, draws


# ---- seeded synthetic AIRs ----
def synthetic(seed, log_fri, nregs=3):
    """(Params, constraints as {exponent tuple: int}, trace rows, boundary) of a valid AIR whose FRI domain has
    2^log_fri points: register i's next value is a seeded polynomial in the current row (register 0's cubic,
    register 1's linear with an x term, the others quadratic), 2 colinearity checks, expansion factor 4"""
    rng = random.Random(seed)
    n = 1 << log_fri
    ncycles = n // 16 - 8  # randomized length n / 16, times 3 below n / 4: omicron domain n / 4
    stark = sa_stark.Params(T.field, 4, 2, 4, nregs, ncycles, transition_constraints_degree=3)
    assert stark.fri_domain_length == n
    nvars = 1 + 2 * nregs
    cons, maps = [], []
    for i in range(nregs):
        degree = 3 if i == 0 else 1 if i == 1 else 2
        terms = {}
        for _ in range(1 + rng.randrange(3)):
            e = [0] * nvars
            for _ in range(rng.randrange(degree + 1)):
                e[1 + rng.randrange(nregs)] += 1
            terms[tuple(e)] = rng.randrange(1, P)
        top = [0] * nvars
        for _ in range(degree):
            top[1 + rng.randrange(nregs)] += 1
        terms[tuple(top)] = rng.randrange(1, P)
        if i == 1:
            terms[tuple([1] + [0] * (nvars - 1))] = rng.randrange(1, P)
        maps.append(terms)
        nxt = [0] * nvars
        nxt[1 + nregs + i] = 1
        d = {tuple(nxt): 1}
        for k, v in terms.items():
            d[k] = (d.get(k, 0) - v) % P
        cons.append(d)
    w = stark.omicron.value
    row = [rng.randrange(P) for _ in range(nregs)]
    rows = [row]
    for c in range(ncycles - 1):
        x = pow(w, c, P)
        nxt = []
        for terms in maps:
            acc = 0
            for k, v in terms.items():
                t = v * pow(x, k[0], P)
                for j, e in enumerate(k[1:1 + nregs]):
                    t = t * pow(row[j], e, P)
                acc += t
            nxt.append(acc % P)
        row = nxt
        rows.append(row)
    boundary = [(0, s, rows[0][s]) for s in range(nregs)] + [(ncycles - 1, 0, rows[-1][0])]
    boundary += [(c, 1, rows[c][1]) for c in rng.sample(range(1, ncycles - 1), 2)]
    trace = [T.elems(r) for r in rows]
    return stark, cons, trace, [(c, r, T.fe(v)) for c, r, v in boundary]


def synthetic_prove(seed, log_fri, nregs=3):
    """a synthetic case's proof with os.urandom from random.Random(seed): (proof, draws)"""
    stark, cons, trace, boundary = synthetic(seed, log_fri, nregs)
    zpoly, zvals = zerofier(stark)
    rng = random.Random(seed)
    draws = Urandom([rng.randrange(P) for _ in range(nregs * stark.num_randomizers + stark.fri_domain_length)])
    proof, _ = run(stark, trace, cons, boundary, zpoly, zerofier_codeword(zvals, True), draws)
    return proof, draws.count
