"""Cases of the plain prover tests (sa_stark.PlainStarkPlan), shared by the CPU suite (tests/test_stark_plain_cpu.py)
and the GPU suite (tests/test_gpu_stark_plain.py): tests/stark_cases.py's test double extended with the exact
transition quotients, a stand-in for the reference's Stark, the fixture tests/golden/stark_plain.json and a way to
run one of its cases.

The double's exact apply restates sa_air_quotients_exact from its definition: the coset quotient's row U_c at the
plan's order, and the flag set where U_c has a non-zero coefficient from n - deg Z on."""
import copy
import hashlib
import json
import os
import pickle
import random

import numpy as np

import stark_cases as C
import sa_stark
from sa_engine import REMAINDER, SA_ERRORS, SaError

P = C.P
T = C.T


class PlainStarkEngine(C.StarkEngine):
    name = "oracle-test-double-stark-plain"

    def air_plan(self, constraints, nregs, zerofier, max_ncoef, log_n, root, offset, step):
        plan = C.StarkEngine.air_plan(self, constraints, nregs, zerofier, max_ncoef, log_n, root, offset, step)
        plan.zdeg = zerofier.shape[0] - 1
        return plan

    def air_quotients_exact(self, plan, trace, qlen, check=True):
        self._log("air_quotients_exact", *trace.shape[:-1], qlen)
        n = 1 << plan.log_n
        if trace.ndim != 3 or trace.shape[0] != plan.nregs or not 1 <= trace.shape[1] <= plan.max_ncoef \
                or not 1 <= qlen <= n or plan.zdeg is None:
            raise SaError(SA_ERRORS[-6])
        air, z, step = plan.plan
        rows = [C.O.from_np(r) for r in trace]
        out = np.zeros((len(air), qlen, 2), np.uint64)
        flags = np.zeros(len(air), np.int32)
        for c, d in enumerate(air):
            _, u = C._coset_quotient(C.numerator(d, rows, step) or [0], z, n, plan.root, plan.offset)
            out[c] = C.O.scale_np(u[:qlen], C.O.inverse(plan.offset))
            flags[c] = int(u[n - plan.zdeg:].any())
        if check:
            bad = [c for c, f in enumerate(flags.tolist()) if f]
            if bad:
                raise SaError("%s (constraints %s)" % (REMAINDER, bad))
        return out, flags


# ---- a stand-in for the reference's Stark ----
def plain_stark(params):
    """a copy of a Params turned into what Stark keeps: the omicron domain as a list, and none of the derived lengths
    (randomized_trace_length, omicron_domain_length, fri_domain_length) as attributes"""
    params = copy.copy(params)
    params.omicron_domain = [T.fe(pow(params.omicron.value, i, P)) for i in range(params.omicron_domain_length)]
    del params.omicron_domain_length, params.fri_domain_length, params.randomized_trace_length
    return params


def stark(rec):
    return plain_stark(C.params(rec))


# ---- the fixture ----
def golden():
    """the fixture, with each signature's draw_stream [seed, skip, count] expanded into its draws (the seeded stream
    of make_golden_stark.Draws: 17 bytes of random.Random(seed).getrandbits(8) per value, reduced mod p) and air_of
    into the named case's AIR"""
    with open(os.path.join(C.HERE, "golden", "stark_plain.json")) as f:
        g = json.load(f)
    for rec in g.values():
        if "draw_stream" in rec:
            seed, skip, count = rec["draw_stream"]
            rng = random.Random(seed)
            values = [int.from_bytes(bytes(rng.getrandbits(8) for _ in range(17)), "big") % P
                      for _ in range(skip + count)]
            rec["draws"] = [str(v) for v in values[skip:]]
        if "air_of" in rec:
            rec["air"] = g[rec["air_of"]]["air"]
    return g


def run(stark, trace, constraints, boundary, draws, stream=None, plan=None):
    """one plain prove with os.urandom replaced by `draws`: the proof bytes or the AssertionError"""
    real = os.urandom
    os.urandom = draws
    try:
        if plan is not None:
            return plan.prove(trace, boundary, stream)
        return sa_stark.prove_plain(stark, trace, constraints, boundary, stream)
    except AssertionError as e:
        return e
    finally:
        os.urandom = real


def prefix_digests(objects, nregs, nquad):
    """make_golden_stark_plain.py's: after the boundary roots, the randomizer root, FRI and each of the nregs + 1
    opening blocks"""
    block = 2 * nquad
    after_fri = len(objects) - (nregs + 1) * block
    cuts = [nregs, nregs + 1, after_fri] + [after_fri + block * (j + 1) for j in range(nregs + 1)]
    return [hashlib.sha256(pickle.dumps(objects[:k])).hexdigest() for k in cuts]


def check(rec, proof, ps, draws):
    """a plain prove's result against the recorded one"""
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


def run_case(rec, plan=None, st=None):
    """(proof or AssertionError, stream, draws) of a fixture case through the current engine"""
    st = st or stark(rec)
    trace, boundary = C.inputs(rec)
    draws = C.Urandom(rec["draws"])
    ps = C.stream(rec)
    return run(st, trace, C.air(rec), boundary, draws, ps, plan), ps, draws


# ---- both provers on one AIR ----
def pair(params, cons, trace, boundary, values, zcw=None, zpoly=None):
    """(plain proof, FastStark proof) of one AIR, both drawing `values`: the plain proof's objects are the FastStark
    proof's without its zerofier openings.  zpoly / zcw default to stark_cases.zerofier's"""
    if zpoly is None:
        zpoly, zvals = C.zerofier(params)
        zcw = C.zerofier_codeword(zvals, True)
    fast = C.run(params, trace, cons, boundary, zpoly, zcw, C.Urandom(values))[0]
    plain = run(plain_stark(params), trace, cons, boundary, C.Urandom(values))
    return plain, fast


def without_zerofier_openings(fast, checks):
    """FastStark's proof objects minus the last 2 * 4 * checks: a value and a path per quadrupled index of the
    zerofier"""
    return pickle.loads(fast)[:-2 * 4 * checks]
