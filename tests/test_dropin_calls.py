"""Pin on the engine calls the drop-in modules make (no GPU).

Every workload below runs on a fresh tests/fake_engine.OracleEngine and its call log is compared with
tests/golden/dropin_calls.json as a multiset: the same calls with the same sizes, in any order.  A change
to the Python layer that adds a host<->device crossing (an upload, a download, a whole-tree download)
or drops a kernel shows up here even when every value it returns is still right.  After a deliberate
change to the calls, ``python tests/test_dropin_calls.py`` re-records the fixture.
"""
import collections
import hashlib
import json
import os
import pickle

import pytest

import dropin_cases as C
import sa_devlist
import sa_engine
from conftest import GOLDEN, load_golden
from fake_engine import OracleEngine

T, N, F = C.T, C.N, C.F
FIXTURE = os.path.join(GOLDEN, "dropin_calls.json")


def _record(run):
    """the engine calls `run` makes, as {"name arg ...": count}"""
    eng = sa_engine.set_engine(OracleEngine())
    run()
    return dict(collections.Counter(" ".join(str(a) for a in call) for call in eng.calls))


def _fri_prove(n, resident):
    c = [c for c in load_golden("fri.json")["prove"] if c["n"] == n][0]
    omega, g = T.field.primitive_nth_root(n), T.field.generator()
    codeword = N.fast_coset_evaluate(T.poly(c["coeffs"]), g, omega, n)
    if not resident:
        codeword = codeword.tolist()

    def run():
        ps = F.ProofStream()
        ps.push(b"prior-object")
        assert F.Fri(g, omega, n, c["ef"], c["tests"]).prove(codeword, ps) == c["indices"]
        assert hashlib.sha256(pickle.dumps(ps.objects)).hexdigest() == c["transcript_sha256"]
    return _record(run)


def _merkle_opens(resident):
    xs = C.seeded(61, 1024)
    data = F.DeviceCodeword(sa_devlist.to_device(xs), None, T.field) if resident else xs
    host = F._HostMerkle

    def run():
        paths = [F.Merkle.open(i, data) for i in range(1024)]
        assert paths[0] == host.open(0, xs) and paths[777] == host.open(777, xs)
    return _record(run)


def _products():
    w, g = T.field.primitive_nth_root(64), T.field.generator()
    lhs, rhs = T.Polynomial(C.seeded(62, 40)), T.Polynomial(C.seeded(63, 23))
    zero_at_coset = T.poly([(-g).value, 1]) * T.poly([1] * 9)  # X - g vanishes at g*w^0

    def run():
        product = N.fast_multiply(lhs, rhs, w, 64)
        assert product == lhs * rhs
        assert N.fast_coset_divide(product, rhs, g, w, 64) == lhs
        with pytest.raises(AssertionError, match="divide by zero"):
            N.fast_coset_divide(product, zero_at_coset, g, w, 64)
    return _record(run)


WORKLOADS = {
    "faststark_trace_replay": lambda: _record(C.case_faststark_trace_replay),
    "fri_prove_64_list": lambda: _fri_prove(64, False),
    "fri_prove_64_device": lambda: _fri_prove(64, True),
    "fri_prove_1024_list": lambda: _fri_prove(1024, False),
    "fri_prove_1024_device": lambda: _fri_prove(1024, True),
    "merkle_open_1024_list": lambda: _merkle_opens(False),
    "merkle_open_1024_device": lambda: _merkle_opens(True),
    "fast_multiply_and_coset_divide": _products,
    "accel_polymul": lambda: _record(C.case_accel_polymul),
    "poly_golden": lambda: _record(C.case_poly),
    "device_list": lambda: _record(C.case_device_list),
}


@pytest.fixture(autouse=True)
def double_engine():
    prev = sa_engine._ENGINE
    sa_engine.set_engine(OracleEngine())
    yield
    sa_engine.set_engine(prev)


@pytest.mark.parametrize("name", sorted(WORKLOADS))
def test_engine_calls(name):
    with open(FIXTURE) as f:
        want = json.load(f)[name]
    assert WORKLOADS[name]() == want


if __name__ == "__main__":
    prev = sa_engine._ENGINE
    try:
        logs = {name: WORKLOADS[name]() for name in sorted(WORKLOADS)}
    finally:
        sa_engine.set_engine(prev)
    with open(FIXTURE, "w") as f:
        json.dump(logs, f, indent=1, sort_keys=True)
        f.write("\n")
