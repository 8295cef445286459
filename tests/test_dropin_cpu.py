"""Host-logic tests of the drop-in modules (no GPU): the engine is replaced by the
oracle-backed test double from tests/fake_engine.py.  Everything here is checked
against the reference's own outputs in tests/golden/."""
import pytest

import dropin_cases as C
import sa_engine
from fake_engine import OracleEngine


@pytest.fixture(autouse=True)
def double_engine():
    prev = sa_engine._ENGINE
    sa_engine.set_engine(OracleEngine())
    yield
    sa_engine.set_engine(prev)


def test_ntt_vectors():
    C.case_ntt_vectors()


def test_ntt_asserts():
    C.case_ntt_asserts()


def test_ntt_digests():
    C.case_ntt_digests(1 << 14)


def test_poly():
    C.case_poly()


def test_poly_asserts():
    C.case_poly_asserts()


def test_coset_offset_zero():
    C.case_coset_offset_zero()


def test_poly_split_recursion():
    C.case_poly_split_recursion()


def test_fast_multiply_4096():
    C.case_fast_multiply_big(1 << 12)


def test_fri_commit():
    C.case_fri_commit(1 << 12)


def test_fri_prove_and_verify():
    C.case_fri_prove(1 << 12)


def test_faststark_trace_replay():
    C.case_faststark_trace_replay()


def test_merkle_class():
    C.case_merkle_class()


def test_accel_polymul():
    C.case_accel_polymul()


def test_device_list():
    C.case_device_list()


def test_reference_style_properties():
    C.case_reference_style_properties()


def test_engine_use_is_recorded():
    """the drop-in really goes through the engine object (no hidden host arithmetic)"""
    eng = sa_engine.get_engine()
    C.N.ntt(C.T.field.primitive_nth_root(16), C.seeded(1, 16))
    assert ("ntt", 4, False, 1) in eng.calls


def test_merkle_tree_cache_is_per_engine():
    """a tree cached by fri.Merkle belongs to the engine that built it: after set_engine the new engine
    builds its own (a CUDA engine must never be handed a tree the test double made)"""
    xs = C.seeded(11, 64)
    first = sa_engine.get_engine()
    root = C.F.Merkle.commit(xs)
    assert ("merkle_tree", 64) in first.calls
    second = sa_engine.set_engine(OracleEngine())
    assert C.F.Merkle.commit(xs) == root
    assert ("merkle_tree", 64) in second.calls


def test_default_engine_fails_loudly_without_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    sa_engine.set_engine(None)
    with pytest.raises(RuntimeError, match="no CUDA device"):
        C.N.ntt(C.T.field.primitive_nth_root(16), C.seeded(1, 16))
