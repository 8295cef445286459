"""Cases of the batched prover tests (StarkPlan.prove_batch, PlainStarkPlan.prove_batch, sa_stark.sign_batch),
shared by the CPU suite (tests/test_stark_batch_cpu.py) and the GPU suite (tests/test_gpu_stark_batch.py): the test
double of tests/stark_plain_cases.py extended with the batch forms of its calls, each restated as the single call per
trace, row or group; the batch draw streams assembled from per-proof draws; and a stand-in signer."""
import os

import numpy as np

import stark_cases as C
import stark_plain_cases as S
import sa_stark
from sa_engine import SA_ERRORS, SaError


class BatchStarkEngine(S.PlainStarkEngine):
    name = "oracle-test-double-stark-batch"

    def air_quotients(self, plan, trace, qlen):
        if trace.ndim != 4:
            return S.PlainStarkEngine.air_quotients(self, plan, trace, qlen)
        return np.stack([S.PlainStarkEngine.air_quotients(self, plan, t, qlen) for t in trace])

    def air_quotients_exact(self, plan, trace, qlen, check=True):
        if trace.ndim != 4:
            return S.PlainStarkEngine.air_quotients_exact(self, plan, trace, qlen, check)
        got = [S.PlainStarkEngine.air_quotients_exact(self, plan, t, qlen, False) for t in trace]
        flags = np.stack([f for _, f in got])
        if check and flags.any():
            raise SaError("%s (constraints %s)" % (C.REMAINDER, np.argwhere(flags).tolist()))
        return np.stack([q for q, _ in got]), flags

    def coset_combine_evaluate_batch(self, terms, nrows, log_n, root, offset):
        self._log("coset_combine_evaluate_batch", len(terms), nrows, log_n)
        for t in terms:
            if not 0 <= int(t[3]) < nrows:
                raise SaError(SA_ERRORS[-6])
        return np.stack([self.coset_combine_evaluate([t[:3] for t in terms if t[3] == r], log_n, root, offset)
                         for r in range(nrows)])

    @staticmethod
    def _sets(batch, indices, group):
        if group is None:
            return [list(indices)] * batch
        sets = [list(s) for s in indices]
        if group < 1 or len(sets) != max(1, -(-batch // group)) or len({len(s) for s in sets}) > 1:
            raise SaError(SA_ERRORS[-6])
        return [sets[b // group] for b in range(batch)]

    def gather_batch(self, vecs, indices, group=None):
        sets = self._sets(vecs.shape[0], indices, group)
        self._log("gather_batch", vecs.shape[0], len(sets[0]) if sets else 0)
        return np.stack([v[s] for v, s in zip(vecs, sets)]) if sets else np.zeros((0, 0, 2), np.uint64)

    def merkle_open_batch(self, trees, indices, group=None):
        sets = self._sets(trees.shape[0], indices, group)
        self._log("merkle_open_batch", trees.shape[0], len(sets[0]) if sets else 0)
        n = trees.shape[1] // 2
        for s in sets:
            for i in s:
                if not 0 <= i < n:
                    raise SaError(SA_ERRORS[-5])
        return [[C.O.merkle_open(t, i) if n > 1 else [] for i in s] for t, s in zip(trees, sets)]


def batch_draws(draws, ntrace):
    """the batch's draw stream from each proof's own: every proof's first ntrace draws (its trace randomizers), then
    every proof's remaining ones (its randomizer coefficients)"""
    return [d for ds in draws for d in ds[:ntrace]] + [d for ds in draws for d in ds[ntrace:]]


def run_batch(plan, traces, boundaries, draws, streams=None, zcw=None):
    """plan.prove_batch with os.urandom replaced by `draws`: the proof list or the AssertionError"""
    real = os.urandom
    os.urandom = draws
    try:
        if zcw is None:
            return plan.prove_batch(traces, boundaries, streams)
        return plan.prove_batch(traces, boundaries, zcw, streams)
    except (AssertionError, IndexError) as e:
        return e
    finally:
        os.urandom = real


def ntrace(rec):
    p = rec["params"]
    return p["num_registers"] * p["num_randomizers"]


class Signer:
    """a stand-in for RPSSS / FastRPSSS over a fixture case: rp gives the case's trace, boundary and AIR, stark is its
    Params (or its plain-Stark restatement), and sign(sk, d) proves one document with the case's draws installed by
    the caller.  Its module is stark_cases, whose SignatureProofStream sign_batch picks up."""
    __module__ = C.__name__

    def __init__(self, rec, fast):
        self.rec = rec
        self.stark = C.params(rec) if fast else S.stark(rec)
        trace, boundary = C.inputs(rec)
        air = C.air(rec)
        self.rp = type("RP", (), {
            "hash": staticmethod(lambda sk: "out"),
            "trace": staticmethod(lambda sk: trace),
            "boundary_constraints": staticmethod(lambda out: boundary),
            "transition_constraints": staticmethod(lambda omicron: air),
        })()
        if fast:
            zpoly, zvals = C.zerofier(self.stark)
            self.transition_zerofier = zpoly
            self.transition_zerofier_codeword = C.zerofier_codeword(zvals, True)

    def sign(self, sk, document):
        ps = C.SignatureProofStream(document)
        if hasattr(self, "transition_zerofier"):
            return sa_stark.prove(self.stark, self.rp.trace(sk), self.rp.transition_constraints(None),
                                  self.rp.boundary_constraints(None), self.transition_zerofier,
                                  self.transition_zerofier_codeword, ps)
        return sa_stark.prove_plain(self.stark, self.rp.trace(sk), self.rp.transition_constraints(None),
                                    self.rp.boundary_constraints(None), ps)
