"""Cases of the seeded prover tests, shared by the CPU suite (tests/test_stark_seeded_cpu.py) and the GPU suite
(tests/test_gpu_stark_seeded.py): the batch test double of tests/stark_batch_cases.py plus sample_seeded on the CPU
emulation of csrc/sample.cuh, and the two ways to prove with seeds: the seeded provers with os.urandom refused, and
the host route, each proof alone with os.urandom = sa_stark.seeded_urandom(its seed)."""
import ctypes
import hashlib
import os

import numpy as np

import __graft_entry__ as G
import stark_batch_cases as SB
import sa_stark
from sa_engine import SA_ERRORS, SaError

_EMU = None


def emu():
    global _EMU
    if _EMU is None:
        lib = ctypes.CDLL(G.build_emu_sample())
        lib.emu_sample_seeded.restype = ctypes.c_int
        lib.emu_sample_seeded.argtypes = [ctypes.c_void_p, ctypes.c_char_p] + [ctypes.c_size_t] * 2 + \
            [ctypes.c_uint64] + [ctypes.c_size_t] * 3 + [ctypes.c_longlong]
        _EMU = lib
    return _EMU


class SeededStarkEngine(SB.BatchStarkEngine):
    name = "oracle-test-double-stark-seeded"

    def upload_seeds(self, seeds):
        if not all(isinstance(s, bytes) and len(s) == 32 for s in seeds):
            raise SaError(SA_ERRORS[-6])
        self._log("upload_seeds", len(seeds))
        return np.frombuffer(b"".join(seeds), dtype=np.uint8).reshape(-1, 32).copy()

    def sample_seeded(self, out, seeds, first, count, width=1, lane_stride=1, seed_stride=None, offset=0):
        """CudaEngine.sample_seeded's checks, then the emulated kernel over a grid of 37 threads"""
        if not isinstance(seeds, np.ndarray):
            seeds = self.upload_seeds(list(seeds))
        seed_stride = count if seed_stride is None else seed_stride
        self._log("sample_seeded", seeds.shape[0], first, count, width)
        if width < 1 or out.dtype != np.uint64 or not out.flags.c_contiguous:
            raise SaError(SA_ERRORS[-6])
        if seeds.shape[0] == 0 or count == 0:
            return out
        last = offset + (seeds.shape[0] - 1) * seed_stride + (min(count, width) - 1) * lane_stride + \
            (count - 1) // width
        if last >= out.size // 2:
            raise SaError(SA_ERRORS[-6])
        rc = emu().emu_sample_seeded(out.ctypes.data + 16 * offset, seeds.tobytes(), seeds.shape[0], seed_stride,
                                     first, count, width, lane_stride, 37)
        if rc:
            raise SaError(SA_ERRORS[rc])
        return out


def seed(*tag):
    """a 32-byte seed named by `tag`"""
    return hashlib.blake2b(repr(tag).encode(), digest_size=32).digest()


def refuse_urandom(n):
    raise AssertionError("os.urandom called by a seeded proof")


def _call(fn):
    try:
        return fn()
    except (AssertionError, IndexError) as e:
        return e


def seeded(plan, traces, boundaries, seeds, zcw=None, streams=None):
    """plan.prove_batch with `seeds` and os.urandom refused: the proof list or the exception"""
    real = os.urandom
    os.urandom = refuse_urandom
    try:
        if zcw is None:
            return _call(lambda: plan.prove_batch(traces, boundaries, streams, seeds=seeds))
        return _call(lambda: plan.prove_batch(traces, boundaries, zcw, streams, seeds=seeds))
    finally:
        os.urandom = real


def route(plan, traces, boundaries, seeds, zcw=None, streams=None):
    """the host route: each proof alone and unseeded with os.urandom = seeded_urandom(its seed), in order: the proof
    list, or the first exception with its proof's index as proof_index"""
    real = os.urandom
    proofs = []
    try:
        for b, (trace, boundary, s) in enumerate(zip(traces, boundaries, seeds)):
            os.urandom = sa_stark.seeded_urandom(s)
            ps = None if streams is None else streams[b]
            got = _call(lambda: plan.prove(trace, boundary, ps) if zcw is None else
                        plan.prove(trace, boundary, zcw, ps))
            if not isinstance(got, bytes):
                got.proof_index = b
                return got
            proofs.append(got)
    finally:
        os.urandom = real
    return proofs


def same(a, b):
    """two results agree: equal proof lists, or exceptions of one type, message and proof_index"""
    if isinstance(a, list) or isinstance(b, list):
        return a == b
    return (type(a), str(a), getattr(a, "proof_index", None)) == (type(b), str(b), getattr(b, "proof_index", None))
