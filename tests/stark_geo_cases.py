"""Cases of the geometric-route prover tests (tests/test_stark_geo_cpu.py, tests/test_gpu_stark_geo.py): the batch
test double of tests/stark_batch_cases.py with a tree cap of its own and the geometric calls, each run through the CPU
emulation of the library's geo.cuh schedules (tests/emu/emu_geo.cpp), so that a small AIR takes the route a trace
above 2^20 rows takes on the device."""
import ctypes

import numpy as np

import __graft_entry__ as G
import stark_batch_cases as SB
from sa_engine import SA_ERRORS, GeoInterpPlan, SaError

O = SB.C.O
_vp, _sz, _ci = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
_EMU = None


def emu():
    global _EMU
    if _EMU is None:
        lib = ctypes.CDLL(G.build_emu_geo())
        for name, res, args in [("emu_geo_plan_bytes", _sz, [_sz]), ("emu_geo_plan", _ci, [_vp, _vp, _sz]),
                                ("emu_geo_interp_batch", _ci, [_vp, _vp, _vp, _sz, _sz, _sz]),
                                ("emu_geo_zerofier", _ci, [_vp, _vp, _sz])]:
            getattr(lib, name).restype = res
            getattr(lib, name).argtypes = args
        _EMU = lib
    return _EMU


def _check(rc):
    if rc:
        raise SaError(SA_ERRORS[rc])


class GeoStarkEngine(SB.BatchStarkEngine):
    """the batch double whose subproduct tree takes at most `cap` points"""
    name = "oracle-test-double-stark-geo"

    def __init__(self, cap):
        SB.BatchStarkEngine.__init__(self)
        self.cap = cap

    def tree_fits(self, k):
        return 1 <= k <= self.cap

    def geo_interp_plan(self, step, k):
        self._log("geo_interp_plan", k)
        step = int(step) % O.P
        plan = np.zeros(max(16, emu().emu_geo_plan_bytes(k)) // 8, np.uint64)
        _check(emu().emu_geo_plan(O._ptr(plan), O._ptr(O._fe(step)), k))
        return GeoInterpPlan(plan, step, k)

    def geo_interp_apply(self, plan, values):
        self._log("geo_interp_apply", *values.shape[:-1])
        if values.ndim not in (2, 3) or tuple(values.shape[-2:]) != (plan.k, 2):
            raise SaError(SA_ERRORS[-6])
        values = np.ascontiguousarray(values, dtype=np.uint64)
        out = np.zeros(values.shape, np.uint64)
        batch = values.shape[0] if values.ndim == 3 else 1
        _check(emu().emu_geo_interp_batch(O._ptr(out), O._ptr(plan.plan), O._ptr(values), plan.k, batch, 0))
        return out

    def geo_zerofier(self, step, k):
        self._log("geo_zerofier", k)
        out = np.zeros((k + 1, 2), np.uint64)
        _check(emu().emu_geo_zerofier(O._ptr(out), O._ptr(O._fe(int(step) % O.P)), k))
        return out
