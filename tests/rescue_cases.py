"""Cases of the Rescue-Prime kernel tests, shared by the CPU suite (tests/test_rescue_cpu.py) and the GPU suite
(tests/test_gpu_rescue.py): the fixture tests/golden/rescue.json (the reference's constants, hashes and traces), the
CPU emulation of csrc/rescue.cuh and the independent oracle (tests/emu/rescue_oracle.cpp), both in
libsa_emu_rescue.so, and a restatement in Python ints for small cross-checks."""
import ctypes
import json
import os

import numpy as np

import __graft_entry__ as G

P = (407 << 119) + 1
HERE = os.path.dirname(os.path.abspath(__file__))
MAX_ROUNDS = 512  # SA_RESCUE_MAX_ROUNDS
_GOLDEN = None
_LIB = None


def golden():
    global _GOLDEN
    if _GOLDEN is None:
        with open(os.path.join(HERE, "golden", "rescue.json")) as f:
            _GOLDEN = json.load(f)
    return _GOLDEN


def constants(g=None):
    """the fixture's constant block in sa_rescue's order, as ints"""
    g = g or golden()
    return [int(v) for v in g["mds"]] + [int(v) for v in g["round_constants"]]


def exponents(g=None):
    g = g or golden()
    return int(g["alpha"]), int(g["alphainv"])


def to_np(values):
    a = np.zeros((len(values), 2), dtype=np.uint64)
    for i, v in enumerate(values):
        a[i, 0], a[i, 1] = v & 0xFFFFFFFFFFFFFFFF, v >> 64
    return a


def from_np(a):
    a = np.asarray(a, dtype=np.uint64).reshape(-1, 2)
    return [int(lo) | int(hi) << 64 for lo, hi in a.tolist()]


def _u128(e):
    return (ctypes.c_uint64 * 2)(e & 0xFFFFFFFFFFFFFFFF, e >> 64)


def lib():
    global _LIB
    if _LIB is None:
        lib = ctypes.CDLL(G.build_emu_rescue())
        lib.emu_rescue.restype = ctypes.c_int
        lib.emu_rescue.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t] + \
            [ctypes.c_void_p] * 2 + [ctypes.c_size_t] * 2 + [ctypes.c_longlong]
        lib.rescue_oracle.restype = None
        lib.rescue_oracle.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t] + \
            [ctypes.c_void_p] * 2
        lib.rescue_oracle_pow.restype = None
        lib.rescue_oracle_pow.argtypes = [ctypes.c_void_p] * 3
        _LIB = lib
    return _LIB


def _ptr(a):
    return None if a is None else a.ctypes.data


def emu(hashes, trace, inputs, consts, rounds, alpha, alphainv, inst_stride, lane_stride, threads=7):
    """sa_rescue on the emulation over host arrays (hashes and trace (n, 2) uint64 arrays or None): its return code"""
    return lib().emu_rescue(_ptr(hashes), _ptr(trace), _ptr(inputs), inputs.shape[0], _ptr(consts), rounds,
                            _u128(alpha), _u128(alphainv), inst_stride, lane_stride, threads)


def oracle(inputs, consts, rounds, alpha, alphainv, trace=True):
    """(hashes (count, 2), traces (count, 2, rounds + 1, 2) or None) of the (count, 2) uint64 inputs"""
    inputs = np.ascontiguousarray(inputs, dtype=np.uint64).reshape(-1, 2)
    consts = np.ascontiguousarray(consts, dtype=np.uint64).reshape(-1, 2)
    count = inputs.shape[0]
    hashes = np.zeros((count, 2), np.uint64)
    tr = np.zeros((count, 2, rounds + 1, 2), np.uint64) if trace else None
    lib().rescue_oracle(_ptr(hashes), _ptr(tr), _ptr(inputs), count, _ptr(consts), rounds, _u128(alpha),
                        _u128(alphainv))
    return hashes, tr


def oracle_pow(x, e):
    out = np.zeros(2, np.uint64)
    lib().rescue_oracle_pow(out.ctypes.data, _u128(x), _u128(e))
    return int(out[0]) | int(out[1]) << 64


def python_rescue(x, consts, rounds, alpha, alphainv):
    """(hash, trace rows [s0, s1]) in Python ints, rescue_prime.py's loops restated with pow()"""
    mds, rc = consts[:4], consts[4:]
    state, rows = [x, 0], [[x, 0]]
    for r in range(rounds):
        for half, e in ((0, alpha), (1, alphainv)):
            s = [pow(v, e, P) for v in state]
            state = [(mds[2 * i] * s[0] + mds[2 * i + 1] * s[1] + rc[4 * r + 2 * half + i]) % P for i in range(2)]
        rows.append(list(state))
    return state[0], rows


def dense_trace(traces):
    """(count, 2, rows, 2) uint64 -> per input the list of rows [s0, s1] as ints"""
    count, _, rows, _ = traces.shape
    vals = from_np(traces)
    return [[[vals[(b * 2 + s) * rows + r] for s in range(2)] for r in range(rows)] for b in range(count)]
