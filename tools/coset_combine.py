#!/usr/bin/env python3
"""Coset combinations: the weighted, degree-shifted sum of a prover's quotients and its coset codeword
(fast_stark.py:125-148), through the host as a caller does it without sa_coset_combine_evaluate, and in one call.

Per FRI domain n = 2^log_n and term set (C, R), on FastStark-shaped terms (expansion factor 4, max_degree = n/4 - 1):
a randomizer of n/4 coefficients, C transition quotients of 3n/16 coefficients (rows of one tensor, as
coset_div_apply returns them) and R boundary quotients of n/4 - 1 - r coefficients (separate tensors), each as the
pair (q, x^s * q) with FastStark's shift s = max_degree - deg q: T = 1 + 2C + 2R terms.

  host_ms          download the rows, sum the combination with Python ints, upload it, coset_evaluate; one call
                   timed with a host clock that ends in a device synchronise (it runs for seconds at the larger sizes)
  combine_ms       one CudaEngine.coset_combine_evaluate (the C call and the engine's Python), CUDA events around a
                   window of at least --window seconds after a warm-up call
  ntt_ms           one in-place sa_ntt of n elements, the transform inside combine_ms, timed the same way
  combine_fri_ms   coset_combine_evaluate followed by fri_commit of its codeword (4, 16 colinearity tests: rounds as
                   Fri's), with a constant challenge callback, timed the same way
  rows_mib         the bytes of the distinct source rows a call reads

One JSON line per (size, term set), then one naming the device and its power limit (read in the same run).  Every
line checks that the host route and the device call give the same codeword."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "stark-anatomy_b200"), os.path.join(ROOT, "oracle"), ROOT]
import numpy as np  # noqa: E402
import torch  # noqa: E402

import oracle as O  # noqa: E402
import sa_engine  # noqa: E402

LOGS = [12, 14, 16, 18, 20, 22]
SETS = [(2, 2), (8, 8), (32, 32)]
P = sa_engine.P


def power_limit_w(index):
    """the board's enforced power limit in W as nvidia-smi reports it (a read-only query), or None"""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out)
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


def rand_vec(shape, dev):
    x = torch.randint(0, 1 << 62, tuple(shape) + (2,), dtype=torch.int64, device=dev)
    x[..., 1] &= (1 << 61) - 1  # < 2^125 < p
    return x


def timed_ms(fn, st, window_s):
    """ms per call of fn over a window of at least window_s seconds (one warm-up call first)"""
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 1
    while True:
        e0.record(st)
        for _ in range(reps):
            fn()
        e1.record(st)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        if ms >= window_s * 1e3:
            return ms / reps
        reps = max(reps * 2, int(reps * window_s * 1e3 / max(ms, 1e-3)) + 1)


def faststark_terms(log_n, C, R, dev, seed):
    n, m = 1 << log_n, 1 << (log_n - 2)
    rng = np.random.default_rng(seed)
    weights = [int.from_bytes(rng.bytes(16), "little") % P for _ in range(1 + 2 * C + 2 * R)]
    quotients = rand_vec((C, 3 * m // 4), dev)
    rows = [rand_vec((m,), dev)] + [quotients[c] for c in range(C)] + [rand_vec((m - 1 - r,), dev) for r in range(R)]
    terms = [(rows[0], 0, weights[0])]
    for k, q in enumerate(rows[1:]):
        terms += [(q, 0, weights[1 + 2 * k]), (q, m - q.shape[0], weights[2 + 2 * k])]
    assert max(s + v.shape[0] for v, s, _ in terms) <= n // 4
    return rows, terms


def host_route(eng, terms, log_n, root, offset):
    """what a caller does today: every row to the host, the sum in Python ints, the combination back, coset_evaluate"""
    m = max(s + v.shape[0] for v, s, _ in terms)
    c = [0] * m
    host = {}
    for vec, shift, w in terms:
        key = vec.data_ptr()
        if key not in host:
            host[key] = O.from_np(vec.cpu().numpy().view(np.uint64))
        row = host[key]
        c[shift:shift + len(row)] = [(a + w * b) % P for a, b in zip(c[shift:shift + len(row)], row)]
    comb = eng.upload(O.to_np(c).view(np.int64))
    return eng.coset_evaluate(comb, log_n, root, offset)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--window", type=float, default=0.3, help="seconds per timed window")
    ap.add_argument("--logs", type=int, nargs="*", default=LOGS, help="log2 of the FRI domain sizes")
    args = ap.parse_args()

    eng = sa_engine.get_engine()
    dev = eng.device
    st = torch.cuda.current_stream(dev)
    torch.manual_seed(0)
    for log_n in args.logs:
        n = 1 << log_n
        root, offset = O.primitive_nth_root(n), O.GENERATOR
        rounds = O.fri_num_rounds(n, 4, 16)
        x = rand_vec((n,), dev)
        for C, R in SETS:
            rows, terms = faststark_terms(log_n, C, R, dev, seed=log_n * 100 + C)
            got = eng.coset_combine_evaluate(terms, log_n, root, offset)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            want = host_route(eng, terms, log_n, root, offset)
            torch.cuda.synchronize()
            host_ms = (time.perf_counter() - t0) * 1e3
            assert bool((got == want).all()), "host route and device call differ at 2^%d, (C, R) = (%d, %d)" % (
                log_n, C, R)

            def combine_fri():
                eng.fri_commit(eng.coset_combine_evaluate(terms, log_n, root, offset), rounds, offset, root,
                               lambda r, rt, want_alpha: 12345)

            row = {"log_n": log_n, "C": C, "R": R, "terms": len(terms),
                   "rows_mib": round(sum(16 * v.shape[0] for v in rows) / (1 << 20), 3),
                   "host_ms": host_ms,
                   "combine_ms": timed_ms(lambda: eng.coset_combine_evaluate(terms, log_n, root, offset), st,
                                          args.window),
                   "ntt_ms": timed_ms(lambda: eng.ntt_into(x, x, log_n, root), st, args.window),
                   "combine_fri_ms": timed_ms(combine_fri, st, args.window)}
            print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in row.items()}), flush=True)
            del rows, terms, got, want
        del x
        torch.cuda.synchronize(dev)
        torch.cuda.empty_cache()
        assert eng.lib.sa_release_workspaces() == 0
    print(json.dumps({"device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index),
                      "window_s": args.window}), flush=True)


if __name__ == "__main__":
    main()
