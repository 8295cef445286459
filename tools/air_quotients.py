#!/usr/bin/env python3
"""Transition quotients: a prover's numerators and their division by the transition zerofier (fast_stark.py:108-113),
through the host as a caller does it without sa_air_quotients, and as one plan plus one apply.

Rescue-shaped AIRs: the exponent structure of tests/golden/air.json (two registers, 2 x 272 terms, x exponents up
to 78, trace degree 3) with seeded random coefficients.  Per trace length T (coefficients per trace polynomial) the
coset has order n = the smallest power of two above 78 + 3 (T - 1), as FastStark's omicron domain, and a zerofier of
28 seeded coefficients; qlen = n - 27.

  plan_ms     one CudaEngine.air_plan (it synchronises): host clock
  apply_ms    one CudaEngine.air_quotients, CUDA events around a window of at least --window seconds after a warm-up
  host_ms     download the trace polynomials, evaluate_symbolic restated over the host Polynomial type (schoolbook
              products), then the drop-in fast_coset_divide per constraint; one call, host clock (up to --host-max)
  accel_ms    the same with sa_accel.enable() (the products on the device; up to --accel-max)

One JSON line per size, then one naming the device and its power limit (read in the same run).  Every line checks
that the host route and the device call give the same quotients where the host route ran."""
import argparse
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "stark-anatomy_b200"), os.path.join(ROOT, "oracle"), ROOT]
import numpy as np  # noqa: E402
import torch  # noqa: E402

import oracle as O  # noqa: E402
import sa_engine  # noqa: E402

LOGS = list(range(8, 19, 2))
P = sa_engine.P


def power_limit_w(index):
    """the board's enforced power limit in W as nvidia-smi reports it (a read-only query), or None"""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out)
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


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


def rescue_shaped_air(seed):
    with open(os.path.join(ROOT, "tests", "golden", "air.json")) as f:
        rec = json.load(f)["faststark"]
    rng = random.Random(seed)
    return [{tuple(t["e"]): rng.randrange(P) for t in cons} for cons in rec["air"]]


def host_route(eng, air, trace_dev, zerofier, omicron, n):
    """what a caller does today: the trace polynomials to the host, evaluate_symbolic (MPolynomial's loop, restated
    over the host Polynomial type), the drop-in fast_coset_divide"""
    import ntt as N
    import sa_host
    Polynomial = sa_host.univariate.Polynomial
    field = sa_host.algebra.Field.main()
    fe = lambda v: sa_host.algebra.FieldElement(int(v), field)  # noqa: E731
    tps = [Polynomial([fe(v) for v in O.from_np(eng.download(r).view(np.uint64))]) for r in trace_dev]
    om = fe(omicron)
    point = [Polynomial([field.zero(), field.one()])] + tps + [tp.scale(om) for tp in tps]
    z = Polynomial([fe(v) for v in zerofier])
    out = []
    for a in air:
        acc = Polynomial([])
        for k, v in a.items():
            prod = Polynomial([fe(v)])
            for i in range(len(k)):
                prod = prod * (point[i] ^ k[i])
            acc = acc + prod
        out.append([c.value for c in N.fast_coset_divide(acc, z, fe(O.GENERATOR), om, n).coefficients])
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--window", type=float, default=0.3, help="seconds per timed window")
    ap.add_argument("--logs", type=int, nargs="*", default=LOGS, help="log2 of the trace lengths")
    ap.add_argument("--host-max", type=int, default=8, help="largest log2 trace length the host route runs at")
    ap.add_argument("--accel-max", type=int, default=10, help="largest log2 trace length the sa_accel route runs at")
    args = ap.parse_args()

    import sa_accel
    eng = sa_engine.get_engine()
    dev = eng.device
    st = torch.cuda.current_stream(dev)
    air = rescue_shaped_air(0)
    for lt in args.logs:
        T = 1 << lt
        n = 1 << (78 + 3 * (T - 1)).bit_length()
        log_n = n.bit_length() - 1
        rng = random.Random(lt)
        trace = [[rng.randrange(P) for _ in range(T)] for _ in range(2)]
        zerofier = [rng.randrange(P) for _ in range(28)]
        omicron = O.primitive_nth_root(n)
        trace_dev = eng.upload(O.to_np(trace[0] + trace[1]).view(np.int64)).reshape(2, T, 2)
        zdev = eng.upload(O.to_np(zerofier).view(np.int64))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        plan = eng.air_plan(air, 2, zdev, T, log_n, omicron, O.GENERATOR, omicron)
        plan_ms = (time.perf_counter() - t0) * 1e3
        qlen = n - 27
        got = eng.air_quotients(plan, trace_dev, qlen)
        row = {"trace_len": T, "log_n": log_n, "terms": sum(len(a) for a in air), "plan_ms": plan_ms,
               "apply_ms": timed_ms(lambda: eng.air_quotients(plan, trace_dev, qlen), st, args.window)}
        got_rows = [O.from_np(eng.download(got[c]).view(np.uint64)) for c in range(len(air))]
        for name, top, accel in (("host_ms", args.host_max, False), ("accel_ms", args.accel_max, True)):
            if lt > top:
                continue
            if accel:
                sa_accel.enable()
            try:
                t0 = time.perf_counter()
                want = host_route(eng, air, trace_dev, zerofier, omicron, n)
                row[name] = (time.perf_counter() - t0) * 1e3
            finally:
                if accel:
                    sa_accel.disable()
            # the reference truncates at deg N - deg Z + 1 = qlen
            assert all(g[:len(w)] == w for g, w in zip(got_rows, want)), (name, lt)
        print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in row.items()}), flush=True)
        del plan, got, trace_dev, zdev
        torch.cuda.synchronize(dev)
        torch.cuda.empty_cache()
        assert eng.lib.sa_release_workspaces() == 0
    print(json.dumps({"device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index),
                      "window_s": args.window}), flush=True)


if __name__ == "__main__":
    main()
