#!/usr/bin/env python3
"""Boundary quotients: each register's (T_s - I_s) / Z_s and its codeword on the FRI domain (fast_stark.py:92-106),
through the host as a caller does it without sa_boundary_quotients, and as one plan plus one apply.

FastStark shapes at expansion factor 4: per FRI domain of n points the omicron domain has n / 4 points and the trace
polynomials T = n / 16 coefficients; 2 and 8 registers, each with boundary points at cycles 0 and T - 1 (seeded
values) and seeded trace polynomials I + Z R, so every division is clean.

  plan_ms     one CudaEngine.boundary_plan (zerofiers and interpolants on the device; it synchronises): host clock
  apply_ms    one CudaEngine.boundary_quotients with check=True (quotients, codewords, flags and the flags' read),
              CUDA events around a window of at least --window seconds after a warm-up
  host_ms     download the trace polynomials, host Polynomial subtraction and division by the boundary zerofier,
              then the drop-in fast_coset_evaluate per register; one call, host clock (up to --host-max: the
              reference's long division is quadratic in T)

One JSON line per shape, then one naming the device and its power limit (read in the same run).  Every line checks
that the host route and the device call give the same quotients and codewords where the host route ran."""
import argparse
import json
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "stark-anatomy_b200"), os.path.join(ROOT, "oracle"), ROOT,
                os.path.dirname(os.path.abspath(__file__))]
import numpy as np  # noqa: E402
import torch  # noqa: E402

import oracle as O  # noqa: E402
import sa_engine  # noqa: E402
from air_quotients import power_limit_w, timed_ms  # noqa: E402  (the same clock and power query)

LOGS = list(range(12, 23, 2))
P = sa_engine.P


def clean_trace(eng, boundary, nregs, omicron, T, seed):
    """I_s + Z_s R_s of T coefficients per register, R_s seeded on the device, Z_s and I_s from the engine"""
    g = torch.Generator(device=eng.device).manual_seed(seed)
    out = torch.empty((nregs, T, 2), dtype=torch.int64, device=eng.device)
    m = 1 << (T + 2).bit_length()
    root = O.primitive_nth_root(m)
    for s in range(nregs):
        pts = [(pow(omicron, c, P), v) for c, r, v in boundary if r == s]
        dom = eng.upload(O.to_np([x for x, _ in pts]).view(np.int64))
        z = eng.zerofier(dom)
        i = O.from_np(eng.download(eng.interpolate(dom, eng.upload(O.to_np([v for _, v in pts]).view(np.int64))))
                      .view(np.uint64))
        r = torch.randint(-(1 << 63), (1 << 63) - 1, (T - len(pts), 2), dtype=torch.int64, device=eng.device,
                          generator=g)
        r[:, 1] &= (1 << 55) - 1  # below 2^119 < p: canonical
        lg = m.bit_length() - 1
        zr = eng.ntt(eng.pointwise_mul(eng.ntt(eng.pad(z, m), lg, root), eng.ntt(eng.pad(r, m), lg, root)), lg, root,
                     inverse=True)
        head = O.from_np(eng.download(zr[:len(i)]).view(np.uint64))
        zr[:len(i)] = eng.upload(O.to_np([(a + b) % P for a, b in zip(head, i)]).view(np.int64))
        out[s] = zr[:T]
    return out


def host_route(eng, boundary, nregs, trace_dev, omicron, n):
    """what a caller does today: the trace polynomials to the host, the boundary zerofiers and interpolants, host
    Polynomial subtraction and division, the drop-in fast_coset_evaluate"""
    import ntt as N
    import sa_host
    Polynomial = sa_host.univariate.Polynomial
    field = sa_host.algebra.Field.main()
    fe = lambda v: sa_host.algebra.FieldElement(int(v), field)  # noqa: E731
    om = fe(omicron)
    quots, cws = [], []
    for s in range(nregs):
        tp = Polynomial([fe(v) for v in O.from_np(eng.download(trace_dev[s]).view(np.uint64))])
        pts = [(om ^ c, fe(v)) for c, r, v in boundary if r == s]
        z = Polynomial.zerofier_domain([x for x, _ in pts])
        i = Polynomial.interpolate_domain([x for x, _ in pts], [v for _, v in pts])
        q = (tp - i) / z
        quots.append([c.value for c in q.coefficients])
        cws.append([c.value for c in N.fast_coset_evaluate(q, fe(O.GENERATOR), fe(O.primitive_nth_root(n)), n)])
    return quots, cws


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--window", type=float, default=0.3, help="seconds per timed window")
    ap.add_argument("--logs", type=int, nargs="*", default=LOGS, help="log2 of the FRI domain lengths")
    ap.add_argument("--regs", type=int, nargs="*", default=[2, 8], help="register counts")
    ap.add_argument("--host-max", type=int, default=16, help="largest log2 FRI domain the host route runs at")
    args = ap.parse_args()

    eng = sa_engine.get_engine()
    dev = eng.device
    st = torch.cuda.current_stream(dev)
    for lg in args.logs:
        n = 1 << lg
        T = n // 16
        omicron = O.primitive_nth_root(n // 4)
        for nregs in args.regs:
            rng = random.Random(1000 * lg + nregs)
            boundary = [(c, s, rng.randrange(P)) for s in range(nregs) for c in (0, T - 1)]
            trace_dev = clean_trace(eng, boundary, nregs, omicron, T, lg)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            plan = eng.boundary_plan(boundary, nregs, omicron, lg, O.primitive_nth_root(n), O.GENERATOR)
            plan_ms = (time.perf_counter() - t0) * 1e3
            quot, cw, _ = eng.boundary_quotients(plan, trace_dev)
            row = {"fri_log_n": lg, "nregs": nregs, "trace_len": T, "plan_ms": plan_ms,
                   "apply_ms": timed_ms(lambda: eng.boundary_quotients(plan, trace_dev), st, args.window)}
            if lg <= args.host_max:
                t0 = time.perf_counter()
                want_q, want_cw = host_route(eng, boundary, nregs, trace_dev, omicron, n)
                row["host_ms"] = (time.perf_counter() - t0) * 1e3
                for s in range(nregs):
                    got_q = O.from_np(eng.download(quot[s]).view(np.uint64))
                    assert got_q == want_q[s] + [0] * (T - len(want_q[s])), (lg, nregs, s)
                    assert O.from_np(eng.download(cw[s]).view(np.uint64)) == want_cw[s], (lg, nregs, s)
            print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in row.items()}), flush=True)
            del plan, quot, cw, trace_dev
            torch.cuda.synchronize(dev)
            torch.cuda.empty_cache()
            assert eng.lib.sa_release_workspaces() == 0
    print(json.dumps({"device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index),
                      "window_s": args.window}), flush=True)


if __name__ == "__main__":
    main()
