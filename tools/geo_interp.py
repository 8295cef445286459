#!/usr/bin/env python3
"""Geometric interpolation plans against the subproduct tree, and the prover above the tree's cap.

Per domain size k (the domain step^0 .. step^(k-1), step a root of unity of order 2^(ceil(log2 k) + 1), as the
prover's trace domain), timed with CUDA events around windows of at least --window seconds after one warm-up call of
the same shape:

  geo_plan_ms, tree_plan_ms        one sa_geo_plan / one sa_interp_plan of the explicit domain (both synchronise)
  geo_apply_ms, tree_apply_ms      one apply of one vector
  geo_apply_b8_ms, tree_apply_b8_ms  one batched apply of 8 vectors
  geo_zerofier_ms, tree_zerofier_ms  sa_geo_zerofier / sa_zerofier of the explicit domain
  geo_plan_bytes, tree_plan_bytes

The tree's columns stop at its cap (2^20); above, the geometric route alone.  Each size up to the cap checks that
both routes give the same bytes.  Then one line for StarkPlan at a randomized trace of 2^20 + 1 rows (2^24 FRI
domain, tests/test_gpu_stark_geo.py's two-register AIR): plan build, prove and the summed CUDA-event time of the
device stages inside prove (tools/stark_prove.py's device_ms).  Last, one line naming the device and its power limit
(read in the same run)."""
import argparse
import json
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.join(os.path.dirname(ROOT), "stark-anatomy_b200"), os.path.dirname(ROOT),
                os.path.join(os.path.dirname(ROOT), "tests"), os.path.join(os.path.dirname(ROOT), "oracle"), ROOT]
import torch  # noqa: E402

import sa_engine  # noqa: E402
import interp_plan as IP  # noqa: E402
import stark_prove as SP  # noqa: E402

P = sa_engine.P
SIZES = [1 << 10, 1 << 12, 1 << 16, 1 << 20, 1 << 22, 1 << 24]


def root(order):
    g = 85408008396924667383611388730472331217  # order 2^119
    return pow(g, (1 << 119) // order, P)


def domain(eng, q, k):
    x, out = 1, bytearray()
    for _ in range(k):
        out += x.to_bytes(16, "little")
        x = x * q % P
    return eng.upload(out)


def size_line(eng, k, window):
    st = torch.cuda.current_stream(eng.device)
    q = root(1 << max(1, (2 * k - 1).bit_length()))
    line = {"k": k, "geo_plan_bytes": eng.lib.sa_geo_plan_bytes(k), "tree_plan_bytes": eng.lib.sa_interp_plan_bytes(k)}
    v8 = IP.rand_vec(8 * k, eng.device).reshape(8, k, 2)
    gplan = eng.geo_interp_plan(q, k)
    line["geo_plan_ms"] = IP.timed_ms(lambda: eng.geo_interp_plan(q, k), st, window)
    line["geo_apply_ms"] = IP.timed_ms(lambda: eng.geo_interp_apply(gplan, v8[0]), st, window)
    line["geo_apply_b8_ms"] = IP.timed_ms(lambda: eng.geo_interp_apply(gplan, v8), st, window)
    line["geo_zerofier_ms"] = IP.timed_ms(lambda: eng.geo_zerofier(q, k), st, window)
    if eng.tree_fits(k):
        dom = domain(eng, q, k)
        tplan = eng.interp_plan(dom)
        line["tree_plan_ms"] = IP.timed_ms(lambda: eng.interp_plan(dom), st, window)
        line["tree_apply_ms"] = IP.timed_ms(lambda: eng.interp_apply(tplan, v8[0]), st, window)
        line["tree_apply_b8_ms"] = IP.timed_ms(lambda: eng.interp_apply(tplan, v8), st, window)
        line["tree_zerofier_ms"] = IP.timed_ms(lambda: eng.zerofier(dom), st, window)
        line["same_bytes"] = bool((eng.geo_interp_apply(gplan, v8) == eng.interp_apply(tplan, v8)).all()) and \
            bool((eng.geo_zerofier(q, k) == eng.zerofier(dom)).all())
        del tplan, dom
    del gplan, v8
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    eng.lib.sa_release_workspaces()
    return {key: round(v, 3) if isinstance(v, float) else v for key, v in line.items()}


def prover_line(eng):
    import numpy as np
    import oracle as O
    import stark_cases as C
    import sa_devlist
    import sa_stark
    import test_gpu_stark_geo as TG
    st, cons, rows, boundary = TG.air24()
    n = st.fri_domain_length
    z = eng.geo_zerofier(st.omicron.value, TG.NCYCLES - 1)
    zpoly = O.from_np(eng.download(z).view(np.uint64))
    zcw = sa_devlist.DeviceCodeword(eng.coset_evaluate(z, n.bit_length() - 1, st.omega.value, st.generator.value),
                                    None, C.T.field, n)
    t0 = time.perf_counter()
    plan = sa_stark.StarkPlan(st, cons, zpoly)
    torch.cuda.synchronize()
    plan_ms = (time.perf_counter() - t0) * 1e3
    rng = random.Random(6)
    values = [rng.randrange(P) for _ in range(st.num_registers * st.num_randomizers + plan.max_degree + 1)]
    trace, bnd = TG.fe_trace(rows), TG.fe_boundary(boundary)

    def one():
        return C.run(st, trace, None, bnd, zpoly, zcw, C.Urandom(values), plan=plan)[0]
    first = one()
    t0 = time.perf_counter()
    again = one()
    torch.cuda.synchronize()
    prove_ms = (time.perf_counter() - t0) * 1e3
    SP.STAGES = SP.STAGES + ["geo_interp_apply"]
    dev = SP.device_ms(eng, one)
    return {"stark_plan": "T=2^20+1, FRI 2^24, 2 registers", "plan_ms": round(plan_ms, 1),
            "prove_ms": round(prove_ms, 1), "device_ms": round(dev, 1), "same_bytes": first == again,
            "proof_bytes": len(first)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--window", type=float, default=0.3, help="seconds per timed window")
    ap.add_argument("--sizes", type=int, nargs="*", default=SIZES)
    ap.add_argument("--no-prover", action="store_true", help="skip the StarkPlan line")
    args = ap.parse_args()
    eng = sa_engine.get_engine()
    for k in args.sizes:
        print(json.dumps(size_line(eng, k, args.window)), flush=True)
    if not args.no_prover:
        print(json.dumps(prover_line(eng)), flush=True)
    idx = eng.device.index
    print(json.dumps({"device": torch.cuda.get_device_name(idx), "power_limit_w": IP.power_limit_w(idx)}))


if __name__ == "__main__":
    main()
