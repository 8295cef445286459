#!/usr/bin/env python3
"""Batched proofs (StarkPlan.prove_batch, PlainStarkPlan.prove_batch, sa_stark.sign_batch) against the same proofs
one at a time, on the fixture's FastRPSSS and RPSSS instances (tests/golden/stark.json and stark_plain.json: FRI
domain 4096, 2 registers, 64 colinearity checks) and on the seeded synthetic AIR of tests/stark_cases.synthetic at
FRI domains 2^12 and 2^16.  For B in --batches, per proof:

  batch_ms     one prove_batch of B proofs, divided by B: host clock around the call (it ends in the proofs' bytes,
               so in synchronising reads), median of --reps
  seq_ms       B plan.prove calls fed the same draws rearranged into per-proof order, divided by B, timed alternately
               with batch_ms in the same run
  pre_fri_launches   kernel launches (sa_launch_count) from the start of the call to the first proof's FRI, divided by B
  sign_batch_ms / sign_ms   (the fixture instances) sa_stark.sign_batch against B calls of a sign rebound to the device
               prover (a plan built per call, as the rebound reference sign runs), on a stand-in signer replaying the
               fixture's trace, boundary and AIR

Every batch's bytes are checked against the sequential proofs of the same run.  One JSON line per (instance, B),
then one naming the device and its power limit (read in the same run)."""
import argparse
import json
import os
import random
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "stark-anatomy_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"),
                ROOT]
import torch  # noqa: E402

import sa_engine  # noqa: E402
import stark_batch_cases as SB  # noqa: E402
import stark_cases as C  # noqa: E402
import stark_plain_cases as S  # noqa: E402
import sa_stark  # noqa: E402
from stark_prove import power_limit_w  # noqa: E402

P = C.P


def instances(which):
    """(name, plan, traces source, boundary, zerofier codeword or None, signer or None)"""
    out = []
    if "fast_rpsss" in which:
        rec = C.golden()["rpsss"]
        st = C.params(rec)
        zpoly, zvals = C.zerofier(st)
        trace, boundary = C.inputs(rec)
        out.append(("fast_rpsss", sa_stark.StarkPlan(st, C.air(rec), zpoly), trace, boundary,
                    C.zerofier_codeword(zvals, True), SB.Signer(rec, True), rec))
    if "rpsss" in which:
        rec = S.golden()["rpsss"]
        trace, boundary = C.inputs(rec)
        out.append(("rpsss", sa_stark.PlainStarkPlan(S.stark(rec), C.air(rec)), trace, boundary, None,
                    SB.Signer(rec, False), rec))
    for log_fri in (12, 16):
        if "synthetic_%d" % log_fri in which:
            st, cons, trace, boundary = C.synthetic(log_fri, log_fri)
            zpoly, zvals = C.zerofier(st)
            out.append(("synthetic_2^%d" % log_fri, sa_stark.StarkPlan(st, cons, zpoly), trace, boundary,
                        C.zerofier_codeword(zvals, True), None, None))
    return out


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batches", default="1,4,16,64")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--which", default="fast_rpsss,rpsss,synthetic_12,synthetic_16")
    args = ap.parse_args()
    eng = sa_engine.get_engine()
    for name, plan, trace, boundary, zcw, signer, rec in instances(args.which.split(",")):
        nt = plan.nregs * plan.stark.num_randomizers
        for B in [int(b) for b in args.batches.split(",")]:
            rng = random.Random(B)
            per = [[rng.randrange(P) for _ in range(nt + plan.max_degree + 1)] for _ in range(B)]
            launches = {}
            fri_prove = plan.fri.prove

            def first_fri(codeword, ps):
                launches.setdefault("pre", eng.launch_count() - launches["start"])
                return fri_prove(codeword, ps)

            def batch():
                launches.clear()
                launches["start"] = eng.launch_count()
                plan.fri.prove = first_fri
                try:
                    return SB.run_batch(plan, [trace] * B, [boundary] * B, C.Urandom(SB.batch_draws(per, nt)), None,
                                        zcw)
                finally:
                    del plan.fri.prove

            def sequential():
                if zcw is None:
                    return [S.run(None, trace, None, boundary, C.Urandom(ds), plan=plan) for ds in per]
                return [C.run(None, trace, None, boundary, None, zcw, C.Urandom(ds), plan=plan)[0] for ds in per]
            batch(), sequential()  # warm: workspaces, caches
            tb, ts = [], []
            for _ in range(args.reps if B <= 16 else 1):
                got, t = timed(batch)
                tb.append(t / B)
                want, t = timed(sequential)
                ts.append(t / B)
            assert got == want, "%s B=%d: batch bytes differ from sequential proofs" % (name, B)
            row = {"instance": name, "B": B, "batch_ms": round(statistics.median(tb), 3),
                   "seq_ms": round(statistics.median(ts), 3),
                   "pre_fri_launches": round(launches["pre"] / B, 1), "bytes_equal": True}
            if signer is not None:
                docs = [bytes([b % 256, b // 256]) for b in range(B)]
                real = sa_stark.os.urandom
                try:
                    sa_stark.os.urandom = C.Urandom(SB.batch_draws(per, nt))
                    sigs, t = timed(lambda: sa_stark.sign_batch(signer, 1, docs))
                    row["sign_batch_ms"] = round(t / B, 3)
                    one = []
                    t0 = time.perf_counter()
                    for d, ds in zip(docs, per):
                        sa_stark.os.urandom = C.Urandom(ds)
                        one.append(signer.sign(1, d))
                    torch.cuda.synchronize()
                    row["sign_ms"] = round((time.perf_counter() - t0) * 1e3 / B, 3)
                finally:
                    sa_stark.os.urandom = real
                assert sigs == one, "%s B=%d: sign_batch differs from sign" % (name, B)
            print(json.dumps(row), flush=True)
    index = torch.cuda.current_device()
    print(json.dumps({"device": torch.cuda.get_device_name(index), "power_limit_w": power_limit_w(index)}))


if __name__ == "__main__":
    main()
