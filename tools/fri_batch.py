#!/usr/bin/env python3
"""Batched FRI (Fri.prove_batch, sa_fri_commit_batch) against FRI proof by proof.

Prover lines: per-proof time of the same batch proven with the default route (Fri.prove per proof) and with
fri_batch=True, for B = 1, 16 and 64: seeded SignerPlan.sign on the stand-in FastRPSSS and RPSSS of
tests/stark_rescue_cases.py, and seeded StarkPlan.prove_batch on synthetic three-register AIRs at 2^12 and 2^16 FRI
domains.  Median of --reps calls after a warm-up, host clock around a call whose result is bytes on the host; the
bytes of both routes are asserted equal.

FRI lines: the FRI stage alone on the signatures' shape (domain 4096, expansion factor 4, 64 checks, 4 rounds) and
at 2^16, B random codewords already on the device: B Fri.prove calls against one Fri.prove_batch, the commit alone (B
sa_fri_commit calls against one sa_fri_commit_batch), and the queries as the rest; kernel launches and host waits (one
per round and call) of each.

Split lines: where the time of one FastRPSSS / RPSSS signature (B = 1, default route) goes: the whole call, the time
inside Fri.prove, inside prover_fiat_shamir and inside serialize (pickling, which Fiat-Shamir calls), each of the last
two outside and inside FRI (the *_in_fri keys); the device stages and the rest of the host are the whole call minus
FRI and minus Fiat-Shamir outside FRI.  Median of --reps.  A last line names the device and its power limit, read in
the same run."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "stark-anatomy_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"),
                os.path.join(ROOT, "tools"), ROOT]
import numpy as np  # noqa: E402
import torch  # noqa: E402

import fri as dropin_fri  # noqa: E402
import sa_devlist  # noqa: E402
import sa_engine  # noqa: E402
import sa_host  # noqa: E402
import sa_stark  # noqa: E402
import stark_cases as C  # noqa: E402
import stark_plain_cases as S  # noqa: E402
import stark_prove as SP  # noqa: E402
import stark_rescue_cases as SR  # noqa: E402

BATCHES = (1, 16, 64)


def runs_s(fn, reps):
    fn()
    times = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t)
    return times


def per_proof(times, B):
    return {"median_ms": round(1e3 * statistics.median(times) / B, 3),
            "min_ms": round(1e3 * min(times) / B, 3), "max_ms": round(1e3 * max(times) / B, 3)}


def signers():
    g, gp = C.golden(), S.golden()
    for fast, rec in ((True, g["rpsss"]), (False, gp["rpsss"])):
        yield ("FastRPSSS" if fast else "RPSSS"), SR.Signer(rec, fast)


def prover_lines(reps):
    for name, signer in signers():
        plan = sa_stark.SignerPlan(signer)
        for B in BATCHES:
            sks = [C.T.fe(3 + 7 * b) for b in range(B)]
            docs = [b"document %d" % b for b in range(B)]
            seeds = [bytes([b]) * 32 for b in range(B)]
            assert plan.sign(sks, docs, seeds) == plan.sign(sks, docs, seeds, fri_batch=True), name
            for route in (False, True):
                times = runs_s(lambda: plan.sign(sks, docs, seeds, fri_batch=route), reps)
                print(json.dumps({"prover": name, "B": B, "fri": "batched" if route else "per proof", "runs": reps,
                                  **per_proof(times, B)}), flush=True)
    for log_fri in (12, 16):
        st, cons, trace, boundary = C.synthetic(log_fri, log_fri)
        zpoly, zvals = C.zerofier(st)
        zcw = C.zerofier_codeword(zvals, True)
        plan = sa_stark.StarkPlan(st, cons, zpoly)
        for B in BATCHES:
            seeds = [bytes([b]) * 32 for b in range(B)]

            def prove(route):
                return plan.prove_batch([trace] * B, [boundary] * B, zcw, seeds=seeds, fri_batch=route)
            assert prove(False) == prove(True), log_fri
            for route in (False, True):
                times = runs_s(lambda: prove(route), reps)
                print(json.dumps({"prover": "synthetic 2^%d" % log_fri, "B": B,
                                  "fri": "batched" if route else "per proof", "runs": reps, **per_proof(times, B)}),
                      flush=True)


def fri_lines(eng, reps):
    field = C.T.field
    rng = np.random.default_rng(0)
    for log_n, k in ((12, 64), (16, 32)):
        n = 1 << log_n
        f = dropin_fri.Fri(field.generator(), field.primitive_nth_root(n), n, 4, k)
        rounds = f.num_rounds()
        for B in BATCHES:
            x = rng.integers(0, 1 << 64, size=(B, n, 2), dtype=np.uint64)
            x[:, :, 1] %= np.uint64(407 << 55)
            vecs = torch.from_numpy(x.view(np.int64)).to(eng.device)

            def per_proof_prove():
                for b in range(B):
                    f.prove(sa_devlist.DeviceCodeword(vecs[b], None, field, n), sa_host.ip.ProofStream())

            def batched_prove():
                f.prove_batch(vecs, [sa_host.ip.ProofStream() for _ in range(B)])

            def per_proof_commit():
                for b in range(B):
                    f.commit(sa_devlist.DeviceCodeword(vecs[b], None, field, n), sa_host.ip.ProofStream())

            def batched_commit():
                f.commit_batch(vecs, [sa_host.ip.ProofStream() for _ in range(B)])
            out = {"fri": "2^%d, %d checks, %d rounds" % (log_n, k, rounds), "B": B, "runs": reps}
            for name, fn, waits in (("per proof", per_proof_prove, B * rounds), ("batched", batched_prove, rounds),
                                    ("per proof commit", per_proof_commit, B * rounds),
                                    ("batched commit", batched_commit, rounds)):
                eng.synchronize()
                before = eng.launch_count()
                fn()
                eng.synchronize()
                launches = eng.launch_count() - before
                times = runs_s(fn, reps)
                out[name] = {**per_proof(times, B), "launches": launches, "host_waits": waits}
            for route in ("per proof", "batched"):
                out[route + " queries"] = {"median_ms": round(out[route]["median_ms"] -
                                                              out[route + " commit"]["median_ms"], 3)}
            print(json.dumps(out), flush=True)
            del vecs


def split_lines(reps):
    for name, signer in signers():
        plan = sa_stark.SignerPlan(signer)
        args = ([C.T.fe(11)], [b"document"], [bytes(32)])
        plan.sign(*args)
        stream, base, fri = plan.stream, sa_host.ip.ProofStream, plan.plan.fri
        rows = []
        for _ in range(reps):
            spent, where = {}, {"fri": False}

            def timed(key, fn):
                def call(*a, **kw):
                    t = time.perf_counter()
                    outer = key == "fri"
                    where["fri"] |= outer
                    try:
                        return fn(*a, **kw)
                    finally:
                        if outer:
                            where["fri"] = False
                        k = key + ("_in_fri" if where["fri"] else "")
                        spent[k] = spent.get(k, 0.0) + time.perf_counter() - t
                return call
            saved = [(stream, "prover_fiat_shamir", stream.__dict__.get("prover_fiat_shamir")),
                     (base, "serialize", base.__dict__.get("serialize"))]
            stream.prover_fiat_shamir = timed("fiat_shamir", stream.prover_fiat_shamir)
            base.serialize = timed("pickling", base.serialize)
            fri.prove = timed("fri", fri.prove)
            try:
                t = time.perf_counter()
                plan.sign(*args)
                total = time.perf_counter() - t
            finally:
                del fri.prove
                for owner, attr, old in saved:
                    if old is None:
                        delattr(owner, attr)
                    else:
                        setattr(owner, attr, old)
            rows.append({"total": total, **spent,
                         "device_stages_and_rest": total - spent.get("fri", 0.0) - spent.get("fiat_shamir", 0.0)})
        med = {k: round(1e3 * statistics.median(r.get(k, 0.0) for r in rows), 3) for k in rows[0]}
        print(json.dumps({"split": name, "B": 1, "runs": reps, "ms": med}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    eng = sa_engine.get_engine()
    assert eng.name == "cuda", "needs the CUDA engine"
    prover_lines(args.reps)
    fri_lines(eng, args.reps)
    split_lines(args.reps)
    idx = eng.device.index
    print(json.dumps({"device": torch.cuda.get_device_name(idx), "power_limit_w": SP.power_limit_w(idx)}), flush=True)


if __name__ == "__main__":
    main()
