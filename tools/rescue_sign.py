#!/usr/bin/env python3
"""Rescue-Prime on the device and signatures from a kept SignerPlan.

Kernel lines (sa_rescue, the fixture's constants from tests/golden/rescue.json, random inputs): for 2^10, 2^14, 2^18
and 2^22 inputs, hash-only and trace launches, CUDA events over --reps launches after a warm-up:

  ms              one launch
  hashes_per_s    inputs / ms
  products_per_s  field products / ms, where one hash costs, per round and for each exponent e of the two half-rounds,
                  2 (bits(e) - 1) squarings and 2 (popcount(e) - 1) multiplies (two registers, left to right from the
                  top bit), plus 4 MDS products per half-round, one conversion of the input into Montgomery form and
                  one out of it per element written (the hash, or 2 per trace row after row 0)

Signing lines (the stand-in FastRPSSS and RPSSS of tests/stark_rescue_cases.py: the recorded case's AIR and the
fixture's constants): the plan build once, then for B = 1, 16 and 64 distinct keys the per-signature time of one
seeded SignerPlan.sign call (median of --reps after a warm-up, host clock around a call whose result is bytes on the
host) against B sign_batch calls, one per key, each fed its key's trace by the host oracle (C, not the reference's
Python; sign_batch builds a plan per call).  Both routes' bytes are asserted equal.  A last line names the device
and its power limit, read in the same run."""
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

import rescue_cases as R  # noqa: E402
import sa_engine  # noqa: E402
import sa_stark  # noqa: E402
import stark_cases as C  # noqa: E402
import stark_plain_cases as S  # noqa: E402
import stark_prove as SP  # noqa: E402
import stark_rescue_cases as SR  # noqa: E402


def products_per_hash(rounds, alpha, alphainv, trace):
    sbox = sum(2 * (e.bit_length() - 1) + 2 * (bin(e).count("1") - 1) for e in (alpha, alphainv))
    return rounds * (sbox + 2 * 4) + 1 + (2 * rounds if trace else 1)


def kernel_lines(eng, reps):
    alpha, alphainv = R.exponents()
    kc = eng.upload(R.to_np(R.constants()).view(np.int64))
    rng = np.random.default_rng(0)
    for log_n in (10, 14, 18, 22):
        n = 1 << log_n
        xs = rng.integers(0, 1 << 64, size=(n, 2), dtype=np.uint64)
        xs[:, 1] %= np.uint64(407 << 55)
        inputs = eng.upload(xs.view(np.int64))
        for trace in (False, True):
            out = eng.empty(n * 56 if trace else n)
            kw = {"trace": out} if trace else {"hashes": out}
            for _ in range(3):
                eng.rescue(inputs, kc, 27, alpha, alphainv, **kw)
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(reps):
                eng.rescue(inputs, kc, 27, alpha, alphainv, **kw)
            end.record()
            end.synchronize()
            ms = start.elapsed_time(end) / reps
            per = products_per_hash(27, alpha, alphainv, trace)
            print(json.dumps({"kernel": "trace" if trace else "hash", "inputs": n, "ms": round(ms, 4),
                              "hashes_per_s": round(n / ms * 1e3), "products_per_hash": per,
                              "products_per_s": round(n * per / ms * 1e3)}), flush=True)
            del out
        del inputs


def median_s(fn, reps):
    fn()
    times = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t)
    return statistics.median(times)


def signing_lines(eng, reps):
    g, gp = C.golden(), S.golden()
    for fast, rec in ((True, g["rpsss"]), (False, gp["rpsss"])):
        name = "FastRPSSS" if fast else "RPSSS"
        signer = SR.Signer(rec, fast)
        t = time.perf_counter()
        plan = sa_stark.SignerPlan(signer)
        torch.cuda.synchronize()
        print(json.dumps({"signer": name, "plan_build_ms": round(1e3 * (time.perf_counter() - t), 2)}), flush=True)
        for B in (1, 16, 64):
            sks = [C.T.fe(3 + 7 * b) for b in range(B)]
            docs = [b"document %d" % b for b in range(B)]
            seeds = [bytes([b]) * 32 for b in range(B)]
            got = plan.sign(sks, docs, seeds)
            want = [sa_stark.sign_batch(signer, sk, [d], [s])[0] for sk, d, s in zip(sks, docs, seeds)]
            assert got == want, "SignerPlan.sign differs from sign_batch"
            plan_s = median_s(lambda: plan.sign(sks, docs, seeds), reps)
            batch_s = median_s(lambda: [sa_stark.sign_batch(signer, sk, [d], [s]) for sk, d, s in
                                        zip(sks, docs, seeds)], 1 if B > 16 else reps)
            print(json.dumps({"signer": name, "keys": B, "signer_plan_ms_per_sig": round(1e3 * plan_s / B, 3),
                              "sign_batch_ms_per_sig": round(1e3 * batch_s / B, 3)}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    eng = sa_engine.get_engine()
    assert eng.name == "cuda", "needs the CUDA engine"
    kernel_lines(eng, max(args.reps, 10))
    signing_lines(eng, args.reps)
    idx = eng.device.index
    print(json.dumps({"device": torch.cuda.get_device_name(idx), "power_limit_w": SP.power_limit_w(idx)}), flush=True)


if __name__ == "__main__":
    main()
