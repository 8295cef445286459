#!/usr/bin/env python3
"""The device prover (sa_stark) end to end: FastStark.prove's result from a trace, on the fixture's FastRPSSS
instance (tests/golden/stark.json, FRI domain 4096) and on seeded synthetic AIRs (tests/stark_cases.synthetic: three
registers, a cubic, a linear and a quadratic constraint, expansion factor 4) at FRI domains 2^12 ... 2^20.

  plan_ms      one StarkPlan build (interpolation plan, AIR plans, zerofier upload; it synchronises): host clock
  prove_ms     StarkPlan.prove, median of --reps calls after one warm-up: host clock around a call that ends in a
               synchronising read
  oneshot_ms   sa_stark.prove (a plan built for the call, as the rebound FastStark.prove runs), median of --reps
  device_ms    inside one StarkPlan.prove: CUDA events around each engine call of the device stages (interpolation,
               boundary and transition quotients, coset evaluation, trees, combination, the FRI commit, openings and
               gathers), summed; host_ms = prove_ms - device_ms is the Python side (draws, packing, Fiat-Shamir,
               pickling, FRI's queries)

The drop-in route (the reference's own fast_stark.py on the drop-in modules) needs the reference's code and is not
run here: BASELINE config 5 gives 29.4 s for FastRPSSS.sign on the reference alone.  One JSON line per instance, then
one naming the device and its power limit (read in the same run).  The RPSSS line checks the proof against the
recorded SHA-256.

--plain times the plain prover (sa_stark.PlainStarkPlan, Stark.prove's device route) instead, with the same columns:
the fixture's first RPSSS signature (tests/golden/stark_plain.json, replayed from its recorded trace, AIR and draws,
checked against the recorded SHA-256), the synthetic AIRs on a Stark stand-in, and per synthetic size the exact
transition quotients against the unchecked ones (exact_ms / unchecked_ms: CUDA events around one apply of every
division order's plan, median of --reps after a warm call)."""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "stark-anatomy_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"),
                ROOT]
import torch  # noqa: E402

import sa_engine  # noqa: E402
import stark_cases as C  # noqa: E402
import stark_plain_cases as S  # noqa: E402
import sa_devlist  # noqa: E402
import sa_stark  # noqa: E402

STAGES = ["interp_apply", "boundary_plan", "boundary_quotients", "air_quotients", "air_quotients_exact", "zerofier",
          "coset_evaluate", "merkle_trees",
          "coset_combine_evaluate", "fri_commit", "merkle_open_batch", "merkle_open", "gather_batch", "gather"]


def power_limit_w(index):
    """the board's enforced power limit in W as nvidia-smi reports it (a read-only query), or None"""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out)
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


def device_ms(eng, call):
    """the summed CUDA-event time of the engine's device stages during call()"""
    spans, saved = [], {}
    for name in STAGES:
        fn = getattr(eng, name)
        saved[name] = fn

        def timed(*a, _fn=fn, **k):
            st = torch.cuda.current_stream(eng.device)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            try:
                return _fn(*a, **k)
            finally:
                e1.record(st)
                spans.append((e0, e1))
        setattr(eng, name, timed)
    try:
        call()
    finally:
        for name in STAGES:
            delattr(eng, name)
    torch.cuda.synchronize()
    return sum(a.elapsed_time(b) for a, b in spans)


def measure(eng, label, stark, constraints, trace, boundary, zpoly, zcw, draws, reps, stream=None, want=None,
            plain=False):
    def one(plan=None):
        d = C.Urandom(draws)
        ps = stream() if stream else None
        if plain:
            proof = S.run(stark, trace, constraints, boundary, d, ps, plan)
        else:
            proof, _ = C.run(stark, trace, constraints, boundary, zpoly, zcw, d, ps, plan)
        torch.cuda.synchronize()
        assert isinstance(proof, bytes), proof
        return proof

    t0 = time.perf_counter()
    plan = sa_stark.PlainStarkPlan(stark, constraints) if plain else sa_stark.StarkPlan(stark, constraints, zpoly)
    torch.cuda.synchronize()
    plan_ms = 1e3 * (time.perf_counter() - t0)
    proof = one(plan)
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        one(plan)
        times.append(1e3 * (time.perf_counter() - t0))
    oneshot = []
    for _ in range(reps):
        t0 = time.perf_counter()
        one()
        oneshot.append(1e3 * (time.perf_counter() - t0))
    dev = device_ms(eng, lambda: one(plan))
    prove_ms = statistics.median(times)
    line = {"instance": label, "fri_domain": 1 << plan.log_n, "registers": stark.num_registers,
            "trace_length": plan.trace_length, "plan_ms": round(plan_ms, 2), "prove_ms": round(prove_ms, 2),
            "prove_ms_min_max": [round(min(times), 2), round(max(times), 2)],
            "oneshot_ms": round(statistics.median(oneshot), 2), "device_ms": round(dev, 2),
            "host_ms": round(prove_ms - dev, 2), "proof_bytes": len(proof),
            "proof_sha256": hashlib.sha256(proof).hexdigest()}
    if want is not None:
        line["matches_reference"] = line["proof_sha256"] == want
    if plain:
        line.update(exact_against_unchecked(eng, plan, trace, reps))
    print(json.dumps(line), flush=True)
    return plan


def exact_against_unchecked(eng, plan, trace, reps):
    """CUDA-event medians of one air_quotients_exact and one air_quotients per division order of a plain plan, on
    the plan's trace polynomials (interpolated once, without randomizers)"""
    T = plan.trace_length
    rows = [list(r) for r in trace] + [[0] * plan.nregs] * (T - len(trace))
    cols = eng.upload(sa_devlist.pack([rows[c][s] for s in range(plan.nregs) for c in range(T)]))
    polys = eng.interp_apply(plan.interp, cols.reshape(plan.nregs, T, 2))
    out = {}
    for name, call in (("exact_ms", lambda p, q: eng.air_quotients_exact(p, polys, q, check=False)),
                       ("unchecked_ms", lambda p, q: eng.air_quotients(p, polys, q))):
        times = []
        for _ in range(reps + 1):
            st = torch.cuda.current_stream(eng.device)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for p, _, q in plan.groups:
                call(p, q)
            e1.record(st)
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        out[name] = round(statistics.median(times[1:]), 3)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--logs", default="12,14,16,18,20", help="synthetic FRI domains (log2), comma separated")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--plain", action="store_true", help="time the plain prover (Stark.prove's route) instead")
    args = ap.parse_args()
    eng = sa_engine.get_engine()
    if args.plain:
        return main_plain(eng, args)

    rec = C.golden()["rpsss"]
    stark = C.params(rec)
    zpoly, zvals = C.zerofier(stark)
    trace, boundary = C.inputs(rec)
    measure(eng, "rpsss_sign", stark, C.air(rec), trace, boundary, zpoly, C.zerofier_codeword(zvals, True),
            rec["draws"], args.reps, stream=lambda: C.stream(rec), want=rec["proof_sha256"])

    for lg in [int(x) for x in args.logs.split(",") if x]:
        stark, cons, trace, boundary = C.synthetic(lg, lg)
        zpoly, zvals = C.zerofier(stark)
        draws = list(range(1, stark.num_registers * stark.num_randomizers + stark.fri_domain_length + 1))
        measure(eng, "synthetic", stark, cons, trace, boundary, zpoly, C.zerofier_codeword(zvals, True), draws,
                args.reps)

    idx = eng.device.index
    print(json.dumps({"device": torch.cuda.get_device_name(idx), "power_limit_w": power_limit_w(idx),
                      "drop_in_route_ms": "not measured (needs the reference's fast_stark.py)",
                      "reference_sign_s_baseline_config5": 29.4}), flush=True)


def main_plain(eng, args):
    rec = S.golden()["rpsss"]
    trace, boundary = C.inputs(rec)
    measure(eng, "rpsss_sign_plain", S.stark(rec), C.air(rec), trace, boundary, None, None, rec["draws"], args.reps,
            stream=lambda: C.stream(rec), want=rec["proof_sha256"], plain=True)
    for lg in [int(x) for x in args.logs.split(",") if x]:
        params, cons, trace, boundary = C.synthetic(lg, lg)
        draws = list(range(1, params.num_registers * params.num_randomizers + params.fri_domain_length + 1))
        measure(eng, "synthetic_plain", S.plain_stark(params), cons, trace, boundary, None, None, draws, args.reps,
                plain=True)
    idx = eng.device.index
    print(json.dumps({"device": torch.cuda.get_device_name(idx), "power_limit_w": power_limit_w(idx),
                      "reference_rpsss_sign_s": "182 (one run of the unmodified reference on a CPU machine)"}),
          flush=True)


if __name__ == "__main__":
    main()
