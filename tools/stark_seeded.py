#!/usr/bin/env python3
"""Seeded proofs (sa_stark with seeds: the randomizers drawn on the device by sa_sample_seeded) against the unseeded
prover fed the same draws on the host through os.urandom = sa_stark.seeded_urandom(seed), on the fixture's FastRPSSS
and RPSSS signatures, synthetic three-register AIRs at FRI domains 2^16 and 2^20 (tests/stark_cases.synthetic), and
the two-register AIR of a 2^20 + 1-row randomized trace at a 2^24 FRI domain (tests/test_gpu_stark_geo.air24).  Each
instance asserts that both routes give the same bytes, then reports:

  seeded_ms, unseeded_ms  one proof with a kept plan, median of --reps after a warm-up: host clock around a call that
                          ends in a synchronising read (the unseeded one includes its host draws)
  device_ms               inside one seeded proof: CUDA events around each engine call of the device stages, summed
  host_ms                 seeded_ms - device_ms: the Python side that is left
  draws_ms                the host draws alone: field.sample(seeded_urandom(seed)(17)) as many times as a proof draws

then one line for the sampler kernel alone (2^21 draws, CUDA events over 20 launches after a warm-up), and one naming
the device and its power limit (read in the same run)."""
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

import oracle as O  # noqa: E402
import sa_devlist  # noqa: E402
import sa_engine  # noqa: E402
import sa_stark  # noqa: E402
import stark_cases as C  # noqa: E402
import stark_plain_cases as S  # noqa: E402
import stark_prove as SP  # noqa: E402

if "sample_seeded" not in SP.STAGES:
    SP.STAGES.append("sample_seeded")


def measure(eng, label, plan, trace, boundary, zcw, reps, stream=None):
    seed = bytes(range(32))

    def prove(seeded):
        ps = stream() if stream else None
        real = os.urandom
        os.urandom = sa_stark.seeded_urandom(seed)
        try:
            s = [seed] if seeded else None
            if zcw is None:
                proof = plan.prove_batch([trace], [boundary], None if ps is None else [ps], seeds=s)[0]
            else:
                proof = plan.prove_batch([trace], [boundary], zcw, None if ps is None else [ps], seeds=s)[0]
        finally:
            os.urandom = real
        torch.cuda.synchronize()
        return proof

    def median_ms(fn):
        fn()
        times = []
        for _ in range(reps):
            t0 = time.perf_counter()
            fn()
            times.append(1e3 * (time.perf_counter() - t0))
        return statistics.median(times)

    seeded = prove(True)
    assert seeded == prove(False), "%s: the seeded proof differs from the seeded_urandom route" % label
    seeded_ms = median_ms(lambda: prove(True))
    unseeded_ms = median_ms(lambda: prove(False))
    dev = SP.device_ms(eng, lambda: prove(True))
    ndraws = plan.nregs * plan.stark.num_randomizers + plan.max_degree + 1
    t0 = time.perf_counter()
    urandom, field = sa_stark.seeded_urandom(seed), plan.stark.field
    for _ in range(ndraws):
        field.sample(urandom(17))
    draws_ms = 1e3 * (time.perf_counter() - t0)
    line = {"instance": label, "fri_domain": 1 << plan.log_n, "trace_length": plan.trace_length, "draws": ndraws,
            "seeded_ms": round(seeded_ms, 2), "unseeded_ms": round(unseeded_ms, 2), "device_ms": round(dev, 2),
            "host_ms": round(seeded_ms - dev, 2), "draws_ms": round(draws_ms, 2), "bytes_equal": True}
    print(json.dumps(line), flush=True)


def kernel_ms(eng, count=1 << 21, launches=20):
    out = eng.empty(count)
    seeds = eng.upload_seeds([bytes(32)])
    eng.sample_seeded(out, seeds, 0, count)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        eng.sample_seeded(out, seeds, 0, count)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / launches
    print(json.dumps({"kernel": "k_sample_seeded", "draws": count, "ms": round(ms, 4),
                      "draws_per_s": round(count / ms * 1e3)}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip24", action="store_true", help="leave out the 2^24 FRI domain instance")
    args = ap.parse_args()
    eng = sa_engine.get_engine()
    g, gp = C.golden(), S.golden()

    rec = g["rpsss"]
    st = C.params(rec)
    zpoly, zvals = C.zerofier(st)
    trace, boundary = C.inputs(rec)
    measure(eng, "FastRPSSS", sa_stark.StarkPlan(st, C.air(rec), zpoly), trace, boundary,
            C.zerofier_codeword(zvals, True), args.reps, stream=lambda: C.stream(rec))
    rec = gp["rpsss"]
    trace, boundary = C.inputs(rec)
    measure(eng, "RPSSS", sa_stark.PlainStarkPlan(S.stark(rec), C.air(rec)), trace, boundary, None, args.reps,
            stream=lambda: C.stream(rec))
    for log_fri in (16, 20):
        st, cons, trace, boundary = C.synthetic(log_fri, log_fri)
        zpoly, zvals = C.zerofier(st)
        measure(eng, "synthetic_2^%d" % log_fri, sa_stark.StarkPlan(st, cons, zpoly), trace, boundary,
                C.zerofier_codeword(zvals, True), args.reps)
    if not args.skip24:
        from test_gpu_stark_geo import NCYCLES, air24, fe_boundary, fe_trace
        st, cons, rows, boundary = air24()
        n = st.fri_domain_length
        z = eng.geo_zerofier(st.omicron.value, NCYCLES - 1)
        zpoly = O.from_np(eng.download(z).view(np.uint64))
        cw = eng.coset_evaluate(z, n.bit_length() - 1, st.omega.value, st.generator.value)
        zcw = sa_devlist.DeviceCodeword(cw, None, C.T.field, n)
        measure(eng, "air24_T=2^20+1", sa_stark.StarkPlan(st, cons, zpoly), fe_trace(rows), fe_boundary(boundary),
                zcw, args.reps)
    kernel_ms(eng)
    props = torch.cuda.get_device_properties(eng.device)
    print(json.dumps({"device": props.name, "power_limit_w": SP.power_limit_w(eng.device.index)}), flush=True)


if __name__ == "__main__":
    main()
