#!/usr/bin/env python3
"""Batched verification on the device (sa_stark.VerifierPlan, SignerPlan.verify; DESIGN sections 3.15 and 3.17).

Per-signature verify time of SignerPlan.verify at B = 1, 16, 64 and 256 seeded signatures from one SignerPlan.sign,
for the stand-in FastRPSSS and RPSSS of tests/stark_rescue_cases.py, through the device route (proofs read from their
bytes on the device) and the host route (unpickled and packed on the host) in the same process, alternating (median
of --reps calls after a warm-up call that builds the verifier plan; host clock around a call, whose verdicts are host
booleans, so it ends in a device synchronise).  Beside each device-route row: the transcript kernels' CUDA-event
time on their own (sa_transcript_sections for the whole batch), the route's own upload of the chunk (upload_bytes,
host clock to a device synchronise) and the host time left per signature (the call minus both).  Then the time of one
VerifierPlan.verify of a synthetic proof at 2^12, 2^16 and 2^20 FRI domains.
Beside the synthetic proofs, the host route: tests/stark_verify.py, a restatement of FastStark.verify on the drop-in
Fri.verify (the last codeword's degree by an inverse transform).  Every verdict
is checked True.  Not measured: the unmodified reference's verify (it does not run on the GPU machine; BASELINE gives
205.8 s for FastRPSSS and 444 s for RPSSS on a CPU), and a host route for plain Stark proofs.  Prints one JSON line per measurement with the device name and power limit.

    python tools/stark_verify.py [--reps 5]
"""
import argparse
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

import oracle as O  # noqa: E402
import sa_engine  # noqa: E402
import sa_stark  # noqa: E402
import stark_cases as C  # noqa: E402
import stark_plain_cases as S  # noqa: E402
import stark_rescue_cases as SR  # noqa: E402
import stark_verify as SV  # noqa: E402
import verify_cases as V  # noqa: E402


def device():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, reps):
    out = fn()  # warm-up
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        times.append(time.perf_counter() - t0)
    return statistics.median(times), out


def transcript_times(eng, vp, sigs, docs, pks, plan):
    """(ms of sa_transcript_sections over the batch as one chunk by CUDA events, ms of the route's own upload of that
    chunk: upload_bytes from pageable host memory, host clock to a device synchronise)"""
    items = [(p, vp._fs_prefix(plan.stream(d)), vp._statement(plan.rp.boundary_constraints(pk)))
             for p, d, pk in zip(sigs, docs, pks)]
    raw, parts, L, nstat = vp._transcript_chunk(items)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    buf = eng.upload_bytes(raw)
    eng.transcript_sections(buf, parts, L, nstat, len(items), vp.transcript)  # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    buf = eng.upload_bytes(raw)
    torch.cuda.synchronize()
    upload = time.perf_counter() - t0
    ev[1].record()
    eng.transcript_sections(buf, parts, L, nstat, len(items), vp.transcript)
    ev[2].record()
    torch.cuda.synchronize()
    return ev[1].elapsed_time(ev[2]), 1e3 * upload


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batches", default="1,16,64,256", help="comma-separated signature counts")
    ap.add_argument("--no-synthetic", action="store_true")
    a = ap.parse_args()
    import __graft_entry__ as G
    G.build()
    eng = sa_engine.get_engine()
    dev = device()
    min_proofs = sa_stark.DEVICE_ROUTE_MIN_PROOFS
    for fast in (True, False):
        rec = (C.golden() if fast else S.golden())["rpsss"]
        signer = SR.Signer(rec, fast)
        if fast:
            signer.transition_zerofier_root = bytes.fromhex(rec["zerofier_root"])
        plan = sa_stark.SignerPlan(signer)
        plan.stream = V.SignatureProofStream
        for B in [int(x) for x in a.batches.split(",")]:
            sks = [C.T.fe(11 + 5 * d) for d in range(B)]
            docs = [b"document %d" % d for d in range(B)]
            sigs = plan.sign(sks, docs, [bytes([d % 256]) * 32 for d in range(B)])
            pks = [signer.rp.hash(sk) for sk in sks]
            assert plan.verify(pks, docs, sigs) == [True] * B  # builds the verifier plan
            vp = plan._verifier
            shape = vp.transcript
            routes = {"device": [], "host": []}
            sa_stark.DEVICE_ROUTE_MIN_PROOFS = 1  # both routes at every B; the default selects by B
            for _ in range(a.reps):
                for route in ("device", "host"):
                    vp.transcript = shape if route == "device" else None
                    t, got = timed(lambda: plan.verify(pks, docs, sigs), 1)
                    assert got == [True] * B
                    routes[route].append(t)
            vp.transcript = shape
            sa_stark.DEVICE_ROUTE_MIN_PROOFS = min_proofs
            kernel_ms, upload_ms = transcript_times(eng, vp, sigs, docs, pks, plan)
            dev_t = statistics.median(routes["device"])
            line = {"what": "SignerPlan.verify", "signer": "FastRPSSS" if fast else "RPSSS", "B": B,
                    "device_route_ms_per_signature": 1e3 * dev_t / B,
                    "host_route_ms_per_signature": 1e3 * statistics.median(routes["host"]) / B,
                    "transcript_kernels_ms": kernel_ms, "upload_ms": upload_ms,
                    "signature_bytes": len(sigs[0]),
                    "host_left_ms_per_signature": (1e3 * dev_t - kernel_ms - upload_ms) / B, "device": dev}
            print(json.dumps(line), flush=True)
    for log_fri in () if a.no_synthetic else (12, 16, 20):
        stark, cons, _, boundary = C.synthetic(0, log_fri)
        proof, _ = C.synthetic_prove(0, log_fri)
        root = O.merkle_tree_np(O.to_np(C.zerofier(stark)[1]))[1].tobytes()
        plan = sa_stark.VerifierPlan(stark, cons, root)
        t, got = timed(lambda: plan.verify(proof, boundary), a.reps)
        assert got is True
        t0 = time.perf_counter()
        assert SV.verify(stark, proof, cons, boundary, root) is True
        host = time.perf_counter() - t0
        print(json.dumps({"what": "VerifierPlan.verify", "fri_domain": 1 << log_fri, "ms": 1e3 * t,
                          "host_route_ms": 1e3 * host, "device": dev}), flush=True)
    eng.synchronize()


if __name__ == "__main__":
    main()
