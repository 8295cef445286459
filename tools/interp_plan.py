#!/usr/bin/env python3
"""Interpolation plans against the one-shot call: how much of sa_interpolate depends on the values.

Per domain size k, on random device-resident points and values, timed with CUDA events around windows of at least
--window seconds after one warm-up call of the same shape (workspaces grown, twiddle plans cached):

  interpolate_ms     one sa_interpolate (builds the domain's plan, synchronises, applies)
  plan_ms            one sa_interp_plan (zerofier tree, M'(d_i) and its inverses; synchronises)
  apply_ms           one sa_interp_apply (the value-dependent part; asynchronous)
  apply_x8_ms        8 applies of one plan to 8 value vectors, queued back to back (FastStark's 8 columns)
  interpolate_x8_ms  8 sa_interpolate calls on the same 8 vectors
  apply_batchB_ms    one sa_interp_apply_batch of B vectors (--batch, default 8: the same 8 vectors as apply_x8_ms)
  plan_bytes         sa_interp_plan_bytes(k)

apply_over_interpolate = apply_ms / interpolate_ms.  One JSON line per size, then one naming the device and its
power limit (read in the same run).  Each size checks apply == sa_interpolate on its first vector, and the batch's
first and last rows against single applies."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "stark-anatomy_b200"), ROOT]
import torch  # noqa: E402

import sa_engine  # noqa: E402

SIZES = [284, 1024, 1025, 1 << 13, 1 << 16, (1 << 16) + 256, 1 << 18, 1 << 20]


def power_limit_w(index):
    """the board's enforced power limit in W as nvidia-smi reports it (a read-only query), or None"""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out)
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


def rand_vec(n, dev):
    x = torch.randint(0, 1 << 62, (n, 2), dtype=torch.int64, device=dev)
    x[:, 1] &= (1 << 61) - 1  # < 2^125 < p
    return x


def timed_ms(fn, st, window_s):
    """ms per call of fn over a window of at least window_s seconds (one warm-up call first)"""
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps, ms = 1, 0.0
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


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--window", type=float, default=0.5, help="seconds per timed window")
    ap.add_argument("--sizes", type=int, nargs="*", default=SIZES)
    ap.add_argument("--batch", type=int, default=8, help="vectors per sa_interp_apply_batch call")
    args = ap.parse_args()

    eng = sa_engine.get_engine()
    lib, dev = eng.lib, eng.device
    st = torch.cuda.current_stream(dev)
    stream = ctypes.c_void_p(st.cuda_stream)
    torch.manual_seed(0)
    for k in args.sizes:
        dom = rand_vec(k, dev)
        vals = [rand_vec(k, dev) for _ in range(8)]
        out = eng.empty(k)
        nbytes = lib.sa_interp_plan_bytes(k)
        plan = torch.empty(nbytes, dtype=torch.uint8, device=dev)

        def interpolate(v=vals[0]):
            assert lib.sa_interpolate(out.data_ptr(), dom.data_ptr(), v.data_ptr(), k, stream) == 0

        def build():
            assert lib.sa_interp_plan(plan.data_ptr(), dom.data_ptr(), k, stream) == 0

        def apply(v=vals[0]):
            assert lib.sa_interp_apply(out.data_ptr(), plan.data_ptr(), v.data_ptr(), k, stream) == 0

        build()
        apply()
        got = out.clone()
        interpolate()
        assert bool((got == out).all()), "apply differs from sa_interpolate at k = %d" % k
        row = {"k": k, "plan_bytes": nbytes,
               "interpolate_ms": timed_ms(interpolate, st, args.window),
               "plan_ms": timed_ms(build, st, args.window),
               "apply_ms": timed_ms(apply, st, args.window),
               "apply_x8_ms": timed_ms(lambda: [apply(v) for v in vals], st, args.window),
               "interpolate_x8_ms": timed_ms(lambda: [interpolate(v) for v in vals], st, args.window)}
        # after the single-vector columns, which thus run on the memory and workspaces they had before the batch
        vbatch = torch.stack((vals + [rand_vec(k, dev) for _ in range(args.batch - 8)])[:args.batch])
        obatch = torch.empty_like(vbatch)

        def apply_batch():
            assert lib.sa_interp_apply_batch(obatch.data_ptr(), plan.data_ptr(), vbatch.data_ptr(), k, args.batch,
                                             stream) == 0

        apply_batch()
        for b in (0, args.batch - 1):
            apply(vbatch[b])
            assert bool((obatch[b] == out).all()), "batch row %d differs from a single apply at k = %d" % (b, k)
        row["apply_batch%d_ms" % args.batch] = timed_ms(apply_batch, st, args.window)
        row["apply_over_interpolate"] = row["apply_ms"] / row["interpolate_ms"]
        print(json.dumps({key: (round(v, 4) if isinstance(v, float) else v) for key, v in row.items()}), flush=True)
        del plan, dom, vals, out, vbatch, obatch
        torch.cuda.synchronize(dev)
        torch.cuda.empty_cache()
        assert lib.sa_release_workspaces() == 0
    print(json.dumps({"device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index),
                      "window_s": args.window}), flush=True)


if __name__ == "__main__":
    main()
