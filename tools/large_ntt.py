#!/usr/bin/env python3
"""One in-place transform per size, 2^24 ... 2^30, forward and inverse, timed with CUDA events after warm-up.

2^24 ... 2^26 run the three-pass plan with the full n-entry pass-1 matrix, 2^27 ... 2^30 the plan with factored
pass-1 twiddles (one more Montgomery product per element in pass 1), so the output shows both sides of that
choice.  One JSON line per size and direction, then one line naming the device and its power limit.

  butterflies_per_s  (n/2) log2 n butterflies / time
  alg_GB_per_s       32 n algorithmic bytes (read + write of every element, 16 bytes each) / time
  plan_bytes         growth of sa_cache_bytes when the size's plan was built (twiddle tables)
  workspace_bytes    device memory the first call kept besides its plan (the n-element intermediate)

A size is skipped, before anything is allocated for it, when the vector and the intermediate (2 * 16 n bytes)
plus a margin do not fit in the device's free memory.  Workspaces are released between sizes."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "stark-anatomy_b200"), os.path.join(ROOT, "oracle"), ROOT]
import torch  # noqa: E402

import oracle as O  # noqa: E402
import sa_engine  # noqa: E402

MARGIN = 2 << 30


def power_limit_w(index):
    """the board's enforced power limit in W as nvidia-smi reports it (a read-only query), or None"""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out)
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--min-log", type=int, default=24)
    ap.add_argument("--max-log", type=int, default=30)
    ap.add_argument("--reps", type=int, default=5, help="timed transforms per size and direction")
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    eng = sa_engine.get_engine()
    lib, dev = eng.lib, eng.device
    st = torch.cuda.current_stream(dev)
    stream = ctypes.c_void_p(st.cuda_stream)
    for log_n in range(args.min_log, args.max_log + 1):
        n = 1 << log_n
        torch.cuda.synchronize(dev)
        torch.cuda.empty_cache()
        assert lib.sa_release_workspaces() == 0
        free, _ = torch.cuda.mem_get_info(dev)
        need = 2 * 16 * n + MARGIN
        if free < need:
            print(json.dumps({"log_n": log_n, "skipped": "needs %d bytes free, %d are" % (need, free)}), flush=True)
            continue
        x = torch.randint(0, 1 << 62, (n, 2), dtype=torch.int64, device=dev)
        x[:, 1] &= (1 << 61) - 1
        root = sa_engine._limbs(O.primitive_nth_root(n))
        for inverse in (0, 1):
            call = lambda: lib.sa_ntt(x.data_ptr(), x.data_ptr(), log_n, root, inverse, 1, stream)
            torch.cuda.synchronize(dev)
            free0, cache0 = torch.cuda.mem_get_info(dev)[0], lib.sa_cache_bytes()
            assert call() == 0
            torch.cuda.synchronize(dev)
            plan = lib.sa_cache_bytes() - cache0
            kept = free0 - torch.cuda.mem_get_info(dev)[0]
            for _ in range(args.warmup - 1):
                assert call() == 0
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for _ in range(args.reps):
                call()
            e1.record(st)
            torch.cuda.synchronize(dev)
            s = e0.elapsed_time(e1) / args.reps * 1e-3
            print(json.dumps({"log_n": log_n, "inverse": bool(inverse),
                              "pass1_twiddles": "factored" if log_n > 26 else "full matrix",
                              "ms": round(s * 1e3, 4), "butterflies_per_s": (n // 2) * log_n / s,
                              "alg_GB_per_s": 32 * n / s / 1e9, "plan_bytes": plan,
                              "workspace_bytes": max(kept - plan, 0) if inverse == 0 else None}), flush=True)
        del x
    print(json.dumps({"device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index),
                      "reps": args.reps, "warmup": args.warmup}), flush=True)


if __name__ == "__main__":
    main()
