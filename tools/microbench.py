#!/usr/bin/env python3
"""Field-arithmetic microbenchmark on the GPU (sa_microbench): per-op issue cost in SM cycles.
Output: one JSON line per (op, ilp)."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "stark-anatomy_b200"), ROOT]
import sa_engine
lib = sa_engine.load_library()
import torch
torch.cuda.init()
sm_count = torch.cuda.get_device_properties(0).multi_processor_count
names = {0: "montmul", 1: "add", 2: "sub", 3: "butterfly", 5: "tile butterfly"}
iters, blocks, threads = 2000, sm_count * 4, 256
for op in (0, 1, 2, 3, 5):
    for ilp in (1, 2, 4, 8):
        ms = lib.sa_microbench(op, ilp, iters, blocks, threads)
        ops = iters * ilp * blocks * threads
        print(json.dumps({"op": names[op], "ilp": ilp, "ms": ms, "Gops_per_s": ops / ms / 1e6,
                          "warp_ops_per_sm_per_us": ops / 32 / sm_count / (ms * 1e3)}))
