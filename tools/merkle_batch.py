#!/usr/bin/env python3
"""Batched Merkle commitments and openings against one call per codeword: what a prover that commits to B codewords
of one length, and later opens the same leaves in all of them, gains from the batch entry points.

Per size n = 2^log_n and batch B (--batches), on random device-resident codewords, timed with CUDA events around
windows of at least --window seconds after one warm-up call of the same shape:

  trees_single_ms   B sa_merkle_tree calls, one per codeword, queued back to back
  trees_batch_ms    one sa_merkle_tree_batch of the B codewords
  open_single_ms    B merkle_open + B gather engine calls of the same 64 sorted leaf indices (each uploads the
                    indices and downloads its result)
  open_batch_ms     one merkle_open_batch + one gather_batch engine call of those indices

Each shape first checks that the batched trees, paths and values equal the single calls'.  One JSON line per
(size, batch), then one naming the device and its power limit (read in the same run).

--guard LIB runs, after that, the regression guard: sa_fri_commit (12 rounds, constant challenge) and sa_merkle_tree
at 2^20 timed in fresh processes, alternating this tree's library with LIB (SA_B200_LIB selects the build),
--guard-reps times each, one JSON line per run and a summary line with each library's range and whether the two
computed the same roots."""
import argparse
import ctypes
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "stark-anatomy_b200"), os.path.join(ROOT, "oracle"), ROOT]

LOGS = [10, 12, 14, 16, 18, 20]
BATCHES = [8, 32]
GUARD_LOG = 20
GUARD_ROUNDS = 12  # Fri(ef 4, 64 colinearity tests).num_rounds() at 2^20, as bench.py
GENERATOR = 85408008396924667383611388730472331217  # algebra.py:100-102, order 2^119
P = 1 + 407 * (1 << 119)


def power_limit_w(index):
    """the board's enforced power limit in W as nvidia-smi reports it (a read-only query), or None"""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out)
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


def rand_vec(shape, dev):
    import torch
    x = torch.randint(0, 1 << 62, tuple(shape) + (2,), dtype=torch.int64, device=dev)
    x[..., 1] &= (1 << 61) - 1  # < 2^125 < p
    return x


def timed_ms(fn, st, window_s):
    """ms per call of fn over a window of at least window_s seconds (one warm-up call first)"""
    import torch
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


def measure(args):
    import torch
    import sa_engine
    eng = sa_engine.get_engine()
    lib, dev = eng.lib, eng.device
    st = torch.cuda.current_stream(dev)
    stream = ctypes.c_void_p(st.cuda_stream)
    torch.manual_seed(0)
    rng = random.Random(0)
    for log_n in args.logs:
        n = 1 << log_n
        for batch in args.batches:
            vecs = rand_vec((batch, n), dev)
            trees = torch.empty((batch, 2 * n, 64), dtype=torch.uint8, device=dev)
            ptrs = [(trees[b].data_ptr(), vecs[b].data_ptr()) for b in range(batch)]
            idx = sorted(rng.sample(range(n), min(64, n)))

            def trees_single():
                for t, v in ptrs:
                    assert lib.sa_merkle_tree(t, v, n, stream) == 0

            def trees_batch():
                assert lib.sa_merkle_tree_batch(trees.data_ptr(), vecs.data_ptr(), n, batch, stream) == 0

            def open_single():
                return ([eng.merkle_open(trees[b], idx) for b in range(batch)],
                        [eng.gather(vecs[b], idx) for b in range(batch)])

            def open_batch():
                return eng.merkle_open_batch(trees, idx), eng.gather_batch(vecs, idx)

            trees_single()
            want = trees.clone()
            trees.zero_()
            trees_batch()
            assert bool((trees == want).all()), "batched trees differ at 2^%d x %d" % (log_n, batch)
            (ps, gs), (pb, gb) = open_single(), open_batch()
            assert ps == pb and all((gs[b] == gb[b]).all() for b in range(batch)), "openings differ"
            row = {"log_n": log_n, "batch": batch,
                   "trees_single_ms": timed_ms(trees_single, st, args.window),
                   "trees_batch_ms": timed_ms(trees_batch, st, args.window),
                   "open_single_ms": timed_ms(open_single, st, args.window),
                   "open_batch_ms": timed_ms(open_batch, st, args.window)}
            row["trees_speedup"] = row["trees_single_ms"] / row["trees_batch_ms"]
            row["open_speedup"] = row["open_single_ms"] / row["open_batch_ms"]
            print(json.dumps({key: (round(v, 4) if isinstance(v, float) else v) for key, v in row.items()}), flush=True)
            del vecs, trees, want, ptrs
            torch.cuda.synchronize(dev)
            torch.cuda.empty_cache()
    print(json.dumps({"device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index),
                      "window_s": args.window}), flush=True)


def guard_child(window_s):
    """one guard run in this process, on the library SA_B200_LIB names: prints one JSON line"""
    import hashlib
    import torch
    import sa_engine
    present = ctypes.CDLL(sa_engine.LIB_PATH)
    # an older build lacks the batch entry points: bind what it has
    sa_engine.SYMBOLS = [s for s in sa_engine.SYMBOLS if hasattr(present, s[0])]
    eng = sa_engine.get_engine()
    dev = eng.device
    st = torch.cuda.current_stream(dev)
    stream = ctypes.c_void_p(st.cuda_stream)
    n = 1 << GUARD_LOG
    torch.manual_seed(1)
    cw = rand_vec((n,), dev)
    tree = torch.empty((2 * n, 64), dtype=torch.uint8, device=dev)
    omega = GENERATOR
    for _ in range(119 - GUARD_LOG):
        omega = omega * omega % P

    def fri_commit():
        roots = []
        eng.fri_commit(cw, GUARD_ROUNDS, GENERATOR, omega, lambda r, root, want: (roots.append(root), 12345678901)[1])
        return roots

    def merkle_tree():
        assert eng.lib.sa_merkle_tree(tree.data_ptr(), cw.data_ptr(), n, stream) == 0

    roots = fri_commit()
    merkle_tree()
    torch.cuda.synchronize()
    digest = hashlib.blake2b(b"".join(roots) + tree.cpu().numpy().tobytes()).hexdigest()[:32]
    t0, reps = time.perf_counter(), 0
    while time.perf_counter() - t0 < window_s:  # host-synchronous: every round waits for its root
        fri_commit()
        reps += 1
    torch.cuda.synchronize()
    fri_ms = (time.perf_counter() - t0) / reps * 1e3
    print(json.dumps({"fri_commit_ms": round(fri_ms, 4), "merkle_tree_ms": round(timed_ms(merkle_tree, st, window_s), 4),
                      "result_digest": digest}), flush=True)


def guard(other_lib, reps, window_s):
    ours = os.path.join(ROOT, "stark-anatomy_b200", "libsa_b200.so")
    libs = {"this": ours, "other": os.path.abspath(other_lib)}
    runs = {"this": [], "other": []}
    for rep in range(reps):
        for label in (("this", "other") if rep % 2 == 0 else ("other", "this")):  # alternate which goes first
            env = dict(os.environ, SA_B200_LIB=libs[label])
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--guard-child", "--window", str(window_s)],
                                 env=env, capture_output=True, text=True, check=True).stdout
            line = json.loads(out.strip().splitlines()[-1])
            runs[label].append(line)
            print(json.dumps(dict(line, lib=label, rep=rep)), flush=True)
    summary = {"guard": "fri_commit and merkle_tree at 2^%d" % GUARD_LOG, "same_results":
               len({r["result_digest"] for rs in runs.values() for r in rs}) == 1}
    for label, rs in runs.items():
        for key in ("fri_commit_ms", "merkle_tree_ms"):
            vals = sorted(r[key] for r in rs)
            summary["%s_%s" % (label, key)] = [vals[0], vals[len(vals) // 2], vals[-1]]  # min, median, max
    print(json.dumps(summary), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--window", type=float, default=0.3, help="seconds per timed window")
    ap.add_argument("--logs", type=int, nargs="*", default=LOGS, help="log2 of the codeword lengths")
    ap.add_argument("--batches", type=int, nargs="*", default=BATCHES, help="codewords per batch")
    ap.add_argument("--guard", metavar="LIB", help="another build of libsa_b200.so to alternate with at 2^20")
    ap.add_argument("--guard-reps", type=int, default=4, help="guard runs per library")
    ap.add_argument("--guard-child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.guard_child:
        return guard_child(args.window)
    measure(args)
    if args.guard:
        guard(args.guard, args.guard_reps, args.window)


if __name__ == "__main__":
    main()
