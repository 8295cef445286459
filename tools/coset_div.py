#!/usr/bin/env python3
"""Coset division plans and evaluations, through the engine and through the drop-in: how much of fast_coset_divide
depends on the numerator, and what a caller of the drop-in pays.

Per size n = 2^log_n, on random device-resident operands (numerators of n coefficients, a divisor of n/2 + 1, so
quotients of n/2; polynomials of n/4 coefficients to evaluate), timed with CUDA events around windows of at least
--window seconds after one warm-up call of the same shape (workspaces grown, twiddle plans cached):

  oneshot_ms           one numerator through the engine calls the drop-in's fast_coset_divide makes: coset_div_plan
                       (synchronises) and coset_div_apply of one row
  plan_ms              one sa_coset_div_plan (offset^i, offset^-i, the divisor's transform and its inverses;
                       synchronises)
  apply_ms             one sa_coset_div_apply_batch of 1 row (asynchronous)
  oneshot_x8_ms        8 one-shot divisions of 8 numerators by the same divisor
  apply_x8_ms          8 single applies of one plan to the same 8 numerators, queued back to back
  apply_batchB_ms      one sa_coset_div_apply_batch of B rows (--batch, default 8: the same 8 numerators)
  evaluate_x8_ms       8 coset_evaluate calls of one polynomial each, the engine call of the drop-in's
                       fast_coset_evaluate
  evaluate_batchB_ms   one sa_coset_evaluate_batch of B rows (the same 8 polynomials)
  dropin_divide_ms     ntt.fast_coset_divide of the first numerator by the divisor as Polynomials: the uploads, the
                       engine calls and the quotient's download into FieldElements
  dropin_evaluate_ms   ntt.fast_coset_evaluate of the first polynomial as a Polynomial: its upload and the engine
                       call (the codeword stays on the device, as the drop-in returns it)
  plan_bytes           sa_coset_div_plan_bytes(log_n)

The C calls are timed as such; the engine columns include the engine's Python and allocations, which the drop-in
pays too.  One JSON line per size, then one naming the device and its power limit (read in the same run).  Each size
checks the division and the evaluation of the first numerator and polynomial against the oracle up to 2^20, and
above by the property ntt(U) * R == L of a full row, and checks that the drop-in, the single calls and the first and
last batched rows agree."""
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
import sa_devlist  # noqa: E402
import sa_engine  # noqa: E402
import sa_host  # noqa: E402
import ntt as dropin  # noqa: E402

LOGS = [10, 14, 16, 18, 20, 22]
ORACLE_MAX_LOG = 20
P = sa_engine.P
GENERATOR = 85408008396924667383611388730472331217  # algebra.py:100-102, order 2^119


def power_limit_w(index):
    """the board's enforced power limit in W as nvidia-smi reports it (a read-only query), or None"""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out)
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


def rand_vec(shape, dev):
    x = torch.randint(0, 1 << 62, tuple(shape) + (2,), dtype=torch.int64, device=dev)
    x[..., 1] &= (1 << 61) - 1  # < 2^125 < p
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


def check(eng, log_n, root, offset, divisor, num, poly):
    """the division of num by divisor at order n, and the evaluation of poly, against the oracle up to ORACLE_MAX_LOG,
    else a full row U * offset^-j of the division by ntt(U) * R == L on the coset"""
    n = 1 << log_n
    if log_n <= ORACLE_MAX_LOG:
        rows = [O.from_np(v.cpu().numpy().view("<u8")) for v in (num, divisor, poly)]
        q = eng.coset_div_apply(eng.coset_div_plan(divisor, log_n, root, offset), num, n // 2)
        assert O.from_np(q.cpu().numpy().view("<u8")) == O.fast_coset_divide(rows[0], rows[1], offset, root, n)
        ev = eng.coset_evaluate(poly, log_n, root, offset)
        assert O.from_np(ev.cpu().numpy().view("<u8")) == O.fast_coset_evaluate(rows[2], offset, root, n)
    else:
        full = eng.coset_div_apply(eng.coset_div_plan(divisor, log_n, root, offset), num, n)
        R = eng.coset_evaluate(divisor, log_n, root, offset)
        got = eng.pointwise_mul(eng.coset_evaluate(full, log_n, root, offset), R)
        assert bool((got == eng.coset_evaluate(num, log_n, root, offset)).all())


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--window", type=float, default=0.5, help="seconds per timed window")
    ap.add_argument("--logs", type=int, nargs="*", default=LOGS, help="log2 of the coset sizes")
    ap.add_argument("--batch", type=int, default=8, help="rows per batched call")
    args = ap.parse_args()

    eng = sa_engine.get_engine()
    lib, dev = eng.lib, eng.device
    st = torch.cuda.current_stream(dev)
    stream = ctypes.c_void_p(st.cuda_stream)
    field = sa_host.algebra.Field.main()
    FE = sa_host.algebra.FieldElement
    torch.manual_seed(0)
    for log_n in args.logs:
        n, qlen, ncoef_eval = 1 << log_n, (1 << log_n) // 2, (1 << log_n) // 4
        root = GENERATOR
        for _ in range(119 - log_n):
            root = root * root % P
        offset = GENERATOR
        root_l = sa_engine._limbs(root)
        divisor = rand_vec((qlen + 1,), dev)
        nums = [rand_vec((n,), dev) for _ in range(8)]
        polys = [rand_vec((ncoef_eval,), dev) for _ in range(8)]
        nbytes = lib.sa_coset_div_plan_bytes(log_n)
        plan = eng.coset_div_plan(divisor, log_n, root, offset)
        out = eng.empty(qlen)
        check(eng, log_n, root, offset, divisor, nums[0], polys[0])
        lhs_poly = sa_host.univariate.Polynomial(sa_devlist.from_device(nums[0], field))
        rhs_poly = sa_host.univariate.Polynomial(sa_devlist.from_device(divisor, field))
        eval_poly = sa_host.univariate.Polynomial(sa_devlist.from_device(polys[0], field))
        offset_fe, root_fe = FE(offset, field), FE(root, field)

        def oneshot(lhs=nums[0]):
            return eng.coset_div_apply(eng.coset_div_plan(divisor, log_n, root, offset), lhs, qlen)

        def build():
            assert lib.sa_coset_div_plan(plan.plan.data_ptr(), divisor.data_ptr(), qlen + 1, log_n, root_l,
                                         sa_engine._limbs(offset), stream) == 0

        def apply(lhs=nums[0]):
            assert lib.sa_coset_div_apply_batch(out.data_ptr(), plan.plan.data_ptr(), lhs.data_ptr(), n, qlen, log_n,
                                                root_l, 1, stream) == 0

        def evaluate(coeffs=polys[0]):
            return eng.coset_evaluate(coeffs, log_n, root, offset)

        def dropin_divide():
            return dropin.fast_coset_divide(lhs_poly, rhs_poly, offset_fe, root_fe, n)

        def dropin_evaluate():
            return dropin.fast_coset_evaluate(eval_poly, offset_fe, root_fe, n)

        apply()
        assert bool((out == oneshot()).all()), "apply differs from plan + apply at 2^%d" % log_n
        quotient = sa_devlist.to_device(dropin_divide().coefficients)
        assert bool((quotient == out).all()), "the drop-in's quotient differs at 2^%d" % log_n
        assert bool((sa_devlist.to_device(dropin_evaluate()) == evaluate()).all()), "the drop-in's codeword differs"
        row = {"log_n": log_n, "plan_bytes": nbytes,
               "oneshot_ms": timed_ms(oneshot, st, args.window),
               "plan_ms": timed_ms(build, st, args.window),
               "apply_ms": timed_ms(apply, st, args.window),
               "oneshot_x8_ms": timed_ms(lambda: [oneshot(v) for v in nums], st, args.window),
               "apply_x8_ms": timed_ms(lambda: [apply(v) for v in nums], st, args.window),
               "evaluate_x8_ms": timed_ms(lambda: [evaluate(c) for c in polys], st, args.window),
               "dropin_divide_ms": timed_ms(dropin_divide, st, args.window),
               "dropin_evaluate_ms": timed_ms(dropin_evaluate, st, args.window)}
        # after the single-row columns, which thus run on the memory and workspaces they had before the batch
        extra = args.batch - 8
        lbatch = torch.stack((nums + [rand_vec((n,), dev) for _ in range(extra)])[:args.batch])
        cbatch = torch.stack((polys + [rand_vec((ncoef_eval,), dev) for _ in range(extra)])[:args.batch])
        obatch = torch.empty((args.batch, qlen, 2), dtype=torch.int64, device=dev)
        ebatch = torch.empty((args.batch, n, 2), dtype=torch.int64, device=dev)

        def apply_batch():
            assert lib.sa_coset_div_apply_batch(obatch.data_ptr(), plan.plan.data_ptr(), lbatch.data_ptr(), n, qlen,
                                                log_n, root_l, args.batch, stream) == 0

        def evaluate_batch():
            assert lib.sa_coset_evaluate_batch(ebatch.data_ptr(), cbatch.data_ptr(), ncoef_eval, log_n, root_l,
                                               sa_engine._limbs(offset), args.batch, stream) == 0

        apply_batch()
        evaluate_batch()
        for b in (0, args.batch - 1):
            assert bool((obatch[b] == oneshot(lbatch[b])).all()), "batch row %d differs at 2^%d" % (b, log_n)
            assert bool((ebatch[b] == evaluate(cbatch[b])).all()), "evaluation row %d differs at 2^%d" % (b, log_n)
        row["apply_batch%d_ms" % args.batch] = timed_ms(apply_batch, st, args.window)
        row["evaluate_batch%d_ms" % args.batch] = timed_ms(evaluate_batch, st, args.window)
        print(json.dumps({key: (round(v, 4) if isinstance(v, float) else v) for key, v in row.items()}), flush=True)
        del plan, divisor, nums, polys, out, lbatch, cbatch, obatch, ebatch, lhs_poly, rhs_poly, eval_poly, quotient
        torch.cuda.synchronize(dev)
        torch.cuda.empty_cache()
        assert lib.sa_release_workspaces() == 0
    print(json.dumps({"device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index),
                      "window_s": args.window}), flush=True)


if __name__ == "__main__":
    main()
