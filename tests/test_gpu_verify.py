"""Batched verification on the device: the fixture cases' proofs and every tamper kind get the verdicts and printed
messages recorded from the unmodified reference (tests/golden/verify.json); synthetic batches at 2^12 x 16, 2^16 x 4
and 2^20 x 2 are accepted as the test-side verifier accepts them; the tamper matrix at 2^16 equals the Python
restatement of the device checks; 64 seeded FastRPSSS and RPSSS signatures verify in one call; and per kernel: a grid
past its wrap, a batch across chunks, a fixed launch count per chunk, errors before any launch, graph replay and no
spills."""
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import stark_cases as C
import stark_plain_cases as S
import stark_rescue_cases as SR
import stark_verify as SV
import verify_cases as V
from test_gpu_air import release

import sa_engine  # noqa: E402
import sa_stark  # noqa: E402

pytestmark = pytest.mark.gpu
G = C.golden()
GP = S.golden()
PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "stark-anatomy_b200")


@pytest.fixture(scope="module")
def eng():
    sa_engine.set_engine(None)
    e = sa_engine.get_engine()
    assert e.name == "cuda"
    return e


@pytest.fixture(autouse=True)
def _cuda_engine(eng):
    sa_engine.set_engine(eng)
    yield
    release(eng)


def with_double(fn):
    prev = sa_engine._ENGINE
    sa_engine.set_engine(V.VerifyEngine())
    try:
        return fn()
    finally:
        sa_engine.set_engine(prev)


@pytest.mark.parametrize("name", V.FAST)
def test_fast_verdicts_recorded_from_the_reference(name):
    assert V.check_recorded(name, True) == 1 + len(V.kinds(True))


@pytest.mark.parametrize("name", V.PLAIN)
def test_plain_verdicts_recorded_from_the_reference(name):
    assert V.check_recorded(name, False) == 1 + len(V.kinds(False))


def synthetic_batch(log_fri, count):
    """count seeded proofs of one synthetic AIR's statement from one prove_batch call (each proof its own
    randomizers): ([(stark, constraints, boundary, proof)], the zerofier root)"""
    stark, cons, trace, boundary = C.synthetic(0, log_fri)
    zpoly, zvals = C.zerofier(stark)
    plan = sa_stark.StarkPlan(stark, cons, zpoly)
    proofs = plan.prove_batch([trace] * count, [boundary] * count, C.zerofier_codeword(zvals, True),
                              seeds=[bytes([log_fri, b]) * 16 for b in range(count)])
    root = V.O.merkle_tree_np(V.O.to_np(zvals))[1].tobytes()
    return [(stark, cons, boundary, p) for p in proofs], root


@pytest.mark.parametrize("log_fri,count", [(12, 16), (16, 4), (20, 2)])
def test_synthetic_batches_accepted(log_fri, count):
    batch, root = synthetic_batch(log_fri, count)
    stark, cons, boundary = batch[0][:3]
    assert len({p for *_, p in batch}) == count
    plan = sa_stark.VerifierPlan(stark, cons, root)
    got = plan.verify_batch([p for *_, p in batch], [boundary] * count, reasons=True)
    assert got == [(True, None)] * count
    for b in (0, count - 1):
        assert SV.verify(stark, batch[b][3], cons, boundary, root) is True


def test_tamper_matrix_at_2_16():
    batch, root = synthetic_batch(16, 1)
    stark, cons, boundary, proof = batch[0]
    k, rounds = stark.fri.num_colinearity_tests, stark.fri.num_rounds()
    proofs = [proof] + [V.tamper(proof, stark.num_registers, rounds, k, t) for t in V.kinds(True)]
    got = sa_stark.VerifierPlan(stark, cons, root).verify_batch(proofs, [boundary] * len(proofs), reasons=True)
    want = with_double(lambda: sa_stark.VerifierPlan(stark, cons, root).verify_batch(
        proofs, [boundary] * len(proofs), reasons=True))
    assert got == want
    assert got[0] == (True, None) and all(v is False for v, _ in got[1:])


def test_batch_across_chunks_and_launches_per_chunk(eng, monkeypatch):
    stark, cons, boundary, root, proof = V.case("three_register", True)
    plan = sa_stark.VerifierPlan(stark, cons, root)
    k, rounds = stark.fri.num_colinearity_tests, stark.fri.num_rounds()
    proofs = [proof, V.tamper(proof, stark.num_registers, rounds, k, "boundary_leaf"), proof,
              V.tamper(proof, stark.num_registers, rounds, k, "last_codeword")]
    whole = plan.verify_batch(proofs, [boundary] * 4, reasons=True)
    before = eng.launch_count()
    plan.verify_batch(proofs[:1], [boundary], reasons=True)
    one = eng.launch_count() - before
    monkeypatch.setattr(sa_stark, "CHUNK_BYTES", plan._bytes(plan._parse(proof, boundary, None)) + 1)
    before = eng.launch_count()
    assert plan.verify_batch(proofs, [boundary] * 4, reasons=True) == whole
    assert eng.launch_count() - before == 4 * one  # one chunk per proof, each chunk the same launches


@pytest.mark.parametrize("fast", [True, False], ids=["fastrpsss", "rpsss"])
def test_64_seeded_signatures_in_one_call(eng, fast):
    g = G if fast else GP
    first = g["rpsss"]
    signer = SR.Signer(first, fast)
    if fast:
        signer.transition_zerofier_root = bytes.fromhex(first["zerofier_root"])
    plan = sa_stark.SignerPlan(signer)
    plan.stream = V.SignatureProofStream
    sks = [C.T.fe(7 + 3 * d) for d in range(64)]
    docs = [b"document %d" % d for d in range(64)]
    sigs = plan.sign(sks, docs, [bytes([d]) * 32 for d in range(64)])
    pks = [signer.rp.hash(sk) for sk in sks]
    assert plan.verify(pks, docs, sigs) == [True] * 64  # the first call builds the verifier plan
    counts = []
    for p, d in ((pks, docs), (pks, docs[1:] + docs[:1]), (pks[1:] + pks[:1], docs)):
        before = eng.launch_count()
        assert plan.verify(p, d, sigs) == [d is docs and p is pks] * 64
        counts.append(eng.launch_count() - before)
    assert len(set(counts)) == 1  # a fixed launch count per chunk, whatever the verdicts


# ---- per kernel ----
def colinear_items(eng, count, seed):
    """count FRI items of round seed % 3 on a 2^12 domain, every third not colinear: device buffers and the flags
    the Lagrange test in ints gives"""
    rng = np.random.default_rng(seed)
    P = C.P
    offset, n = C.T.field.generator().value, 1 << 12
    omega = C.T.field.primitive_nth_root(n).value
    r = seed % 3
    a = [int(v) for v in rng.integers(0, n >> (r + 1), count)]
    s, t = 3, 5
    ax = [pow(offset, 1 << r, P) * pow(omega, (1 << r) * x, P) % P for x in a]
    alpha = [(x * 7 + seed) % P for x in range(count)]
    ay = [(s * x + t) % P for x in ax]
    by = [(s * (P - x) + t) % P for x in ax]
    cy = [(s * al + t + (j % 3 == 2)) % P for j, al in enumerate(alpha)]
    want = [int(not V.colinear(x, y0, P - x, y1, al, y2)) for x, y0, y1, al, y2 in zip(ax, ay, by, alpha, cy)]
    up = lambda v: eng.upload(bytearray(b"".join((int(x) % P).to_bytes(16, "little") for x in v)))  # noqa: E731
    import torch
    dev = dict(ay=up(ay), by=up(by), cy=up(cy), alpha=up(alpha),
               a=torch.tensor(a, dtype=torch.int64, device=eng.device),
               r=torch.full((count,), r, dtype=torch.int32, device=eng.device))
    return dev, want, offset, omega


def launch_colinear(eng, flags, dev, offset, omega, count):
    return eng.lib.sa_fri_colinear_batch(flags.data_ptr(), dev["ay"].data_ptr(), dev["by"].data_ptr(),
                                         dev["cy"].data_ptr(), dev["a"].data_ptr(), dev["alpha"].data_ptr(),
                                         dev["r"].data_ptr(), sa_engine._limbs(offset), sa_engine._limbs(omega),
                                         count, eng._stream())


def test_colinear_grid_past_its_wrap(eng):
    import torch
    count = 16 * 132 * 128 + 4097  # past grid_for's cap of 16 blocks of 128 per SM
    dev, want, offset, omega = colinear_items(eng, count, 1)
    flags = torch.full((count,), 7, dtype=torch.int32, device=eng.device)
    assert launch_colinear(eng, flags, dev, offset, omega, count) == 0
    assert flags.cpu().tolist() == want


def test_merkle_grid_past_its_wrap(eng):
    import hashlib
    import torch
    count = 16 * 132 * 128 + 999
    P = C.P
    values = [(7919 * j) % P for j in range(count)]
    sib = bytes(range(64))
    roots = b"".join(hashlib.blake2b((sib + hashlib.blake2b(str(v).encode()).digest()) if j & 1 else
                                     (hashlib.blake2b(str(v).encode()).digest() + sib)).digest()
                     if j % 5 else bytes(64) for j, v in enumerate(values))
    idx = torch.tensor([j & 1 for j in range(count)], dtype=torch.int64, device=eng.device)
    depth = torch.ones(count, dtype=torch.int32, device=eng.device)
    poff = torch.zeros(count, dtype=torch.int64, device=eng.device)
    r = eng.upload_bytes(roots)
    leaves = eng.upload(bytearray(b"".join(v.to_bytes(16, "little") for v in values)))
    paths = eng.upload_bytes(sib)
    flags = torch.full((count,), 7, dtype=torch.int32, device=eng.device)
    assert eng.lib.sa_merkle_verify_batch(flags.data_ptr(), r.data_ptr(), leaves.data_ptr(), idx.data_ptr(),
                                          depth.data_ptr(), paths.data_ptr(), poff.data_ptr(), count,
                                          eng._stream()) == 0
    assert flags.cpu().tolist() == [int(j % 5 == 0) for j in range(count)]


def test_errors_before_any_launch(eng):
    import torch
    lib = eng.lib
    before = eng.launch_count()
    x = torch.zeros(64, dtype=torch.int64, device=eng.device).data_ptr()
    lim = 1 << 59
    z = sa_engine._limbs(0)
    st = eng._stream()
    assert lib.sa_merkle_verify_batch(x, x, x, x, x, x, x, lim, st) == -6
    assert lib.sa_merkle_verify_batch(x, None, x, x, x, x, x, 1, st) == -6
    assert lib.sa_fri_colinear_batch(x, x, x, x, x, x, x, z, z, lim, st) == -6
    assert lib.sa_fri_colinear_batch(x, x, None, x, x, x, x, z, z, 1, st) == -6
    for k, nb, ncons, nregs, blen, log_n, ef in [(1, 1, 1, 0, 1, 4, 1), (1, 1, 1, 17, 1, 4, 1),
                                                 (1, 1, 0, 1, 1, 4, 1), (1, 1, 1, 1, 0, 4, 1),
                                                 (1, 1, 1, 1, 1, 31, 1), (1, 1, 1, 1, 1, 4, 16),
                                                 (lim, 1, 1, 1, 1, 4, 1)]:
        assert lib.sa_verify_combination(x, x, x, k, nb, x, ncons, nregs, blen, None, 0, z, z, log_n, ef, st) == -6
    assert lib.sa_verify_combination(x, x, x, 1, 1, x, 1, 1, 1, x, 0, z, z, 4, 1, st) == -6  # zcoef of length 0
    assert lib.sa_poly_degree_batch(x, x, 3, 1, st) == -6
    assert lib.sa_poly_degree_batch(x, x, 0, 1, st) == -6
    assert lib.sa_poly_degree_batch(x, x, 1 << 20, lim >> 10, st) == -6
    for fn in (lib.sa_merkle_verify_batch, lib.sa_fri_colinear_batch):
        args = [x] * (9 if fn is lib.sa_merkle_verify_batch else 7)
        args = args[:7] + ([0, st] if fn is lib.sa_merkle_verify_batch else [z, z, 0, st])
        assert fn(*args) == 0  # an empty batch: no launch
    assert eng.launch_count() == before


def test_graph_replay(eng):
    import torch
    count = 5000
    dev, want, offset, omega = colinear_items(eng, count, 2)
    flags = torch.zeros(count, dtype=torch.int32, device=eng.device)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        assert launch_colinear(eng, flags, dev, offset, omega, count) == 0
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        launch_colinear(eng, flags, dev, offset, omega, count)
    for seed in (5, 8):  # seed % 3 == 2: the captured round
        fresh, want, _, _ = colinear_items(eng, count, seed)
        for key in dev:
            dev[key].copy_(fresh[key])
        flags.fill_(9)
        g.replay()
        torch.cuda.synchronize()
        assert flags.cpu().tolist() == want


def test_kernels_have_no_spills():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-diag-suppress",
                              "550", "-c", "-Xptxas", "-v", "-o", os.path.join(tmp, "verify.o"),
                              os.path.join(PKG, "csrc", "verify.cu")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    lines = res.stderr.splitlines()
    for kernel in ("k_merkle_verify", "k_fri_colinear", "k_verify_combination", "k_poly_degree"):
        at = [i for i, line in enumerate(lines) if "Compiling entry function" in line and kernel in line]
        assert len(at) == 1, kernel
        report = " ".join(lines[at[0]:at[0] + 4])
        spills = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", report)
        assert spills and spills.groups() == ("0", "0"), report


def test_degrees_of_many_rows(eng):
    import torch
    rows, n = 5, 1 << 10
    vals = torch.zeros((rows * n, 2), dtype=torch.int64, device=eng.device)
    want = [-1, 0, n - 1, 17, 513]
    for b, d in enumerate(want):
        if d >= 0:
            vals[b * n + d, 0] = 3
            vals[b * n + d // 2, 1] = 1
    out = torch.empty(rows, dtype=torch.int64, device=eng.device)
    assert eng.lib.sa_poly_degree_batch(out.data_ptr(), vals.data_ptr(), n, rows, eng._stream()) == 0
    assert out.cpu().tolist() == want
