"""sa_engine -- ctypes binding of the C ABI (include/sa_b200.h) plus device memory.

This is the "reference-side binding a maintainer would add" (INTEGRATION.md):
plain pointers and sizes go to ``libsa_b200.so``; PyTorch is used only for
device memory (``torch.empty(..., device="cuda")``), host<->device copies and the
current CUDA stream.  There is no CPU fallback: creating the engine without a
CUDA device or without the built library raises.

Vectors are ``torch.int64`` tensors of shape [n, 2] on the GPU holding the
(lo, hi) limbs of canonical residues mod p = 1 + 407*2^119 (16 bytes/element).
"""
import ctypes
import os

P = 1 + 407 * (1 << 119)
_HERE = os.path.dirname(os.path.abspath(__file__))
# SA_B200_LIB: another build of the same C ABI (kernel experiments); default = the in-tree library
LIB_PATH = os.environ.get("SA_B200_LIB") or os.path.join(_HERE, "libsa_b200.so")

# include/sa_b200.h error codes -> the reference's assertion messages
SA_ERRORS = {
    -1: "cannot compute ntt of non-power-of-two sequence",                                   # ntt.py:4
    -2: "primitive root must be nth root of unity, where n is len(values)",                  # ntt.py:10
    -3: "primitive root is not primitive nth root of unity, where n is len(values)",         # ntt.py:11
    -4: "divide by zero",                                                                    # algebra.py:92
    -5: "cannot open invalid index",                                                         # merkle.py:18
    -6: "unsupported size",
}
FRI_CHALLENGE_FN = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                    ctypes.POINTER(ctypes.c_uint64), ctypes.c_int)

# every symbol include/sa_b200.h declares: (name, restype, argtypes)
_vp, _sz, _ci, _u64p = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.POINTER(ctypes.c_uint64)
SYMBOLS = [
    ("sa_version", ctypes.c_char_p, []),
    ("sa_last_error", ctypes.c_char_p, []),
    ("sa_launch_count", ctypes.c_uint64, []),
    ("sa_ntt", _ci, [_vp, _vp, _ci, _u64p, _ci, _sz, _vp]),
    ("sa_ntt_multi", _ci, [ctypes.POINTER(ctypes.c_void_p), _ci, _sz, _vp, _ci, _u64p, _ci, _sz, _vp]),
    ("sa_ntt_mcast", _ci, [_vp, _vp, _sz, _vp, _ci, _u64p, _ci, _sz, _vp]),
    ("sa_push_mcast", _ci, [_vp, _vp, _sz, _vp]),
    ("sa_enable_peer_access", _ci, [_ci]),
    ("sa_peer_alloc", _ci, [ctypes.POINTER(ctypes.c_void_p), _sz, ctypes.c_char_p]),
    ("sa_peer_open", _ci, [ctypes.POINTER(ctypes.c_void_p), ctypes.c_char_p]),
    ("sa_peer_close", _ci, [_vp]),
    ("sa_peer_free", _ci, [_vp]),
    ("sa_copy_async", _ci, [_vp, _vp, _sz, _vp]),
    ("sa_push", _ci, [ctypes.POINTER(ctypes.c_void_p), _ci, _vp, _sz, _vp]),
    ("sa_ntt_host", _ci, [_vp, _vp, _ci, _u64p, _ci, _sz, _vp]),
    ("sa_host_alloc", _vp, [_sz]),
    ("sa_host_free", _ci, [_vp]),
    ("sa_pointwise_mul", _ci, [_vp, _vp, _vp, _sz, _vp]),
    ("sa_poly_eval", _ci, [_vp, _vp, _sz, _vp, _sz, _vp]),
    ("sa_poly_eval_mode", _ci, [_vp, _vp, _sz, _vp, _sz, _ci, _vp]),
    ("sa_zerofier", _ci, [_vp, _vp, _sz, _vp]),
    ("sa_interpolate", _ci, [_vp, _vp, _vp, _sz, _vp]),
    ("sa_interp_plan_bytes", _sz, [_sz]),
    ("sa_interp_plan", _ci, [_vp, _vp, _sz, _vp]),
    ("sa_interp_apply", _ci, [_vp, _vp, _vp, _sz, _vp]),
    ("sa_interp_apply_batch", _ci, [_vp, _vp, _vp, _sz, _sz, _vp]),
    ("sa_interp_batch_max", _sz, [_sz]),
    ("sa_geo_plan_bytes", _sz, [_sz]),
    ("sa_geo_plan", _ci, [_vp, _u64p, _sz, _vp]),
    ("sa_geo_interp_batch", _ci, [_vp, _vp, _vp, _sz, _sz, _vp]),
    ("sa_geo_batch_max", _sz, [_sz]),
    ("sa_geo_zerofier", _ci, [_vp, _u64p, _sz, _vp]),
    ("sa_coset_div_plan_bytes", _sz, [_ci]),
    ("sa_coset_div_plan", _ci, [_vp, _vp, _sz, _ci, _u64p, _u64p, _vp]),
    ("sa_coset_div_apply_batch", _ci, [_vp, _vp, _vp, _sz, _sz, _ci, _u64p, _sz, _vp]),
    ("sa_coset_evaluate_batch", _ci, [_vp, _vp, _sz, _ci, _u64p, _u64p, _sz, _vp]),
    ("sa_coset_batch_max", _sz, [_ci]),
    ("sa_coset_combine_evaluate", _ci, [_vp, _ci, _u64p, _u64p, ctypes.POINTER(ctypes.c_void_p),
                                        ctypes.POINTER(_sz), ctypes.POINTER(_sz), _u64p, _sz, _vp]),
    ("sa_coset_combine_evaluate_batch", _ci, [_vp, _sz, _ci, _u64p, _u64p, ctypes.POINTER(ctypes.c_void_p),
                                              ctypes.POINTER(_sz), ctypes.POINTER(_sz), ctypes.POINTER(_sz), _u64p,
                                              _sz, _vp]),
    ("sa_air_plan_bytes", _sz, [_ci, _sz, _sz, _sz]),
    ("sa_air_plan", _ci, [_vp, _u64p, ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(_sz), _sz, _sz, _sz, _vp, _sz,
                          _ci, _u64p, _u64p, _u64p, _vp]),
    ("sa_air_quotients", _ci, [_vp, _vp, _vp, _sz, _sz, _sz, _sz, _ci, _u64p, _vp]),
    ("sa_air_quotients_exact", _ci, [_vp, ctypes.POINTER(ctypes.c_uint32), _vp, _vp, _sz, _sz, _sz, _sz, _sz, _ci,
                                     _u64p, _vp]),
    ("sa_air_quotients_batch", _ci, [_vp, _vp, _vp, _sz, _sz, _sz, _sz, _sz, _ci, _u64p, _vp]),
    ("sa_air_quotients_exact_batch", _ci, [_vp, ctypes.POINTER(ctypes.c_uint32), _vp, _vp, _sz, _sz, _sz, _sz, _sz,
                                           _sz, _ci, _u64p, _vp]),
    ("sa_air_batch_max", _sz, [_sz, _sz, _ci]),
    ("sa_boundary_plan_bytes", _sz, [_ci, _sz]),
    ("sa_boundary_plan", _ci, [_vp, ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(_sz),
                               ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(_sz), _sz, _ci, _u64p, _u64p, _vp]),
    ("sa_boundary_quotients", _ci, [_vp, _vp, ctypes.POINTER(ctypes.c_uint32), _vp, _vp, _sz, _sz, _ci, _u64p, _vp]),
    ("sa_merkle_tree", _ci, [_vp, _vp, _sz, _vp]),
    ("sa_merkle_open", _ci, [_vp, _vp, _sz, _u64p, _sz, _vp]),
    ("sa_gather", _ci, [_vp, _vp, _sz, _u64p, _sz, _vp]),
    ("sa_merkle_tree_batch", _ci, [_vp, _vp, _sz, _sz, _vp]),
    ("sa_merkle_open_batch", _ci, [_vp, _vp, _sz, _sz, _u64p, _sz, _vp]),
    ("sa_gather_batch", _ci, [_vp, _vp, _sz, _sz, _u64p, _sz, _vp]),
    ("sa_merkle_open_batch_sets", _ci, [_vp, _vp, _sz, _sz, _sz, _u64p, _sz, _vp]),
    ("sa_gather_batch_sets", _ci, [_vp, _vp, _sz, _sz, _sz, _u64p, _sz, _vp]),
    ("sa_sample_seeded", _ci, [_vp, _vp, _sz, _sz, ctypes.c_uint64, _sz, _sz, _sz, _vp]),
    ("sa_rescue", _ci, [_vp, _vp, _vp, _sz, _vp, _sz, _u64p, _u64p, _sz, _sz, _vp]),
    ("sa_merkle_verify_batch", _ci, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    ("sa_fri_colinear_batch", _ci, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _u64p, _u64p, _sz, _vp]),
    ("sa_verify_combination", _ci, [_vp, _vp, _vp, _sz, _sz, _vp, _sz, _sz, _sz, _vp, _sz, _u64p, _u64p, _ci, _sz,
                                    _vp]),
    ("sa_poly_degree_batch", _ci, [_vp, _vp, _sz, _sz, _vp]),
    ("sa_air_program_bytes", _sz, [_sz, _sz]),
    ("sa_transcript_bytes", _sz, [_u64p]),
    ("sa_transcript_sections", _ci, [_vp, _u64p, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp, _sz, _u64p, _vp]),
    ("sa_air_program", _ci, [_vp, _u64p, ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(_sz), _sz, _sz, _vp]),
    ("sa_fri_fold", _ci, [_vp, _vp, _sz, _u64p, _u64p, _u64p, _vp]),
    ("sa_fri_round", _ci, [_vp, _vp, _vp, _sz, _u64p, _u64p, _u64p, _vp]),
    ("sa_fri_commit", _ci, [_vp, _vp, _vp, _sz, _ci, _u64p, _u64p, _vp, _vp, _vp]),
    ("sa_fri_commit_batch", _ci, [_vp, _vp, _vp, _sz, _sz, _ci, _u64p, _u64p, _vp, _vp, _vp]),
    ("sa_cache_limit", _sz, [_sz]),
    ("sa_cache_bytes", _sz, []),
    ("sa_release_workspaces", _ci, []),
    ("sa_selftest_field", ctypes.c_longlong, [_sz, ctypes.c_uint64]),
    ("sa_selftest_tile", ctypes.c_longlong, [_sz, ctypes.c_uint64, _u64p, _sz]),
    ("sa_microbench", ctypes.c_double, [_ci, _ci, _ci, _ci, _ci]),
]


def load_library(path=LIB_PATH):
    """dlopen the C-ABI library and type every entry point (works without a GPU)."""
    if not os.path.exists(path):
        raise RuntimeError(
            "stark-anatomy_b200: %s is missing -- build it with `python -c 'import __graft_entry__ as g; "
            "g.build()'` (nvcc, sm_90a). There is no CPU fallback." % path)
    lib = ctypes.CDLL(path)
    for name, restype, argtypes in SYMBOLS:
        fn = getattr(lib, name)
        fn.restype = restype
        fn.argtypes = argtypes
    return lib


def _limbs(x):
    x = int(x)
    return (ctypes.c_uint64 * 2)(x & 0xFFFFFFFFFFFFFFFF, x >> 64)


class SaError(AssertionError):
    """Raised with the reference's assertion message for SA_E* codes."""


class InterpPlan:
    """An interpolation plan (CudaEngine.interp_plan): the device buffer sa_interp_plan filled (torch.uint8) for a
    domain of k points."""
    __slots__ = ("plan", "k")

    def __init__(self, plan, k):
        self.plan = plan
        self.k = k


class GeoInterpPlan:
    """A geometric interpolation plan (CudaEngine.geo_interp_plan): the device buffer sa_geo_plan filled (torch.uint8)
    for the domain step^0 .. step^(k-1)."""
    __slots__ = ("plan", "step", "k")

    def __init__(self, plan, step, k):
        self.plan = plan
        self.step = step
        self.k = k


class CosetDivPlan:
    """A coset division plan (CudaEngine.coset_div_plan): the device buffer sa_coset_div_plan filled (torch.uint8)
    for one divisor on the coset offset * <root> of order 2^log_n, with the scalars every apply passes again"""
    __slots__ = ("plan", "log_n", "root", "offset")

    def __init__(self, plan, log_n, root, offset):
        self.plan = plan
        self.log_n = log_n
        self.root = root
        self.offset = offset


class AirPlan:
    """A transition quotient plan (CudaEngine.air_plan): the device buffer sa_air_plan filled (torch.uint8) for one
    AIR and zerofier on the coset offset * <root> of order 2^log_n, with the values every apply passes again and the
    zerofier's degree (its length - 1; None where unknown), which the exact apply's tail needs"""
    __slots__ = ("plan", "log_n", "root", "offset", "nregs", "ncons", "max_ncoef", "zdeg")

    def __init__(self, plan, log_n, root, offset, nregs, ncons, max_ncoef, zdeg=None):
        self.plan = plan
        self.log_n = log_n
        self.root = root
        self.offset = offset
        self.nregs = nregs
        self.ncons = ncons
        self.max_ncoef = max_ncoef
        self.zdeg = zdeg


class BoundaryPlan:
    """A boundary quotient plan (CudaEngine.boundary_plan): the device buffer sa_boundary_plan filled (torch.uint8)
    for one boundary on the coset offset * <root> of order 2^log_n, with the values every apply passes again and the
    degree of each register's boundary zerofier (its number of boundary points)"""
    __slots__ = ("plan", "log_n", "root", "offset", "nregs", "degrees")

    def __init__(self, plan, log_n, root, offset, nregs, degrees):
        self.plan = plan
        self.log_n = log_n
        self.root = root
        self.offset = offset
        self.nregs = nregs
        self.degrees = degrees

    def degree_bounds(self, trace_length):
        """FastStark.boundary_quotient_degree_bounds for trace polynomials of trace_length coefficients"""
        return [trace_length - 1 - d for d in self.degrees]


REMAINDER = "cannot perform polynomial division because remainder is not zero"  # univariate.py:52


def _air_arrays(constraints, nregs):
    """the C ABI's coefficient limbs, exponents and term_start of constraints given as objects with a `.dictionary`
    (MPolynomial) or as {exponent tuple: value} dicts, values ints or anything with `.value`; tuples shorter than
    1 + 2 nregs are zero-padded (as MPolynomial.__add__ pads) and terms that meet there are added"""
    nvars = 1 + 2 * nregs
    coeffs, exps, starts = [], [], [0]
    for a in constraints:
        terms = {}
        for k, v in getattr(a, "dictionary", a).items():
            k = tuple(int(e) for e in k)
            if len(k) > nvars or any(not 0 <= e < 1 << 32 for e in k):
                raise SaError(SA_ERRORS[-6])
            k += (0,) * (nvars - len(k))
            terms[k] = (terms.get(k, 0) + int(getattr(v, "value", v))) % P
        for k, v in terms.items():
            coeffs += [v & 0xFFFFFFFFFFFFFFFF, v >> 64]
            exps += k
        starts.append(len(exps) // nvars)
    return coeffs, exps, starts


class CudaEngine:
    """Device-resident operations; one instance per process (one process per GPU)."""

    name = "cuda"

    def __init__(self, device=None):
        import torch
        if not torch.cuda.is_available():
            raise RuntimeError("stark-anatomy_b200: no CUDA device visible; the engine has no CPU fallback")
        self.torch = torch
        self.lib = load_library()
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        # host<->device traffic this engine object has caused (calls and bytes); tools/config5.py and the
        # tests use it to show which boundary crossings are left (SURVEY 8 f3)
        self.stats = {"h2d_calls": 0, "h2d_bytes": 0, "d2h_calls": 0, "d2h_bytes": 0}

    def _count(self, kind, nbytes):
        self.stats[kind + "_calls"] += 1
        self.stats[kind + "_bytes"] += int(nbytes)

    # ------------------------------------------------------------ plumbing
    def _stream(self):
        # the C library works on the CURRENT device; make sure that is this engine's (a peer tensor rebuilt from
        # an IPC handle, or user code, may have left another device current)
        cuda = self.torch.cuda
        if cuda.current_device() != self.device.index:
            cuda.set_device(self.device)
        return ctypes.c_void_p(cuda.current_stream(self.device).cuda_stream)

    def _check(self, rc):
        if rc == 0:
            return
        if rc in SA_ERRORS:
            raise SaError(SA_ERRORS[rc])
        if rc == -7:
            raise RuntimeError("sa_b200: the challenge callback failed")
        raise RuntimeError("sa_b200: CUDA error: %s" % self.lib.sa_last_error().decode())

    def empty(self, n):
        return self.torch.empty((n, 2), dtype=self.torch.int64, device=self.device)

    def zeros(self, n):
        return self.torch.zeros((n, 2), dtype=self.torch.int64, device=self.device)

    def length(self, vec):
        return vec.shape[0]

    def upload(self, buf):
        """packed 16-byte elements (bytearray / numpy / pinned tensor) -> device vector"""
        torch = self.torch
        if isinstance(buf, torch.Tensor):
            if not buf.is_cuda:
                self._count("h2d", buf.numel() * buf.element_size())
            return buf.reshape(-1, 2).to(self.device, non_blocking=True)
        if len(buf) == 0:
            return self.empty(0)
        host = torch.frombuffer(buf, dtype=torch.int64).reshape(-1, 2)
        self._count("h2d", host.numel() * 8)
        return host.to(self.device)

    def download(self, vec):
        """device vector -> numpy uint64[n, 2] (buffer protocol, 16 bytes/element)"""
        self._count("d2h", vec.numel() * 8)
        return vec.contiguous().cpu().numpy()

    def pad(self, vec, n):
        """zero-extend to n elements"""
        if vec.shape[0] == n:
            return vec
        out = self.zeros(n)
        out[:vec.shape[0]] = vec
        return out

    def slice(self, vec, lo, hi):
        return vec[lo:hi]

    def concat(self, vecs):
        return self.torch.cat(vecs, dim=0)

    # ------------------------------------------------------------------ ntt
    @staticmethod
    def _check_ntt_length(vec, log_n, batch):
        """the library reads batch << log_n elements of the input: a shorter vector is refused here, before any
        device work (the library cannot see a buffer's length)"""
        if log_n >= 0 and vec.shape[0] < batch << log_n:
            raise SaError(SA_ERRORS[-6])

    def ntt(self, vec, log_n, root, inverse=False, batch=1):
        self._check_ntt_length(vec, log_n, batch)
        vec = vec.contiguous()
        out = self.empty(vec.shape[0])
        self._check(self.lib.sa_ntt(out.data_ptr(), vec.data_ptr(), log_n, _limbs(root), int(bool(inverse)),
                                    batch, self._stream()))
        return out

    def ntt_into(self, out, vec, log_n, root, inverse=False, batch=1):
        """sa_ntt into a caller-provided device vector (a slice of a larger buffer); out may alias vec"""
        assert out.is_contiguous() and vec.is_contiguous() and out.shape[0] == vec.shape[0]
        self._check_ntt_length(vec, log_n, batch)
        self._check(self.lib.sa_ntt(out.data_ptr(), vec.data_ptr(), log_n, _limbs(root), int(bool(inverse)), batch,
                                    self._stream()))
        return out

    def ntt_multi(self, outs, out_offset, vec, log_n, root, inverse=False, batch=1):
        """sa_ntt_multi: transform `vec` and store the result at element offset `out_offset` of every buffer in
        `outs` (outs[0] on this device, the others peer-mapped buffers of other GPUs; tensors or raw pointers)"""
        self._check_ntt_length(vec, log_n, batch)
        vec = vec.contiguous()
        ptrs = (ctypes.c_void_p * len(outs))(*[int(t) if isinstance(t, int) else int(t.data_ptr()) for t in outs])
        self._check(self.lib.sa_ntt_multi(ptrs, len(outs), out_offset, vec.data_ptr(), log_n, _limbs(root),
                                          int(bool(inverse)), batch, self._stream()))

    def ntt_mcast(self, mc_ptr, local, out_offset, vec, log_n, root, inverse=False, batch=1):
        """sa_ntt_mcast: transform `vec`, store the result through the multicast address `mc_ptr` (every rank's
        buffer receives it, this rank's `local` included) at element offset `out_offset`"""
        self._check_ntt_length(vec, log_n, batch)
        vec = vec.contiguous()
        self._check(self.lib.sa_ntt_mcast(ctypes.c_void_p(int(mc_ptr)), local.data_ptr(), out_offset, vec.data_ptr(),
                                          log_n, _limbs(root), int(bool(inverse)), batch, self._stream()))

    def wrap_pointer(self, ptr, nelems):
        """a device vector (torch.int64[n, 2]) over memory this process got from the C library"""
        class _Raw:
            __cuda_array_interface__ = {"shape": (nelems, 2), "typestr": "<i8", "data": (int(ptr), False), "version": 2}
        return self.torch.as_tensor(_Raw(), device=self.device)

    def pointwise_mul(self, a, b):
        out = self.empty(a.shape[0])
        self._check(self.lib.sa_pointwise_mul(out.data_ptr(), a.contiguous().data_ptr(),
                                              b.contiguous().data_ptr(), a.shape[0], self._stream()))
        return out

    def poly_eval(self, coeffs, points, mode=0):
        """values of the polynomial at the points; mode 0 = the library chooses, 1 = Horner kernel, 2 = walk down
        the subproduct tree of the points (sa_poly_eval_mode)"""
        coeffs, points = coeffs.contiguous(), points.contiguous()
        out = self.empty(points.shape[0])
        self._check(self.lib.sa_poly_eval_mode(out.data_ptr(), coeffs.data_ptr(), coeffs.shape[0], points.data_ptr(),
                                               points.shape[0], int(mode), self._stream()))
        return out

    MAX_DIRECT_POINTS = 1 << 20  # sa_zerofier / sa_interpolate handle this many points per call

    def zerofier(self, domain):
        domain = domain.contiguous()
        out = self.empty(domain.shape[0] + 1)
        self._check(self.lib.sa_zerofier(out.data_ptr(), domain.data_ptr(), domain.shape[0], self._stream()))
        return out

    def interpolate(self, domain, values):
        domain, values = domain.contiguous(), values.contiguous()
        out = self.empty(domain.shape[0])
        self._check(self.lib.sa_interpolate(out.data_ptr(), domain.data_ptr(), values.data_ptr(), domain.shape[0],
                                            self._stream()))
        return out

    def interp_plan(self, domain):
        """sa_interp_plan: what interpolation over `domain` needs of the domain alone, kept on the device for
        interp_apply (synchronises; "divide by zero" when two points coincide)"""
        domain = domain.contiguous()
        k = domain.shape[0]
        plan = self.torch.empty(self.lib.sa_interp_plan_bytes(k), dtype=self.torch.uint8, device=self.device)
        self._check(self.lib.sa_interp_plan(plan.data_ptr(), domain.data_ptr(), k, self._stream()))
        return InterpPlan(plan, k)

    def interp_apply(self, plan, values):
        """sa_interp_apply_batch: the coefficients `interpolate` gives for `values` over the plan's domain, for one
        vector (k, 2) or a batch of them (B, k, 2) in one call; asynchronous, the plan is only read"""
        # the library cannot see the vectors' shape
        if values.dim() not in (2, 3) or tuple(values.shape[-2:]) != (plan.k, 2):
            raise SaError(SA_ERRORS[-6])
        values = values.contiguous()
        out = self.torch.empty(values.shape, dtype=self.torch.int64, device=self.device)
        batch = values.shape[0] if values.dim() == 3 else 1
        if batch:
            self._check(self.lib.sa_interp_apply_batch(out.data_ptr(), plan.plan.data_ptr(), values.data_ptr(), plan.k,
                                                       batch, self._stream()))
        return out

    def tree_fits(self, k):
        """whether the subproduct tree takes k points (sa_interp_plan_bytes(k) != 0; sa_zerofier has the same cap,
        2^20): host-only, no CUDA call.  Above it, geometric domains take geo_interp_plan and geo_zerofier."""
        return self.lib.sa_interp_plan_bytes(k) != 0

    def geo_interp_plan(self, step, k):
        """sa_geo_plan: what interpolation over step^0 .. step^(k-1) needs of the domain alone, kept on the device for
        geo_interp_apply (synchronises; "unsupported size" outside 1 <= k <= 2^26, "divide by zero" from k = 2 on
        when step is 0 or step^d = 1 for some d <= k)"""
        step = int(step) % P
        plan = self.torch.empty(max(1, self.lib.sa_geo_plan_bytes(k)), dtype=self.torch.uint8, device=self.device)
        self._check(self.lib.sa_geo_plan(plan.data_ptr(), _limbs(step), k, self._stream()))
        return GeoInterpPlan(plan, step, k)

    def geo_interp_apply(self, plan, values):
        """sa_geo_interp_batch: the coefficients interp_apply gives over the explicit domain, for one vector (k, 2) or
        a batch of them (B, k, 2) in one call; asynchronous, the plan is only read"""
        if values.dim() not in (2, 3) or tuple(values.shape[-2:]) != (plan.k, 2):
            raise SaError(SA_ERRORS[-6])
        values = values.contiguous()
        out = self.torch.empty(values.shape, dtype=self.torch.int64, device=self.device)
        batch = values.shape[0] if values.dim() == 3 else 1
        if batch:
            self._check(self.lib.sa_geo_interp_batch(out.data_ptr(), plan.plan.data_ptr(), values.data_ptr(), plan.k,
                                                     batch, self._stream()))
        return out

    def geo_zerofier(self, step, k):
        """sa_geo_zerofier: the k + 1 coefficients of prod_{i<k} (x - step^i), as zerofier gives them over the explicit
        domain (synchronises once; the refusals of geo_interp_plan)"""
        out = self.empty(k + 1)
        self._check(self.lib.sa_geo_zerofier(out.data_ptr(), _limbs(int(step) % P), k, self._stream()))
        return out

    @staticmethod
    def _rows(vecs, n):
        """the batch of a (ncoef, 2) or (B, ncoef, 2) tensor with 1 <= ncoef <= n; "unsupported size" otherwise (the
        library cannot see the tensors' shape)"""
        if vecs.dim() not in (2, 3) or vecs.shape[-1] != 2 or not 1 <= vecs.shape[-2] <= n:
            raise SaError(SA_ERRORS[-6])
        return vecs.shape[0] if vecs.dim() == 3 else 1

    def coset_div_plan(self, divisor, log_n, root, offset):
        """sa_coset_div_plan: what dividing by `divisor` (dlen, 2) on the coset offset * <root> of order 2^log_n needs
        of the divisor alone, kept on the device for coset_div_apply (synchronises; "divide by zero" when the divisor
        vanishes somewhere on the coset, the zero divisor included)"""
        nbytes = self.lib.sa_coset_div_plan_bytes(log_n)
        if nbytes == 0 or divisor.dim() != 2:
            raise SaError(SA_ERRORS[-6])
        self._rows(divisor, 1 << log_n)
        divisor = divisor.contiguous()
        plan = self.torch.empty(nbytes, dtype=self.torch.uint8, device=self.device)
        self._check(self.lib.sa_coset_div_plan(plan.data_ptr(), divisor.data_ptr(), divisor.shape[0], log_n,
                                               _limbs(root), _limbs(offset), self._stream()))
        return CosetDivPlan(plan, log_n, int(root), int(offset))

    def coset_div_apply(self, plan, lhs, qlen):
        """sa_coset_div_apply_batch: the first qlen coefficients of U(X) * offset^-j, U = intt(L / R) on the plan's
        coset, for one numerator (ncoef, 2) -> (qlen, 2) or a batch of them (B, ncoef, 2) -> (B, qlen, 2) in one
        call; asynchronous, the plan is only read"""
        n = 1 << plan.log_n
        batch = self._rows(lhs, n)
        if not 1 <= qlen <= n:
            raise SaError(SA_ERRORS[-6])
        lhs = lhs.contiguous()
        out = self.torch.empty(tuple(lhs.shape[:-2]) + (qlen, 2), dtype=self.torch.int64, device=self.device)
        if batch:
            self._check(self.lib.sa_coset_div_apply_batch(out.data_ptr(), plan.plan.data_ptr(), lhs.data_ptr(),
                                                          lhs.shape[-2], qlen, plan.log_n, _limbs(plan.root), batch,
                                                          self._stream()))
        return out

    def _out(self, out, shape):
        """a caller's output buffer: a contiguous int64 tensor of exactly `shape` on this device (a row range of a
        larger buffer qualifies); a new tensor when out is None"""
        torch = self.torch
        if out is None:
            return torch.empty(shape, dtype=torch.int64, device=self.device)
        if (not isinstance(out, torch.Tensor) or out.dtype != torch.int64 or out.device != self.device
                or tuple(out.shape) != tuple(shape) or not out.is_contiguous()):
            raise SaError(SA_ERRORS[-6])
        return out

    def coset_evaluate(self, coeffs, log_n, root, offset, out=None):
        """sa_coset_evaluate_batch: fast_coset_evaluate at order 2^log_n of one polynomial (ncoef, 2) -> (n, 2) or of
        a batch (B, ncoef, 2) -> (B, n, 2) in one call; asynchronous.  `out`, when given, is the contiguous (n, 2) /
        (B, n, 2) tensor the values are written to (and returned)"""
        if self.lib.sa_coset_batch_max(log_n) == 0:
            raise SaError(SA_ERRORS[-6])
        n = 1 << log_n
        batch = self._rows(coeffs, n)
        coeffs = coeffs.contiguous()
        out = self._out(out, tuple(coeffs.shape[:-2]) + (n, 2))
        if batch:
            self._check(self.lib.sa_coset_evaluate_batch(out.data_ptr(), coeffs.data_ptr(), coeffs.shape[-2], log_n,
                                                         _limbs(root), _limbs(offset), batch, self._stream()))
        return out

    def coset_combine_evaluate(self, terms, log_n, root, offset):
        """sa_coset_combine_evaluate: fast_coset_evaluate at order 2^log_n of sum_t weight_t * X^shift_t * vec_t over
        terms (vec, shift, weight), each vec a contiguous int64 (len, 2) tensor on this device -> (n, 2) in one call
        (the combination of fast_stark.py:125-148); asynchronous, nothing is uploaded"""
        torch = self.torch
        if self.lib.sa_coset_batch_max(log_n) == 0:
            raise SaError(SA_ERRORS[-6])
        n = 1 << log_n
        ptrs, lens, shifts, weights = [], [], [], []
        for vec, shift, weight in terms:  # the library cannot see the tensors' shape, device or layout
            if (not isinstance(vec, torch.Tensor) or vec.dtype != torch.int64 or vec.dim() != 2 or vec.shape[1] != 2
                    or vec.device != self.device or not vec.is_contiguous()):
                raise SaError(SA_ERRORS[-6])
            shift = int(shift)
            if shift < 0 or shift + vec.shape[0] > n:
                raise SaError(SA_ERRORS[-6])
            weight = int(weight) % P
            ptrs.append(vec.data_ptr())
            lens.append(vec.shape[0])
            shifts.append(shift)
            weights += [weight & 0xFFFFFFFFFFFFFFFF, weight >> 64]
        t = len(ptrs)
        out = self.empty(n)
        self._check(self.lib.sa_coset_combine_evaluate(
            out.data_ptr(), log_n, _limbs(root), _limbs(offset), (ctypes.c_void_p * t)(*ptrs),
            (ctypes.c_size_t * t)(*lens), (ctypes.c_size_t * t)(*shifts), (ctypes.c_uint64 * (2 * t))(*weights), t,
            self._stream()))
        return out

    def coset_combine_evaluate_batch(self, terms, nrows, log_n, root, offset):
        """sa_coset_combine_evaluate_batch: nrows combinations in one call -> (nrows, n, 2), row r the codeword
        coset_combine_evaluate gives for the terms (vec, shift, weight, row) with row == r (zeros for a row without
        terms), each vec a contiguous int64 (len, 2) tensor on this device; asynchronous, nothing is uploaded"""
        torch = self.torch
        nrows = int(nrows)
        if self.lib.sa_coset_batch_max(log_n) == 0 or nrows < 0:
            raise SaError(SA_ERRORS[-6])
        n = 1 << log_n
        ptrs, lens, shifts, rows, weights = [], [], [], [], []
        for vec, shift, weight, row in terms:  # the library cannot see the tensors' shape, device or layout
            if (not isinstance(vec, torch.Tensor) or vec.dtype != torch.int64 or vec.dim() != 2 or vec.shape[1] != 2
                    or vec.device != self.device or not vec.is_contiguous()):
                raise SaError(SA_ERRORS[-6])
            shift, row = int(shift), int(row)
            if shift < 0 or shift + vec.shape[0] > n or not 0 <= row < nrows:
                raise SaError(SA_ERRORS[-6])
            weight = int(weight) % P
            ptrs.append(vec.data_ptr())
            lens.append(vec.shape[0])
            shifts.append(shift)
            rows.append(row)
            weights += [weight & 0xFFFFFFFFFFFFFFFF, weight >> 64]
        t = len(ptrs)
        out = torch.empty((nrows, n, 2), dtype=torch.int64, device=self.device)
        self._check(self.lib.sa_coset_combine_evaluate_batch(
            out.data_ptr(), nrows, log_n, _limbs(root), _limbs(offset), (ctypes.c_void_p * t)(*ptrs),
            (ctypes.c_size_t * t)(*lens), (ctypes.c_size_t * t)(*shifts), (ctypes.c_size_t * t)(*rows),
            (ctypes.c_uint64 * (2 * t))(*weights), t, self._stream()))
        return out

    def air_plan(self, constraints, nregs, zerofier, max_ncoef, log_n, root, offset, step):
        """sa_air_plan: the transition constraints (MPolynomials or {exponent tuple: value} dicts over x, the nregs
        trace rows and the nregs next rows T(step * x)) compiled with the zerofier's (zlen, 2) coset division plan on
        the coset offset * <root> of order 2^log_n, for trace polynomials of up to max_ncoef coefficients
        (synchronises; "unsupported size" when a term's degree bound reaches n, "divide by zero" when the zerofier
        vanishes on the coset)"""
        nregs, max_ncoef = int(nregs), int(max_ncoef)
        constraints = list(constraints)
        if nregs < 1 or not constraints or zerofier.dim() != 2:
            raise SaError(SA_ERRORS[-6])
        if self.lib.sa_air_plan_bytes(log_n, max_ncoef, nregs, 0) == 0:
            raise SaError(SA_ERRORS[-6])
        self._rows(zerofier, 1 << log_n)
        coeffs, exps, starts = _air_arrays(constraints, nregs)
        nbytes = self.lib.sa_air_plan_bytes(log_n, max_ncoef, nregs, starts[-1])
        if nbytes == 0:
            raise SaError(SA_ERRORS[-6])
        zerofier = zerofier.contiguous()
        plan = self.torch.empty(nbytes, dtype=self.torch.uint8, device=self.device)
        ncons = len(constraints)
        self._check(self.lib.sa_air_plan(
            plan.data_ptr(), (ctypes.c_uint64 * max(len(coeffs), 1))(*coeffs),
            (ctypes.c_uint32 * max(len(exps), 1))(*exps), (ctypes.c_size_t * (ncons + 1))(*starts), ncons, nregs,
            max_ncoef, zerofier.data_ptr(), zerofier.shape[0], log_n, _limbs(root), _limbs(offset), _limbs(step),
            self._stream()))
        return AirPlan(plan, log_n, int(root), int(offset), nregs, ncons, max_ncoef, zerofier.shape[0] - 1)

    def _air_trace(self, plan, trace, qlen):
        """the batch of a (nregs, ncoef, 2) trace (None) or of a (B, nregs, ncoef, 2) batch of traces; "unsupported
        size" otherwise (the library cannot see the tensor's shape, dtype or device)"""
        torch = self.torch
        if (not isinstance(trace, torch.Tensor) or trace.dtype != torch.int64 or trace.device != self.device
                or trace.dim() not in (3, 4) or trace.shape[-3] != plan.nregs or trace.shape[-1] != 2
                or not 1 <= trace.shape[-2] <= plan.max_ncoef or not 1 <= int(qlen) <= 1 << plan.log_n):
            raise SaError(SA_ERRORS[-6])
        return trace.shape[0] if trace.dim() == 4 else None

    def air_quotients(self, plan, trace, qlen):
        """sa_air_quotients_batch: the first qlen coefficients of every constraint's quotient for the trace
        polynomials (nregs, ncoef, 2), ncoef <= the plan's max_ncoef -> (ncons, qlen, 2), or for a batch of traces
        (B, nregs, ncoef, 2) -> (B, ncons, qlen, 2), in one call; asynchronous, the plan is only read"""
        torch = self.torch
        batch = self._air_trace(plan, trace, qlen)
        trace = trace.contiguous()
        out = torch.empty(tuple(trace.shape[:-3]) + (plan.ncons, int(qlen), 2), dtype=torch.int64, device=self.device)
        self._check(self.lib.sa_air_quotients_batch(out.data_ptr(), plan.plan.data_ptr(), trace.data_ptr(),
                                                    plan.nregs, trace.shape[-2], int(qlen), plan.ncons,
                                                    1 if batch is None else batch, plan.log_n, _limbs(plan.root),
                                                    self._stream()))
        return out

    def air_quotients_exact(self, plan, trace, qlen, check=True):
        """sa_air_quotients_exact_batch: air_quotients' rows (ncons, qlen, 2) and the remainder flags (ncons,) int32,
        non-zero exactly where Z does not divide the constraint's numerator (the reference's Polynomial.__truediv__
        test), with the tail n - deg Z; for a batch of traces (B, nregs, ncoef, 2) the rows (B, ncons, qlen, 2) and
        flags (B, ncons).  The zerofier's top coefficient must be non-zero (deg Z = its length - 1, as air_plan takes
        it).  check=True reads the flags (one synchronisation) and raises the reference's remainder message naming the
        constraints (for a batch, the (trace, constraint) pairs); check=False stays asynchronous.  The plan is only
        read."""
        torch = self.torch
        batch = self._air_trace(plan, trace, qlen)
        if plan.zdeg is None:
            raise SaError(SA_ERRORS[-6])
        trace = trace.contiguous()
        lead = tuple(trace.shape[:-3])
        out = torch.empty(lead + (plan.ncons, int(qlen), 2), dtype=torch.int64, device=self.device)
        flags = torch.empty(lead + (plan.ncons,), dtype=torch.int32, device=self.device)
        self._check(self.lib.sa_air_quotients_exact_batch(
            out.data_ptr(), ctypes.cast(flags.data_ptr(), ctypes.POINTER(ctypes.c_uint32)), plan.plan.data_ptr(),
            trace.data_ptr(), plan.nregs, trace.shape[-2], int(qlen), plan.ncons, 1 if batch is None else batch,
            (1 << plan.log_n) - plan.zdeg, plan.log_n, _limbs(plan.root), self._stream()))
        if check:
            self._count("d2h", 4 * flags.numel())
            if batch is None:
                bad = [c for c, f in enumerate(flags.tolist()) if f]
            else:
                bad = [(b, c) for b, row in enumerate(flags.tolist()) for c, f in enumerate(row) if f]
            if bad:
                raise SaError("%s (constraints %s)" % (REMAINDER, bad))
        return out, flags

    def _ints(self, values):
        """a list of ints -> device vector (n, 2)"""
        return self.upload(bytearray(b"".join((int(v) % P).to_bytes(16, "little") for v in values)))

    def boundary_plan(self, boundary, nregs, omicron, log_n, root, offset):
        """sa_boundary_plan: for FastStark's boundary, a list of (cycle, register, value) with values ints or
        FieldElements, register s's points omicron^cycle, its zerofier Z_s (`zerofier`) and interpolant I_s
        (`interpolate`) on the device, planned on the coset offset * <root> of order 2^log_n (synchronises).
        "unsupported size" before any device work for offset 0, a register outside 0..nregs-1, a register without
        boundary points (the reference's interpolate_domain refuses those) or one with n or more; "divide by zero"
        when two of a register's cycles give one point, or when a zerofier vanishes on the coset"""
        nregs = int(nregs)
        if nregs < 1 or self.lib.sa_boundary_plan_bytes(log_n, nregs) == 0 or int(offset) % P == 0:
            raise SaError(SA_ERRORS[-6])
        w = int(getattr(omicron, "value", omicron))
        points = [[] for _ in range(nregs)]
        for c, r, v in boundary:
            if not 0 <= int(r) < nregs:
                raise SaError(SA_ERRORS[-6])
            points[int(r)].append((pow(w, int(c), P), int(getattr(v, "value", v))))
        if any(not 1 <= len(pts) < 1 << log_n for pts in points):
            raise SaError(SA_ERRORS[-6])
        zs, its = [], []
        for pts in points:
            domain = self._ints([x for x, _ in pts])
            its.append(self.interpolate(domain, self._ints([v for _, v in pts])))
            zs.append(self.zerofier(domain))
        plan = self.torch.empty(self.lib.sa_boundary_plan_bytes(log_n, nregs), dtype=self.torch.uint8,
                                device=self.device)
        vp, sz = ctypes.c_void_p * nregs, ctypes.c_size_t * nregs
        self._check(self.lib.sa_boundary_plan(
            plan.data_ptr(), vp(*[z.data_ptr() for z in zs]), sz(*[z.shape[0] for z in zs]),
            vp(*[i.data_ptr() for i in its]), sz(*[i.shape[0] for i in its]), nregs, log_n, _limbs(root),
            _limbs(int(offset) % P), self._stream()))
        return BoundaryPlan(plan, log_n, int(root), int(offset) % P, nregs, [len(pts) for pts in points])

    def boundary_quotients(self, plan, trace, check=True, out=None):
        """sa_boundary_quotients: for the trace polynomials (nregs, ncoef, 2), each register's boundary quotient
        (T_s - I_s) / Z_s followed by zeros (nregs, ncoef, 2), its codeword on the plan's coset (nregs, n, 2) and the
        remainder flags (nregs,) int32, non-zero where the division is not clean.  check=True reads the flags (one
        synchronisation) and raises the reference's remainder message naming the registers; check=False stays
        asynchronous.  `out`, when given, is the contiguous (nregs, n, 2) tensor the codewords are written to (and
        returned), e.g. the first rows of a buffer that more codewords share.  The plan is only read."""
        torch = self.torch
        n = 1 << plan.log_n
        # the library cannot see the tensor's shape, dtype or device
        if (not isinstance(trace, torch.Tensor) or trace.dtype != torch.int64 or trace.device != self.device
                or trace.dim() != 3 or trace.shape[0] != plan.nregs or trace.shape[2] != 2
                or not 1 <= trace.shape[1] <= n):
            raise SaError(SA_ERRORS[-6])
        trace = trace.contiguous()
        ncoef = trace.shape[1]
        quot = torch.empty((plan.nregs, ncoef, 2), dtype=torch.int64, device=self.device)
        codewords = self._out(out, (plan.nregs, n, 2))
        flags = torch.empty(plan.nregs, dtype=torch.int32, device=self.device)
        self._check(self.lib.sa_boundary_quotients(
            quot.data_ptr(), codewords.data_ptr(), ctypes.cast(flags.data_ptr(), ctypes.POINTER(ctypes.c_uint32)),
            plan.plan.data_ptr(), trace.data_ptr(), plan.nregs, ncoef, plan.log_n, _limbs(plan.root), self._stream()))
        if check:
            self._count("d2h", 4 * plan.nregs)
            bad = [s for s, f in enumerate(flags.tolist()) if f]
            if bad:
                raise SaError("%s (registers %s)" % (REMAINDER, bad))
        return quot, codewords, flags

    # --------------------------------------------------------------- merkle
    def _new_tree(self, n):
        return self.torch.empty((2 * n, 64), dtype=self.torch.uint8, device=self.device)

    def merkle_tree(self, vec):
        vec = vec.contiguous()
        n = vec.shape[0]
        tree = self._new_tree(n)
        self._check(self.lib.sa_merkle_tree(tree.data_ptr(), vec.data_ptr(), n, self._stream()))
        return tree

    def tree_root(self, tree):
        self._count("d2h", 64)
        return bytes(tree[1].cpu().numpy().tobytes())

    def download_tree(self, tree):
        """the whole heap-ordered tree as a host array uint8[2n, 64] (small trees: paths are then read on
        the host, O(log n) per opened index and no device round trip)"""
        self._count("d2h", tree.numel())
        return tree.cpu().numpy()

    def merkle_open(self, tree, indices):
        """authentication paths (lists of 64-byte digests, bottom-up) for leaf indices"""
        n = tree.shape[0] // 2
        k = len(indices)
        depth = n.bit_length() - 1
        if k == 0:
            return []
        if depth == 0:
            for i in indices:
                if not 0 <= i < n:
                    raise SaError(SA_ERRORS[-5])
            return [[] for _ in indices]
        for i in indices:
            if not 0 <= i < n:
                raise SaError(SA_ERRORS[-5])
        out = self.torch.empty((k, depth, 64), dtype=self.torch.uint8, device=self.device)
        idx = (ctypes.c_uint64 * k)(*indices)
        self._check(self.lib.sa_merkle_open(out.data_ptr(), tree.data_ptr(), n, idx, k, self._stream()))
        self._count("h2d", 8 * k)
        self._count("d2h", k * depth * 64)
        raw = out.cpu().numpy().tobytes()
        return [[raw[(q * depth + l) * 64:(q * depth + l + 1) * 64] for l in range(depth)] for q in range(k)]

    def gather(self, vec, indices):
        """values at `indices` -> numpy uint64[k, 2] on the host"""
        vec = vec.contiguous()
        k = len(indices)
        out = self.empty(k)
        if k:
            idx = (ctypes.c_uint64 * k)(*indices)
            self._check(self.lib.sa_gather(out.data_ptr(), vec.data_ptr(), vec.shape[0], idx, k, self._stream()))
            self._count("h2d", 8 * k)
            self._count("d2h", 16 * k)
        return out.cpu().numpy()

    def merkle_trees(self, vecs):
        """sa_merkle_tree_batch: the trees of B codewords of one length n, (B, n, 2) -> (B, 2n, 64) uint8, in one
        launch ladder; asynchronous"""
        if vecs.dim() != 3 or vecs.shape[-1] != 2:  # the library cannot see the tensor's shape
            raise SaError(SA_ERRORS[-6])
        vecs = vecs.contiguous()
        batch, n = vecs.shape[0], vecs.shape[1]
        trees = self.torch.empty((batch, 2 * n, 64), dtype=self.torch.uint8, device=self.device)
        self._check(self.lib.sa_merkle_tree_batch(trees.data_ptr(), vecs.data_ptr(), n, batch, self._stream()))
        return trees

    def tree_roots(self, trees):
        """the roots of a (B, 2n, 64) batch of trees as B 64-byte strings, from one device-to-host copy"""
        if trees.dim() != 3 or trees.shape[1] < 2 or trees.shape[1] % 2 or trees.shape[2] != 64:
            raise SaError(SA_ERRORS[-6])
        self._count("d2h", 64 * trees.shape[0])
        raw = trees[:, 1].cpu().numpy().tobytes()
        return [raw[64 * b:64 * (b + 1)] for b in range(trees.shape[0])]

    @staticmethod
    def _index_sets(batch, n, indices, group):
        """(the group, k, the flat index list) of a call's index sets: one set `indices` when group is None, else
        indices is a list of ceil(batch / group) sets of one length k, set g for rows g * group .. g * group + group;
        "unsupported size" or "cannot open invalid index" before any device work"""
        if group is None:
            sets, group = [list(indices)], max(batch, 1)
        else:
            group, sets = int(group), [list(s) for s in indices]
            if group < 1 or len(sets) != max(1, -(-batch // group)) or len({len(s) for s in sets}) > 1:
                raise SaError(SA_ERRORS[-6])
        flat = [i for s in sets for i in s]
        for i in flat:
            if not 0 <= i < n:
                raise SaError(SA_ERRORS[-5])
        return group, len(sets[0]), flat

    def merkle_open_batch(self, trees, indices, group=None):
        """sa_merkle_open_batch_sets: for each tree of a (B, 2n, 64) batch, the authentication paths of the same leaf
        indices, or with `group`, of its group's own set indices[b // group] (B lists of k lists of 64-byte digests,
        bottom-up), with one upload and one download"""
        if trees.dim() != 3 or trees.shape[1] < 2 or trees.shape[1] % 2 or trees.shape[2] != 64:
            raise SaError(SA_ERRORS[-6])
        trees = trees.contiguous()
        batch, n = trees.shape[0], trees.shape[1] // 2
        group, k, flat = self._index_sets(batch, n, indices, group)
        depth = n.bit_length() - 1
        out = self.torch.empty((batch, k, depth, 64), dtype=self.torch.uint8, device=self.device)
        idx = (ctypes.c_uint64 * max(len(flat), 1))(*flat)
        self._check(self.lib.sa_merkle_open_batch_sets(out.data_ptr(), trees.data_ptr(), n, batch, group, idx, k,
                                                       self._stream()))
        if out.numel() == 0:  # no tree, no index or no sibling: nothing was launched
            return [[[] for _ in range(k)] for _ in range(batch)]
        self._count("h2d", 8 * len(flat))
        self._count("d2h", out.numel())
        raw = out.cpu().numpy().tobytes()
        digests = [raw[i:i + 64] for i in range(0, len(raw), 64)]
        paths = [digests[i:i + depth] for i in range(0, len(digests), depth)]
        return [paths[b * k:(b + 1) * k] for b in range(batch)]

    def gather_batch(self, vecs, indices, group=None):
        """sa_gather_batch_sets: the values at the same indices in each row of a (B, n, 2) batch, or with `group`, at
        the row's group's own set indices[b // group] -> numpy (B, k, 2) on the host (the int64 limbs `gather`
        returns), with one upload and one download"""
        if vecs.dim() != 3 or vecs.shape[-1] != 2:
            raise SaError(SA_ERRORS[-6])
        vecs = vecs.contiguous()
        batch, n = vecs.shape[0], vecs.shape[1]
        if group is None:  # the library checks a lone set's indices itself
            group, k, flat = max(batch, 1), len(indices), list(indices)
        else:
            group, k, flat = self._index_sets(batch, n, indices, group)
        out = self.torch.empty((batch, k, 2), dtype=self.torch.int64, device=self.device)
        idx = (ctypes.c_uint64 * max(len(flat), 1))(*flat)
        self._check(self.lib.sa_gather_batch_sets(out.data_ptr(), vecs.data_ptr(), n, batch, group, idx, k,
                                                  self._stream()))
        if out.numel():
            self._count("h2d", 8 * len(flat))
            self._count("d2h", out.numel() * 8)
        return out.cpu().numpy()

    # --------------------------------------------------------------- sample
    def upload_seeds(self, seeds):
        """a list of 32-byte `bytes` -> one (nseeds, 32) uint8 device tensor (one upload); "unsupported size" for
        anything else"""
        if not all(isinstance(s, bytes) and len(s) == 32 for s in seeds):
            raise SaError(SA_ERRORS[-6])
        torch = self.torch
        if not seeds:
            return torch.empty((0, 32), dtype=torch.uint8, device=self.device)
        host = torch.frombuffer(bytearray(b"".join(seeds)), dtype=torch.uint8).reshape(-1, 32)
        self._count("h2d", host.numel())
        return host.to(self.device)

    def sample_seeded(self, out, seeds, first, count, width=1, lane_stride=1, seed_stride=None, offset=0):
        """sa_sample_seeded into the contiguous int64 tensor `out` (..., 2) from element `offset` on: for seed b and
        j < count, the element of draw first + j (DESIGN section 3.13) at offset + b seed_stride + (j % width)
        lane_stride + j // width.  `seeds` is a list of 32-byte bytes (upload_seeds) or the (nseeds, 32) uint8 device
        tensor it gives; seed_stride defaults to count.  Asynchronous; "unsupported size" before any device work for
        width 0 or when the largest offset falls outside `out`.  Returns out."""
        torch = self.torch
        if not isinstance(seeds, torch.Tensor):
            seeds = self.upload_seeds(list(seeds))
        if (seeds.dtype != torch.uint8 or seeds.dim() != 2 or seeds.shape[1] != 32 or not seeds.is_contiguous()
                or out.dtype != torch.int64 or out.shape[-1] != 2 or not out.is_contiguous()):
            raise SaError(SA_ERRORS[-6])
        nseeds = seeds.shape[0]
        seed_stride = count if seed_stride is None else seed_stride
        if width < 1 or min(first, count, lane_stride, seed_stride, offset) < 0 or first + count > 1 << 64:
            raise SaError(SA_ERRORS[-6])
        if nseeds == 0 or count == 0:
            return out
        last = offset + (nseeds - 1) * seed_stride + (min(count, width) - 1) * lane_stride + (count - 1) // width
        if last >= out.numel() // 2:
            raise SaError(SA_ERRORS[-6])
        self._check(self.lib.sa_sample_seeded(out.data_ptr() + 16 * offset, seeds.data_ptr(), nseeds, seed_stride,
                                              first, count, width, lane_stride, self._stream()))
        return out

    # --------------------------------------------------------------- rescue
    RESCUE_MAX_ROUNDS = 512  # SA_RESCUE_MAX_ROUNDS

    def rescue(self, inputs, constants, rounds, alpha, alphainv, hashes=None, trace=None, inst_stride=None,
               lane_stride=None):
        """sa_rescue (DESIGN section 3.14): the Rescue-Prime permutation of width 2 over the (count, 2) canonical
        `inputs` with `rounds` rounds, the exponents alpha and alphainv (ints below 2^128) and the device `constants`
        (the MDS matrix row-major, then 4 rounds round constants).  hashes[b] gets input b's hash; the contiguous
        int64 tensor `trace` (..., 2) gets register s of row r <= rounds at b inst_stride + s lane_stride + r
        (default: dense, lane_stride = rounds + 1 and inst_stride = 2 lane_stride).  Either output may be None, not
        both.  Asynchronous; "unsupported size" before any device work for both outputs None, rounds outside
        1..RESCUE_MAX_ROUNDS, an exponent outside 0..2^128 - 1, or a buffer shorter than the call reads or writes.
        Returns (hashes, trace)."""
        lane_stride = rounds + 1 if lane_stride is None else lane_stride
        inst_stride = 2 * lane_stride if inst_stride is None else inst_stride
        vecs = [v for v in (inputs, constants, hashes, trace) if v is not None]
        if (any(v.dtype != self.torch.int64 or v.shape[-1] != 2 or not v.is_contiguous() for v in vecs)
                or (hashes is None and trace is None) or not 1 <= rounds <= self.RESCUE_MAX_ROUNDS
                or not all(0 <= int(e) < 1 << 128 for e in (alpha, alphainv)) or min(inst_stride, lane_stride) < 0
                or constants.numel() // 2 < 4 + 4 * rounds):
            raise SaError(SA_ERRORS[-6])
        count = inputs.numel() // 2
        if hashes is not None and hashes.numel() // 2 < count:
            raise SaError(SA_ERRORS[-6])
        if trace is not None and count and (count - 1) * inst_stride + lane_stride + rounds >= trace.numel() // 2:
            raise SaError(SA_ERRORS[-6])
        if count == 0:
            return hashes, trace
        self._check(self.lib.sa_rescue(None if hashes is None else hashes.data_ptr(),
                                       None if trace is None else trace.data_ptr(), inputs.data_ptr(), count,
                                       constants.data_ptr(), rounds, _limbs(alpha), _limbs(alphainv), inst_stride,
                                       lane_stride, self._stream()))
        return hashes, trace

    # --------------------------------------------------------------- verify
    def air_program(self, constraints, nregs):
        """sa_air_program: the transition constraints (as air_plan takes them) compiled into the program the
        combination walks, a uint8 device tensor (synchronises)"""
        nregs, constraints = int(nregs), list(constraints)
        if nregs < 1 or not constraints:
            raise SaError(SA_ERRORS[-6])
        coeffs, exps, starts = _air_arrays(constraints, nregs)
        nbytes = self.lib.sa_air_program_bytes(starts[-1], nregs)
        if nbytes == 0:
            raise SaError(SA_ERRORS[-6])
        prog = self.torch.empty(nbytes, dtype=self.torch.uint8, device=self.device)
        ncons = len(constraints)
        self._check(self.lib.sa_air_program(
            prog.data_ptr(), (ctypes.c_uint64 * max(len(coeffs), 1))(*coeffs),
            (ctypes.c_uint32 * max(len(exps), 1))(*exps), (ctypes.c_size_t * (ncons + 1))(*starts), ncons, nregs,
            self._stream()))
        return prog

    def upload_bytes(self, buf):
        """a host bytes-like object -> one uint8 device tensor (one upload)"""
        torch = self.torch
        host = torch.frombuffer(bytearray(buf), dtype=torch.uint8) if len(buf) else torch.empty(0, dtype=torch.uint8)
        self._count("h2d", host.numel())
        return host.to(self.device)

    def transcript_bytes(self, shape):
        """sa_transcript_bytes: one proof's workspace for a plan shape (SA_TRANSCRIPT_SHAPE ints), 0 if refused"""
        return self.lib.sa_transcript_bytes((ctypes.c_uint64 * 10)(*shape))

    def transcript_sections(self, buf, parts, L, nstat, nproofs, shape):
        """sa_transcript_sections over the chunk VerifierPlan._transcript_chunk laid out: `buf` its uploaded uint8
        tensor, parts the byte offsets of its proofs, proof_at, prefixes, statement and zerofier root, and
        L["section_at"] the sections' byte offsets in include/sa_b200.h's order.  Returns the
        zeroed-then-written sections (a uint8 tensor of L["bytes"]) and the per-proof out bytes (a uint8 tensor), no
        synchronisation"""
        torch = self.torch
        sec = torch.zeros(max(L["bytes"], 16), dtype=torch.uint8, device=self.device)
        out = torch.empty(80 * max(nproofs, 1), dtype=torch.uint8, device=self.device)
        ws = torch.empty(max(self.transcript_bytes(shape) * nproofs, 16), dtype=torch.uint8, device=self.device)
        ptr = buf.data_ptr()
        at = (ctypes.c_uint64 * len(L["section_at"]))(*L["section_at"])
        zroot = ptr + parts["zroot"] if shape[5] == shape[0] + 2 else None
        self._check(self.lib.sa_transcript_sections(
            sec.data_ptr(), at, out.data_ptr(), ws.data_ptr(), ptr + parts["proofs"], ptr + parts["proof_at"],
            ptr + parts["prefixes"], ptr + parts["statement"], nstat, zroot, nproofs,
            (ctypes.c_uint64 * 10)(*shape), self._stream()))
        return sec, out

    def verify_chunk(self, buf, L, extra=None):
        """The device checks of one chunk of proofs (DESIGN section 3.15) from `buf`, the chunk's one uploaded uint8
        tensor, whose sections start at the byte offsets of the layout L (sa_stark.VerifierPlan._pack):
        sa_merkle_verify_batch over L["paths"] paths, sa_fri_colinear_batch over L["colinear"] items,
        sa_verify_combination over L["k"] indices of L["proofs"] proofs, and for the proofs' last codewords one
        sa_merkle_tree_batch, one batched inverse sa_ntt and sa_poly_degree_batch.  Everything lands in one result
        buffer read with one download: (Merkle flags, colinearity flags, combination flags, the last codewords'
        degrees, their tree roots as bytes), and with `extra`, a uint8 device tensor read back in the same
        download, its bytes last."""
        torch, st = self.torch, self._stream()
        lib = self.lib
        ptr = buf.data_ptr()
        at = lambda name: ptr + L[name]  # noqa: E731
        npath, ncol, B, k, m = L["paths"], L["colinear"], L["proofs"], L["k"], L["last_len"]
        nflag = npath + ncol + B * k
        nextra = 0 if extra is None else extra.numel()
        res = torch.empty(4 * nflag + 8 * B + 64 * B + 8 + nextra, dtype=torch.uint8, device=self.device)
        flags = res.data_ptr()
        deg_at = 4 * nflag + (-4 * nflag) % 8
        self._check(lib.sa_merkle_verify_batch(flags, at("roots"), at("leaves"), at("leaf_index"), at("depth"),
                                               at("digests"), at("path_offset"), npath, st))
        self._check(lib.sa_fri_colinear_batch(flags + 4 * npath, at("ay"), at("by"), at("cy"), at("a_index"),
                                              at("alpha"), at("round"), _limbs(L["fri_offset"]),
                                              _limbs(L["fri_omega"]), ncol, st))
        zcoef = L.get("zcoef")
        self._check(lib.sa_verify_combination(flags + 4 * (npath + ncol), at("items"), at("proof_data"), k, B,
                                              L["prog"].data_ptr(), L["ncons"], L["nregs"], L["blen"],
                                              None if zcoef is None else zcoef.data_ptr(),
                                              0 if zcoef is None else zcoef.shape[0], _limbs(L["offset"]),
                                              _limbs(L["omega"]), L["log_n"], L["ef"], st))
        if B:
            last = buf[L["last"]:L["last"] + 16 * B * m].view(torch.int64).reshape(B, m, 2)
            trees = self.merkle_trees(last)
            coeffs = self.ntt(last.reshape(B * m, 2), m.bit_length() - 1, L["last_omega"], inverse=True, batch=B)
            self._check(lib.sa_poly_degree_batch(flags + deg_at, coeffs.data_ptr(), m, B, st))
            res[deg_at + 8 * B:deg_at + 72 * B].view(B, 64).copy_(trees[:, 1])
        if nextra:
            res[deg_at + 72 * B:deg_at + 72 * B + nextra].copy_(extra)
        host = res.cpu().numpy()
        self._count("d2h", res.numel())
        import numpy as np
        got = (host[:4 * npath].view(np.uint32), host[4 * npath:4 * (npath + ncol)].view(np.uint32),
               host[4 * (npath + ncol):4 * nflag].view(np.uint32), host[deg_at:deg_at + 8 * B].view(np.int64),
               host[deg_at + 8 * B:deg_at + 72 * B].tobytes())
        return got if extra is None else got + (host[deg_at + 72 * B:deg_at + 72 * B + nextra].tobytes(),)

    # ------------------------------------------------------------------ fri
    def fri_fold(self, vec, alpha, offset, omega):
        vec = vec.contiguous()
        n = vec.shape[0]
        out = self.empty(n // 2)
        self._check(self.lib.sa_fri_fold(out.data_ptr(), vec.data_ptr(), n, _limbs(alpha), _limbs(offset),
                                         _limbs(omega), self._stream()))
        return out

    def fri_round(self, vec, alpha, offset, omega):
        """fold (fri.py:85) + Merkle tree of the folded codeword, one fused kernel"""
        vec = vec.contiguous()
        n = vec.shape[0]
        out = self.empty(n // 2)
        tree = self._new_tree(n // 2)
        self._check(self.lib.sa_fri_round(out.data_ptr(), tree.data_ptr(), vec.data_ptr(), n, _limbs(alpha),
                                          _limbs(offset), _limbs(omega), self._stream()))
        return out, tree

    def fri_commit(self, vec, rounds, offset, omega, on_root):
        """code/fri.py:56-96 round loop in one C call (sa_fri_commit).

        on_root(round, root_bytes, want_alpha) is called after every round with the 64-byte
        Merkle root; it returns the challenge alpha (int) when want_alpha.  Returns
        (layers, trees): device vectors / trees of layers 0 .. rounds-1 (layer 0 is `vec`)."""
        vec = vec.contiguous()
        n = vec.shape[0]
        layers = self.empty(max(n - (n >> (rounds - 1)), 1))
        trees = self.torch.empty((4 * n - ((4 * n) >> rounds), 64), dtype=self.torch.uint8, device=self.device)
        errors = []

        def challenge(_user, r, root_ptr, alpha_out, want):
            try:
                alpha = on_root(r, ctypes.string_at(root_ptr, 64), bool(want))
                if want:
                    alpha_out[0] = alpha & 0xFFFFFFFFFFFFFFFF
                    alpha_out[1] = alpha >> 64
                return 0
            except BaseException as exc:  # re-raised below, outside the C frame
                errors.append(exc)
                return 1
        cb = FRI_CHALLENGE_FN(challenge)
        rc = self.lib.sa_fri_commit(layers.data_ptr(), trees.data_ptr(), vec.data_ptr(), n, rounds, _limbs(offset),
                                    _limbs(omega), cb, None, self._stream())
        if errors:
            raise errors[0]
        self._check(rc)
        out_layers, out_trees = [vec], []
        lo, to, ln = 0, 0, n
        for r in range(rounds):
            out_trees.append(trees[to:to + 2 * ln])
            to += 2 * ln
            if r + 1 < rounds:
                out_layers.append(layers[lo:lo + ln // 2])
                lo += ln // 2
                ln //= 2
        return out_layers, out_trees

    def fri_commit_batch(self, vecs, rounds, offset, omega, on_roots):
        """sa_fri_commit_batch: fri_commit for the B rows of a (B, n, 2) device tensor in one launch ladder.

        on_roots(round, roots, want_alpha) is called once per round with the B 64-byte roots of the round (a list of
        bytes, from one host wait); it returns the B challenges (ints) when want_alpha.  Returns (layers, trees):
        layers[r] the (B, n >> r, 2) rows of round r (layers[0] is `vecs`), trees[r] their (B, 2 (n >> r), 64) trees,
        views of one layer buffer and one tree buffer laid out as the library lays them."""
        torch = self.torch
        if vecs.dim() != 3 or vecs.shape[-1] != 2 or vecs.dtype != torch.int64:
            raise SaError(SA_ERRORS[-6])
        vecs = vecs.contiguous()
        batch, n = vecs.shape[0], vecs.shape[1]
        if n < 1 or n & (n - 1) or not 1 <= rounds <= n.bit_length():
            raise SaError(SA_ERRORS[-6])
        layers = self.empty(max(batch * (n - (n >> (rounds - 1))), 1))
        trees = torch.empty((max(batch * (4 * n - ((4 * n) >> rounds)), 1), 64), dtype=torch.uint8, device=self.device)
        errors = []

        def challenge(_user, r, roots_ptr, alphas_out, want):
            try:
                self._count("d2h", 64 * batch)  # the round's roots, from the mapped landing pads
                raw = ctypes.string_at(roots_ptr, 64 * batch)
                alphas = on_roots(r, [raw[64 * b:64 * (b + 1)] for b in range(batch)], bool(want))
                if want:
                    alphas = list(alphas)
                    if len(alphas) != batch:
                        raise ValueError("fri_commit_batch: %d challenges for %d codewords" % (len(alphas), batch))
                    for b, alpha in enumerate(alphas):
                        alphas_out[2 * b] = alpha & 0xFFFFFFFFFFFFFFFF
                        alphas_out[2 * b + 1] = alpha >> 64
                return 0
            except BaseException as exc:  # re-raised below, outside the C frame
                errors.append(exc)
                return 1
        cb = FRI_CHALLENGE_FN(challenge)
        rc = self.lib.sa_fri_commit_batch(layers.data_ptr(), trees.data_ptr(), vecs.data_ptr(), n, batch, rounds,
                                          _limbs(offset), _limbs(omega), cb, None, self._stream())
        if errors:
            raise errors[0]
        self._check(rc)
        out_layers, out_trees = [vecs], []
        lo, to, ln = 0, 0, n
        for r in range(rounds):
            out_trees.append(trees[to:to + batch * 2 * ln].view(batch, 2 * ln, 64))
            to += batch * 2 * ln
            if r + 1 < rounds:
                out_layers.append(layers[lo:lo + batch * (ln // 2)].view(batch, ln // 2, 2))
                lo += batch * (ln // 2)
                ln //= 2
        return out_layers, out_trees

    def synchronize(self):
        self.torch.cuda.synchronize(self.device)

    def launch_count(self):
        return int(self.lib.sa_launch_count())


_ENGINE = None


def get_engine():
    """The process-wide engine; created on first use.  Raises without CUDA."""
    global _ENGINE
    if _ENGINE is None:
        _ENGINE = CudaEngine()
    return _ENGINE


def set_engine(engine):
    """Install an engine object (tests use this to exercise the host logic with a
    test double; the product never calls it)."""
    global _ENGINE
    _ENGINE = engine
    return engine
