"""sa_accel -- opt-in acceleration of the caller's ``Polynomial.__mul__`` (SURVEY.md section 8 f2).

With the hot-path surfaces on the GPU, one ``FastRPSSS.sign`` still spends ~90 % of its time in
the schoolbook ``Polynomial.__mul__`` (code/univariate.py:38-48) called from
``MPolynomial.evaluate_symbolic`` and from ``fast_stark.py:137-145`` -- code outside ntt.py /
fri.py.  ``enable()`` rebinds ``univariate.Polynomial.__mul__`` so that products above a size
threshold go through the device NTT (zero-pad to a power of two, two transforms, Hadamard
product, inverse transform).  The result is the same object the schoolbook loop builds: exactly
``len(a) + len(b) - 1`` coefficients (untrimmed), ``Polynomial([])`` when either list is empty,
every coefficient the exact product coefficient mod p.  Small products, and polynomials over any
other field, keep the original method.

Off by default -- the drop-in never changes the caller's classes on its own.  Turn it on with
``import sa_accel; sa_accel.enable()`` or by exporting SA_B200_ACCEL_POLYMUL=1 before importing
the drop-in ``ntt`` module.
"""
import os

import sa_host
import sa_engine
import sa_devlist
import ntt  # the drop-in, which imports this module in turn; device_mul only runs once both are loaded

Polynomial = sa_host.univariate.Polynomial

_original_mul = None
THRESHOLD = 2048  # len(a) * len(b) below this stays on the host loop


def _root_of_unity(n):
    # algebra.py:104-114 for the main field: generator^(2^119 / n)
    return pow(85408008396924667383611388730472331217, (1 << 119) // n, sa_engine.P)


def device_mul(self, other):
    a, b = self.coefficients, other.coefficients
    if a == [] or b == []:
        return Polynomial([])
    if len(a) * len(b) < THRESHOLD or a[0].field.p != sa_engine.P:
        return _original_mul(self, other)
    out_len = len(a) + len(b) - 1
    n = 1 << max((out_len - 1).bit_length(), 1)
    eng = sa_engine.get_engine()
    fa, fb = eng.pad(sa_devlist.to_device(a), n), eng.pad(sa_devlist.to_device(b), n)
    prod = ntt._ntt_product(fa, fb, _root_of_unity(n))
    return Polynomial(sa_devlist.from_device(eng.slice(prod, 0, out_len), a[0].field))


def enable(threshold=None):
    """rebind univariate.Polynomial.__mul__ to the device product (idempotent)"""
    global _original_mul, THRESHOLD
    if threshold is not None:
        THRESHOLD = threshold
    if _original_mul is None:
        _original_mul = Polynomial.__mul__
        Polynomial.__mul__ = device_mul


def disable():
    global _original_mul
    if _original_mul is not None:
        Polynomial.__mul__ = _original_mul
        _original_mul = None


if os.environ.get("SA_B200_ACCEL_POLYMUL") == "1":
    enable()
