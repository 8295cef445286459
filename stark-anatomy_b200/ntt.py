"""Drop-in for the reference's code/ntt.py, backed by the H100 engine.

Put this directory ahead of the reference's code/ directory on sys.path and
``from ntt import *`` (code/fast_stark.py:4, code/fri.py:4) resolves here.  Same
names, signatures, value types (lists of ``algebra.FieldElement``,
``univariate.Polynomial``), assertion messages and list-length semantics as the
reference; every transform, Hadamard product, coset evaluation and coset division
runs in the sm_90a kernels behind include/sa_b200.h.  No CPU fallback:
without the CUDA library the first call raises.

Known divergence, in misuse only: when ``root_order`` is too small for the operands (degree >= root_order)
the reference's NTT product wraps around silently (ntt.py:47-64 has no check) or trips an assert deep inside a
recursive call, depending on the sizes; ``fast_zerofier`` / ``fast_evaluate`` / ``fast_interpolate`` here do not go
through ``fast_multiply`` and return the mathematically correct polynomial / values in those cases (the two
asserts on ``primitive_root`` / ``root_order`` themselves are the reference's).  ``fast_multiply`` and
``fast_coset_divide`` wrap exactly like the reference.

Reference lines mirrored: ntt :3-18, intt :20-30, fast_multiply :32-64,
fast_zerofier :66-80, fast_evaluate :82-100, fast_interpolate :102-130,
fast_coset_evaluate :132-135, fast_coset_divide :137-176.
"""
import sa_host  # noqa: F401  (resolves algebra/univariate: the reference's, else the host mirror)
from univariate import *  # noqa: F401,F403  re-exported exactly like code/ntt.py:1
from univariate import Polynomial

import sa_engine
import sa_devlist
import sa_accel  # noqa: F401  (opt-in Polynomial.__mul__ acceleration; inert unless enabled)

_P = sa_engine.P

_ORDER_MSG = "supplied root does not have supplied order"
_PRIM_MSG = "supplied root is not primitive root of supplied order"


def _engine():
    return sa_engine.get_engine()


def _check_field(field):
    if field.p != _P:
        raise NotImplementedError("the engine implements the field p = 1 + 407*2^119 only")


def _check_root(primitive_root, root_order):
    """the two asserts every fast_* function of the reference starts with"""
    p = primitive_root.field.p
    assert pow(primitive_root.value, root_order, p) == 1 % p, _ORDER_MSG
    assert pow(primitive_root.value, root_order // 2, p) != 1 % p, _PRIM_MSG


def _log2(n):
    return n.bit_length() - 1


# --------------------------------------------------------------------- ntt --
# ntt / intt / fast_coset_evaluate return a sa_devlist.DeviceCodeword: a list-like whose values stay in
# HBM (len, indexing, iteration, ==, slicing, + ... work; elements are created when read).  Handing it
# back to ntt / intt / Merkle.commit / Merkle.open / Fri.commit / Fri.prove costs no pack and no upload
# (SURVEY 8 f3); SA_B200_DEVICE_LISTS=0 returns plain lists instead.
def ntt(primitive_root, values):
    assert(len(values) & (len(values) - 1) == 0), "cannot compute ntt of non-power-of-two sequence"
    if len(values) <= 1:
        return values
    field = sa_devlist.field_of(values)
    _check_field(field)
    eng = _engine()
    out = eng.ntt(sa_devlist.to_device(values), _log2(len(values)), primitive_root.value)
    return sa_devlist.wrap(out, field)


def intt(primitive_root, values):
    assert(len(values) & (len(values) - 1) == 0), "cannot compute intt of non-power-of-two sequence"
    if len(values) == 1:
        return values
    field = sa_devlist.field_of(values)
    _check_field(field)
    eng = _engine()
    out = eng.ntt(sa_devlist.to_device(values), _log2(len(values)), primitive_root.value, inverse=True)
    return sa_devlist.wrap(out, field)


def _shrink(root, order, degree, p):
    """ntt.py:47-49 / :155-157: halve the order while the degree still fits"""
    while degree < order // 2:
        root = root * root % p
        order = order // 2
    return root, order


def _transform_length(ncoef, order):
    """length of `coefficients[:deg+1]` after the reference's zero-padding loop; the
    reference's ntt then asserts on it (non power of two / wrong root order)"""
    total = max(ncoef, order)
    assert(total & (total - 1) == 0), "cannot compute ntt of non-power-of-two sequence"
    return total


def _ntt_product(a, b, root):
    """ntt.py:52-64 on two zero-padded coefficient vectors: transform both, multiply the codewords, transform back"""
    eng = _engine()
    ln, rn = eng.length(a), eng.length(b)
    a = eng.ntt(a, _log2(ln), root)
    b = eng.ntt(b, _log2(rn), root)
    if ln != rn:  # the reference's zip() truncates to the shorter codeword (ntt.py:61)
        k = min(ln, rn)
        a, b = eng.slice(a, 0, k), eng.slice(b, 0, k)
        assert(k & (k - 1) == 0), "cannot compute intt of non-power-of-two sequence"
    product = eng.pointwise_mul(a, b)
    return eng.ntt(product, _log2(eng.length(product)), root, inverse=True)


def fast_multiply(lhs, rhs, primitive_root, root_order):
    _check_root(primitive_root, root_order)
    if lhs.is_zero() or rhs.is_zero():
        return Polynomial([])
    field = lhs.coefficients[0].field
    _check_field(field)
    lhs_degree, rhs_degree = lhs.degree(), rhs.degree()
    degree = lhs_degree + rhs_degree
    if degree < 8:
        return lhs * rhs
    root, order = _shrink(primitive_root.value, root_order, degree, field.p)
    eng = _engine()
    ln = _transform_length(lhs_degree + 1, order)
    rn = _transform_length(rhs_degree + 1, order)
    a = eng.pad(sa_devlist.to_device(lhs.coefficients[:lhs_degree + 1]), ln)
    b = eng.pad(sa_devlist.to_device(rhs.coefficients[:rhs_degree + 1]), rn)
    product = _ntt_product(a, b, root)
    return Polynomial(sa_devlist.from_device(eng.slice(product, 0, degree + 1), field))


def fast_zerofier(domain, primitive_root, root_order):
    _check_root(primitive_root, root_order)
    if len(domain) == 0:
        return Polynomial([])
    field = primitive_root.field
    if len(domain) == 1:
        return Polynomial([-domain[0], field.one()])
    eng = _engine()
    if len(domain) <= eng.MAX_DIRECT_POINTS:
        # prod (X - d): the subproduct tree of ntt.py:76-80 yields this same monic polynomial,
        # len(domain) + 1 coefficients; one device kernel builds it
        _check_field(field)
        return Polynomial(sa_devlist.from_device(eng.zerofier(sa_devlist.to_device(domain)), field))
    half = len(domain) // 2
    left = fast_zerofier(domain[:half], primitive_root, root_order)
    right = fast_zerofier(domain[half:], primitive_root, root_order)
    return fast_multiply(left, right, primitive_root, root_order)


def fast_evaluate(polynomial, domain, primitive_root, root_order):
    _check_root(primitive_root, root_order)
    if len(domain) == 0:
        return []
    field = domain[0].field
    _check_field(field)
    if len(polynomial.coefficients) == 0:
        return [field.zero() for _ in domain]
    # the remainder tree of the reference (ntt.py:94-100) only re-expresses
    # polynomial(d) for every d in the domain; one Horner kernel gives the same values
    eng = _engine()
    values = eng.poly_eval(sa_devlist.to_device(polynomial.coefficients), sa_devlist.to_device(domain))
    return sa_devlist.from_device(values, field)


def fast_interpolate(domain, values, primitive_root, root_order):
    _check_root(primitive_root, root_order)
    assert(len(domain) == len(values)), "cannot interpolate over domain of different length than values list"
    if len(domain) == 0:
        return Polynomial([])
    if len(domain) == 1:
        return Polynomial([values[0]])
    eng = _engine()
    if len(domain) <= eng.MAX_DIRECT_POINTS:
        # the interpolant of degree < len(domain) is unique, so the device Lagrange kernels
        # return exactly the len(domain) coefficients the recursion of ntt.py:113-130 produces;
        # coinciding domain points raise "divide by zero" like the division at ntt.py:124-125
        field = values[0].field
        _check_field(field)
        coeffs = eng.interpolate(sa_devlist.to_device(domain), sa_devlist.to_device(values))
        return Polynomial(sa_devlist.from_device(coeffs, field))
    half = len(domain) // 2
    left_zerofier = fast_zerofier(domain[:half], primitive_root, root_order)
    right_zerofier = fast_zerofier(domain[half:], primitive_root, root_order)
    left_offset = fast_evaluate(right_zerofier, domain[:half], primitive_root, root_order)
    right_offset = fast_evaluate(left_zerofier, domain[half:], primitive_root, root_order)
    if not all(not v.is_zero() for v in left_offset):
        print("left_offset:", " ".join(str(v) for v in left_offset))
    left_targets = [n / d for (n, d) in zip(values[:half], left_offset)]
    right_targets = [n / d for (n, d) in zip(values[half:], right_offset)]
    left_interpolant = fast_interpolate(domain[:half], left_targets, primitive_root, root_order)
    right_interpolant = fast_interpolate(domain[half:], right_targets, primitive_root, root_order)
    return left_interpolant * right_zerofier + right_interpolant * left_zerofier


def fast_coset_evaluate(polynomial, offset, generator, order):
    field = offset.field
    _check_field(field)
    ncoef = len(polynomial.coefficients)
    total = ncoef + max(0, order - ncoef)  # ntt.py:134 pads with (order - len) zeros
    assert(total & (total - 1) == 0), "cannot compute ntt of non-power-of-two sequence"
    eng = _engine()
    if total <= 1:
        return polynomial.scale(offset).coefficients + [field.zero()] * (order - ncoef)
    coeffs = sa_devlist.to_device(polynomial.coefficients) if ncoef else eng.zeros(1)
    return sa_devlist.wrap(eng.coset_evaluate(coeffs, _log2(total), generator.value, offset.value), field)


def fast_coset_divide(lhs, rhs, offset, primitive_root, root_order):  # clean division only!
    _check_root(primitive_root, root_order)
    assert(not rhs.is_zero()), "cannot divide by zero polynomial"
    if lhs.is_zero():
        return Polynomial([])
    lhs_degree, rhs_degree = lhs.degree(), rhs.degree()
    assert(rhs_degree <= lhs_degree), "cannot divide by polynomial of larger degree"
    field = lhs.coefficients[0].field
    _check_field(field)
    degree = max(lhs_degree, rhs_degree)
    if degree < 8:
        return lhs / rhs
    root, order = _shrink(primitive_root.value, root_order, degree, field.p)
    eng = _engine()
    ln = _transform_length(lhs_degree + 1, order)
    _transform_length(rhs_degree + 1, order)
    # ntt.py:159-176 is the plan's apply at order ln, truncated to the quotient.  ln == order unless
    # degree >= root_order; then the plan's root check raises what the reference's first ntt asserts.
    numerator = sa_devlist.to_device(lhs.coefficients[:lhs_degree + 1])
    divisor = sa_devlist.to_device(rhs.coefficients[:rhs_degree + 1])
    plan = eng.coset_div_plan(divisor, _log2(ln), root, offset.value)  # raises "divide by zero" like algebra.py:92
    quotient = eng.coset_div_apply(plan, numerator, lhs_degree - rhs_degree + 1)
    return Polynomial(sa_devlist.from_device(quotient, field))
