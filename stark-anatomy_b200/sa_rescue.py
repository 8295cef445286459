"""sa_rescue -- RescuePrime.hash and RescuePrime.trace (code/rescue_prime.py) over many inputs on the device.

``hash_batch(rp, inputs)`` is ``[rp.hash(x) for x in inputs]`` and ``trace_batch(rp, inputs)`` is
``[rp.trace(x) for x in inputs]``, each as one upload of the instance's constants and the inputs and one sa_rescue
launch (DESIGN section 3.14).  The constants, the round count and the exponents are read from the caller's `rp`
(rp.MDS, rp.round_constants, rp.N, rp.alpha, rp.alphainv): the library holds none of its own, so any RescuePrime
instance of state width 2 works.  A batch keygen is the caller's secret-key draws followed by one ``hash_batch``.

The AIR (``transition_constraints``) stays host algebra: ``sa_stark.SignerPlan`` builds it once per signer."""
import sa_devlist
import sa_engine
import sa_marshal

P = sa_engine.P


def values(elements, what="input"):
    """the ints of field elements (FieldElement or int), each asserted to be a residue of p"""
    out = [getattr(x, "value", x) for x in elements]
    assert all(type(v) is int and 0 <= v < P for v in out), "sa_rescue: every %s must be an element of p" % what
    return out


def constants(rp):
    """rp's constant block in sa_rescue's order: the MDS matrix row-major, then the 4 N round constants.  Asserts a
    state width of 2 and a round count the kernel takes."""
    assert rp.m == 2, "sa_rescue: the kernel takes state width 2, not %r" % (rp.m,)
    assert 1 <= rp.N <= sa_engine.CudaEngine.RESCUE_MAX_ROUNDS, "sa_rescue: %r rounds" % (rp.N,)
    assert 0 <= rp.alpha < 1 << 128 and 0 <= rp.alphainv < 1 << 128, "sa_rescue: exponents are below 2^128"
    return values([v for row in rp.MDS for v in row] + list(rp.round_constants[:4 * rp.N]), "constant")


def _upload(eng, block, xs):
    """one upload of a constant block followed by the inputs: (the constant block, the inputs) as device views"""
    buf = eng.upload(sa_devlist.pack(block + xs))
    return buf[:len(block)], buf[len(block):]


def upload_constants(eng, rp):
    """rp's constant block on the device (one upload), for callers that keep it between launches"""
    return _upload(eng, constants(rp), [])[0]


def _elements(rp, raw):
    return sa_marshal.unpack(raw, rp.field, type(rp.round_constants[0]))


def hash_batch(rp, inputs):
    """[rp.hash(x) for x in inputs] from one upload and one launch"""
    block, xs = constants(rp), values(inputs)
    if not xs:
        return []
    eng = sa_engine.get_engine()
    kc, dev = _upload(eng, block, xs)
    hashes = eng.empty(len(xs))
    eng.rescue(dev, kc, rp.N, rp.alpha, rp.alphainv, hashes=hashes)
    return _elements(rp, eng.download(hashes))


def trace_batch(rp, inputs):
    """[rp.trace(x) for x in inputs] (each a list of N + 1 rows [register 0, register 1]) from one upload and one
    launch"""
    block, xs = constants(rp), values(inputs)
    if not xs:
        return []
    eng = sa_engine.get_engine()
    kc, dev = _upload(eng, block, xs)
    rows = rp.N + 1
    trace = eng.empty(len(xs) * 2 * rows)
    eng.rescue(dev, kc, rp.N, rp.alpha, rp.alphainv, trace=trace)
    flat = _elements(rp, eng.download(trace))
    return [[[flat[2 * rows * b + r], flat[2 * rows * b + rows + r]] for r in range(rows)] for b in range(len(xs))]
