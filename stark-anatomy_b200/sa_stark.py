"""sa_stark -- FastStark.prove and Stark.prove on the device: from the trace to the serialized proof through the
planned stages.

The reference's prover (code/fast_stark.py:76-178) interpolates the trace, divides out the boundary and the
transition zerofiers, commits, combines and runs FRI in Python.  ``StarkPlan.prove`` runs the same schedule through
the engine's planned calls, and only roots, challenges and opened leaves cross to the host:

  1. the trace randomizers are drawn with the caller's ``field.sample(os.urandom(17))``, in the reference's order;
  2. the columns are packed and uploaded once, and one batched ``interp_apply`` gives the trace polynomials;
  3. ``boundary_quotients`` gives each register's quotient and codeword, and raises the reference's remainder
     message when a boundary value is false;
  4. ``air_quotients`` divides every transition constraint at the order the reference divides it at (one AIR plan
     per order), and the divisions the reference refuses are refused with its messages;
  5. the randomizer polynomial is drawn where the reference draws it, its codeword is written next to the boundary
     codewords, and one ``merkle_trees`` call commits all of them;
  6. the weights come from the caller's ``prover_fiat_shamir()``; the degree check reads one coefficient per
     constraint; one ``coset_combine_evaluate`` gives the combined codeword;
  7. the drop-in ``Fri.prove`` runs on that codeword where it lies;
  8. the openings are one gather and one path read for the boundary and randomizer codewords, and the zerofier
     codeword's own.

The proof bytes are the reference's (DESIGN section 3.9 gives the argument), or an AssertionError: inputs this
schedule cannot decide exactly are refused rather than proven differently.

``PlainStarkPlan.prove`` is the same schedule for stark.py's plain prover (Stark.prove, stark.py:73-170, and so
RPSSS.sign): the stages above are shared code, the transition quotients come from ``air_quotients_exact``, whose
per-constraint flag is exactly the reference's exact-division test (DESIGN section 3.10), and there are no zerofier
openings.

``prove_batch`` proves many statements of one plan's AIR in one call: the stages before FRI run once for the whole
batch (one interpolation, one boundary apply, one transition apply per division order, one commitment, one
combination into one codeword per proof, one gather and one path read for all openings), FRI runs per proof, and each
proof is the bytes ``prove`` gives from the same draws (DESIGN section 3.11); ``prove`` is ``prove_batch`` of one.
``sign_batch`` signs many documents with one key on an RPSSS or FastRPSSS instance; ``SignerPlan`` keeps a signer's
AIR, plan and Rescue constants and signs under many keys per call, each key's trace computed on the device straight
into the prover's column buffer (DESIGN section 3.14).

With a 32-byte ``seed`` per proof (``prove(..., seed=)``, ``prove_batch(..., seeds=)``, ``sign_batch(..., seeds=)``)
the randomizers are expanded from the seed on the device (``sample_seeded``, DESIGN section 3.13) and nothing calls
os.urandom: the proof is the one the unseeded prover gives with os.urandom = ``seeded_urandom(seed)``.

``enable(cls)`` rebinds ``cls.prove`` (FastStark's) to ``prove``, ``enable_plain(cls)`` rebinds Stark's to
``prove_plain``; ``disable()`` restores both.  Off by default, as ``sa_accel``.  Nothing here imports torch or holds
device state outside a plan.
"""
import hashlib
import itertools
import os
import pickle
from hashlib import blake2b

import sa_host
import sa_engine
import sa_devlist
import sa_marshal
import sa_rescue
import fri as _fri

P = sa_engine.P
FieldElement = sa_host.algebra.FieldElement
REMAINDER = sa_engine.REMAINDER
DEGREE_MISMATCH = "transition quotient degrees do not match with expectation"      # fast_stark.py:127
LARGER_DEGREE = "cannot divide by polynomial of larger degree"                     # ntt.py:145
ZERO_DIVISOR = "cannot divide by zero polynomial"                                  # ntt.py:140
LONG_DIVISION_BELOW = 8  # ntt.py:152: below this degree the reference divides by long division


def _bits(x):
    """the number of binary digits FastStark counts for x: len(bin(x)) without its two-character prefix"""
    return max(1, x.bit_length()) if x >= 0 else x.bit_length() + 1


def _terms(constraint):
    """a constraint's (exponent tuple, int coefficient) pairs, from an MPolynomial or an {exponent tuple: value}
    dict, with zero coefficients kept (FastStark's degree bounds count them)"""
    return [(tuple(int(e) for e in k), int(getattr(v, "value", v)) % P)
            for k, v in getattr(constraint, "dictionary", constraint).items()]


def _term_degree(k, trace_degree):
    """degree of a term's numerator with x of degree 1 and every trace row of degree trace_degree"""
    return sum(e * (1 if i == 0 else trace_degree) for i, e in enumerate(k))


def _ints(values):
    return [int(getattr(v, "value", v)) for v in values]


def _value(lo, hi):
    """the residue of one element's two 64-bit limbs (signed or unsigned, as the engine returns them)"""
    return (int(lo) & 0xFFFFFFFFFFFFFFFF) | (int(hi) & 0xFFFFFFFFFFFFFFFF) << 64


def _tree_fits(eng, k):
    """whether the engine's subproduct tree takes k points; an engine without the query takes every k up to its
    MAX_DIRECT_POINTS"""
    fits = getattr(eng, "tree_fits", None)
    return fits(k) if fits is not None else k <= eng.MAX_DIRECT_POINTS


def _degree(values):
    d = -1
    for i, v in enumerate(values):
        if v:
            d = i
    return d


def _seeds(seeds, count):
    """None, or the list of one 32-byte ``bytes`` seed (a list or tuple) for each of `count` proofs"""
    assert seeds is None or (isinstance(seeds, (list, tuple)) and len(seeds) == count and
                             all(isinstance(s, bytes) and len(s) == 32 for s in seeds)), \
        "sa_stark: seeds must be a list of one 32-byte bytes object per proof"
    return None if seeds is None else list(seeds)


def seeded_urandom(seed):
    """os.urandom for one seeded proof: the n-th call returns blake2b(seed || n as 8 little-endian bytes)'s first 17
    bytes, the draw the device expands for draw n (DESIGN section 3.13).  With os.urandom replaced by it, the unseeded
    prover (or the reference's own prove) gives the seeded proof's bytes.  Only os.urandom(17) is served."""
    assert isinstance(seed, bytes) and len(seed) == 32, "sa_stark: a seed is 32 bytes"
    counter = itertools.count()

    def urandom(n):
        assert n == 17, "sa_stark: seeded_urandom serves the provers' 17-byte draws only, not %r bytes" % (n,)
        return blake2b(seed + next(counter).to_bytes(8, "little")).digest()[:17]
    return urandom


class Params:
    """What FastStark.__init__ derives from its arguments, with its degree bounds and weight sampling, restated from
    the reference's behaviour so that a prove needs no reference checkout; ``fri`` is a drop-in ``fri.Fri``."""

    def __init__(self, field, expansion_factor, num_colinearity_checks, security_level, num_registers, num_cycles,
                 transition_constraints_degree=2):
        assert len(bin(field.p)) - 2 >= security_level, "p must have at least as many bits as security level"
        assert expansion_factor & (expansion_factor - 1) == 0, "expansion factor must be a power of 2"
        assert expansion_factor >= 4, "expansion factor must be 4 or greater"
        assert num_colinearity_checks * 2 >= security_level, \
            "number of colinearity checks must be at least half of security level"
        self.field = field
        self.expansion_factor = expansion_factor
        self.num_colinearity_checks = num_colinearity_checks
        self.security_level = security_level
        self.num_randomizers = 4 * num_colinearity_checks
        self.num_registers = num_registers
        self.original_trace_length = num_cycles
        self.randomized_trace_length = num_cycles + self.num_randomizers
        self.omicron_domain_length = 1 << _bits(self.randomized_trace_length * transition_constraints_degree)
        self.fri_domain_length = self.omicron_domain_length * expansion_factor
        self.generator = field.generator()
        self.omega = field.primitive_nth_root(self.fri_domain_length)
        self.omicron = field.primitive_nth_root(self.omicron_domain_length)
        self.fri = _fri.Fri(self.generator, self.omega, self.fri_domain_length, expansion_factor,
                            num_colinearity_checks)

    def transition_degree_bounds(self, transition_constraints):
        trace_degree = self.original_trace_length + self.num_randomizers - 1
        return [max(_term_degree(k[:1 + 2 * self.num_registers], trace_degree) for k, _ in _terms(a))
                for a in transition_constraints]

    def transition_quotient_degree_bounds(self, transition_constraints):
        return [d - (self.original_trace_length - 1) for d in self.transition_degree_bounds(transition_constraints)]

    def max_degree(self, transition_constraints):
        return (1 << _bits(max(self.transition_quotient_degree_bounds(transition_constraints)))) - 1

    def boundary_quotient_degree_bounds(self, randomized_trace_length, boundary):
        """randomized_trace_length - 1 minus each register's number of boundary points (its zerofier's degree)"""
        if any(all(r != s for _, r, _ in boundary) for s in range(self.num_registers)):
            raise IndexError("list index out of range")  # the reference's zerofier_domain of no points
        return [randomized_trace_length - 1 - sum(1 for _, r, _ in boundary if r == s)
                for s in range(self.num_registers)]

    def sample_weights(self, number, randomness):
        return [self.field.sample(blake2b(randomness + bytes(i)).digest()) for i in range(number)]


class _Constraint:
    __slots__ = ("index", "degree", "bound", "top", "kind", "order")


class _Stages:
    """The stages FastStark's and Stark's provers share (fast_stark.py:82-106, 116-125, 129-169; stark.py:79-104,
    113-123, 127-167): the trace randomizers and one batched interpolation (over the subproduct tree's plan up to its
    cap, the geometric plan of (omicron, T) above it), the boundary quotients into the first nregs rows of the
    commitment buffer, the randomizer polynomial next to them and one commitment of all nregs + 1 codewords, the
    weights, the combination, FRI on the device codeword and the openings of the committed codewords.  A plan sets
    stark, fri, nregs, ncycles, trace_length, log_n, max_degree and interp."""

    def _setup(self, stark, n):
        """fri (the drop-in Fri of the FRI domain of n points) and interp (the randomized trace domain's plan)"""
        eng = sa_engine.get_engine()
        fri = getattr(stark, "fri", None)
        self.fri = fri if isinstance(fri, _fri.Fri) else _fri.Fri(
            stark.generator, stark.omega, n, stark.expansion_factor, stark.num_colinearity_checks)
        omicron = stark.omicron.value
        if _tree_fits(eng, self.trace_length):
            domain = [FieldElement(pow(omicron, i, P), stark.field) for i in range(self.trace_length)]
            self.interp = eng.interp_plan(eng.upload(sa_devlist.pack(domain)))
        else:
            # above the tree's cap the domain's closed forms: no list of points (DESIGN section 3.12)
            self.interp = eng.geo_interp_plan(omicron, self.trace_length)

    def _trace_polynomials(self, eng, traces, seeds=None, columns=None):
        """every proof's trace randomizers, drawn proof by proof and row by row in the reference's order (the
        callers' lists are not touched), one upload of all columns and one batched interpolation: the (B nregs, T, 2)
        trace polynomials, proof b's register s in row b nregs + s.  With `seeds` (the (B, 32) device seeds) only the
        callers' rows are uploaded, and one sample_seeded launch writes row k of register s of proof b as draw
        k nregs + s of seed b (DESIGN section 3.13).  With `columns`, the (B nregs, T, 2) column buffer whose first
        ncycles rows are already filled on the device, no trace element is uploaded: only its randomizer rows are
        written, from the same draws"""
        stark, field, nregs, T = self.stark, self.stark.field, self.nregs, self.trace_length
        ncycles, nrand = self.ncycles, stark.num_randomizers
        if columns is None:
            for trace in traces:
                assert len(trace) == self.ncycles, \
                    "sa_stark: a trace of %d rows, the plan is for %d cycles" % (len(trace), self.ncycles)
            if seeds is None:
                values = []
                for trace in traces:
                    rows = list(trace) + [[field.sample(os.urandom(17)) for s in range(nregs)]
                                          for k in range(nrand)]
                    values += [rows[c][s] for s in range(nregs) for c in range(T)]
                columns = eng.upload(sa_devlist.pack(values)).reshape(len(traces) * nregs, T, 2)
            else:
                values = [trace[c][s] for trace in traces for s in range(nregs) for c in range(ncycles)]
                columns = eng.empty(len(traces) * nregs * T).reshape(len(traces) * nregs, T, 2)
                columns[:, :ncycles] = eng.upload(sa_devlist.pack(values)).reshape(len(traces) * nregs, ncycles, 2)
        elif seeds is None:
            B = columns.shape[0] // nregs
            draws = [[field.sample(os.urandom(17)) for s in range(nregs)] for b in range(B) for k in range(nrand)]
            values = [draws[b * nrand + k][s] for b in range(B) for s in range(nregs) for k in range(nrand)]
            columns[:, ncycles:] = eng.upload(sa_devlist.pack(values)).reshape(B * nregs, nrand, 2)
        if seeds is not None:
            eng.sample_seeded(columns, seeds, 0, nrand * nregs, width=nregs, lane_stride=T, seed_stride=nregs * T,
                              offset=ncycles)
        if isinstance(self.interp, sa_engine.GeoInterpPlan):
            return eng.geo_interp_apply(self.interp, columns)
        return eng.interp_apply(self.interp, columns)

    def _boundary(self, eng, polys, boundaries, failed):
        """(the (B, nregs + 1, n, 2) commitment buffer with each proof's boundary codewords in its first rows, the
        boundary quotients, each proof's degree bounds) from one boundary plan of B nregs registers, register
        b nregs + s being proof b's register s; a proof whose boundary value is false gets the reference's remainder
        message in `failed`.  None when the plan of all boundaries is refused (``_refused`` finds the proof)."""
        stark, nregs, log_n, B = self.stark, self.nregs, self.log_n, len(boundaries)
        n = 1 << log_n
        merged = [(c, b * nregs + int(r), v) for b, boundary in enumerate(boundaries) for c, r, v in boundary]
        try:
            bplan = eng.boundary_plan(merged, B * nregs, stark.omicron, log_n, stark.omega.value,
                                      stark.generator.value)
        except AssertionError:
            return None
        committed = eng.empty(B * (nregs + 1) << log_n).reshape(B, nregs + 1, n, 2)
        # a proof's rows are contiguous in the buffer, so a batch of one writes its codewords there directly
        bquot, bcw, flags = eng.boundary_quotients(bplan, polys, check=False,
                                                   out=committed[0, :nregs] if B == 1 else None)
        if B > 1:
            committed[:, :nregs] = bcw.reshape(B, nregs, n, 2)
        flags = flags.tolist()
        for b in range(B):
            bad = [s for s in range(nregs) if flags[b * nregs + s]]
            if bad:
                failed.setdefault(b, sa_engine.SaError("%s (registers %s)" % (REMAINDER, bad)))
        bounds = bplan.degree_bounds(self.trace_length)
        return committed, bquot, [bounds[b * nregs:(b + 1) * nregs] for b in range(B)]

    def _refused(self, eng, boundaries):
        """the lowest proof whose own boundary plan is refused, and its exception"""
        stark = self.stark
        for b, boundary in enumerate(boundaries):
            try:
                eng.boundary_plan(boundary, self.nregs, stark.omicron, self.log_n, stark.omega.value,
                                  stark.generator.value)
            except AssertionError as e:
                return b, e
        raise AssertionError("sa_stark: the boundary plan of the batch was refused, and no proof's own")

    def _randomizers(self, count):
        """the randomizer polynomials of the first `count` proofs, drawn proof by proof where the reference draws
        each proof's"""
        field = self.stark.field
        return [[field.sample(os.urandom(17)) for i in range(self.max_degree + 1)] for b in range(count)]

    def _seeded_randomizers(self, eng, seeds):
        """the (B, max_degree + 1, 2) randomizer polynomials from one sample_seeded launch: coefficient i of proof b
        is draw num_randomizers nregs + i of seed b, the draw after its trace randomizers"""
        width = self.max_degree + 1
        rvec = eng.empty(seeds.shape[0] * width).reshape(seeds.shape[0], width, 2)
        eng.sample_seeded(rvec, seeds, self.stark.num_randomizers * self.nregs, width)
        return rvec

    def _commit(self, eng, committed, rvec, proof_streams):
        """every proof's randomizer codeword from the (B, max_degree + 1, 2) randomizers `rvec` in its last row of the
        buffer (one batched coset_evaluate), one commitment of all B (nregs + 1) rows, and each proof's roots pushed in
        order into its stream: the trees"""
        stark, nregs, log_n, B = self.stark, self.nregs, self.log_n, rvec.shape[0]
        if B == 1:
            eng.coset_evaluate(rvec[0], log_n, stark.omega.value, stark.generator.value, out=committed[0, nregs])
        else:
            committed[:, nregs] = eng.coset_evaluate(rvec, log_n, stark.omega.value, stark.generator.value)
        trees = eng.merkle_trees(committed.reshape(B * (nregs + 1), 1 << log_n, 2))
        roots = eng.tree_roots(trees)
        for b, ps in enumerate(proof_streams):
            for root in roots[b * (nregs + 1):(b + 1) * (nregs + 1)]:
                ps.push(root)
        return trees

    def _weights(self, proof_stream):
        """1 + 2 ncons + 2 nregs weights from the caller's prover_fiat_shamir()"""
        number = 1 + 2 * len(self.constraints) + 2 * self.nregs
        return [w.value for w in self.stark.sample_weights(number, proof_stream.prover_fiat_shamir())]

    def _combine_prove_open(self, eng, rvec, rows, bquot, bounds_b, weights, committed, trees, proof_streams,
                            fri_batch=False):
        """for each proof b the combination of its randomizer, each transition quotient row (rows[b]: (the row
        truncated to its bound + 1, the bound)) and each boundary quotient at shift 0 and at max_degree - bound, all
        B codewords from one call; FRI on each proof's codeword, proof by proof, or with fri_batch on all B rows of
        the combination at once (Fri.prove_batch); then one gather and one path read of every proof's committed
        codewords at that proof's own indices.  An empty row (a zero quotient) adds nothing and is left out.
        Returns each proof's quadrupled indices."""
        stark, field, nregs, log_n, B = self.stark, self.stark.field, self.nregs, self.log_n, len(proof_streams)
        n = 1 << log_n
        terms = []
        for b in range(B):
            w = weights[b]
            terms.append((rvec[b], 0, w[0], b))
            for c, (q, bound) in enumerate(rows[b]):
                if bound >= 0:
                    terms += [(q, 0, w[1 + 2 * c], b), (q, self.max_degree - bound, w[2 + 2 * c], b)]
            base = 1 + 2 * len(rows[b])
            for s, bound in enumerate(bounds_b[b]):
                q = bquot[b * nregs + s, :bound + 1]
                terms += [(q, 0, w[base + 2 * s], b), (q, self.max_degree - bound, w[base + 2 * s + 1], b)]
        args = (log_n, stark.omega.value, stark.generator.value)
        # a batch of one is the single-codeword call: nrows = 1 of the same kernel
        if B == 1:
            combined = eng.coset_combine_evaluate([t[:3] for t in terms], *args).reshape(1, n, 2)
        else:
            combined = eng.coset_combine_evaluate_batch(terms, B, *args)

        if fri_batch:
            tops = self.fri.prove_batch(combined, proof_streams, field)
        else:
            tops = [self.fri.prove(sa_devlist.DeviceCodeword(combined[b], None, field, n), ps)
                    for b, ps in enumerate(proof_streams)]
        quadrupled = []
        for indices in tops:
            duplicated = list(indices) + [(i + stark.expansion_factor) % n for i in indices]
            quadrupled.append(sorted(duplicated + [(i + n // 2) % n for i in duplicated]))
        # each proof's distinct indices, padded with its last one to a common length
        distinct = [sorted(set(q)) for q in quadrupled]
        width = max(len(d) for d in distinct)
        distinct = [d + d[-1:] * (width - len(d)) for d in distinct]
        rows2d = committed.reshape(B * (nregs + 1), n, 2)
        if B == 1:
            raw = eng.gather_batch(rows2d, distinct[0])
            paths = eng.merkle_open_batch(trees, quadrupled[0])
        else:
            raw = eng.gather_batch(rows2d, distinct, group=nregs + 1)
            paths = eng.merkle_open_batch(trees, quadrupled, group=nregs + 1)
        for b, ps in enumerate(proof_streams):
            for r in range(b * (nregs + 1), (b + 1) * (nregs + 1)):
                # a repeated index pushes the same element object, as indexing one list does; every path is its own
                values = dict(zip(distinct[b], sa_marshal.unpack(raw[r], field, FieldElement)))
                for q, i in enumerate(quadrupled[b]):
                    ps.push(values[i])
                    ps.push(paths[r][q])
        return quadrupled

    def _prove_batch(self, traces, boundaries, proof_streams, transition, seeds=None, columns=None, fri_batch=False):
        """the schedule both provers share: (the proof streams, each proof's quadrupled indices).  transition(eng,
        polys, failed, B) runs the plan's transition quotients and their checks for every proof not yet in `failed`
        and returns (rows_of, degree_check): rows_of(b) gives proof b's combination rows, degree_check(eng, live,
        failed) checks the proofs below `live`.  With `seeds` (one 32-byte seed per proof) every draw comes from the
        device expansion of its proof's seed and nothing calls os.urandom.  With `columns` (the (B nregs, T, 2)
        device column buffer with every proof's trace in its first ncycles rows) `traces` is None.  fri_batch runs FRI
        on the whole batch at once (_combine_prove_open)."""
        B = len(traces) if columns is None else len(boundaries)
        seeds = _seeds(seeds, B)
        eng = sa_engine.get_engine()
        assert len(boundaries) == B, "sa_stark: %d traces and %d boundaries" % (B, len(boundaries))
        if proof_streams is None:
            proof_streams = [sa_host.ip.ProofStream() for b in range(B)]
        assert len(proof_streams) == B, "sa_stark: %d traces and %d proof streams" % (B, len(proof_streams))
        if B == 0:
            return [], []

        seeds_dev = None if seeds is None else eng.upload_seeds(seeds)
        polys = self._trace_polynomials(eng, traces, seeds_dev, columns)
        failed = {}  # proof -> the exception proving it alone raises first
        stage = self._boundary(eng, polys, boundaries, failed)
        if stage is None:
            # a boundary the plan refuses: the proofs before the lowest such proof run as a batch of their own
            b, exc = self._refused(eng, boundaries)
            self._prove_batch(None if columns is not None else traces[:b], boundaries[:b], proof_streams[:b],
                              transition, None if seeds is None else seeds[:b],
                              None if columns is None else columns[:b * self.nregs], fri_batch)
            exc.proof_index = b
            raise exc
        committed, bquot, bounds_b = stage
        rows_of, degree_check = transition(eng, polys, failed, B)

        # the proofs before the lowest failed one go on: their randomizers, and their degree checks
        live = min(failed) if failed else B
        if seeds is None:
            randomizers = self._randomizers(live)
        if not failed:
            if seeds is None:
                rvec = eng.upload(sa_devlist.pack([r for rs in randomizers for r in rs]))
                rvec = rvec.reshape(B, self.max_degree + 1, 2)
            else:
                rvec = self._seeded_randomizers(eng, seeds_dev)
            trees = self._commit(eng, committed, rvec, proof_streams)
            weights = [self._weights(ps) for ps in proof_streams]
        degree_check(eng, live, failed)
        if failed:
            b = min(failed)
            failed[b].proof_index = b
            raise failed[b]

        quadrupled = self._combine_prove_open(eng, rvec, [rows_of(b) for b in range(B)], bquot, bounds_b, weights,
                                              committed, trees, proof_streams, fri_batch)
        return proof_streams, quadrupled


class StarkPlan(_Stages):
    """What does not change between proofs of one AIR on one FastStark (or ``Params``): the interpolation plan of
    the randomized trace domain, one AIR plan per division order with the zerofier uploaded once, and the
    constraints' degrees, bounds and shifts.  Only read by ``prove``."""

    def __init__(self, stark, transition_constraints, transition_zerofier):
        eng = sa_engine.get_engine()
        self.stark = stark
        field = stark.field
        nregs = stark.num_registers
        self.nregs = nregs
        self.ncycles = stark.original_trace_length
        self.trace_length = self.ncycles + stark.num_randomizers
        odl, n = stark.omicron_domain_length, stark.fri_domain_length
        self.log_n = n.bit_length() - 1
        omicron = stark.omicron.value
        T = self.trace_length
        self._setup(stark, n)

        zerofier = _ints(getattr(transition_zerofier, "coefficients", transition_zerofier))
        zdeg = _degree(zerofier)
        assert zdeg >= 0, ZERO_DIVISOR
        # the bounds subtract original_trace_length - 1 where the quotients' lengths subtract deg Z: the two agree
        # only for the zerofier FastStark.preprocess builds
        assert zdeg == self.ncycles - 1, \
            "sa_stark: the transition zerofier has degree %d, not original_trace_length - 1 = %d" % (zdeg, self.ncycles - 1)

        self.constraints = list(transition_constraints)
        self.cons = []
        for c, a in enumerate(self.constraints):
            terms = [(k, v) for k, v in _terms(a)]
            if any(len(k) > 1 + 2 * nregs for k, _ in terms):
                raise AssertionError(sa_engine.SA_ERRORS[-6])
            k = _Constraint()
            k.index = c
            degs = [_term_degree(e, T - 1) for e, _ in terms]
            k.degree = max(degs)  # ValueError for a constraint without terms, as the reference's max()
            k.bound = k.degree - (self.ncycles - 1)
            k.top = [(e, v) for (e, v), d in zip(terms, degs) if d == k.degree]
            if k.degree < zdeg:
                k.kind, k.order = "larger", None
            elif k.degree < LONG_DIVISION_BELOW:
                # long division in the reference: a clean quotient is the coset quotient at any order above the
                # degree; the whole row is read to check the division is clean
                k.kind, k.order = "long", 1 << max(_bits(k.degree), (T - 1).bit_length())
            else:
                assert k.degree < odl, "sa_stark: transition constraint %d has degree %d, at or above the omicron " \
                    "domain's length %d (the reference's transform aliases there)" % (c, k.degree, odl)
                order = odl
                while k.degree < order // 2:
                    order //= 2
                assert order >= T, "sa_stark: transition constraint %d divides at order %d, below the randomized " \
                    "trace length %d" % (c, order, T)
                k.kind, k.order = "transform", order
            self.cons.append(k)
        bounds = [k.bound for k in self.cons]
        self.max_degree = (1 << _bits(max(bounds))) - 1

        # one AIR plan per division order, the zerofier uploaded once
        self.zerofier = eng.upload(sa_devlist.pack([FieldElement(v, field) for v in zerofier[:zdeg + 1]]))
        self.groups = []  # (order, AirPlan, constraint indices, qlen)
        for order in sorted({k.order for k in self.cons if k.order is not None}):
            idx = [k.index for k in self.cons if k.order == order]
            long = self.cons[idx[0]].kind == "long"
            plan = eng.air_plan([self.constraints[c] for c in idx], nregs, self.zerofier, T, order.bit_length() - 1,
                                pow(omicron, odl // order, P), stark.generator.value, omicron)
            self.groups.append((order, plan, idx, order if long else max(self.cons[c].bound for c in idx) + 1))

    def _where(self):
        """constraint index -> (its group, its row in the group)"""
        return {c: (g, j) for g, (_, _, idx, _) in enumerate(self.groups) for j, c in enumerate(idx)}

    def _top_coefficient(self, k, tops):
        """the coefficient of x^degree in constraint k's numerator: its maximal-degree terms on the trace
        polynomials' top coefficients (a next-row variable's top coefficient carries omicron^(T - 1))"""
        nregs = self.nregs
        shift = pow(self.stark.omicron.value, self.trace_length - 1, P)
        acc = 0
        for e, v in k.top:
            t = v
            for i, x in enumerate(e[1:]):
                if x:
                    top = tops[i] if i < nregs else tops[i - nregs] * shift % P
                    t = t * pow(top, x, P) % P
            acc += t
        return acc % P

    def prove(self, trace, boundary, transition_zerofier_codeword, proof_stream=None, seed=None):
        """FastStark.prove(trace, constraints, boundary, zerofier, zerofier_codeword, proof_stream) for this plan's
        constraints and zerofier: proof_stream.serialize().  It is prove_batch of one; `seed` (32 bytes) draws the
        randomizers from its device expansion instead of os.urandom."""
        return self.prove_batch([trace], [boundary], transition_zerofier_codeword,
                                None if proof_stream is None else [proof_stream], None if seed is None else [seed])[0]

    def prove_batch(self, traces, boundaries, transition_zerofier_codeword, proof_streams=None, seeds=None,
                    fri_batch=False):
        """FastStark.prove for each (traces[b], boundaries[b], proof_streams[b]) with this plan's constraints and
        zerofier, the pre-FRI stages of all proofs in one schedule: the list of proof bytes, proof b's the bytes
        proving it alone gives from the same draws (DESIGN section 3.11 gives the draw order).  The exception is the
        one proving the proofs one at a time in order raises first, with the failing proof's index as
        ``proof_index``.  With `seeds`, one 32-byte seed per proof, proof b's draws are the device expansion of
        seeds[b] (DESIGN section 3.13): its bytes are those proving it alone with os.urandom = seeded_urandom(seeds[b])
        gives, whatever the batch.  With fri_batch, FRI runs on all proofs at once (Fri.prove_batch: one host wait per
        round for the whole batch) and the proofs are the same bytes."""
        return self._prove(list(traces), list(boundaries), transition_zerofier_codeword, proof_streams, seeds,
                           fri_batch=fri_batch)

    def _prove(self, traces, boundaries, transition_zerofier_codeword, proof_streams, seeds, columns=None,
               fri_batch=False):
        """prove_batch, or with `columns` (traces None) the proofs of the traces already in that column buffer"""
        T, nregs = self.trace_length, self.nregs
        where = self._where()

        def transition(eng, polys, failed, B):
            # transition quotients (:108-113), each constraint at the order the reference divides it at
            tops = [_value(lo, hi) for lo, hi in eng.gather_batch(polys, [T - 1]).reshape(B * nregs, 2).tolist()]
            batched = polys if B == 1 else polys.reshape(B, nregs, T, 2)
            quots = [eng.air_quotients(plan, batched, qlen) for _, plan, _, qlen in self.groups]
            quots = [q.reshape((B,) + tuple(q.shape[-3:])) for q in quots]
            long_rows = {}
            for b in range(B):
                for k in self.cons:
                    if b in failed:
                        break
                    # a non-zero top coefficient makes the numerator's degree k.degree, so the reference's order is
                    # k.order
                    if not self._top_coefficient(k, tops[b * nregs:(b + 1) * nregs]):
                        failed[b] = AssertionError("sa_stark: the numerator of transition constraint %d is below its "
                                                   "degree bound %d; its division order cannot be decided exactly"
                                                   % (k.index, k.degree))
                    elif k.kind == "larger":
                        failed[b] = AssertionError(LARGER_DEGREE)
                    elif k.kind == "long":
                        g, j = where[k.index]
                        if g not in long_rows:  # one download of the group's rows for every proof
                            long_rows[g] = sa_marshal.unpack(eng.download(quots[g].reshape(-1, 2)), self.stark.field,
                                                             FieldElement)
                        qlen, ng = self.groups[g][3], len(self.groups[g][2])
                        at = (b * ng + j) * qlen
                        if any(v.value for v in long_rows[g][at + k.bound + 1:at + qlen]):
                            failed[b] = AssertionError(REMAINDER)

            def degree_check(eng, live, failed):
                # the degree check (:127): each quotient's coefficient at its bound is non-zero
                for g, (_, _, idx, qlen) in enumerate(self.groups):
                    if self.cons[idx[0]].kind == "transform" and live:
                        at = [(b * len(idx) + j) * qlen + self.cons[c].bound for b in range(live)
                              for j, c in enumerate(idx)]
                        vals = eng.gather_batch(quots[g].reshape(1, -1, 2), at).reshape(-1, 2).tolist()
                        for b in range(live):
                            chunk = vals[b * len(idx):(b + 1) * len(idx)]
                            if not all(int(lo) or int(hi) for lo, hi in chunk):
                                failed.setdefault(b, AssertionError(DEGREE_MISMATCH))

            def rows_of(b):
                return [(quots[where[k.index][0]][b, where[k.index][1], :k.bound + 1], k.bound) for k in self.cons]
            return rows_of, degree_check

        streams, quadrupled = self._prove_batch(traces, boundaries, proof_streams, transition, seeds, columns,
                                                fri_batch)

        # ... and the zerofier's openings (:171-175), proof by proof: the codeword is the caller's
        zc = transition_zerofier_codeword
        for ps, quad in zip(streams, quadrupled):
            if isinstance(zc, sa_devlist.DeviceCodeword):
                zc.prefetch(quad)
                zpaths = zc.open_paths(quad)
            else:
                tree = _fri.Merkle._device_tree(zc)
                zpaths = ([_fri.Merkle.open(i, zc) for i in quad] if tree is None or len(zc) < 2
                          else sa_engine.get_engine().merkle_open(tree, quad))
            for q, i in enumerate(quad):
                ps.push(zc[i])
                ps.push(zpaths[q])
        return [ps.serialize() for ps in streams]


def prove(stark, trace, transition_constraints, boundary, transition_zerofier, transition_zerofier_codeword,
          proof_stream=None):
    """FastStark.prove's signature and result through a StarkPlan built for this one call (no plan is cached)"""
    plan = StarkPlan(stark, transition_constraints, transition_zerofier)
    return plan.prove(trace, boundary, transition_zerofier_codeword, proof_stream)


class PlainStarkPlan(_Stages):
    """What does not change between proofs of one AIR on one Stark (stark.py's plain prover): the interpolation plan
    of the randomized trace domain, the transition zerofier built on the device over omicron^0 .. omicron^(ncycles -
    2) (Stark has no preprocess; by the tree up to its cap, by geo_zerofier above), one AIR plan per division order,
    and the constraints' bounds.  Stark keeps neither the omicron domain's nor the FRI domain's length as attributes:
    they come from len(stark.omicron_domain) and stark.fri.domain_length.  Only read by ``prove``.

    The reference divides each transition numerator by Polynomial.__truediv__, an exact division, so the division
    order never changes its result: constraint c (numerator degree bound D_c, T the randomized trace length) divides
    at 2^max(bits(D_c), bits(T - 1)) with an exact-division flag, and a flag raises the remainder message.  Refused
    with an AssertionError rather than proven otherwise: a division order above 2^30, a combination of max_degree + 1
    coefficients above the FRI domain (the reference evaluates it there, but it does not fold), and the boundary
    lists the boundary plan refuses."""

    def __init__(self, stark, transition_constraints):
        eng = sa_engine.get_engine()
        self.stark = stark
        field = stark.field
        nregs = stark.num_registers
        self.nregs = nregs
        self.ncycles = stark.original_trace_length
        self.trace_length = T = self.ncycles + stark.num_randomizers
        n = stark.fri.domain_length
        self.log_n = n.bit_length() - 1
        omicron = stark.omicron.value
        self._setup(stark, n)

        self.constraints = list(transition_constraints)
        zdeg = self.ncycles - 1
        self.bounds, orders = [], []
        for c, a in enumerate(self.constraints):
            terms = _terms(a)
            if any(len(k) > 1 + 2 * nregs for k, _ in terms):
                raise AssertionError(sa_engine.SA_ERRORS[-6])
            degree = max(_term_degree(e, T - 1) for e, _ in terms)  # ValueError without terms, as the reference's
            self.bounds.append(degree - zdeg)
            order = 1 << max(_bits(degree), _bits(T - 1))
            assert order <= 1 << 30, "sa_stark: transition constraint %d has degree %d; its division order %d is " \
                "above 2^30" % (c, degree, order)
            orders.append(order)
        self.max_degree = (1 << _bits(max(self.bounds))) - 1
        assert self.max_degree + 1 <= n, "sa_stark: the combination has max_degree + 1 = %d coefficients, above " \
            "the FRI domain's %d" % (self.max_degree + 1, n)

        # the zerofier of omicron^0 .. omicron^(ncycles - 2) on the device; none for one cycle, where the reference's
        # transition_zerofier raises IndexError at the division (prove raises it there)
        self.groups = []  # (AirPlan, constraint indices, qlen)
        if self.ncycles < 2:
            return
        if _tree_fits(eng, self.ncycles - 1):
            points = [FieldElement(pow(omicron, i, P), field) for i in range(self.ncycles - 1)]
            self.zerofier = eng.zerofier(eng.upload(sa_devlist.pack(points)))
        else:
            self.zerofier = eng.geo_zerofier(omicron, self.ncycles - 1)
        for order in sorted(set(orders)):
            idx = [c for c, o in enumerate(orders) if o == order]
            plan = eng.air_plan([self.constraints[c] for c in idx], nregs, self.zerofier, T, order.bit_length() - 1,
                                field.primitive_nth_root(order).value, stark.generator.value, omicron)
            self.groups.append((plan, idx, max(1, max(self.bounds[c] for c in idx) + 1)))

    def prove(self, trace, boundary, proof_stream=None, seed=None):
        """Stark.prove(trace, constraints, boundary, proof_stream) for this plan's constraints:
        proof_stream.serialize().  It is prove_batch of one; `seed` as StarkPlan.prove's."""
        return self.prove_batch([trace], [boundary], None if proof_stream is None else [proof_stream],
                                None if seed is None else [seed])[0]

    def prove_batch(self, traces, boundaries, proof_streams=None, seeds=None, fri_batch=False):
        """Stark.prove for each (traces[b], boundaries[b], proof_streams[b]) with this plan's constraints, the
        pre-FRI stages of all proofs in one schedule: the list of proof bytes, proof b's the bytes proving it alone
        gives from the same draws (DESIGN section 3.11).  The exception is the one proving the proofs one at a time
        in order raises first, with the failing proof's index as ``proof_index``.  `seeds` as
        StarkPlan.prove_batch's, and fri_batch as there."""
        return self._prove(list(traces), list(boundaries), proof_streams, seeds, fri_batch=fri_batch)

    def _prove(self, traces, boundaries, proof_streams, seeds, columns=None, fri_batch=False):
        """prove_batch, or with `columns` (traces None) the proofs of the traces already in that column buffer"""
        T, nregs = self.trace_length, self.nregs

        def transition(eng, polys, failed, B):
            # transition quotients (stark.py:107-111): exact divisions, the remainder message before the randomizer
            # is drawn
            if not self.groups:  # zerofier_domain of no points (univariate.py:123)
                for b in range(B):
                    failed.setdefault(b, IndexError("list index out of range"))
                return None, lambda eng, live, failed: None
            batched = polys if B == 1 else polys.reshape(B, nregs, T, 2)
            quots, flags = [], []
            for plan, _, qlen in self.groups:
                q, f = eng.air_quotients_exact(plan, batched, qlen, check=False)
                quots.append(q.reshape((B,) + tuple(q.shape[-3:])))
                flags.append(f.reshape(B, -1).tolist())
            for b in range(B):
                for f in flags:
                    bad = [j for j, x in enumerate(f[b]) if x]
                    if bad:
                        failed.setdefault(b, sa_engine.SaError("%s (constraints %s)" % (REMAINDER, bad)))
                        break

            def degree_check(eng, live, failed):
                # the degree check (:125).  A clean row U_c vanishes above deg N_c - deg Z <= b_c, so the quotient
                # has degree b_c exactly when U_c[b_c] != 0.  For b_c < 0, deg N_c <= D_c < deg Z and Z | N_c force
                # N_c = 0: the quotient is Polynomial([]), of degree -1 (univariate.py:8-9, 83-84), which matches
                # b_c = -1 only.
                ok = [all(c >= -1 for c in self.bounds)] * live
                for g, (_, idx, qlen) in enumerate(self.groups):
                    js = [j for j, c in enumerate(idx) if self.bounds[c] >= 0]
                    if js and live:
                        at = [(b * len(idx) + j) * qlen + self.bounds[idx[j]] for b in range(live) for j in js]
                        vals = eng.gather_batch(quots[g].reshape(1, -1, 2), at).reshape(-1, 2).tolist()
                        for b in range(live):
                            ok[b] = ok[b] and all(int(lo) or int(hi) for lo, hi in vals[b * len(js):(b + 1) * len(js)])
                for b in range(live):
                    if not ok[b]:
                        failed.setdefault(b, AssertionError(DEGREE_MISMATCH))

            def rows_of(b):
                rows = [None] * len(self.constraints)
                for g, (_, idx, _) in enumerate(self.groups):
                    for j, c in enumerate(idx):
                        rows[c] = (quots[g][b, j, :max(0, self.bounds[c] + 1)], self.bounds[c])
                return rows
            return rows_of, degree_check

        streams, _ = self._prove_batch(traces, boundaries, proof_streams, transition, seeds, columns, fri_batch)
        return [ps.serialize() for ps in streams]


def prove_plain(stark, trace, transition_constraints, boundary, proof_stream=None):
    """Stark.prove's signature and result through a PlainStarkPlan built for this one call (no plan is cached)"""
    return PlainStarkPlan(stark, transition_constraints).prove(trace, boundary, proof_stream)


def sign_batch(signer, sk, documents, seeds=None, fri_batch=False):
    """For an RPSSS or FastRPSSS instance `signer`, [signer.sign(sk, d) for d in documents]: each signature is the
    one signer.sign gives from the same draws, taken in prove_batch's order (signing draws nothing outside its
    prove).  The hash, the trace, the boundary and the transition constraints are computed once, one plan proves
    every document (PlainStarkPlan for a Stark, StarkPlan with the signer's zerofier for a FastStark), and each
    document's stream is the signer module's own SignatureProofStream.  Nothing is kept between calls.  With
    `seeds`, one secret 32-byte seed per document, signature d is signer.sign(sk, documents[d]) with os.urandom =
    seeded_urandom(seeds[d]); a seed must never sign two different documents (DESIGN section 3.13).  fri_batch as
    StarkPlan.prove_batch's."""
    import sys
    documents = list(documents)
    seeds = _seeds(seeds, len(documents))
    if not documents:
        return []
    rp, stark = signer.rp, signer.stark
    output = rp.hash(sk)
    trace = rp.trace(sk)
    transition = rp.transition_constraints(stark.omicron)
    boundary = rp.boundary_constraints(output)
    stream = sys.modules[type(signer).__module__].SignatureProofStream
    streams = [stream(d) for d in documents]
    if hasattr(signer, "transition_zerofier"):
        plan = StarkPlan(stark, transition, signer.transition_zerofier)
        return plan.prove_batch([trace] * len(documents), [boundary] * len(documents),
                                signer.transition_zerofier_codeword, streams, seeds, fri_batch)
    plan = PlainStarkPlan(stark, transition)
    return plan.prove_batch([trace] * len(documents), [boundary] * len(documents), streams, seeds, fri_batch)


class SignerPlan:
    """What does not change between signatures of an RPSSS or FastRPSSS instance `signer`: its transition
    constraints (rp.transition_constraints, built once), the PlainStarkPlan for a Stark or the StarkPlan with the
    signer's zerofier for a FastStark, and the device copy of its Rescue constants (sa_rescue).  ``sign`` signs any
    number of (key, document) pairs per call, and a plan serves any number of calls (DESIGN section 3.14)."""

    def __init__(self, signer):
        import sys
        rp, stark = signer.rp, signer.stark
        assert stark.original_trace_length == rp.N + 1 and stark.num_registers == 2, \
            "sa_stark: the signer's Stark proves %d cycles of %d registers, not the %d rows of 2 of its Rescue trace" \
            % (stark.original_trace_length, stark.num_registers, rp.N + 1)
        self.rp, self.stark = rp, stark
        self.constants = sa_rescue.upload_constants(sa_engine.get_engine(), rp)
        transition = rp.transition_constraints(stark.omicron)
        self.transition = transition
        if hasattr(signer, "transition_zerofier"):
            self.plan = StarkPlan(stark, transition, signer.transition_zerofier)
            self.zerofier_codeword = signer.transition_zerofier_codeword
            self.zerofier_root = getattr(signer, "transition_zerofier_root", None)
        else:
            self.plan = PlainStarkPlan(stark, transition)
            self.zerofier_codeword = self.zerofier_root = None
        self.stream = sys.modules[type(signer).__module__].SignatureProofStream
        self._verifier = None

    def sign(self, sks, documents, seeds=None, fri_batch=False):
        """[signer.sign(sks[d], documents[d]) for each d]: one sa_rescue launch writes every key's trace into rows
        0 .. N of the prover's column buffer, the public keys are read from row N of register 0 with one gather, and
        the batch is proven as prove_batch proves it, each document with its own SignatureProofStream.  No trace
        element crosses to the device.  Unseeded, the draws are taken in prove_batch's order; with `seeds`, one
        secret 32-byte seed per signature, signature d is signer.sign(sks[d], documents[d]) with os.urandom =
        seeded_urandom(seeds[d]), whatever the batch.  Unequal lengths, bad seeds and keys that are not elements of p
        raise an AssertionError before any device work.  fri_batch as StarkPlan.prove_batch's."""
        sks, documents = list(sks), list(documents)
        assert len(sks) == len(documents), "sa_stark: %d keys and %d documents" % (len(sks), len(documents))
        seeds = _seeds(seeds, len(documents))
        keys = sa_rescue.values(sks, "secret key")
        if not keys:
            return []
        eng = sa_engine.get_engine()
        rp, plan, B, N, T = self.rp, self.plan, len(keys), self.rp.N, self.plan.trace_length
        columns = eng.empty(B * 2 * T).reshape(B * 2, T, 2)
        eng.rescue(eng.upload(sa_devlist.pack(keys)), self.constants, N, rp.alpha, rp.alphainv, trace=columns,
                   inst_stride=2 * T, lane_stride=T)
        pks = eng.gather_batch(columns.reshape(1, B * 2 * T, 2), [b * 2 * T + N for b in range(B)])
        element = type(rp.round_constants[0])
        boundaries = [rp.boundary_constraints(element(_value(lo, hi), rp.field)) for lo, hi in pks.reshape(B, 2)]
        streams = [self.stream(d) for d in documents]
        if self.zerofier_codeword is not None:
            return plan._prove(None, boundaries, self.zerofier_codeword, streams, seeds, columns, fri_batch)
        return plan._prove(None, boundaries, streams, seeds, columns, fri_batch)


    def verify(self, pks, documents, signatures, reasons=False):
        """[signer.verify(pks[d], documents[d], signatures[d]) for each d] in one VerifierPlan.verify_batch call: the
        boundary of rp.boundary_constraints(pk) and each document's SignatureProofStream, the verifier plan built on
        the first call and kept"""
        pks, documents, signatures = list(pks), list(documents), list(signatures)
        assert len(pks) == len(documents) == len(signatures), \
            "sa_stark: %d keys, %d documents and %d signatures" % (len(pks), len(documents), len(signatures))
        assert self.zerofier_codeword is None or self.zerofier_root is not None, \
            "sa_stark: the FastStark signer has no transition_zerofier_root to verify against"
        if self._verifier is None:
            self._verifier = VerifierPlan(self.stark, self.transition, self.zerofier_root)
        return self._verifier.verify_batch(signatures, [self.rp.boundary_constraints(pk) for pk in pks],
                                           [self.stream(d) for d in documents], reasons)


# ---- verification (DESIGN section 3.15) ----
FRI_MESSAGES = {"a": "merkle authentication path verification fails for aa",     # fri.py:214-224
                "b": "merkle authentication path verification fails for bb",
                "c": "merkle authentication path verification fails for cc"}
LAST_FORM = "last codeword is not well formed"                                     # fri.py:148
COLINEAR = "colinearity check failure"                                             # fri.py:208
MALFORMED = "malformed"
CHUNK_BYTES = 1 << 30  # one chunk's device buffers, as coset_batch_max bounds a coset call's
SECTIONS = ("roots", "leaves", "leaf_index", "depth", "digests", "path_offset", "ay", "by", "cy", "alpha", "items",
            "proof_data", "last", "a_index", "round")  # _pack's order; sa_transcript_sections writes them in it
# The device route reads a call's proofs when at least this many of them can take it.  Its fixed cost is one thread
# parsing a whole proof (about 35 ms for a 1.1-1.3 MB signature), so below this count the host route is faster:
# per signature, host / device route, FastRPSSS 13.2 / 13.8 ms at 4 and 12.5 / 9.7 ms at 6, RPSSS 8.6 / 10.1 ms
# at 4 and 8.7 / 7.3 ms at 6 (H100 80GB HBM3 at a 700 W limit, tools/stark_verify.py, DESIGN section 3.17).
DEVICE_ROUTE_MIN_PROOFS = 6
TRANSCRIPT_PREFIX, TRANSCRIPT_OUT = 144, 80  # include/sa_b200.h's per-proof prefix and out strides
_transcripts_checked = {}  # (shape, FieldElement class, pickle protocol) -> whether the stand-in check passed


def _xor_exponent(e):
    """the exponent FieldElement.__xor__ (algebra.py:38-45) applies for an int e: e itself from 0 on; for a negative
    e its bits over len(bin(e)) - 2 positions of the two's complement"""
    return e if e >= 0 else e & ((1 << (len(bin(e)) - 2)) - 1)


def _lagrange(xs, ys):
    """Polynomial.interpolate_domain's coefficients (univariate.py:107-120), low to high, with inverse(0) = 0"""
    acc = [0] * len(xs)
    for j, (xj, yj) in enumerate(zip(xs, ys)):
        basis, den = [1], 1
        for m, xm in enumerate(xs):
            if m != j:
                basis = [((basis[t - 1] if t else 0) - xm * (basis[t] if t < len(basis) else 0)) % P
                         for t in range(len(basis) + 1)]
                den = den * (xj - xm) % P
        f = yj * pow(den, P - 2, P) % P
        for t, b in enumerate(basis):
            acc[t] = (acc[t] + f * b) % P
    return acc


def _is_element(v):
    return type(v).__name__ == "FieldElement" and type(getattr(v, "value", None)) is int and 0 <= v.value < P


def _is_digest(d):
    return type(d) is bytes and len(d) == 64


def _is_path(path, depth):
    return type(path) is list and len(path) == depth and all(_is_digest(d) for d in path)


class _Refused(AssertionError):
    """a statement VerifierPlan does not take (DESIGN section 3.15); enable_verify hands it to the original verify"""


class _Parsed:
    """one proof's transcript: what the host reads and derives, and the device items it contributes"""
    __slots__ = ("weights", "fri_roots", "alphas", "last", "top_indices", "top", "triples", "fri_paths", "opened",
                 "statement")


class VerifierPlan:
    """What does not change between verifications of one AIR: the FRI parameters, the compiled AIR program, the
    transition quotients' shifts and, for a plain Stark, its transition zerofier on the device.  With a
    `transition_zerofier_root` the plan verifies FastStark proofs (FastStark.verify, fast_stark.py:180-286; `stark`
    a FastStark or a ``Params``), without one plain ones (Stark.verify, stark.py:172-275), the zerofier of omicron^0
    .. omicron^(ncycles - 2) built as PlainStarkPlan builds it.

    A verdict is the reference's for every proof whose stream has the reference's shape: the number of objects the
    verifier pulls, 64-byte ``bytes`` roots, a last codeword of FieldElements of the length FRI gives, 3-tuples of
    elements for the FRI leaves, lists of 64-byte digests of the tree's depth for paths and elements for opened
    leaves.  A proof outside that shape is False (reason "malformed").  Everything but unpickling, Fiat-Shamir (the
    stream's own verifier_fiat_shamir), the weights and the index sampling runs on the device (DESIGN section
    3.15)."""

    def __init__(self, stark, transition_constraints, transition_zerofier_root=None):
        eng = sa_engine.get_engine()
        self.stark = stark
        self.constraints = list(transition_constraints)
        self.zerofier_root = transition_zerofier_root
        self.nregs = stark.num_registers
        fri = stark.fri
        self.fri = fri
        self.n = fri.domain_length
        self.log_n = self.n.bit_length() - 1
        self.ef = fri.expansion_factor
        self.k = fri.num_colinearity_tests
        self.rounds = fri.num_rounds()
        self.last_len = self.n >> (self.rounds - 1)
        if not 1 <= self.nregs <= 16:
            raise _Refused("sa_stark: the verifier takes 1 to 16 registers, not %d" % self.nregs)
        if 1 << self.log_n != self.n or not 1 <= self.log_n <= 30:
            raise _Refused("sa_stark: a FRI domain of %d points" % self.n)
        self.prog = eng.air_program(self.constraints, self.nregs)
        self.max_degree = stark.max_degree(self.constraints)
        self.tshifts = [_xor_exponent(self.max_degree - b)
                        for b in stark.transition_quotient_degree_bounds(self.constraints)]
        if not all(0 <= s < 1 << 32 for s in self.tshifts):
            raise _Refused("sa_stark: a transition shift at or above 2^32")
        self.zcoef = None
        if transition_zerofier_root is None:
            ncycles = stark.original_trace_length
            if ncycles < 2:
                raise _Refused("sa_stark: a plain Stark of one cycle has no transition zerofier")
            omicron = stark.omicron.value
            if _tree_fits(eng, ncycles - 1):
                points = [FieldElement(pow(omicron, i, P), stark.field) for i in range(ncycles - 1)]
                self.zcoef = eng.zerofier(eng.upload(sa_devlist.pack(points)))
            else:
                self.zcoef = eng.geo_zerofier(omicron, ncycles - 1)
        self._statements = {}
        self.transcript = None
        self.transcript = self._transcript_setup(eng)

    # -- the statement of one boundary: its zerofiers, interpolants and shifts (fast_stark.py:53-67, 272-277) --
    def _statement(self, boundary):
        key = tuple((int(c), int(r), int(getattr(v, "value", v))) for c, r, v in boundary)
        st = self._statements.get(key)
        if st is not None:
            return st
        stark, nregs = self.stark, self.nregs
        rtl = 1 + max(c for c, _, _ in key) + stark.num_randomizers
        omicron = stark.omicron.value
        zs, its = [], []
        for s in range(nregs):
            pts = [(pow(omicron, c, P), v % P) for c, r, v in key if r == s]
            if not pts:
                raise AssertionError("cannot interpolate between zero points")  # univariate.py:109
            z = [1]
            for x, _ in pts:
                z = [((z[t - 1] if t else 0) - x * (z[t] if t < len(z) else 0)) % P for t in range(len(z) + 1)]
            zs.append(z)
            its.append(_lagrange([x for x, _ in pts], [v for _, v in pts]))
        bshifts = [_xor_exponent(self.max_degree - (rtl - 1 - (len(z) - 1))) for z in zs]
        if not all(0 <= s < 1 << 32 for s in bshifts):
            raise _Refused("sa_stark: a boundary shift at or above 2^32")
        blen = max(len(z) for z in zs)
        coef = []
        for z, i in zip(zs, its):
            coef += z + [0] * (blen - len(z)) + i + [0] * (blen - len(i))
        st = (blen, self.tshifts + bshifts, coef)
        self._statements[key] = st
        return st

    # -- one proof's transcript, in the reference's pull order; None outside the shape --
    def _parse(self, proof, boundary, proof_stream):
        stark, fri, nregs, k, rounds, n = self.stark, self.fri, self.nregs, self.k, self.rounds, self.n
        max(c for c, _, _ in boundary)  # fast_stark.py:184: the trace length first (ValueError without points)
        try:
            ps = (proof_stream if proof_stream is not None else sa_host.ip.ProofStream()).deserialize(proof)
        except Exception:
            return None
        objects = getattr(ps, "objects", None)
        nopen = nregs + 1 + (self.zerofier_root is not None)
        top = 2 * k if rounds > 1 else 0
        count = nregs + 1 + rounds + 1 + (rounds - 1) * 4 * k + nopen * 2 * 2 * top
        if type(objects) is not list or len(objects) < count:
            return None
        pr = _Parsed()
        roots = [ps.pull() for _ in range(nregs + 1)]
        # the boundary's interpolants and zerofiers after the roots' pulls (fast_stark.py:192-201), with their
        # exceptions
        pr.statement = self._statement(boundary)
        if not all(_is_digest(r) for r in roots):
            return None
        W = 1 + 2 * len(self.constraints) + 2 * nregs
        pr.weights = [w.value for w in stark.sample_weights(W, ps.verifier_fiat_shamir())]
        pr.fri_roots, pr.alphas = [], []
        for r in range(rounds):
            pr.fri_roots.append(ps.pull())
            pr.alphas.append(stark.field.sample(ps.verifier_fiat_shamir()).value)
        if not all(_is_digest(r) for r in pr.fri_roots):
            return None
        last = ps.pull()
        if type(last) is not list or len(last) != self.last_len or not all(_is_element(v) for v in last):
            return None
        pr.last = last
        pr.top_indices = fri.sample_indices(ps.verifier_fiat_shamir(), n >> 1, n >> (rounds - 1), k) \
            if rounds > 1 else []
        pr.triples, pr.fri_paths = [], []
        for r in range(rounds - 1):
            triples = [ps.pull() for _ in range(k)]
            if not all(type(t) is tuple and len(t) == 3 and all(_is_element(v) for v in t) for t in triples):
                return None
            paths = [ps.pull() for _ in range(3 * k)]
            depth = self.log_n - r
            if not all(_is_path(p, depth - (q % 3 == 2)) for q, p in enumerate(paths)):
                return None
            pr.triples.append(triples)
            pr.fri_paths.append(paths)
        # the combination's indices: FRI's round-0 a and b indices, sorted (fast_stark.py:205-211)
        half = n >> 1
        values = sorted([(i % half, pr.triples[0][s][0]) for s, i in enumerate(pr.top_indices)] +
                        [(i % half + half, pr.triples[0][s][1]) for s, i in enumerate(pr.top_indices)],
                        key=lambda iv: iv[0]) if top else []
        dup = sorted([i for i, _ in values] + [(i + self.ef) % n for i, _ in values])
        pr.opened = []  # (root, [(index, leaf, path)])
        for root in roots + ([self.zerofier_root] if self.zerofier_root is not None else []):
            reads = []
            for i in dup:
                leaf, path = ps.pull(), ps.pull()
                if not _is_element(leaf) or not _is_path(path, self.log_n):
                    return None
                reads.append((i, leaf, path))
            pr.opened.append((root, reads))
        pr.top = values
        return pr

    # -- the packed buffer of a chunk: every section 16-byte aligned --
    def _pack(self, parsed):
        import numpy as np
        nregs, k, rounds = self.nregs, self.k, self.rounds
        roots, leaves, idx, depth, digests, poff = [], [], [], [], [], []
        ay, by, cy, aidx, alpha, rnd = [], [], [], [], [], []
        items, pdata, last = [], [], []
        blen = max(pr.statement[0] for pr in parsed)
        ncons = len(self.constraints)
        ktop = len(parsed[0].top)

        def path(root, i, leaf, p):
            roots.append(root)
            leaves.append(leaf)
            idx.append(i)
            depth.append(len(p))
            poff.append(len(digests))
            digests.extend(p)
        for pr in parsed:
            # FRI round r (fri.py:180-224): c = a = top index mod n / 2^(r+1), b = a + n / 2^(r+1); c opens in the
            # next round's tree
            for r in range(rounds - 1):
                half = self.n >> (r + 1)
                for s, t in enumerate(pr.triples[r]):
                    a = pr.top_indices[s] % half
                    ay.append(t[0])
                    by.append(t[1])
                    cy.append(t[2])
                    aidx.append(a)
                    alpha.append(pr.alphas[r])
                    rnd.append(r)
                for s, t in enumerate(pr.triples[r]):
                    a = pr.top_indices[s] % half
                    ps3 = pr.fri_paths[r][3 * s:3 * s + 3]
                    path(pr.fri_roots[r], a, t[0], ps3[0])
                    path(pr.fri_roots[r], a + half, t[1], ps3[1])
                    path(pr.fri_roots[r + 1], a, t[2], ps3[2])
            for root, reads in pr.opened:
                for i, leaf, p in reads:
                    path(root, i, leaf, p)
            blen_p, shifts, coef = pr.statement
            pdata += pr.weights + shifts
            per = 2 * blen_p
            for s in range(nregs):
                z = coef[s * per:s * per + blen_p]
                it = coef[s * per + blen_p:(s + 1) * per]
                pdata += z + [0] * (blen - blen_p) + it + [0] * (blen - blen_p)
            values = {}
            for root_no, (root, reads) in enumerate(pr.opened):
                for i, leaf, p in reads:
                    values[(root_no, i)] = leaf  # a repeated index keeps the last leaf pulled, as the dict does
            for i, v in pr.top:
                j = (i + self.ef) % self.n
                items += [i, v] + [values[(s, i)] for s in range(nregs)] + [values[(s, j)] for s in range(nregs)]
                items += [values[(nregs, i)], values[(nregs + 1, i)] if self.zerofier_root is not None else 0]
            last += pr.last
        sections, L, size = [], {}, 0

        def add(name, raw):
            nonlocal size
            raw = bytes(raw)
            L[name] = size
            pad = (-len(raw)) % 16
            sections.append(raw + bytes(pad))
            size += len(raw) + pad
        add("roots", b"".join(roots))
        add("leaves", sa_marshal.pack(leaves))
        add("leaf_index", np.array(idx, dtype=np.uint64).tobytes())
        add("depth", np.array(depth, dtype=np.uint32).tobytes())
        add("digests", b"".join(digests))
        add("path_offset", np.array(poff, dtype=np.uint64).tobytes())
        for name, vals in (("ay", ay), ("by", by), ("cy", cy), ("alpha", alpha), ("items", items),
                           ("proof_data", pdata), ("last", last)):
            add(name, sa_marshal.pack(vals))
        add("a_index", np.array(aidx, dtype=np.uint64).tobytes())
        add("round", np.array(rnd, dtype=np.uint32).tobytes())
        self._constants(L, len(idx), len(ay), len(parsed), ktop, blen)
        return b"".join(sections), L

    def _constants(self, L, npath, ncol, nproofs, ktop, blen):
        """the layout's counts and the plan's constants verify_chunk reads beside the section offsets"""
        stark = self.stark
        L.update(paths=npath, colinear=ncol, proofs=nproofs, k=ktop, last_len=self.last_len,
                 fri_offset=self.fri.offset.value, fri_omega=self.fri.omega.value, prog=self.prog,
                 ncons=len(self.constraints), nregs=self.nregs, blen=blen, offset=stark.generator.value,
                 omega=stark.omega.value, log_n=self.log_n, ef=self.ef, zcoef=self.zcoef,
                 last_omega=pow(self.fri.omega.value, 1 << (self.rounds - 1), P))

    def _decide(self, last_root, mflags, cflags, kflags, degree, root):
        """the reference's verdict from one proof's device flags, checks in the reference's order: (verdict, reason,
        whether the zerofier vanished at the failing index); last_root is the proof's last FRI root"""
        k, rounds = self.k, self.rounds
        if root != last_root:
            return False, LAST_FORM
        bound = self.last_len // self.ef - 1
        if degree > bound:
            return False, ("last codeword does not correspond to polynomial of low enough degree\n"
                           "observed degree: %d\nbut should be: %d" % (degree, bound))
        m = 0
        for r in range(rounds - 1):
            for s in range(k):
                if cflags[r * k + s]:
                    return False, COLINEAR
            for q in range(3 * k):
                if mflags[m + q]:
                    return False, FRI_MESSAGES["abc"[q % 3]]
            m += 3 * k
        if any(mflags[m:]):
            return False, "leaf path"
        for f in kflags:
            if f == 2:
                raise AssertionError("divide by zero")  # algebra.py:92
            if f:
                return False, "combination"
        return True, None

    def _bytes(self, pr):
        """the device bytes one proof takes in a chunk: its packed sections, its flags and its last codeword's tree,
        inverse transform, degree and root"""
        npath = (self.rounds - 1) * 3 * self.k + sum(len(reads) for _, reads in pr.opened)
        ndigest = sum(len(p) for paths in pr.fri_paths for p in paths) + sum(
            len(p) for _, reads in pr.opened for _, _, p in reads)
        blen, shifts, _ = pr.statement
        return self._section_bytes(npath, ndigest, len(pr.top), len(pr.weights) + len(shifts) + 2 * self.nregs * blen)

    def _section_bytes(self, npath, ndigest, ntop, ndata):
        ncol = (self.rounds - 1) * self.k
        nitems = ntop * (4 + 2 * self.nregs)
        return (npath * (64 + 16 + 8 + 4 + 8 + 4) + 64 * ndigest + ncol * (4 * 16 + 8 + 4 + 4) +
                16 * (nitems + ndata) + 4 * ntop + self.last_len * (16 + 128 + 16) + 8 + 64 + 11 * 16)

    def _chunks(self, parsed):
        """runs of consecutive proofs whose device buffers (_bytes) stay within CHUNK_BYTES; a proof above the bound
        on its own is a chunk of its own"""
        chunks, cur, used = [], [], 0
        for b, pr in parsed:
            size = self._bytes(pr)
            if cur and used + size > CHUNK_BYTES:
                chunks.append(cur)
                cur, used = [], 0
            cur.append((b, pr))
            used += size
        return chunks + ([cur] if cur else [])

    def verify_batch(self, proofs, boundaries, proof_streams=None, reasons=False):
        """The reference's verdict for each (proofs[b], boundaries[b], proof_streams[b]) (each proof's stream
        deserializes it, so a SignatureProofStream's prefix enters its Fiat-Shamir): a list of bool, or with
        `reasons` of (bool, reason) pairs, the reason None for an accepted proof, else the message the reference
        prints for the first failing check (its three lines for the last codeword's degree), "leaf path" for an
        opened leaf's path, "combination" for the combination and "malformed" for a stream outside the shape.  A
        zero transition zerofier value at a checked index raises the reference's AssertionError("divide by zero")
        with the proof's index as ``proof_index``, as verifying the proofs one at a time in order would.

        A proof whose bytes are the canonical pickle of a stream of the plan's shape, with a stream whose Fiat-Shamir
        the device replays, is read on the device (the device route, DESIGN section 3.17) when the call has at least
        DEVICE_ROUTE_MIN_PROOFS such proofs; every other proof is unpickled and packed on the host.  Both routes give
        the same verdicts and exceptions."""
        proofs, boundaries = list(proofs), list(boundaries)
        B = len(proofs)
        assert len(boundaries) == B, "sa_stark: %d proofs and %d boundaries" % (B, len(boundaries))
        streams = [None] * B if proof_streams is None else list(proof_streams)
        assert len(streams) == B, "sa_stark: %d proofs and %d proof streams" % (B, len(streams))
        eng = sa_engine.get_engine()
        decided = self._verify_on_device(eng, proofs, boundaries, streams)  # b -> verdict or exception
        out = [None] * B
        parsed = []
        for b in range(B):
            try:
                if b in decided:
                    # what _parse raises for a stream it deserializes with enough objects, in the same order
                    max(c for c, _, _ in boundaries[b])
                    self._statement(boundaries[b])
                    continue
                pr = self._parse(proofs[b], boundaries[b], streams[b])
            except Exception as exc:
                exc.proof_index = b
                raise
            if pr is None:
                out[b] = (False, MALFORMED)
            else:
                parsed.append((b, pr))
        for chunk in self._chunks(parsed):
            raw, L = self._pack([pr for _, pr in chunk])
            mflags, cflags, kflags, degrees, roots = eng.verify_chunk(eng.upload_bytes(raw), L)
            m = c = q = 0
            ktop = L["k"]
            for j, (b, pr) in enumerate(chunk):
                nm = (self.rounds - 1) * 3 * self.k + sum(len(reads) for _, reads in pr.opened)
                nc = (self.rounds - 1) * self.k
                decided[b] = self._outcome(pr.fri_roots[-1], mflags[m:m + nm], cflags[c:c + nc], kflags[q:q + ktop],
                                           degrees[j], roots[64 * j:64 * (j + 1)])
                m, c, q = m + nm, c + nc, q + ktop
        for b in sorted(decided):
            if isinstance(decided[b], BaseException):
                decided[b].proof_index = b
                raise decided[b]
            out[b] = decided[b]
        return out if reasons else [v for v, _ in out]

    def _outcome(self, *args):
        try:
            return self._decide(*args)
        except AssertionError as exc:
            return exc

    # -- the device route (DESIGN section 3.17) --
    def _transcript_counts(self, nopen):
        k, rounds, log_n = self.k, self.rounds, self.log_n
        fri_digests = sum(k * (3 * (log_n - r) - 1) for r in range(rounds - 1))
        path_digests = fri_digests + 4 * nopen * k * log_n
        nroots = self.nregs + 1 + rounds
        nvalues = self.last_len + 3 * (rounds - 1) * k + 4 * nopen * k
        npaths = 3 * (rounds - 1) * k + 4 * nopen * k
        memo = 2 + 3 * (rounds - 1) * k + 4 * nopen * k + (rounds - 1) * k + nroots + path_digests + 2 * nvalues + 10
        return npaths, path_digests, memo

    def _transcript_setup(self, eng):
        """the shape sa_transcript_sections reads this plan's proofs with, or None (the host route only): an engine
        without the entry point, a shape it refuses, or a pickler whose output on a stand-in stream of the shape the
        device does not read, or whose Fiat-Shamir prefixes it does not hash as pickle.dumps writes them"""
        if not hasattr(eng, "transcript_sections") or self.rounds < 2 or self.k > self.last_len:
            return None
        shape = self._transcript_shape()
        if eng.transcript_bytes(shape) == 0:
            return None
        key = (shape, sa_host.algebra.FieldElement, pickle.DEFAULT_PROTOCOL)
        if key not in _transcripts_checked:
            self.transcript = shape
            _transcripts_checked[key] = self._transcript_check(eng)
        return shape if _transcripts_checked[key] else None

    def _transcript_shape(self):
        """include/sa_b200.h's SA_TRANSCRIPT_SHAPE words for this plan at the running pickle protocol"""
        nopen = self.nregs + 1 + (self.zerofier_root is not None)
        W = 1 + 2 * len(self.constraints) + 2 * self.nregs
        return (self.nregs, self.rounds, self.k, self.last_len, self.log_n, nopen, W, pickle.DEFAULT_PROTOCOL,
                self.ef, self._transcript_counts(nopen)[2])

    def _standin(self, seed=0):
        """a stream of the plan's shape with random digests and elements of every int encoding's size"""
        import random
        rng = random.Random(seed)
        field, FE = self.stark.field, sa_host.algebra.FieldElement
        el = lambda: FE(rng.choice([rng.randrange(1 << 8), rng.randrange(1 << 16), rng.randrange(1 << 31),  # noqa
                                    rng.randrange(P)]), field)
        dg = lambda: rng.randbytes(64)  # noqa: E731
        objs = [dg() for _ in range(self.nregs + 1 + self.rounds)] + [[el() for _ in range(self.last_len)]]
        for r in range(self.rounds - 1):
            objs += [(el(), el(), el()) for _ in range(self.k)]
            objs += [[dg() for _ in range(self.log_n - r - (q % 3 == 2))] for q in range(3 * self.k)]
        for _ in range(self.nregs + 1 + (self.zerofier_root is not None)):
            for _ in range(4 * self.k):
                objs += [el(), [dg() for _ in range(self.log_n)]]
        return objs

    def _transcript_check(self, eng):
        """the stand-in's pickle is accepted, and its weights, alphas and indices are the ones the host draws from
        shake_256(pickle.dumps(objects[:j]))"""
        objs = self._standin()
        fs = lambda j: hashlib.shake_256(pickle.dumps(objs[:j])).digest(32)  # noqa: E731
        j0 = self.nregs + 1
        weights = [w.value for w in self.stark.sample_weights(1 + 2 * len(self.constraints) + 2 * self.nregs, fs(j0))]
        alphas = [self.stark.field.sample(fs(j0 + 1 + r)).value for r in range(self.rounds)]
        top = self.fri.sample_indices(fs(j0 + self.rounds + 1), self.n >> 1, self.last_len, self.k)
        stat = (1, [0] * (len(self.constraints) + self.nregs), [0] * (2 * self.nregs))
        raw, parts, L, nstat = self._transcript_chunk([(pickle.dumps(objs), b"", stat)])
        sec, out = eng.transcript_sections(eng.upload_bytes(raw), parts, L, nstat, 1, self.transcript)
        sec, out = sec.cpu().numpy().tobytes(), out.cpu().numpy().tobytes()
        fe = lambda name, n: [int.from_bytes(sec[L[name] + 16 * i:L[name] + 16 * (i + 1)], "little")  # noqa: E731
                              for i in range(n)]
        ncol = (self.rounds - 1) * self.k
        aidx = [int.from_bytes(sec[L["a_index"] + 8 * i:L["a_index"] + 8 * (i + 1)], "little") for i in range(ncol)]
        return (out[0] == 1 and fe("proof_data", len(weights)) == weights and
                fe("alpha", ncol) == [a for a in alphas[:-1] for _ in range(self.k)] and
                aidx == [i % (self.n >> (r + 1)) for r in range(self.rounds - 1) for i in top])

    def _transcript_chunk(self, items):
        """one device chunk's upload (the proofs, their offsets and prefixes, the statements at the chunk's blen and
        the zerofier root), the byte offsets of its parts, the sections' layout L as _pack would give it, and the
        statement elements per proof.  items: (proof bytes, prefix, statement or None)"""
        nregs, k, B = self.nregs, self.k, len(items)
        nopen = nregs + 1 + (self.zerofier_root is not None)
        npaths, path_digests, _ = self._transcript_counts(nopen)
        blen = max([st[0] for _, _, st in items if st is not None], default=1)
        nstat = len(self.constraints) + nregs + 2 * nregs * blen
        proofs, at, prefixes, stat = [], [], [], []
        used = 0
        for proof, prefix, st in items:
            at += [used, len(proof)]
            proofs.append(proof + bytes(-len(proof) % 16))
            used += len(proof) + (-len(proof) % 16)
            prefixes.append(len(prefix).to_bytes(8, "little") + bytes(8) + prefix[:128] +
                            bytes(TRANSCRIPT_PREFIX - 16 - len(prefix[:128])))
            if st is None:
                stat += [0] * nstat
                continue
            blen_p, shifts, coef = st
            stat += shifts
            for s in range(nregs):
                z, it = coef[2 * s * blen_p:(2 * s + 1) * blen_p], coef[(2 * s + 1) * blen_p:(2 * s + 2) * blen_p]
                stat += z + [0] * (blen - blen_p) + it + [0] * (blen - blen_p)
        import numpy as np
        parts = {}
        chunks = []
        for name, raw in (("proofs", b"".join(proofs)), ("proof_at", np.array(at, dtype=np.uint64).tobytes()),
                          ("prefixes", b"".join(prefixes)), ("statement", sa_marshal.pack(stat)),
                          ("zroot", self.zerofier_root or b"")):
            parts[name] = sum(len(c) for c in chunks)
            chunks.append(raw + bytes(-len(raw) % 16))
        W = 1 + 2 * len(self.constraints) + 2 * nregs
        ncol = (self.rounds - 1) * k
        sizes = {"roots": 64 * npaths, "leaves": 16 * npaths, "leaf_index": 8 * npaths, "depth": 4 * npaths,
                 "digests": 64 * path_digests, "path_offset": 8 * npaths, "ay": 16 * ncol, "by": 16 * ncol,
                 "cy": 16 * ncol, "alpha": 16 * ncol, "items": 16 * 2 * k * (4 + 2 * nregs),
                 "proof_data": 16 * (W + nstat), "last": 16 * self.last_len, "a_index": 8 * ncol, "round": 4 * ncol}
        L, size = {}, 0
        for name in SECTIONS:
            L[name] = size
            size += B * sizes[name] + (-B * sizes[name]) % 16
        L["bytes"] = size
        L["section_at"] = [L[name] for name in SECTIONS]
        self._constants(L, B * npaths, B * ncol, B, 2 * k, blen)
        return b"".join(chunks), parts, L, nstat

    @staticmethod
    def _fs_prefix(stream):
        """the bytes the stream's verifier_fiat_shamir hashes before pickle.dumps(objects[:read_index]), or None
        where a stand-in transcript of two objects shows it hashes something else"""
        try:
            q = (stream if stream is not None else sa_host.ip.ProofStream()).deserialize(
                pickle.dumps([bytes(64), bytes(range(64))]))
            q.pull()
            q.pull()
            prefix = getattr(q, "prefix", b"")
            if type(prefix) is not bytes or len(prefix) > 128:
                return None
            if q.verifier_fiat_shamir() != hashlib.shake_256(prefix + pickle.dumps(q.objects[:2])).digest(32):
                return None
            return prefix
        except Exception:
            return None

    def _verify_on_device(self, eng, proofs, boundaries, streams):
        """the device route: {b: verdict or exception} for the proofs the device read; the others are left to the
        host route.  Chunks of consecutive such proofs, each within CHUNK_BYTES, one upload, six transcript launches,
        verify_chunk's ladder and one download each"""
        if self.transcript is None:
            return {}
        nopen = self.nregs + 1 + (self.zerofier_root is not None)
        npaths, path_digests, _ = self._transcript_counts(nopen)
        base = eng.transcript_bytes(self.transcript) + TRANSCRIPT_PREFIX + TRANSCRIPT_OUT + 16
        W = 1 + 2 * len(self.constraints) + 2 * self.nregs
        eligible = []
        for b, proof in enumerate(proofs):
            prefix = self._fs_prefix(streams[b]) if type(proof) is bytes else None
            if prefix is not None:
                eligible.append((b, proof, prefix))
        if len(eligible) < DEVICE_ROUTE_MIN_PROOFS:
            return {}
        chunks, cur, used = [], [], 0
        for b, proof, prefix in eligible:
            try:
                max(c for c, _, _ in boundaries[b])
                st = self._statement(boundaries[b])
            except Exception:
                st = None  # the walk in verify_batch raises it where the host route would
            blen = st[0] if st is not None else 1
            size = len(proof) + base + self._section_bytes(npaths, path_digests, 2 * self.k,
                                                           W + len(self.constraints) + self.nregs + 2 * self.nregs * blen)
            if cur and used + size > CHUNK_BYTES:
                chunks.append(cur)
                cur, used = [], 0
            cur.append((b, proof, prefix, st))
            used += size
        chunks += [cur] if cur else []
        decided = {}
        nm, nc = npaths, (self.rounds - 1) * self.k
        ktop = 2 * self.k
        for chunk in chunks:
            raw, parts, L, nstat = self._transcript_chunk([(p, x, st) for _, p, x, st in chunk])
            sec, out = eng.transcript_sections(eng.upload_bytes(raw), parts, L, nstat, len(chunk), self.transcript)
            mflags, cflags, kflags, degrees, roots, out = eng.verify_chunk(sec, L, extra=out)
            for j, (b, _, _, _) in enumerate(chunk):
                if out[TRANSCRIPT_OUT * j] != 1:
                    continue
                last_root = bytes(out[TRANSCRIPT_OUT * j + 16:TRANSCRIPT_OUT * (j + 1)])
                decided[b] = self._outcome(last_root, mflags[j * nm:(j + 1) * nm], cflags[j * nc:(j + 1) * nc],
                                           kflags[j * ktop:(j + 1) * ktop], degrees[j], roots[64 * j:64 * (j + 1)])
        return decided

    def verify(self, proof, boundary, proof_stream=None):
        """verify_batch of one proof: its bool"""
        return self.verify_batch([proof], [boundary], None if proof_stream is None else [proof_stream])[0]


_originals = {}  # class -> its own `prove` attribute before enable (None: inherited)
_verify_originals = {}  # class -> (its own `verify` attribute before enable_verify (None: inherited), the method)


def enable(cls):
    """rebind cls.prove (FastStark's, or a subclass's) to sa_stark.prove (idempotent)"""
    if cls not in _originals:
        _originals[cls] = cls.__dict__.get("prove")
        cls.prove = prove


def enable_plain(cls):
    """rebind cls.prove (Stark's, or a subclass's) to sa_stark.prove_plain (idempotent), so that RPSSS.sign runs
    unmodified"""
    if cls not in _originals:
        _originals[cls] = cls.__dict__.get("prove")
        cls.prove = prove_plain


def _verify_on_plan(original, make_plan, proof, boundary, proof_stream, args):
    """the plan's verdict, the reference's message printed where it prints one.  A Stark the plan refuses (more
    than 16 registers, a shift at or above 2^32, a plain Stark of one cycle) and a malformed stream go to the
    class's original verify, so its behaviour, exceptions included, is the reference's"""
    try:
        plan = make_plan()  # an AIR the program compiler refuses raises SaError, an AssertionError too
    except AssertionError:
        return original(*args)
    try:
        verdict, reason = plan.verify_batch([proof], [boundary], [proof_stream], reasons=True)[0]
    except _Refused:
        return original(*args)
    if reason == MALFORMED:
        return original(*args)
    if reason is not None and reason not in ("leaf path", "combination"):
        print(reason)
    return verdict


def enable_verify(cls):
    """rebind cls.verify (FastStark's, or a subclass's) to a VerifierPlan built for the call (idempotent), so that
    FastRPSSS.verify runs unmodified; a stream outside the shape is verified by the original method"""
    if cls in _verify_originals:
        return
    original = cls.verify

    def verify(self, proof, transition_constraints, boundary, transition_zerofier_root, proof_stream=None):
        plan = lambda: VerifierPlan(self, transition_constraints, transition_zerofier_root)  # noqa: E731
        return _verify_on_plan(original, plan, proof, boundary, proof_stream,
                               (self, proof, transition_constraints, boundary, transition_zerofier_root,
                                proof_stream))
    _verify_originals[cls] = (cls.__dict__.get("verify"), original)
    cls.verify = verify


def enable_verify_plain(cls):
    """rebind cls.verify (Stark's, or a subclass's) to a plain VerifierPlan built for the call (idempotent), so
    that RPSSS.verify runs unmodified; a stream outside the shape is verified by the original method"""
    if cls in _verify_originals:
        return
    original = cls.verify

    def verify(self, proof, transition_constraints, boundary, proof_stream=None):
        plan = lambda: VerifierPlan(self, transition_constraints)  # noqa: E731
        return _verify_on_plan(original, plan, proof, boundary, proof_stream,
                               (self, proof, transition_constraints, boundary, proof_stream))
    _verify_originals[cls] = (cls.__dict__.get("verify"), original)
    cls.verify = verify


def disable():
    """restore every class enable, enable_plain, enable_verify and enable_verify_plain rebound"""
    for cls, orig in _originals.items():
        if orig is None:
            del cls.prove
        else:
            cls.prove = orig
    _originals.clear()
    for cls, (orig, _) in _verify_originals.items():
        if orig is None:
            del cls.verify
        else:
            cls.verify = orig
    _verify_originals.clear()
