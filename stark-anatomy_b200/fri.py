"""Drop-in for the reference's code/fri.py, backed by the H100 engine.

``from fri import *`` (code/fast_stark.py:1) resolves here when this directory is
ahead of the reference's on sys.path.  It re-exports the names the reference's
fri module exports (algebra, merkle, ip, ntt, univariate names, hexlify,
unhexlify, math, blake2b) and provides ``Fri`` with the reference's constructor,
``num_rounds``, ``sample_index(es)``, ``eval_domain``, ``commit``, ``query``,
``prove`` and ``verify``.

Device flow of ``commit`` (code/fri.py:56-96): the codeword is uploaded once; the
Merkle tree of round 0 is built on the GPU; every later round is ONE fused
kernel (fold + leaf hashing + subtree reduction, ``sa_fri_round``).  Per round a
64-byte root comes back to the host because the challenge is
``field.sample(proof_stream.prover_fiat_shamir())`` on the caller's proof stream
object (possibly a subclass, code/fast_rpsss.py:7-17).  Trees stay on the device
for ``query`` (code/fri.py:98-113), which gathers leaf triples and
authentication paths instead of re-hashing whole layers per opened index.

Pushed objects have the reference's types and object identity structure (root
``bytes``, the last codeword as a ``list`` of ``algebra.FieldElement``, tuples of
the SAME element objects a layer list would hold, ``list[bytes]`` paths), so
``pickle.dumps(proof_stream.objects)`` is byte-identical to the reference's.
"""
import sa_host  # noqa: F401
from algebra import *  # noqa: F401,F403
from merkle import *  # noqa: F401,F403
from ip import *  # noqa: F401,F403
from ntt import *  # noqa: F401,F403
from binascii import hexlify, unhexlify  # noqa: F401
import math  # noqa: F401
from hashlib import blake2b

from univariate import *  # noqa: F401,F403
from univariate import Polynomial, test_colinearity
from algebra import FieldElement
from merkle import Merkle as _HostMerkle
from ntt import intt

import sa_engine
import sa_devlist
from sa_devlist import DeviceCodeword
import sa_marshal


class Merkle(_HostMerkle):
    """code/merkle.py's Merkle with ``commit`` / ``open`` on the GPU for field-element data.

    code/fast_stark.py calls ``Merkle.commit(codeword)`` once and then ``Merkle.open(i, codeword)``
    hundreds of times on the same list (fast_stark.py:105,118,162-174); the reference re-hashes
    every leaf per call (merkle.py:26-27).  Here the packed list is fingerprinted (blake2b of the
    16-byte limbs, on the host) and its device tree is kept in a small cache, so an ``open`` is one
    path gather.  Leaves are blake2b(decimal ASCII of the value) exactly as merkle.py:14 +
    algebra.py:53-57.  Data that is not a list of field elements of p = 1 + 407*2^119 (e.g. the raw
    byte strings of code/test_merkle.py) is outside the engine's domain and goes through the
    caller's own host class unchanged.  ``verify`` / ``verify_`` / ``commit_`` / ``open_`` are the
    host class's (verifier side, digests in and out).
    """

    _trees = {}           # fingerprint -> (engine, device tree), insertion ordered
    _cache_bytes = 0
    _CACHE_LIMIT = 1 << 30

    def _device_tree(data_array):
        if isinstance(data_array, DeviceCodeword):
            # values already in HBM (what ntt / fast_coset_evaluate return): the tree is built once and
            # stays attached to the object -- no pack, no upload, no fingerprint
            n = len(data_array)
            return data_array.device_tree() if n and not n & (n - 1) else None
        n = len(data_array)
        if n == 0 or n & (n - 1):
            return None
        first = data_array[0]
        if not isinstance(first, FieldElement) or first.field.p != sa_engine.P:
            return None
        try:
            packed = sa_devlist.pack(data_array)
        except (TypeError, AttributeError, OverflowError):
            return None
        key = blake2b(packed, digest_size=32).digest()
        eng = sa_engine.get_engine()
        hit = Merkle._trees.get(key)
        if hit is not None and hit[0] is eng:
            return hit[1]
        if hit is not None:  # built by an engine that has since been replaced: its tree is not this engine's
            Merkle._cache_bytes -= 64 * Merkle._trees.pop(key)[1].shape[0]
        tree = eng.merkle_tree(sa_devlist.to_device(packed))
        Merkle._trees[key] = (eng, tree)
        Merkle._cache_bytes += 128 * n
        while Merkle._cache_bytes > Merkle._CACHE_LIMIT and len(Merkle._trees) > 1:
            old = next(iter(Merkle._trees))
            Merkle._cache_bytes -= 64 * Merkle._trees.pop(old)[1].shape[0]
        return tree

    def commit(data_array):
        tree = Merkle._device_tree(data_array)
        if tree is None:
            return _HostMerkle.commit(list(data_array) if isinstance(data_array, DeviceCodeword) else data_array)
        if isinstance(data_array, DeviceCodeword):
            return data_array.root()
        return sa_engine.get_engine().tree_root(tree)

    def open(index, data_array):
        tree = Merkle._device_tree(data_array)
        if tree is None or len(data_array) < 2:
            return _HostMerkle.open(index, list(data_array) if isinstance(data_array, DeviceCodeword) else data_array)
        assert(0 <= index and index < len(data_array)), "cannot open invalid index"
        if isinstance(data_array, DeviceCodeword):
            return data_array.open_paths([index])[0]
        return sa_engine.get_engine().merkle_open(tree, [index])[0]


class Fri:
    def __init__(self, offset, omega, initial_domain_length, expansion_factor, num_colinearity_tests):
        self.offset = offset
        self.omega = omega
        self.domain_length = initial_domain_length
        self.field = omega.field
        self.expansion_factor = expansion_factor
        self.num_colinearity_tests = num_colinearity_tests
        self._resident = {}  # id(list) -> (list, device vector, device tree) of the last commit
        assert(self.num_rounds() >= 1), "cannot do FRI with less than one round"

    # ------------------------------------------------------- host helpers --
    def num_rounds(self):
        """code/fri.py:22-28"""
        codeword_length = self.domain_length
        num_rounds = 0
        while codeword_length > self.expansion_factor and 4 * self.num_colinearity_tests < codeword_length:
            codeword_length /= 2
            num_rounds += 1
        return num_rounds

    def sample_index(byte_array, size):
        """code/fri.py:30-34: big-endian integer of the bytes, reduced mod size"""
        return int.from_bytes(bytes(byte_array), "big") % size

    def sample_indices(self, seed, size, reduced_size, number):
        """code/fri.py:36-51 (bytes(counter) is `counter` zero bytes, as in the reference)"""
        assert(number <= reduced_size), f"cannot sample more indices than available in last codeword; requested: {number}, available: {reduced_size}"
        assert(number <= 2 * reduced_size), "not enough entropy in indices wrt last codeword"
        indices, reduced_indices = [], []
        counter = 0
        while len(indices) < number:
            index = Fri.sample_index(blake2b(seed + bytes(counter)).digest(), size)
            reduced_index = index % reduced_size
            counter += 1
            if reduced_index not in reduced_indices:
                indices += [index]
                reduced_indices += [reduced_index]
        return indices

    def eval_domain(self):
        return [self.offset * (self.omega ^ i) for i in range(self.domain_length)]

    # --------------------------------------------------------------- commit --
    def commit(self, codeword, proof_stream, round_index=0):
        eng = sa_engine.get_engine()
        p = self.field.p
        omega, offset = self.omega.value, self.offset.value
        rounds = self.num_rounds()
        self._resident = {}
        N = len(codeword)
        # make sure omega has the right order (fri.py:68; if it holds for round 0 it holds for
        # every squared omega / halved length after it)
        assert(pow(omega, N - 1, p) == pow(omega, -1, p)), "error in commit: omega does not have the right order!"

        def on_root(r, root, want_alpha):
            # compute and send Merkle root (fri.py:71-72); get challenge (fri.py:79)
            proof_stream.push(root)
            if want_alpha:
                return self.field.sample(proof_stream.prover_fiat_shamir()).value
            return None

        # the whole ladder runs on the device: round 0 = leaf hashing + tree, every later round =
        # one fused kernel (split-and-fold fri.py:85 + leaf hashing + tree); only the 64-byte roots
        # come back, through on_root.  A DeviceCodeword (what fast_coset_evaluate returns) is already
        # in HBM: no pack, no upload.
        vecs, trees = eng.fri_commit(sa_devlist.to_device(codeword), rounds, offset, omega, on_root)

        if isinstance(codeword, DeviceCodeword):
            codeword.attach_tree(trees[0])
        codewords = [codeword] + [DeviceCodeword(vecs[r], trees[r], self.field, N >> r) for r in range(1, rounds)]
        # send last codeword (a real list: it is pickled into the transcript)
        if isinstance(codewords[-1], DeviceCodeword):
            codewords[-1] = codewords[-1].tolist()
        proof_stream.push(codewords[-1])
        for layer, vec, tree in zip(codewords, vecs, trees):
            if not isinstance(layer, DeviceCodeword):
                self._resident[id(layer)] = (layer, vec, tree)
        return codewords

    # ---------------------------------------------------------------- query --
    def _open_layer(self, layer, indices):
        """(values, authentication paths) of a layer at `indices`.  A DeviceCodeword opens its own tree.  A
        plain list is opened with one gather from the tree its last commit built, else from a fresh upload
        and tree: the reference re-hashes the list it is given on every Merkle.open (merkle.py:26-27), so a
        list that was modified in place after commit must not be answered from the tree of its old contents;
        the revealed values are compared with the resident vector and a mismatch drops it."""
        if isinstance(layer, DeviceCodeword):
            layer.prefetch(indices)
            return [layer[i] for i in indices], layer.open_paths(indices)
        eng = sa_engine.get_engine()
        values = [layer[i] for i in indices]
        hit = self._resident.get(id(layer))
        fresh = hit is not None and hit[0] is layer and eng.length(hit[1]) == len(layer)
        if fresh and indices:
            resident = bytes(memoryview(eng.gather(hit[1], indices)).cast("B"))
            fresh = resident == bytes(sa_devlist.pack(values))
        if not fresh:
            vec = sa_devlist.to_device(layer)
            hit = self._resident[id(layer)] = (layer, vec, eng.merkle_tree(vec))
        return values, eng.merkle_open(hit[2], indices)

    def query(self, current_codeword, next_codeword, c_indices, proof_stream):
        # infer a and b indices
        a_indices = [index for index in c_indices]
        b_indices = [index + len(current_codeword) // 2 for index in c_indices]
        k = self.num_colinearity_tests
        s_range = range(k)
        ab = [a_indices[s] for s in s_range] + [b_indices[s] for s in s_range]
        cc = [c_indices[s] for s in s_range]
        cur, cur_paths = self._open_layer(current_codeword, ab)
        nxt, nxt_paths = self._open_layer(next_codeword, cc)

        # reveal leafs
        for s in s_range:
            proof_stream.push((cur[s], cur[k + s], nxt[s]))

        # reveal authentication paths
        for s in s_range:
            proof_stream.push(cur_paths[s])
            proof_stream.push(cur_paths[k + s])
            proof_stream.push(nxt_paths[s])

        return a_indices + b_indices

    # ---------------------------------------------------------------- prove --
    def prove(self, codeword, proof_stream):
        assert(self.domain_length == len(codeword)), "initial codeword length does not match length of initial codeword"

        # commit phase
        codewords = self.commit(codeword, proof_stream)

        # get indices
        top_level_indices = self.sample_indices(proof_stream.prover_fiat_shamir(), len(codewords[0]) // 2, len(codewords[-1]), self.num_colinearity_tests)
        indices = [index for index in top_level_indices]

        # query phase
        for i in range(len(codewords) - 1):
            indices = [index % (len(codewords[i]) // 2) for index in indices]  # fold
            self.query(codewords[i], codewords[i + 1], indices, proof_stream)

        return top_level_indices

    # -------------------------------------------------------------- batches --
    def _commit_batch(self, codewords, proof_streams, field):
        """commit_batch, and the (B, N >> r, 2) device layers and (B, 2 (N >> r), 64) trees of every round"""
        eng = sa_engine.get_engine()
        p = self.field.p
        B = len(proof_streams)
        if hasattr(codewords, "shape"):  # one (B, N, 2) device tensor
            vecs = codewords
            assert len(vecs.shape) == 3 and vecs.shape[0] == B, "fri: %d rows and %d proof streams" % (vecs.shape[0], B)
            N = vecs.shape[1]
            if B == 0:
                return [], [], []
            first = [DeviceCodeword(vecs[b], None, field or self.field, N) for b in range(B)]
        else:
            first = list(codewords)
            assert len(first) == B, "fri: %d codewords and %d proof streams" % (len(first), B)
            N = len(first[0]) if first else 0
            assert all(len(cw) == N for cw in first), "fri: the codewords of a batch differ in length"
            if B == 0:
                return [], [], []
            if any(isinstance(cw, DeviceCodeword) for cw in first):
                vecs = eng.concat([sa_devlist.to_device(cw) for cw in first]).reshape(B, N, 2)
            else:  # one upload
                vecs = eng.upload(bytearray().join(sa_devlist.pack(cw) for cw in first)).reshape(B, N, 2)
        self._resident = {}
        rounds = self.num_rounds()
        assert(pow(self.omega.value, N - 1, p) == pow(self.omega.value, -1, p)), "error in commit: omega does not have the right order!"

        def on_roots(r, roots, want_alpha):
            # stream by stream: its root (fri.py:71-72), then its challenge (fri.py:79)
            alphas = []
            for ps, root in zip(proof_streams, roots):
                ps.push(root)
                if want_alpha:
                    alphas.append(self.field.sample(ps.prover_fiat_shamir()).value)
            return alphas

        layers, trees = eng.fri_commit_batch(vecs, rounds, self.offset.value, self.omega.value, on_roots)
        # every proof's last codeword as a real list (it is pickled into the transcript), from one download; a lone
        # round's last codeword is the caller's own
        if rounds > 1 or hasattr(codewords, "shape"):
            raw = eng.download(layers[-1].reshape(-1, 2)).reshape(B, -1, 2)
            last = [sa_marshal.unpack(raw[b], self.field if rounds > 1 else sa_devlist.field_of(first[b]), FieldElement)
                    for b in range(B)]
        else:
            last = [cw.tolist() if isinstance(cw, DeviceCodeword) else cw for cw in first]
        out = []
        for b, ps in enumerate(proof_streams):
            if isinstance(first[b], DeviceCodeword):
                first[b].attach_tree(trees[0][b])
            cws = [first[b]] + [DeviceCodeword(layers[r][b], trees[r][b], self.field, N >> r) for r in range(1, rounds)]
            cws[-1] = last[b]
            ps.push(cws[-1])
            out.append(cws)
        return out, layers, trees

    def commit_batch(self, codewords, proof_streams, field=None):
        """``commit(codewords[b], proof_streams[b])`` for every b as one batched commit (sa_fri_commit_batch): every
        stream receives the objects ``commit`` pushes, the streams visited in order each round, and one host wait per
        round serves the whole batch.  `codewords` is a list of lists or DeviceCodewords of one length, or one
        (B, N, 2) device tensor whose rows hold elements of `field` (default: this Fri's).  Returns each proof's
        codewords as ``commit`` returns them."""
        return self._commit_batch(codewords, proof_streams, field)[0]

    def prove_batch(self, codewords, proof_streams, field=None):
        """``prove(codewords[b], proof_streams[b])`` for every b: each stream receives exactly the objects ``prove``
        pushes (so ``pickle.dumps(ps.objects)`` is the same), with the commit of ``commit_batch`` and, per layer, one
        gather and one path read for the whole batch.  Inputs as ``commit_batch`` takes them.  Returns each proof's
        top-level indices."""
        eng = sa_engine.get_engine()
        B = len(proof_streams)
        if hasattr(codewords, "shape"):
            assert(codewords.shape[1] == self.domain_length), "initial codeword length does not match length of initial codeword"
        else:
            for cw in codewords:
                assert(self.domain_length == len(cw)), "initial codeword length does not match length of initial codeword"
        if B == 0:
            return []
        cws, layers, trees = self._commit_batch(codewords, proof_streams, field)
        rounds = len(cws[0])
        N, k = self.domain_length, self.num_colinearity_tests
        tops = [self.sample_indices(ps.prover_fiat_shamir(), N // 2, len(cws[b][-1]), k)
                for b, ps in enumerate(proof_streams)]
        if rounds == 1:
            return tops
        # the c indices of every query round (fri.py:116), then each layer's openings: c of the round before it, a and
        # b of its own round
        cs = [[[i % ((N >> r) // 2) for i in top] for top in tops] for r in range(rounds - 1)]
        sets = []
        for r in range(rounds):
            sets.append([(cs[r - 1][b] if r else []) + (cs[r][b] + [i + (N >> r) // 2 for i in cs[r][b]]
                                                        if r < rounds - 1 else []) for b in range(B)])
        values, paths = [], []
        for r in range(rounds):
            paths.append(eng.merkle_open_batch(trees[r], sets[r], group=1))
            if r == rounds - 1:  # the pushed last codewords' own elements
                values.append([[cws[b][r][i] for i in sets[r][b]] for b in range(B)])
                continue
            raw = eng.gather_batch(layers[r], sets[r], group=1)
            row = []
            for b in range(B):
                layer = cws[b][r]
                if isinstance(layer, DeviceCodeword):
                    row.append(layer.adopt(sets[r][b], sa_marshal.unpack(raw[b], sa_devlist.field_of(layer),
                                                                         FieldElement)))
                else:
                    row.append([layer[i] for i in sets[r][b]])
            values.append(row)
        for r in range(rounds - 1):
            cur_at = k if r else 0  # layer r's a and b openings follow its c openings of round r - 1
            for b, ps in enumerate(proof_streams):
                cur, cur_paths = values[r][b][cur_at:], paths[r][b][cur_at:]
                nxt, nxt_paths = values[r + 1][b][:k], paths[r + 1][b][:k]
                for s in range(k):
                    ps.push((cur[s], cur[k + s], nxt[s]))
                for s in range(k):
                    ps.push(cur_paths[s])
                    ps.push(cur_paths[k + s])
                    ps.push(nxt_paths[s])
        return tops

    # --------------------------------------------------------------- verify --
    def verify(self, proof_stream, polynomial_values):
        """Verifier (code/fri.py:132-231).  Same accept/reject decisions and the same
        pulls from the proof stream; the low-degree check of the last codeword uses
        the inverse transform the tutorial text describes (docs/faster.md, commented
        out at code/fri.py:165-166) instead of cubic-time Lagrange interpolation."""
        eng = sa_engine.get_engine()
        p = self.field.p
        rounds = self.num_rounds()

        # extract all roots and alphas
        roots, alphas = [], []
        for r in range(rounds):
            roots += [proof_stream.pull()]
            alphas += [self.field.sample(proof_stream.verifier_fiat_shamir())]

        # extract last codeword and check it against the last root
        last_codeword = proof_stream.pull()
        last_vec = sa_devlist.to_device(last_codeword)
        if roots[-1] != eng.tree_root(eng.merkle_tree(last_vec)):
            print("last codeword is not well formed")
            return False

        # check if it is low degree
        degree = (len(last_codeword) // self.expansion_factor) - 1
        last_omega = FieldElement(pow(self.omega.value, 1 << (rounds - 1), p), self.field)
        last_offset = FieldElement(pow(self.offset.value, 1 << (rounds - 1), p), self.field)
        assert(last_omega.inverse() == last_omega ^ (len(last_codeword) - 1)), "omega does not have right order"
        coefficients = intt(last_omega, last_codeword)
        poly = Polynomial(coefficients).scale(last_offset.inverse())
        if poly.degree() > degree:
            print("last codeword does not correspond to polynomial of low enough degree")
            print("observed degree:", poly.degree())
            print("but should be:", degree)
            return False

        # get indices
        top_level_indices = self.sample_indices(proof_stream.verifier_fiat_shamir(), self.domain_length >> 1, self.domain_length >> (rounds - 1), self.num_colinearity_tests)

        omega, offset = self.omega, self.offset
        # for every round, check consistency of subsequent layers
        for r in range(0, rounds - 1):
            half = self.domain_length >> (r + 1)
            c_indices = [index % half for index in top_level_indices]
            a_indices = [index for index in c_indices]
            b_indices = [index + half for index in a_indices]

            # read values and check colinearity
            aa, bb, cc = [], [], []
            for s in range(self.num_colinearity_tests):
                (ay, by, cy) = proof_stream.pull()
                aa += [ay]
                bb += [by]
                cc += [cy]
                # record top-layer values for later verification
                if r == 0:
                    polynomial_values += [(a_indices[s], ay), (b_indices[s], by)]
                ax = offset * (omega ^ a_indices[s])
                bx = offset * (omega ^ b_indices[s])
                cx = alphas[r]
                if test_colinearity([(ax, ay), (bx, by), (cx, cy)]) == False:  # noqa: E712
                    print("colinearity check failure")
                    return False

            # verify authentication paths
            for i in range(self.num_colinearity_tests):
                path = proof_stream.pull()
                if Merkle.verify(roots[r], a_indices[i], path, aa[i]) == False:  # noqa: E712
                    print("merkle authentication path verification fails for aa")
                    return False
                path = proof_stream.pull()
                if Merkle.verify(roots[r], b_indices[i], path, bb[i]) == False:  # noqa: E712
                    print("merkle authentication path verification fails for bb")
                    return False
                path = proof_stream.pull()
                if Merkle.verify(roots[r + 1], c_indices[i], path, cc[i]) == False:  # noqa: E712
                    print("merkle authentication path verification fails for cc")
                    return False

            # square omega and offset to prepare for next round
            omega = omega ^ 2
            offset = offset ^ 2

        # all checks passed
        return True
