"""sa_devlist -- ``DeviceCodeword``: a list of field elements that lives on the GPU (SURVEY.md section 8 f3).

The reference's ``ntt`` / ``intt`` / ``fast_coset_evaluate`` return Python lists of 2^k ``FieldElement``
objects and its callers hand those lists straight back to the hot path
(code/fast_stark.py:104-106,117-119,148-151,154-175: ``fast_coset_evaluate`` -> ``Merkle.commit`` ->
``Fri.prove`` -> ``codeword[i]`` / ``Merkle.open(i, codeword)``).  Turning 2^k residues into 2^k Python
objects and back on every crossing costs 5000x the kernel time at 2^20.  The drop-in therefore returns
this list-like instead: the values stay in HBM, ``Merkle.commit`` / ``Fri.commit`` / ``ntt`` consume the
device vector directly (no pack, no upload, no fingerprint), the Merkle tree built by the first commit
stays attached for ``Merkle.open`` (O(log n) per opened index), and ``FieldElement`` objects are only
created for the indices somebody actually reads.

List semantics that the reference's callers rely on are kept:
  * ``len``, indexing (negative indices, slices), iteration, ``==``, ``in``, ``+`` with lists, ``*``,
    ``index`` / ``count`` / ``copy``, ``reversed``;
  * indexing twice returns the SAME ``FieldElement`` object (pickle's memo sees the difference);
  * every element carries the ``Field`` instance a reference list would carry;
  * mutation works: the first mutating call materialises a real list, the device copy is dropped and
    rebuilt (pack + upload) only if the hot path sees the object again.
``tolist()`` gives the real list (materialised once, identities handed out earlier are kept);
pickling a DeviceCodeword pickles that list.  SA_B200_DEVICE_LISTS=0 makes the drop-in return plain lists
everywhere (the round-1 behaviour).

``to_device`` / ``from_device`` at the end of this module are the drop-in's only conversions between a
sequence of field elements and an engine vector.
"""
import os

import sa_host
import sa_engine
import sa_marshal

FieldElement = sa_host.algebra.FieldElement

ENABLED = os.environ.get("SA_B200_DEVICE_LISTS", "1") != "0"
MIN_LENGTH = 2          # ntt()/intt() of length <= 1 return their argument (ntt.py:5-6, :23-24)
SMALL_VALUES = 1 << 14  # up to this many elements the first element read downloads the whole vector
SMALL_TREE = 1 << 16    # up to this many leaves the first open downloads the whole tree (8 MiB)
GATHER_LIMIT = 4096     # single-element gathers after which a large vector is downloaded as well


class DeviceCodeword:
    __slots__ = ("_vec", "_tree", "_field", "_len", "_cache", "_full", "_host_tree", "_dirty", "_misses")

    def __init__(self, vec, tree, field, length=None):
        self._vec, self._tree, self._field = vec, tree, field
        self._len = sa_engine.get_engine().length(vec) if length is None else length
        self._cache = {}
        self._full = None
        self._host_tree = None
        self._dirty = False
        self._misses = 0

    # ------------------------------------------------------------ device side (used by ntt.py / fri.py)
    def device_vector(self):
        """the values as an engine vector; re-packed and re-uploaded only after a mutation"""
        if self._dirty:
            self._vec = to_device(self._full)
            self._len = len(self._full)
            self._dirty = False
        return self._vec

    def device_tree(self):
        """heap-ordered Merkle tree (code/merkle.py:6-14) of the values, built once and kept"""
        vec = self.device_vector()
        if self._tree is None:
            self._tree = sa_engine.get_engine().merkle_tree(vec)
            self._host_tree = None
        return self._tree

    def attach_tree(self, tree):
        if self._tree is None and not self._dirty:
            self._tree = tree

    def root(self):
        return sa_engine.get_engine().tree_root(self.device_tree())

    def open_paths(self, indices):
        """authentication paths (code/merkle.py:16-27): lists of 64-byte digests, bottom-up"""
        eng = sa_engine.get_engine()
        tree = self.device_tree()
        n = self._len
        # one index at a time (code/fast_stark.py:162-174 opens 1024 positions one by one): fetch a small tree once
        # and read the paths on the host; a batch of indices (Fri.query) is one gather on the device
        indices = list(indices)
        if n <= SMALL_TREE and (self._host_tree is not None or len(indices) <= 2):
            if self._host_tree is None:
                self._host_tree = eng.download_tree(tree)
            host, depth = self._host_tree, n.bit_length() - 1
            out = []
            for i in indices:
                assert(0 <= i and i < n), "cannot open invalid index"
                node = n + i
                out.append([bytes(host[(node >> l) ^ 1]) for l in range(depth)])
            return out
        return eng.merkle_open(tree, indices)

    # ---------------------------------------------------------------------------- element access
    def _field_of(self):
        return self._field

    def prefetch(self, indices):
        if self._full is not None:
            return
        missing = [i for i in dict.fromkeys(indices) if i not in self._cache]
        if not missing:
            return
        self._misses += len(missing)
        if self._len <= SMALL_VALUES or self._misses > GATHER_LIMIT:
            self.tolist()
            return
        raw = sa_engine.get_engine().gather(self._vec, missing)
        for i, el in zip(missing, sa_marshal.unpack(raw, self._field, FieldElement)):
            self._cache[i] = el

    def adopt(self, indices, elements):
        """the element objects at `indices` given their values read elsewhere (`elements`, one per index, e.g. from
        one gather over many device lists): those handed out earlier where there are, else the given ones, which are
        handed out from then on"""
        if self._full is not None:
            return [self._full[i] for i in indices]
        return [self._cache.setdefault(i, el) for i, el in zip(indices, elements)]

    def tolist(self):
        if self._full is None:
            full = from_device(self._vec, self._field)
            for i, el in self._cache.items():  # keep identities handed out earlier
                full[i] = el
            self._full = full
            self._cache = {}
        return self._full

    def __len__(self):
        return len(self._full) if self._dirty else self._len

    def __getitem__(self, i):
        if isinstance(i, slice):
            return self.tolist()[i]
        if self._full is not None:
            return self._full[i]
        i = i.__index__()
        if i < 0:
            i += self._len
        if not 0 <= i < self._len:
            raise IndexError("list index out of range")
        hit = self._cache.get(i)
        if hit is None:
            self.prefetch([i])
            hit = self._full[i] if self._full is not None else self._cache[i]
        return hit

    def __iter__(self):
        return iter(self.tolist())

    def __reversed__(self):
        return reversed(self.tolist())

    def __contains__(self, x):
        return x in self.tolist()

    def __eq__(self, other):
        if isinstance(other, DeviceCodeword):
            if other is self:
                return True
            other = other.tolist()
        if not isinstance(other, list):
            return NotImplemented
        return self.tolist() == other

    def __ne__(self, other):
        r = self.__eq__(other)
        return r if r is NotImplemented else not r

    __hash__ = None

    def __add__(self, other):
        return self.tolist() + (other.tolist() if isinstance(other, DeviceCodeword) else other)

    def __radd__(self, other):
        return other + self.tolist()

    def __mul__(self, k):
        return self.tolist() * k

    __rmul__ = __mul__

    def index(self, *a):
        return self.tolist().index(*a)

    def count(self, x):
        return self.tolist().count(x)

    def copy(self):
        return self.tolist().copy()

    def __repr__(self):
        return "DeviceCodeword(%d elements on %s)" % (len(self), "the device" if not self._dirty else "the host (mutated)")

    def __reduce__(self):
        return (list, (self.tolist(),))

    # --------------------------------------------------------------------------------- mutation
    def _mutable(self):
        """a caller writes to the list: from here on the host list is the truth"""
        full = self.tolist()
        self._dirty = True
        self._tree = None
        self._host_tree = None
        self._vec = None
        return full

    def __setitem__(self, i, v):
        self._mutable()[i] = v

    def __delitem__(self, i):
        del self._mutable()[i]

    def __iadd__(self, other):
        self._mutable().extend(other.tolist() if isinstance(other, DeviceCodeword) else other)
        return self

    def append(self, v):
        self._mutable().append(v)

    def extend(self, it):
        self._mutable().extend(it)

    def insert(self, i, v):
        self._mutable().insert(i, v)

    def pop(self, *a):
        return self._mutable().pop(*a)

    def remove(self, v):
        self._mutable().remove(v)

    def clear(self):
        self._mutable().clear()

    def reverse(self):
        self._mutable().reverse()

    def sort(self, **kw):
        self._mutable().sort(**kw)


def wrap(vec, field, tree=None):
    """what ntt / intt / fast_coset_evaluate return: the device list, or a real list when disabled"""
    if ENABLED:
        return DeviceCodeword(vec, tree, field)
    return from_device(vec, field)


def pack(seq):
    """the host form of a sequence of field elements, 16 little-endian bytes per residue: what
    ``to_device`` uploads, and what fri.py fingerprints and compares revealed values in"""
    return sa_marshal.pack(seq)


def to_device(seq):
    """engine vector of a sequence of field elements: the resident vector of a DeviceCodeword, else
    pack + upload (the bytearray ``pack`` returns is uploaded as it is)"""
    if isinstance(seq, DeviceCodeword):
        return seq.device_vector()
    return sa_engine.get_engine().upload(seq if isinstance(seq, bytearray) else sa_marshal.pack(seq))


def from_device(vec, field):
    """list of ``FieldElement`` of `field` holding the values of an engine vector: download + unpack"""
    return sa_marshal.unpack(sa_engine.get_engine().download(vec), field, FieldElement)


def field_of(seq):
    if isinstance(seq, DeviceCodeword):
        return seq._field
    return seq[0].field
