"""Tampered copies of a serialized FastStark or Stark proof, one change per kind.  Only pickle is used, so the same
function runs beside the unmodified reference (tests/golden/make_golden_verify.py records its verdicts) and beside
the drop-in (the verifier tests), and gives the same bytes from the same proof."""
import pickle

KINDS = ["boundary_root", "randomizer_root", "fri_root", "fri_leaf_a", "fri_leaf_b", "fri_leaf_c", "fri_path",
         "last_codeword", "boundary_leaf", "boundary_path", "randomizer_leaf", "randomizer_path", "zerofier_leaf",
         "zerofier_path", "swapped", "truncated"]


def kinds(fast):
    return [t for t in KINDS if fast or not t.startswith("zerofier")]


def _elem(v):
    p = v.field.p
    return type(v)((v.value + 1) % p, v.field)


def tamper(proof, nregs, rounds, k, kind):
    """a copy of the serialized proof with one change of `kind`, pickled back: every kind keeps the stream's shape
    except "truncated", which drops the last object"""
    objs = pickle.loads(proof)
    fri0 = nregs + 1
    last_at = fri0 + rounds
    q0 = last_at + 1
    opened0 = q0 + (rounds - 1) * 4 * k
    block = 2 * 4 * k  # one opened codeword: 4k (leaf, path) pairs
    if kind == "boundary_root":
        objs[0] = bytes(64)
    elif kind == "randomizer_root":
        objs[nregs] = bytes(64)
    elif kind == "fri_root":
        objs[fri0] = bytes(64)
    elif kind in ("fri_leaf_a", "fri_leaf_b", "fri_leaf_c"):
        pos = "abc".index(kind[-1])
        t = list(objs[q0])
        t[pos] = _elem(t[pos])
        objs[q0] = tuple(t)
    elif kind == "fri_path":
        p = list(objs[q0 + k])
        p[0] = bytes(64)
        objs[q0 + k] = p
    elif kind == "last_codeword":
        last = list(objs[last_at])
        last[0] = _elem(last[0])
        objs[last_at] = last
    elif kind in ("boundary_leaf", "randomizer_leaf", "zerofier_leaf"):
        at = opened0 + {"boundary_leaf": 0, "randomizer_leaf": nregs, "zerofier_leaf": nregs + 1}[kind] * block
        objs[at] = _elem(objs[at])
    elif kind in ("boundary_path", "randomizer_path", "zerofier_path"):
        at = opened0 + {"boundary_path": 0, "randomizer_path": nregs, "zerofier_path": nregs + 1}[kind] * block + 1
        p = list(objs[at])
        p[-1] = bytes(64)
        objs[at] = p
    elif kind == "swapped":
        objs[opened0], objs[opened0 + 2] = objs[opened0 + 2], objs[opened0]
    elif kind == "truncated":
        objs = objs[:-1]
    else:
        raise ValueError(kind)
    return pickle.dumps(objs)
