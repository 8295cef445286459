"""Cases of the coset combination tests, shared by the CPU emulation (tests/test_coset_combine_cpu.py) and the GPU
suite (tests/test_gpu_coset_combine.py): seeded term sets over a few source rows, and the combination
c[i] = sum_t w_t * row_t[i - shift_t] restated with Python ints, whose fast_coset_evaluate is what a call must give.

A term set of T terms at n = 2^log_n mixes, in turn: a row at a random shift; the previous term's row at another
shift (q and x^s * q); a duplicate of the previous (row, shift) pair; a row of 0 or 1 elements; a row that ends
exactly at n.  Weights cycle through 0, 1, p - 1 and random residues."""
import random

import oracle as O

P = O.P
SPECIAL_WEIGHTS = [0, 1, P - 1]


def make_terms(seed, n, T, max_len=None):
    """(rows, terms): rows are lists of ints, terms (row index, shift, weight) with shift + len(row) <= n; max_len
    bounds the rows' lengths (the Python restatement's time at large n)"""
    rng = random.Random(seed)
    top = n if max_len is None else min(n, max_len)
    rows = []

    def new_row(length):
        rows.append([rng.randrange(P) for _ in range(length)])
        return len(rows) - 1

    terms = []
    for t in range(T):
        kind = t % 5
        if kind == 1 and terms:  # the previous term's row, shifted elsewhere
            r = terms[-1][0]
            shift = rng.randrange(n - len(rows[r]) + 1)
        elif kind == 2 and terms:  # the same (row, shift) again
            r, shift = terms[-1][0], terms[-1][1]
        elif kind == 3:  # an empty row or a single element
            r = new_row(t % 2)
            shift = rng.randrange(n - len(rows[r]) + 1)
        elif kind == 4:  # a row that ends exactly at n
            r = new_row(rng.randrange(1, top + 1))
            shift = n - len(rows[r])
        else:
            r = new_row(rng.randrange(1, top + 1))
            shift = rng.randrange(n - len(rows[r]) + 1)
        w = SPECIAL_WEIGHTS[t % 4] if t % 4 < 3 else rng.randrange(P)
        terms.append((r, shift, w))
    return rows, terms


def combination(rows, terms, n):
    """c[0..n) with Python ints"""
    c = [0] * n
    for r, shift, w in terms:
        for j, v in enumerate(rows[r]):
            c[shift + j] = (c[shift + j] + w * v) % P
    return c


def ncomb(rows, terms):
    return max([shift + len(rows[r]) for r, shift, _ in terms], default=0)


def codeword(rows, terms, n, root, offset):
    """the reference's combined_codeword: fast_coset_evaluate of the combination at order n"""
    return O.fast_coset_evaluate(combination(rows, terms, n), offset, root, n)
