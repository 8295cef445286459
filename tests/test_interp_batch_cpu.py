"""sa_interp_batch_max (host-only, no GPU needed) follows the chunk rule documented in include/sa_b200.h: one pass
whatever the batch up to 1024 points (SIZE_MAX), max(1, floor(2^30 / (96 K))) vectors per chunk above, K =
2^ceil(log2 k), and 0 where there is no plan."""
import pytest

import __graft_entry__ as G

SIZE_MAX = (1 << 64) - 1


def chunk_rule(k):
    if k <= 1024:
        return SIZE_MAX
    big_k = 1 << (k - 1).bit_length()
    return max(1, (1 << 30) // (96 * big_k))


@pytest.fixture(scope="module")
def lib():
    G.build_cuda()
    G._paths()
    import sa_engine
    return sa_engine.load_library()


@pytest.mark.parametrize("k", [1, 1024, 1025, 4096, 1 << 16, 1 << 20])
def test_batch_max_follows_the_rule(lib, k):
    assert lib.sa_interp_batch_max(k) == chunk_rule(k)


def test_batch_max_documented_values(lib):
    assert lib.sa_interp_batch_max(1 << 20) == 10
    assert lib.sa_interp_batch_max(1 << 16) == 170
    assert lib.sa_interp_batch_max(1025) == 5461


@pytest.mark.parametrize("k", [0, (1 << 20) + 1])
def test_no_batch_outside_the_range(lib, k):
    assert lib.sa_interp_batch_max(k) == 0
