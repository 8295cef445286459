"""sa_interp_plan_bytes (host-only, no GPU needed) follows the plan layout documented in csrc/poly.cu: sections
padded to 256 bytes (16 elements); up to 1024 points domain | z | 1/z'(d_i), above that the tree's node
transforms (log K * 2K) | 1/M'(d_i) (K), K = 2^ceil(log2 k)."""
import pytest

import __graft_entry__ as G

FE = 16  # bytes per field element
DIRECT_MAX = 1024


def sec(elems):
    return (elems + 15) // 16 * 16


def layout_bytes(k):
    if k <= DIRECT_MAX:
        return FE * (sec(k) + sec(k + 1) + sec(k))
    log_k = (k - 1).bit_length()
    big_k = 1 << log_k
    return FE * (sec(log_k * 2 * big_k) + sec(big_k))


@pytest.fixture(scope="module")
def lib():
    G.build_cuda()
    G._paths()
    import sa_engine
    return sa_engine.load_library()


@pytest.mark.parametrize("k", [1, 2, 1023, 1024, 1025, 4096, 5000, 1 << 20])
def test_plan_bytes_follow_the_layout(lib, k):
    assert lib.sa_interp_plan_bytes(k) == layout_bytes(k)


def test_plan_bytes_at_the_limit(lib):
    assert lib.sa_interp_plan_bytes(1 << 20) == 656 << 20
    assert lib.sa_interp_plan_bytes(1025) == FE * (11 * 4096 + 2048)


@pytest.mark.parametrize("k", [0, (1 << 20) + 1])
def test_no_plan_outside_the_range(lib, k):
    assert lib.sa_interp_plan_bytes(k) == 0
