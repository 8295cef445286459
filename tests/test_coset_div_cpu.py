"""sa_coset_div_plan_bytes and sa_coset_batch_max (host-only, no GPU needed) follow the rules documented in
include/sa_b200.h: a plan is three sections of n = 2^log_n elements, each rounded up to 256 bytes; a chunk is
max(1, floor(2^30 / (32 n))) rows; both are 0 outside log_n 1..30.  The CPU emulation lays plans out the same way."""
import ctypes

import pytest

import __graft_entry__ as G

FE = 16
LOGS = [1, 2, 3, 4, 10, 16, 20, 26, 27, 30]


def plan_rule(log_n):
    n = 1 << log_n
    return 3 * FE * ((n + 15) // 16 * 16)


def chunk_rule(log_n):
    return max(1, (1 << 30) // (32 << log_n))


@pytest.fixture(scope="module")
def lib():
    G.build_cuda()
    G._paths()
    import sa_engine
    return sa_engine.load_library()


@pytest.fixture(scope="module")
def emu():
    e = ctypes.CDLL(G.build_emu_coset())
    e.emu_coset_div_plan_bytes.restype = ctypes.c_size_t
    e.emu_coset_div_plan_bytes.argtypes = [ctypes.c_int]
    return e


@pytest.mark.parametrize("log_n", LOGS)
def test_plan_bytes_and_chunk_follow_the_rules(lib, log_n):
    assert lib.sa_coset_div_plan_bytes(log_n) == plan_rule(log_n)
    assert lib.sa_coset_batch_max(log_n) == chunk_rule(log_n)


def test_documented_values(lib):
    assert lib.sa_coset_div_plan_bytes(20) == 48 << 20
    assert lib.sa_coset_div_plan_bytes(26) == 3 << 30
    assert lib.sa_coset_div_plan_bytes(27) == 6 << 30
    assert lib.sa_coset_div_plan_bytes(30) == 48 << 30
    assert lib.sa_coset_batch_max(20) == 32
    assert lib.sa_coset_batch_max(16) == 512
    assert lib.sa_coset_batch_max(26) == 1
    assert lib.sa_coset_batch_max(30) == 1


@pytest.mark.parametrize("log_n", [0, 31, -1])
def test_nothing_outside_the_range(lib, emu, log_n):
    assert lib.sa_coset_div_plan_bytes(log_n) == 0
    assert lib.sa_coset_batch_max(log_n) == 0
    assert emu.emu_coset_div_plan_bytes(log_n) == 0


@pytest.mark.parametrize("log_n", LOGS)
def test_emulation_plan_is_the_library_s(lib, emu, log_n):
    assert emu.emu_coset_div_plan_bytes(log_n) == lib.sa_coset_div_plan_bytes(log_n)
