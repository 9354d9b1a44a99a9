"""The device-memory budget on the CPU: the slice planner (consecutive greedy slices within an allowance, at least one item each, fewer
than 2^31 anchors each, deterministic) and the parser of MPB_DEVICE_MEM."""
import ctypes as C

import numpy as np
import pytest

import build_hostcheck_mem


@pytest.fixture(scope="module")
def hc():
    L = C.CDLL(build_hostcheck_mem.build())
    L.hc_plan_slices.restype = C.c_int32
    L.hc_plan_slices.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.POINTER(C.c_int32)]
    L.hc_slice_max_count.restype = C.c_int64
    L.hc_parse_mem_size.restype = C.c_int64
    L.hc_parse_mem_size.argtypes = [C.c_char_p]
    return L


def plan(L, bytes_, count, fixed, allowance, max_count=None):
    n = len(bytes_)
    b = np.ascontiguousarray(bytes_, dtype=np.int64)
    c = None if count is None else np.ascontiguousarray(count, dtype=np.int64)
    cut = np.zeros(n + 1, dtype=np.int32)
    over = C.c_int32()
    k = L.hc_plan_slices(n, b.ctypes.data, None if c is None else c.ctypes.data, fixed, allowance,
                         L.hc_slice_max_count() if max_count is None else max_count, cut.ctypes.data, C.byref(over))
    return [int(x) for x in cut[:k + 1]], over.value


def check(cut, over, bytes_, count, fixed, allowance, max_count):
    n = len(bytes_)
    assert cut[0] == 0 and cut[-1] == n
    assert all(a < b for a, b in zip(cut, cut[1:])) or n == 0  # contiguous, ordered, non-empty, covering
    n_over = 0
    for lo, hi in zip(cut, cut[1:]):
        b = fixed + sum(bytes_[lo:hi])
        c = sum(count[lo:hi]) if count is not None else 0
        if hi - lo == 1:
            n_over += b > allowance or c >= max_count
        else:
            assert b <= allowance and c < max_count
        if hi < n:  # greedy: the next item would not have fitted
            assert fixed + sum(bytes_[lo:hi + 1]) > allowance or (count is not None and sum(count[lo:hi + 1]) >= max_count)
    assert n_over == over


@pytest.mark.parametrize("seed", range(20))
def test_plan_random(hc, seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(0, 400))
    count = [int(x) for x in rng.integers(0, 50_000, n)]
    bytes_ = [88 * c + 49_280 for c in count]
    fixed = int(rng.integers(0, 1 << 16))
    allowance = int(rng.choice([1 << 10, 1 << 20, 1 << 24, 1 << 28, 1 << 40]))
    max_count = int(rng.choice([1 << 31, 200_000, 60_000]))
    cut, over = plan(hc, bytes_, count, fixed, allowance, max_count)
    check(cut, over, bytes_, count, fixed, allowance, max_count)
    assert (cut, over) == plan(hc, bytes_, count, fixed, allowance, max_count)  # deterministic


def test_plan_shapes(hc):
    assert plan(hc, [], None, 0, 100) == ([0], 0)
    assert plan(hc, [10] * 5, None, 0, 1 << 30) == ([0, 5], 0)  # room to spare: one slice
    assert plan(hc, [10] * 5, None, 0, 20) == ([0, 2, 4, 5], 0)
    assert plan(hc, [10, 50, 10, 10], None, 5, 30) == ([0, 1, 2, 4], 1)  # 50 + 5 runs alone, over the allowance
    assert plan(hc, [10] * 4, None, 100, 30) == ([0, 1, 2, 3, 4], 4)  # the fixed part alone is over: every item alone and over
    assert plan(hc, [1] * 4, [3, 3, 3, 3], 0, 100, max_count=7) == ([0, 2, 4], 0)
    assert plan(hc, [1, 1], [9, 1], 0, 100, max_count=7) == ([0, 1, 2], 1)


def test_plan_anchor_cap(hc):
    """No slice reaches 2^31 anchors, whatever the allowance."""
    count = [(1 << 29) + 7] * 9
    cut, over = plan(hc, [1] * 9, count, 0, 1 << 62)
    assert over == 0 and all(sum(count[a:b]) < (1 << 31) for a, b in zip(cut, cut[1:])) and cut == [0, 3, 6, 9]


def test_parse_mem_size(hc):
    p = lambda s: hc.hc_parse_mem_size(s.encode())  # noqa: E731
    assert p("0") == 0
    assert p("123") == 123
    assert p("4k") == 4 << 10 and p("4K") == 4 << 10
    assert p("256m") == 256 << 20 and p("256M") == 256 << 20
    assert p("16g") == 16 << 30 and p("16G") == 16 << 30
    for bad in ["", "g", "-1", "1.5g", "12gb", "1t", " 1g", "1g ", "abc", "99999999999999999999", "9999999999999g"]:
        assert p(bad) == -1, bad
    assert hc.hc_parse_mem_size(None) == -1
