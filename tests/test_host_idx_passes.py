"""The pass planner of the device index build on the CPU (plan_bucket_passes): contiguous bucket ranges in order, each within the
allowance unless it is one bucket or the pass minimum forced it, at most the pass cap, fewer than 2^31 pairs per pass, empty buckets
handled; random counts against a brute-force model of the same rules."""
import ctypes as C

import numpy as np
import pytest

import build_hostcheck_idx_passes

PAIR_BYTES = 24  # keys, sort ping-pong and rank (cuda/idx_build.cu)


@pytest.fixture(scope="module")
def hc():
    L = C.CDLL(build_hostcheck_idx_passes.build())
    L.hc_plan_bucket_passes.restype = C.c_int32
    L.hc_plan_bucket_passes.argtypes = [C.c_uint32, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.POINTER(C.c_int32)]
    L.hc_idx_max_passes.restype = C.c_int32
    L.hc_pass_max_pairs.restype = C.c_int64
    return L


def plan(L, cnt, fixed, allowance, max_passes=None, per_pair=PAIR_BYTES):
    c = np.ascontiguousarray(cnt, dtype=np.uint32)
    cut = np.zeros(len(c) + 1, dtype=np.int32)
    over = C.c_int32()
    k = L.hc_plan_bucket_passes(len(c), c.ctypes.data, per_pair, fixed, allowance, L.hc_idx_max_passes() if max_passes is None else max_passes,
                                cut.ctypes.data, C.byref(over))
    return [int(x) for x in cut[:k + 1]], over.value


def model(cnt, per_pair, fixed, allowance, max_passes, max_pairs):
    """Brute force: for each pass start, the longest range whose every step is allowed -- a step takes the next bucket unless the
    pass already holds the pair minimum and the bucket would break the allowance, or it would reach max_pairs pairs; the empty
    buckets after the last pair always join."""
    n, total = len(cnt), sum(cnt)
    pre = [0]
    for x in cnt:
        pre.append(pre[-1] + x)
    min_pairs = -(-total // max(max_passes, 1))
    cut, over, lo, done = [0], 0, 0, 0

    def allowed(lo, h):
        c = pre[h] - pre[lo]
        if done + c == total:
            return True
        nc = c + cnt[h]
        return not (nc >= max_pairs or (c >= min_pairs and fixed + nc * per_pair > allowance))

    while lo < n:
        hi = next(hi for hi in range(n, lo, -1) if all(allowed(lo, h) for h in range(lo + 1, hi)))
        c = sum(cnt[lo:hi])
        over += fixed + c * per_pair > allowance or c >= max_pairs
        cut.append(hi)
        lo, done = hi, done + c
    return cut, over


def check(cut, over, cnt, fixed, allowance, max_passes, max_pairs, per_pair=PAIR_BYTES):
    n, total = len(cnt), sum(cnt)
    min_pairs = -(-total // max(max_passes, 1))
    assert cut[0] == 0 and cut[-1] == n
    assert all(a < b for a, b in zip(cut, cut[1:]))  # contiguous, in order, at least one bucket each
    n_over = 0
    for lo, hi in zip(cut, cut[1:]):
        c = sum(cnt[lo:hi])
        nz = [b for b in range(lo, hi) if cnt[b]]  # the pass's non-empty buckets
        if len(nz) > 1:
            assert c < max_pairs
        if fixed + c * per_pair > allowance or c >= max_pairs:
            n_over += 1
            # one bucket on its own (empty ones around it add nothing), or the pass minimum took the last one past the allowance
            assert len(nz) <= 1 or sum(cnt[lo:nz[-1]]) < min_pairs, (lo, hi, c)
    assert n_over == over
    if total < max_pairs:
        assert len(cut) - 1 <= max_passes


@pytest.mark.parametrize("seed", range(30))
def test_plan_random(hc, seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 300))
    shape = seed % 3
    if shape == 0:
        cnt = [int(x) for x in rng.integers(0, 200, n)]
    elif shape == 1:  # sparse: most buckets empty, a few heavy ones
        cnt = [int(x) if rng.random() < 0.1 else 0 for x in rng.integers(1, 50_000, n)]
    else:  # skewed
        cnt = [int(x) for x in rng.zipf(1.6, n).clip(0, 1 << 20)]
    fixed = int(rng.choice([0, 1 << 16, 1 << 22]))
    allowance = int(rng.choice([1, 1 << 12, 1 << 16, 1 << 20, 1 << 24, 1 << 40]))
    max_passes = int(rng.choice([1, 4, 64]))
    max_pairs = hc.hc_pass_max_pairs()
    cut, over = plan(hc, cnt, fixed, allowance, max_passes)
    check(cut, over, cnt, fixed, allowance, max_passes, max_pairs)
    assert (cut, over) == model(cnt, PAIR_BYTES, fixed, allowance, max_passes, max_pairs)
    assert (cut, over) == plan(hc, cnt, fixed, allowance, max_passes)  # deterministic


def test_plan_shapes(hc):
    assert hc.hc_idx_max_passes() == 64 and hc.hc_pass_max_pairs() == 1 << 31
    assert plan(hc, [3, 1, 4, 1, 5], 0, 1 << 30) == ([0, 5], 0)  # room to spare: one pass over every bucket
    assert plan(hc, [2] * 6, 0, 4 * PAIR_BYTES) == ([0, 2, 4, 6], 0)
    assert plan(hc, [1, 9, 1, 1], 10, 3 * PAIR_BYTES + 10) == ([0, 1, 2, 4], 1)  # the bucket of 9 runs alone, over
    assert plan(hc, [2, 2, 2, 2], 0, 3 * PAIR_BYTES, max_passes=2) == ([0, 2, 4], 2)  # the cap takes 4 pairs per pass, past 3
    assert plan(hc, [5] * 8, 1 << 20, 1) == ([0, 1, 2, 3, 4, 5, 6, 7, 8], 8)  # the fixed part alone is over: a bucket per pass


def test_plan_empty_buckets(hc):
    """All-zero counts and empty buckets at either end: no pass of empty buckets alone, none lost."""
    for n in (1, 2, 1000):
        for allowance in (1, 1 << 30):
            assert plan(hc, [0] * n, 0, allowance) == ([0, n], 0)
    assert plan(hc, [0] * 10, 100, 1) == ([0, 10], 1)  # over by the fixed part alone: one pass all the same
    cnt = [0] * 5 + [4, 4, 4] + [0] * 7
    assert plan(hc, cnt, 0, 4 * PAIR_BYTES) == ([0, 6, 7, 15], 0)  # leading empties join the first pass, trailing ones the last
    assert plan(hc, cnt, 0, 1) == ([0, 6, 7, 15], 3)  # the same ranges when nothing fits: one non-empty bucket each
    cut, over = plan(hc, [0] * 3 + [7] + [0] * 3, 0, 1)
    assert cut == [0, 7] and over == 1


def test_plan_cap(hc):
    """A budget far below the need costs at most the cap's passes, not one per bucket."""
    rng = np.random.default_rng(11)
    cnt = [int(x) for x in rng.integers(0, 40, 50_000)]
    for allowance in (1, 1 << 10, 1 << 14):
        cut, over = plan(hc, cnt, 1 << 16, allowance)
        assert len(cut) - 1 <= 64 and over == len(cut) - 1
        check(cut, over, cnt, 1 << 16, allowance, 64, 1 << 31)
    cut, over = plan(hc, [1] * 1000, 0, 1)
    assert len(cut) - 1 == 63 and all(b - a == 16 for a, b in zip(cut, cut[1:-1]))  # ceil(1000 / 64) = 16 pairs per pass


def test_plan_pair_limit(hc):
    """No pass of several buckets reaches 2^31 pairs, whatever the allowance; a bucket of 2^31 pairs or more runs alone, over."""
    cnt = [(1 << 29) + 7] * 9
    cut, over = plan(hc, cnt, 0, 1 << 62)
    assert over == 0 and cut == [0, 3, 6, 9] and all(sum(cnt[a:b]) < (1 << 31) for a, b in zip(cut, cut[1:]))
    cut, over = plan(hc, [1, (1 << 32) - 1, 1], 0, 1 << 62)
    assert cut == [0, 1, 2, 3] and over == 1


def test_plan_many_buckets(hc):
    """2^24 buckets (the count array of -k 7 -M 4): the planner walks the counts as they are."""
    cnt = np.zeros(1 << 24, dtype=np.uint32)
    cnt[::4096] = 3
    cut, over = plan(hc, cnt, 0, 1 << 40)
    assert cut == [0, 1 << 24] and over == 0
    cut, over = plan(hc, cnt, 0, 1)
    total = int(cnt.sum())
    assert len(cut) - 1 == -(-total // -(-total // 64)) and over == len(cut) - 1
