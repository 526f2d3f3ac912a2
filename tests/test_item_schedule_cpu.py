"""The numpy restatement of k_build_items (tests/item_schedule.py) held to small cases worked out by hand, and its table check held
to tables laid out the way the device may lay them out, and to broken ones."""
import numpy as np
import pytest
import item_schedule as S

HUGE = 50_000_000   # the warp-slot count tests pretend to force splits: the balanced share drops to SPLIT_WORK_MIN


def rows(*r):
    return np.array(r, dtype=np.int64).reshape(-1, 3)


def test_bucket_overflow_raises_thr_past_the_workload():
    """20 000 samples of w = 300 (bucket 37) and 16 384 slots: bucket 37 overflows, THR = max(256, 38 * 8) = 304, nothing split"""
    s = S.schedule(np.full(20000, 300), S.MAX_SPLIT_SLOTS, HUGE)
    assert s["total"] == 6_000_000 and s["thr_share"] == 256
    assert s["raised_bucket"] == 37 and s["thr"] == 304
    assert not s["split"].any() and s["item_count"] == 20000
    assert s["order"] == [37] and np.array_equal(s["buckets"][37][:, 0], np.arange(20000))


def test_top_bucket_overflow_saturates_thr():
    """16 385 samples in the open-ended top bucket (w >= 8184): THR = 0xffffffff, nothing split, one item per sample"""
    w = np.concatenate([np.full(16385, 8184), np.full(10, 100000), [7000, 5]])
    s = S.schedule(w, S.MAX_SPLIT_SLOTS, HUGE)
    assert s["raised_bucket"] == 1023 and s["thr"] == 0xffffffff
    assert not s["split"].any() and s["item_count"] == w.size
    assert s["order"] == [1023, 875, 0] and len(s["buckets"][1023]) == 16395


def test_top_bucket_at_capacity_splits_it_whole():
    """exactly max_split samples in the top bucket: they all fit; bucket 1012 is the first to overflow, THR = 1013 * 8 = 8104"""
    w = np.concatenate([np.full(4, 9000), np.full(3, 8100)])
    s = S.schedule(w, 4, HUGE)
    assert s["raised_bucket"] == 1012 and s["thr"] == 8104
    assert np.array_equal(s["split"], [True] * 4 + [False] * 3)
    assert np.array_equal(s["f"][:4], [2] * 4)                   # 8104 * 2 >= 9000
    assert s["order"] == [1012, 562] and s["item_count"] == 11    # 9000 / 2 = 4500 -> bucket 562


def test_share_below_split_work_min():
    """the balanced share of a huge warp count is ~0: THR = SPLIT_WORK_MIN = 256 and f doubles until THR * f >= w"""
    w = np.array([1000, 200, 100, 256, 255])
    s = S.schedule(w, 16384, HUGE)
    assert s["thr_share"] == 256 and s["thr"] == 256 and s["raised_bucket"] is None
    assert np.array_equal(s["split"], [True, False, False, True, False])
    assert np.array_equal(s["f"], [4, 1, 1, 2, 1])                 # 256 * 2 < 1000 <= 256 * 4; 256 <= 256 * 2
    assert s["order"] == [31, 25, 16, 12] and s["item_count"] == 9  # 1000 / 4 = 250 -> 31; 256 / 2 = 128 -> 16
    assert np.array_equal(s["buckets"][31], rows((0, 0, 8), (0, 8, 16), (0, 16, 24), (0, 24, 32), (4, 0, 32)))
    assert np.array_equal(s["buckets"][16], rows((3, 0, 16), (3, 16, 32)))


def test_share_above_split_work_min():
    """two warps: THR = 0.7 * 12000 / 2 = 4200, only the 10 000 sample is split (f = 4: 4200 * 2 < 10000 <= 4200 * 4)"""
    s = S.schedule(np.array([10000, 1000, 1000]), 3, 2)
    assert s["thr"] == 4200 and s["raised_bucket"] is None
    assert np.array_equal(s["f"], [4, 1, 1])
    assert s["order"] == [312, 125] and s["item_count"] == 6


def test_split_factor_caps_at_32():
    s = S.schedule(np.array([1_000_000, 10]), 16384, HUGE)
    assert s["f"][0] == 32 and s["item_count"] == 33
    assert s["order"] == [1023, 1]                                  # 1e6 / 32 = 31250 -> top bucket


def test_raise_leaves_the_heaviest_split():
    """two slots: the third-heaviest bucket (150) overflows them, THR = 151 * 8 = 1208; 2000 and 1500 split, 1200 not"""
    s = S.schedule(np.array([2000, 1500, 1200, 300]), 2, HUGE)
    assert s["raised_bucket"] == 150 and s["thr"] == 1208
    assert np.array_equal(s["f"], [2, 2, 1, 1])
    assert s["order"] == [150, 125, 93, 37] and s["item_count"] == 6


def test_no_split_slots_analytic_robots():
    """max_split = 0 (analytic shapes): the first non-empty bucket already overflows, nothing is ever split"""
    s = S.schedule(np.array([5000, 300, 0]), 0, HUGE)
    assert s["raised_bucket"] == 625 and s["thr"] == 626 * 8
    assert not s["split"].any() and s["item_count"] == 3 and s["order"] == [625, 37, 0]
    s = S.schedule(np.array([9000, 10]), 0, HUGE)
    assert s["thr"] == 0xffffffff and s["item_count"] == 2
    s = S.schedule(np.zeros(7, dtype=np.uint32), 0, 2112)
    assert s["raised_bucket"] == 0 and s["item_count"] == 7


def random_work(rng, M, hi=20000):
    return np.where(rng.random(M) < 0.3, rng.integers(0, 256, M), rng.integers(256, hi, M)).astype(np.uint32)


@pytest.mark.parametrize("max_split,warp_slots", [(16384, HUGE), (16384, 2112), (40, HUGE), (0, HUGE)])
def test_check_table_accepts_any_device_layout(max_split, warp_slots):
    rng = np.random.default_rng(max_split + warp_slots)
    s = S.schedule(random_work(rng, 3000), max_split, warp_slots)
    for seed in range(3):
        S.check_table(s, S.simulate_table(s, max(max_split, 1), np.random.default_rng(seed)), max_split)


def test_check_table_rejects_broken_tables():
    rng = np.random.default_rng(5)
    s = S.schedule(random_work(rng, 2000, hi=5000), 64, HUGE)
    assert s["split"].sum() > 10
    good = S.simulate_table(s, 64, rng)
    S.check_table(s, good, 64)
    heavy = np.flatnonzero(good[:, 2] >= 0)
    first, last = heavy[0], heavy[-1]
    a, b = good[:, 0] == good[first, 0], good[:, 0] == good[last, 0]
    assert not np.array_equal(a, b)
    broken = []
    t = good.copy(); t[b, 2] = good[first, 2]; broken.append(("two samples share a slot", t))
    t = good.copy(); t[a, 2] = 64; broken.append(("slot out of range", t))
    t = good.copy(); t[first, 1] += 1; broken.append(("class ranges do not tile", t))
    t = np.concatenate([good[-5:], good[:-5]]); broken.append(("buckets out of order", t))
    t = good.copy(); t[-1, 0] = (t[-1, 0] + 1) % 2000; broken.append(("a sample twice, another missing", t))
    t = good.copy(); t[a, 2] = -1; t[a, 1] = -1; broken.append(("split sample listed as whole", t))
    broken.append(("one item short", good[:-1]))
    for what, t in broken:
        try:
            S.check_table(s, t, 64)
        except AssertionError:
            continue
        pytest.fail(f"check_table accepted a table with {what}")
