"""The discrete evaluation's work-item schedule restated in numpy: what k_build_items (implicit-sdf-planner_b200/csrc/isdf_discrete.cuh)
must build from the work values of one evaluation, and a check of a built table against it.

The builder sorts the M local samples into ORDER_BUCKETS buckets by work (w >> 3, the last bucket open-ended) and lays the
buckets out in descending order. A sample with w >= THR is split into f = 2..32 parts, each a contiguous range of ROW_CLASSES / f
row classes, filed under the bucket of w / f. THR is the balanced share 0.7 * total / warp_slots, at least SPLIT_WORK_MIN, raised to
the lower bound of the first bucket above the one where the heaviest samples stop fitting into max_split split slots (first_over),
and saturated to 0xffffffff (nothing split) when the top bucket alone holds more than max_split samples.

Two things depend on shared-memory atomics and are not restated: the order of the items inside a bucket and which split slot a
sample gets. check_table compares the per-bucket multisets instead and checks the slot rules on their own."""
import numpy as np

# mirrors of the constants in isdf_discrete.cuh
ORDER_BUCKETS = 1024
SPLIT_WORK_MIN = 256
ROW_CLASSES = 32
MAX_SPLIT_SLOTS = 16384
THR_SATURATED = 0xffffffff


def order_bucket(w):
    return np.minimum(np.asarray(w, dtype=np.uint64) >> np.uint64(3), np.uint64(ORDER_BUCKETS - 1)).astype(np.int64)


def schedule(work, max_split, warp_slots):
    """the table k_build_items must build: dict(total, thr_share (balanced share before the raise), thr, raised_bucket (b of the
    first_over raise, or None), split (bool per sample), f (parts per sample, 1 = whole), buckets (bucket -> (n, 3) int64 rows
    (m, c0, c1) sorted), order (the non-empty buckets, descending), item_count)"""
    w = np.asarray(work, dtype=np.uint64).reshape(-1)
    M = w.size
    total = int(w.sum())
    share = (total * 7) // (10 * max(int(warp_slots), 1))
    thr = min(max(share, SPLIT_WORK_MIN), THR_SATURATED)
    bucket = order_bucket(w)
    cum = np.cumsum(np.bincount(bucket, minlength=ORDER_BUCKETS)[::-1])   # cum[t]: samples in buckets >= ORDER_BUCKETS - 1 - t
    over = np.flatnonzero(cum > max_split)
    raised = None
    if over.size:
        raised = ORDER_BUCKETS - 1 - int(over[0])
        thr = max(thr, (raised + 1) << 3)
        if raised == ORDER_BUCKETS - 1:
            thr = THR_SATURATED
    split = w >= np.uint64(thr)
    if int(split.sum()) > max_split:
        raise ValueError("more samples qualify than there are split slots: which of them get one depends on the device's atomics")
    f = np.ones(M, dtype=np.int64)
    for m in np.flatnonzero(split):
        k = 2
        while k < ROW_CLASSES and thr * k < int(w[m]):
            k <<= 1
        f[m] = k
    rows, keys = [], []
    for m in range(M):
        if f[m] == 1:
            rows.append((m, 0, ROW_CLASSES))
            keys.append(int(bucket[m]))
        else:
            cw = ROW_CLASSES // int(f[m])
            b = int(order_bucket(int(w[m]) // int(f[m])))
            rows += [(m, p * cw, p * cw + cw) for p in range(int(f[m]))]
            keys += [b] * int(f[m])
    rows = np.array(rows, dtype=np.int64).reshape(-1, 3)
    keys = np.array(keys, dtype=np.int64)
    buckets = {}
    for b in np.unique(keys):
        r = rows[keys == b]
        buckets[int(b)] = r[np.lexsort((r[:, 2], r[:, 1], r[:, 0]))]
    return dict(total=total, thr_share=min(max(share, SPLIT_WORK_MIN), THR_SATURATED), thr=thr, raised_bucket=raised, split=split, f=f,
                buckets=buckets, order=sorted(buckets, reverse=True), item_count=len(rows))


def decode(items):
    """device item rows {m, part, slot} -> (m, c0, c1, slot) with part -1 = all classes"""
    it = np.asarray(items, dtype=np.int64).reshape(-1, 3)
    whole = it[:, 1] < 0
    c0 = np.where(whole, 0, it[:, 1] & 0xff)
    c1 = np.where(whole, ROW_CLASSES, it[:, 1] >> 8)
    return it[:, 0], c0, c1, it[:, 2]


def check_table(sched, items, max_split):
    """assert that a device item table is the one `sched` describes, up to the order inside a bucket and the slot ids"""
    m, c0, c1, slot = decode(items)
    assert len(m) == sched["item_count"], f"{len(m)} items, expected {sched['item_count']}"
    start = 0
    for b in sched["order"]:
        exp = sched["buckets"][b]
        got = np.stack([m, c0, c1], axis=1)[start:start + len(exp)]
        got = got[np.lexsort((got[:, 2], got[:, 1], got[:, 0]))]
        assert np.array_equal(got, exp), f"bucket {b} (items {start}..{start + len(exp)}): contents differ from the restatement"
        start += len(exp)
    # slot rules: whole samples have none; a split sample's parts share one slot, slots are distinct and < max_split, and the
    # parts' class ranges tile [0, ROW_CLASSES) exactly once
    whole = (c0 == 0) & (c1 == ROW_CLASSES)
    assert np.all(slot[whole] == -1) and np.all(slot[~whole] >= 0) and np.all(slot[~whole] < max_split), "split slot out of range"
    seen = {}
    for k in np.flatnonzero(~whole):
        seen.setdefault(int(m[k]), []).append((int(c0[k]), int(c1[k]), int(slot[k])))
    slots = set()
    for s, parts in seen.items():
        ss = {p[2] for p in parts}
        assert len(ss) == 1, f"sample {s}: parts in slots {sorted(ss)}"
        assert not (ss & slots), f"sample {s}: slot {ss} shared with another sample"
        slots |= ss
        assert len(parts) == sched["f"][s], f"sample {s}: {len(parts)} parts, expected {sched['f'][s]}"
        edge = 0
        for a, e, _ in sorted(parts):
            assert a == edge and e > a, f"sample {s}: class ranges {sorted(parts)} do not tile [0, {ROW_CLASSES})"
            edge = e
        assert edge == ROW_CLASSES, f"sample {s}: class ranges {sorted(parts)} do not tile [0, {ROW_CLASSES})"


def simulate_table(sched, max_split, rng):
    """a table as the device may lay it out: buckets in descending order, a random order inside each bucket (a split sample's parts
    kept together) and random distinct slots"""
    f = sched["f"]
    heavy = np.flatnonzero(f > 1)
    slot_of = dict(zip(heavy.tolist(), rng.permutation(max_split)[:len(heavy)].tolist()))
    out = []
    for b in sched["order"]:
        r = sched["buckets"][b]
        groups = {}
        for row in r:
            groups.setdefault(int(row[0]), []).append(row)
        for s in rng.permutation(list(groups)):
            for row in groups[int(s)]:
                whole = row[1] == 0 and row[2] == ROW_CLASSES
                out.append((row[0], -1 if whole else int(row[1]) | int(row[2]) << 8, -1 if whole else slot_of[int(s)]))
    return np.array(out, dtype=np.int32).reshape(-1, 3)
