"""isdf_trajectory_shift / _device: bit for bit the restatement of tests/navigate_oracle.py on ragged batches of random and planned
trajectories, the states of the rest at t equal the input's at t0 + t, junction and end cases, and host = device."""
import numpy as np
import pytest
import isdf_b200 as I
import navigate_oracle as NO

pytestmark = pytest.mark.gpu


def _ragged(rng, counts):
    off = np.zeros(len(counts) + 1, dtype=np.int32)
    off[1:] = np.cumsum(counts)
    T = rng.uniform(0.3, 1.7, off[-1])
    Cc = np.concatenate([rng.normal(0, 2, 18 * n) for n in counts]) if off[-1] else np.zeros(0)
    return off, T, Cc


def _times(rng, off, T):
    t0 = []
    for b in range(len(off) - 1):
        Tb = T[off[b]:off[b + 1]]
        D = float(np.sum(Tb)) if len(Tb) else 1.0
        kind = b % 6
        t0.append([rng.uniform(0, D), 0.0, float(Tb[0]) if len(Tb) else 0.0, D, D + 1, np.nan][kind])
    return np.array(t0)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def test_bit_identical_to_the_restatement_host_and_device():
    import torch
    rng = np.random.default_rng(11)
    ev = I.Evaluator()
    for counts in ([1], [3, 0, 5, 1, 2, 7, 4, 1, 9, 2, 1, 3], list(rng.integers(0, 12, 200))):
        off, T, Cc = _ragged(rng, counts)
        t0 = _times(rng, off, T)
        ro, rT, rC = NO.shift(off, T, Cc, t0)
        ho, hT, hC = ev.trajectory_shift((off, T, Cc), t0)
        assert np.array_equal(ho, ro) and np.array_equal(_bits(hT), _bits(rT)) and np.array_equal(_bits(hC), _bits(rC))
        cu = lambda a, dt=torch.float64: torch.as_tensor(a, dtype=dt, device="cuda")
        d = ev.trajectory_shift_device(cu(off, torch.int32), cu(T), cu(Cc), cu(t0))
        do = d["piece_off"].cpu().numpy()
        P = int(do[-1])
        assert np.array_equal(do, ro) and np.array_equal(_bits(d["T"][:P].cpu().numpy()), _bits(rT))
        assert np.array_equal(_bits(d["coeffs"][:18 * P].cpu().numpy()), _bits(rC))
    ev.close()


def test_states_of_the_rest_follow_the_input():
    rng = np.random.default_rng(12)
    ev = I.Evaluator()
    off, T, Cc = _ragged(rng, [4, 6, 2, 5])
    t0 = np.array([0.7, float(T[4] + T[5]), 0.01, float(np.sum(T[12:17])) - 0.05])
    oo, oT, oC = ev.trajectory_shift((off, T, Cc), t0)
    B = len(t0)
    for b in range(B):
        Db = float(np.sum(oT[oo[b]:oo[b + 1]]))
        ts = np.linspace(0, Db, 23)
        a = ev.trajectory_states((oo, oT, oC), np.full(ts.size, b), ts)
        ref = ev.trajectory_states((off, T, Cc), np.full(ts.size, b), t0[b] + ts)
        for lo, hi in ((0, 3), (3, 6), (6, 9)):
            scale = max(np.abs(ref[:, lo:hi]).max(), 1.0)
            assert np.abs(a[:, lo:hi] - ref[:, lo:hi]).max() <= 1e-9 * scale, (b, lo)
    ev.close()


def test_junction_and_end_cases():
    ev = I.Evaluator()
    rng = np.random.default_rng(13)
    off, T, Cc = _ragged(rng, [3])
    T[:] = [0.5, 0.25, 1.0]
    for t0, n in ((0.0, 3), (0.5, 2), (0.75, 1), (1.0, 1), (1.75, 0), (-0.1, 0), (np.inf, 0)):
        oo, oT, _ = ev.trajectory_shift((off, T, Cc), [t0])
        assert int(oo[1]) == n, t0
    oo, oT, oC = ev.trajectory_shift((off, T, Cc), [0.0])
    assert np.array_equal(_bits(oT), _bits(T)) and np.array_equal(_bits(oC), _bits(Cc))
    # host-form refusals: a non-positive duration, decreasing offsets
    with pytest.raises(I.IsdfError):
        ev.trajectory_shift((off, np.array([0.5, 0.0, 1.0]), Cc), [0.1])
    with pytest.raises(I.IsdfError):
        ev.trajectory_shift((np.array([0, 3, 2], dtype=np.int32), T, Cc), [0.1, 0.1])
    ev.close()
