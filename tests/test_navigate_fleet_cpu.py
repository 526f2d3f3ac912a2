"""Evaluator.navigate's host bookkeeping without a GPU: its ragged trajectory set (_Fleet: gather, replace, adopt; _rows) against a plain
numpy restatement of isdf_plan_batch's ragged layout (vehicle b's pieces at piece_off[b]:piece_off[b + 1] of T, and 18 per piece of
coeffs), on torch CPU tensors; and the summary fields navigate, bench_brake.py and decode_plan_results read by name (_field) against
ctypes' own decoding of records filled with random bytes."""
import ctypes as C

import numpy as np
import pytest
import torch
import isdf_b200 as I

CPU = torch.device("cpu")


def _traj(rng, n):
    """a trajectory of n pieces as numpy (T (n,), coeffs (18 n,))"""
    return rng.random(n), rng.random(18 * n)


def _layout(trajs):
    """the ragged layout of a list of numpy trajectories: (piece_off, T, coeffs)"""
    off = np.zeros(len(trajs) + 1, dtype=np.int64)
    off[1:] = np.cumsum([t.size for t, _ in trajs])
    return off, np.concatenate([t for t, _ in trajs] + [np.zeros(0)]), np.concatenate([c for _, c in trajs] + [np.zeros(0)])


def _torch(traj):
    return torch.from_numpy(traj[0]), torch.from_numpy(traj[1])


def _fleet(trajs):
    f = I._Fleet(len(trajs), CPU)
    f.replace({b: _torch(t) for b, t in enumerate(trajs) if t[0].size})
    return f


def _holds(fleet, trajs):
    """the fleet holds exactly trajs, in the ragged layout"""
    off, T, Cc = _layout(trajs)
    assert np.array_equal(fleet.n, np.diff(off)) and np.array_equal(fleet.offh, off)
    assert fleet.piece_off.dtype == torch.int32 and np.array_equal(fleet.piece_off.numpy(), off)
    assert np.array_equal(fleet.T[:off[-1]].numpy(), T) and np.array_equal(fleet.coeffs[:18 * off[-1]].numpy(), Cc)
    for b, (t, c) in enumerate(trajs):
        pT, pC = fleet.pieces(b)
        assert np.array_equal(pT.numpy(), t) and np.array_equal(pC.numpy(), c)


def _gathered(fleet, trajs, vehicles):
    off, T, Cc = fleet.gather(vehicles)
    eo, eT, eC = _layout([trajs[b] for b in vehicles])
    assert off.dtype == torch.int32 and np.array_equal(off.numpy(), eo)
    if eo[-1]:
        assert np.array_equal(T.numpy(), eT) and np.array_equal(Cc.numpy(), eC)
    else:   # the placeholders of a set without pieces
        assert np.array_equal(T.numpy(), np.zeros(1)) and np.array_equal(Cc.numpy(), np.zeros(18))


def test_a_new_fleet_has_no_pieces():
    f = I._Fleet(3, CPU)
    assert np.array_equal(f.n, np.zeros(3)) and np.array_equal(f.piece_off.numpy(), np.zeros(4))
    assert np.array_equal(f.T.numpy(), np.zeros(1)) and np.array_equal(f.coeffs.numpy(), np.zeros(18))


def test_gather_with_empty_vehicles_between_and_out_of_order():
    rng = np.random.default_rng(1)
    trajs = [_traj(rng, n) for n in (2, 0, 3, 0, 0, 1, 4)]
    f = _fleet(trajs)
    _holds(f, trajs)
    for vehicles in ([0, 2, 5, 6], [6, 0, 5, 2], [1, 3], [4, 2, 1, 0], [3, 6, 3], []):
        _gathered(f, trajs, vehicles)


def test_replace_splices_plans_into_vehicles_with_and_without_pieces():
    rng = np.random.default_rng(2)
    trajs = [_traj(rng, n) for n in (2, 0, 3, 0, 1)]
    f = _fleet(trajs)
    new = {1: _traj(rng, 4), 2: _traj(rng, 1), 4: _traj(rng, 5)}
    # the new pieces come as rows of a ragged output dict, as plans and stops do
    off, T, Cc = _layout(list(new.values()))
    d = dict(piece_off=torch.from_numpy(off.astype(np.int32)), T=torch.from_numpy(T), coeffs=torch.from_numpy(Cc))
    rows = {b: I._rows(d, off, j) for j, b in enumerate(new)}
    for j, b in enumerate(new):
        assert np.array_equal(rows[b][0].numpy(), new[b][0]) and np.array_equal(rows[b][1].numpy(), new[b][1])
    f.replace(rows)
    trajs = [new.get(b, t) for b, t in enumerate(trajs)]
    _holds(f, trajs)
    _gathered(f, trajs, [4, 3, 1])


def test_dropping_vehicles_and_then_every_vehicle():
    rng = np.random.default_rng(3)
    trajs = [_traj(rng, n) for n in (2, 3, 0, 1)]
    f = _fleet(trajs)
    f.replace({b: (f.T[:0], f.coeffs[:0]) for b in (0, 3)})
    trajs = [trajs[b] if b in (1, 2) else (np.zeros(0), np.zeros(0)) for b in range(4)]
    _holds(f, trajs)
    f.replace({b: (f.T[:0], f.coeffs[:0]) for b in range(4)})
    _holds(f, trajs[2:3] * 4)
    assert np.array_equal(f.T.numpy(), np.zeros(1)) and np.array_equal(f.coeffs.numpy(), np.zeros(18))
    _gathered(f, [(np.zeros(0), np.zeros(0))] * 4, [2, 0])


def test_adopt_takes_outputs_with_spare_room():
    rng = np.random.default_rng(4)
    trajs = [_traj(rng, n) for n in (1, 0, 2, 3)]
    off, T, Cc = _layout(trajs)
    spare = 7   # the shift and brake outputs have room past piece_off[B]
    d = dict(piece_off=torch.from_numpy(off.astype(np.int32)), T=torch.from_numpy(np.concatenate([T, rng.random(spare)])),
             coeffs=torch.from_numpy(np.concatenate([Cc, rng.random(18 * spare)])))
    f = I._Fleet(4, CPU)
    f.adopt(d)
    _holds(f, trajs)
    _gathered(f, trajs, [3, 0, 1])
    for j, t in enumerate(trajs):
        rT, rC = I._rows(d, off, j)
        assert np.array_equal(rT.numpy(), t[0]) and np.array_equal(rC.numpy(), t[1])
    new = _traj(rng, 2)
    f.replace({1: _torch(new)})
    trajs[1] = new
    _holds(f, trajs)
    assert f.T.numel() == sum(t.size for t, _ in trajs)   # a splice keeps no spare room


READ = [(I.CertifySummary, ["verdict", "first_hit"]), (I.BrakeSummary, ["status"]), (I.SimSummary, ["diverged"]),
        (I.FrontierGoal, ["kind", "point"]), (I.PlanResult, [n for n, _ in I.PlanResult._fields_])]


@pytest.mark.parametrize("struct,names", READ, ids=[s.__name__ for s, _ in READ])
def test_field_equals_ctypes(struct, names):
    rng = np.random.default_rng(5)
    rows = rng.integers(0, 256, size=(9, C.sizeof(struct)), dtype=np.uint8)
    for name in names:
        got = I._field(torch.from_numpy(rows), struct, name)
        for k, row in enumerate(rows):
            v = getattr(struct.from_buffer_copy(row.tobytes()), name)
            want = np.array(v[:] if hasattr(v, "_length_") else v, dtype=got.numpy().dtype)
            assert got[k].numpy().shape == want.shape and got[k].numpy().tobytes() == want.tobytes(), (struct.__name__, name, k)
    if struct is I.PlanResult:   # decode_plan_results reads every field by name
        res = I.decode_plan_results(torch.from_numpy(rows))
        assert list(res) == names
        for name in names:
            assert res[name].numpy().tobytes() == I._field(torch.from_numpy(rows), struct, name).numpy().tobytes(), name
