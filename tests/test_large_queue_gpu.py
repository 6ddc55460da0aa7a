"""The large-list queue at its bound: every touched cell holds exactly 9 records, so every cell that a call touches is
an entry of the queue of cells with more than 8 records, and a call of max_points points fills that queue to
max_points / 9 entries.  Both the gem_fuse path and the pipelined add (with a scroll clear across cells the fold of the
call before the move still holds) are compared with the oracle bit for bit, and stats() with a numpy bincount."""
import ctypes as C

import numpy as np
import pytest

import fold_cases as fc
import gem_b200
from helpers import assert_layers_equal
from oracle_lib import OracleMap

pytestmark = pytest.mark.gpu

K = 9                       # records per cell: one more than chunk 0 holds
NC = fc.L * fc.L
P = K * NC                  # max_points: the queue's bound is P / 9 = every cell of the map


def _stats_of(keys):
    cnt = np.bincount(keys[keys >= 0], minlength=NC)
    return {"points_binned": int(cnt.sum()), "cells_touched": int(np.count_nonzero(cnt)),
            "max_points_per_cell": int(cnt.max())}


def _keys(xyzi, frame, position=None):
    """the oracle's process_points on a fresh map (moved to `position`): the cell of every point or -1"""
    o = OracleMap(fc.L, fc.RES, compat_box_filter=False)
    if position is not None:
        o.move(position)
    key = o.process_points(xyzi[:, 0], xyzi[:, 1], xyzi[:, 2], frame)[0]
    o.close()
    return key


def _check_stats(g, keys):
    st = g.stats()
    want = _stats_of(keys)
    assert {k: st[k] for k in want} == want, (st, want)


def _fuse_call(rng):
    """P records, K per cell of the whole map, cells interleaved in index order.  Heights near a per-cell level with
    5-sigma jumps in both directions, variances on both sides of the 1e-4 floor, and every fifth record without a
    colour (so the cell's colour and intensity come from a record other than the last one)"""
    key = np.repeat(np.arange(NC, dtype=np.int32), K)
    base = np.repeat(rng.uniform(-1.0, 1.0, NC), K)
    h = base + rng.normal(0.0, 0.02, P)
    jump = rng.random(P) < 0.1
    h[jump] += rng.choice([-0.5, 0.5], int(jump.sum()))
    v = rng.uniform(5e-5, 4e-3, P)
    rgb = rng.integers(1, 256, (P, 3))
    rgb[rng.random(P) < 0.2] = 0
    inten = rng.uniform(0.0, 255.0, P)
    perm = rng.permutation(P)
    return (key[perm], rgb[perm, 0].astype(np.int32), rgb[perm, 1].astype(np.int32), rgb[perm, 2].astype(np.int32),
            inten[perm].astype(np.float32), h[perm].astype(np.float32), v[perm].astype(np.float32))


def test_large_queue_full_gem_fuse():
    """two gem_fuse calls of exactly max_points records: the first folds into empty cells, the second into the state
    the first left (both record parities)"""
    rng = np.random.default_rng(11)
    g = gem_b200.ElevationMap(fc.L, fc.RES, compat_box_filter=False, max_points=P)
    o = OracleMap(fc.L, fc.RES, compat_box_filter=False)
    for call in range(2):
        args = _fuse_call(rng)
        for m in (g, o):
            m.fuse_points(*args)
        assert_layers_equal(g, o, what=f"gem_fuse call {call}")
        _check_stats(g, args[0])
        assert g.stats()["cells_touched"] == NC and g.stats()["points_binned"] == P


def test_large_queue_full_pipelined_add_with_scroll():
    """add_stream_fast of max_points points, K per cell, back to back (both record parities); then a move whose cleared
    rows hold cells the pending fold still has to fold (it runs beside the next call's bin kernel and must write the
    cleared value)"""
    import torch
    sp = gem_b200.LaserSensorProcessor(ignore_points_above=100.0, ignore_points_below=-100.0)
    f = gem_b200.make_frame(np.eye(4), sp)
    rng = np.random.default_rng(12)
    want = {c: K for c in range(NC)}
    xyzi, rgba = fc.place_points(want, rng)
    got, binned = fc.count_cells(xyzi, f)
    assert got == want and binned == P
    g = gem_b200.ElevationMap(fc.L, fc.RES, compat_box_filter=False, max_points=P)
    o = OracleMap(fc.L, fc.RES, compat_box_filter=False)
    xd, rd = torch.from_numpy(xyzi).cuda(), torch.from_numpy(rgba).cuda()
    torch.cuda.synchronize()
    xp, rp = C.c_void_p(xd.data_ptr()), C.c_void_p(rd.data_ptr())
    for _ in range(3):
        g.add_stream_fast(xp, rp, P, C.byref(f))
    g.move([0.3, 0.0, 0.0])
    for _ in range(3):
        g.add_stream_fast(xp, rp, P, C.byref(f))
    g.sync()
    for _ in range(3):
        o.add(xyzi, rgba, f)
    before = o.get_layer("elevation").reshape(-1)
    o.move([0.3, 0.0, 0.0])
    after = o.get_layer("elevation").reshape(-1)
    assert np.count_nonzero((before != -10) & (after == -10)) >= fc.L, "the scroll must clear whole rows of touched cells"
    for _ in range(3):
        o.add(xyzi, rgba, f)
    assert_layers_equal(g, o, what="pipelined add, across the scroll")
    _check_stats(g, _keys(xyzi, f, [0.3, 0.0, 0.0]))
