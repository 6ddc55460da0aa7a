"""Every fold path against the oracle, with crafted per-cell record lists (tests/fold_cases.py).

Value families (gate bands, skip records, magnitude edges, numerator cancellation, non-finite heights, start states,
colours, a state that returns to -10 in the middle of a list) go through gem_fuse; the list-length sweep (1 ... 10921
records in one cell) goes through gem_fuse, gem_fuse_records, the serial add from device memory and the pipelined
add.  Every comparison is all layers, bit for bit."""
import ctypes as C

import numpy as np
import pytest

import fold_cases as fc
import gem_b200
import np_reference
from helpers import assert_layers_equal
from oracle_lib import OracleMap

pytestmark = pytest.mark.gpu

ROUTE_REC = np.dtype([("gkey", "<i4"), ("h", "<f4"), ("var", "<f4"), ("rgb", "<u4"), ("intensity", "<f4")])


def _frame():
    """identity pose, laser model, a height window wide enough for every crafted point"""
    sp = gem_b200.LaserSensorProcessor(ignore_points_above=100.0, ignore_points_below=-100.0)
    return gem_b200.make_frame(np.eye(4), sp)


def _pair(s=None, max_points=0):
    g = gem_b200.ElevationMap(fc.L, fc.RES, compat_box_filter=False, max_points=max_points)
    o = OracleMap(fc.L, fc.RES, compat_box_filter=False)
    if s is not None:
        s.apply_init(g)
        s.apply_init(o)
    return g, o


def _check_stats(g, longest, binned):
    st = g.stats()
    assert st["max_points_per_cell"] == longest, st
    assert st["points_binned"] == binned, st


# ---- value families through gem_fuse ---------------------------------------------------------------------------------
def test_value_families_one_call():
    s = fc.value_families()
    g, o = _pair(s)
    for m in (g, o):
        m.fuse_points(*s.fuse_args())
    assert_layers_equal(g, o, what="value families")
    _check_stats(g, max(s.lists().values()), s.n)


@pytest.mark.parametrize("family", sorted(fc.FAMILIES) + sorted(fc.START_FAMILIES))
def test_value_family(family):
    """one family per call: a difference names its family"""
    s = fc.value_families()
    cells = [c for c, p in s.plans.items() if p.family == family]
    sel = np.isin(s.key, cells)
    args = [a[sel] for a in s.fuse_args()]
    g, o = _pair(s, max_points=1 << 16)
    for m in (g, o):
        m.fuse_points(*args)
    assert_layers_equal(g, o, what=family)
    _check_stats(g, max(s.plans[c].k for c in cells), int(sel.sum()))


# ---- the length sweep ------------------------------------------------------------------------------------------------
def test_length_sweep_gem_fuse():
    s = fc.length_sweep()
    g, o = _pair(s)
    for m in (g, o):
        m.fuse_points(*s.fuse_args())
    assert_layers_equal(g, o, what="length sweep, gem_fuse")
    _check_stats(g, 10921, s.n)


def test_length_sweep_gem_fuse_records():
    """SRC_RECORDS: 20-byte RouteRec {gkey = gx*L + gy, h, var, rgb, intensity} from device memory; the record's slot
    is its point index.  This path also runs the lowest-scan"""
    import torch
    s = fc.length_sweep()
    rec = np.zeros(s.n, ROUTE_REC)
    rec["gkey"], rec["h"], rec["var"], rec["intensity"] = s.key, s.h, s.v, s.I
    rec["rgb"] = (s.R.astype(np.uint32) & 255) | ((s.G.astype(np.uint32) & 255) << 8) | ((s.B.astype(np.uint32) & 255) << 16)
    d = torch.from_numpy(rec.view(np.uint8).copy()).cuda()
    torch.cuda.synchronize()
    g, o = _pair(s)
    g.fuse_records(d, s.n)
    g.sync()
    o.fuse_points(*s.fuse_args())
    o.set_layer("lowest", np_reference.lowest_update(o.get_layer("lowest"), s.key, s.h, s.v))
    assert_layers_equal(g, o, what="length sweep, gem_fuse_records")
    _check_stats(g, 10921, s.n)


def test_length_sweep_serial_add_from_device():
    import torch
    f = _frame()
    ps = fc.sweep_points(f)
    g, o = _pair()
    xd, rd = torch.from_numpy(ps.xyzi).cuda(), torch.from_numpy(ps.rgba).cuda()
    torch.cuda.synchronize()
    g.add(xd, rd, f)
    g.sync()
    o.add(ps.xyzi, ps.rgba, f)
    assert_layers_equal(g, o, what="length sweep, serial add")
    _check_stats(g, 10921, ps.binned)


def test_length_sweep_pipelined_add_with_scroll():
    """add_stream_fast back to back (both record parities), then a move whose cleared rows hold lists longer than 40:
    the fold of the call before the move runs beside the next call's bin kernel and writes the cleared value into
    those cells (in_clear_region on warp-folded cells)"""
    import torch
    f = _frame()
    ps = fc.sweep_points(f)
    n = ps.xyzi.shape[0]
    g, o = _pair()
    xd, rd = torch.from_numpy(ps.xyzi).cuda(), torch.from_numpy(ps.rgba).cuda()
    torch.cuda.synchronize()
    xp, rp = C.c_void_p(xd.data_ptr()), C.c_void_p(rd.data_ptr())
    for _ in range(3):
        g.add_stream_fast(xp, rp, n, C.byref(f))
    g.move([0.3, 0.0, 0.0])
    for _ in range(3):
        g.add_stream_fast(xp, rp, n, C.byref(f))
    g.sync()
    for _ in range(3):
        o.add(ps.xyzi, ps.rgba, f)
    before = o.get_layer("elevation").reshape(-1)
    o.move([0.3, 0.0, 0.0])
    after = o.get_layer("elevation").reshape(-1)
    long_cells = [c for c, k in ps.lists.items() if k > 40]
    cleared = [c for c in long_cells if before[c] != -10 and after[c] == -10]
    assert len(cleared) >= 2, "the scroll must clear cells that hold long lists"
    for _ in range(3):
        o.add(ps.xyzi, ps.rgba, f)
    assert_layers_equal(g, o, what="length sweep, pipelined add")


# ---- the largest launch ------------------------------------------------------------------------------------------------
def test_largest_launch_and_chunked_call():
    """max_points = 2^22 (FOLD_INDEX_BITS): one call of 2^22 points whose cells with 65..1024 records have their records
    at indices close to 2^22 - 1 (the (index << 10 | rank) sort key at its limit), then one call of more than
    max_points points (chunked)"""
    import torch
    P = 1 << 22
    rng = np.random.default_rng(5)
    f = _frame()
    perm = rng.permutation(fc.L * fc.L)
    long_k = {int(c): k for c, k in zip(perm, (65, 100, 128, 129, 200, 256, 257, 512, 513, 700, 1024))}
    others = perm[len(long_k):]
    xl, rl = fc.place_points(long_k, rng)
    nl = xl.shape[0]
    nb = P - nl
    nin = 300000                                        # background points inside the grid, in the other cells
    cc = others[rng.integers(0, others.shape[0], nin)]
    cx, cy = (fc.L / 2 - cc // fc.L - 0.5) * fc.RES, (fc.L / 2 - cc % fc.L - 0.5) * fc.RES
    xin = np.stack([cx + rng.uniform(-0.3, 0.3, nin) * fc.RES, cy + rng.uniform(-0.3, 0.3, nin) * fc.RES,
                    rng.uniform(0.5, 1.5, nin), rng.integers(0, 256, nin)], 1)
    xout = np.stack([rng.uniform(50, 60, nb - nin), rng.uniform(-5, 5, nb - nin), rng.uniform(0.5, 1.5, nb - nin),
                     rng.integers(0, 256, nb - nin)], 1)     # outside the grid
    bg = np.concatenate([xin, xout]).astype(np.float32)[rng.permutation(nb)]
    tail = 4000                                          # the long lists share the last indices with background points
    mix = np.concatenate([bg[nb - tail:], xl])
    mix_rgba = np.concatenate([rng.integers(0, 256, (tail, 4)).astype(np.uint8), rl])
    q = rng.permutation(mix.shape[0])
    xyzi = np.concatenate([bg[:nb - tail], mix[q]]).astype(np.float32)
    rgba = np.concatenate([rng.integers(0, 256, (nb - tail, 4)).astype(np.uint8), mix_rgba[q]])
    assert xyzi.shape[0] == P
    counts, binned = fc.count_cells(xyzi, f)
    assert {c: counts[c] for c in long_k} == long_k
    assert max(counts.values()) == 1024
    o = OracleMap(fc.L, fc.RES, compat_box_filter=False)
    key = o.process_points(xyzi[:, 0], xyzi[:, 1], xyzi[:, 2], f)[0]
    first = np.nonzero(np.isin(key, list(long_k)))[0].min()
    assert first >= P - nl - tail                        # every record of a long list sits near the top of the range
    o.close()

    g, o = _pair(max_points=P)
    xd, rd = torch.from_numpy(xyzi).cuda(), torch.from_numpy(rgba).cuda()
    torch.cuda.synchronize()
    g.add(xd, rd, f)
    g.sync()
    o.add(xyzi, rgba, f)
    assert_layers_equal(g, o, what="2^22 points")
    _check_stats(g, 1024, binned)

    # more than max_points: the call is folded in chunks of max_points, each one like a call of its own
    extra = 3000
    xe, re = fc.place_points({c: extra // len(long_k) + 1 for c in long_k}, rng)
    x2 = np.concatenate([xyzi, xe[:extra]]).astype(np.float32)
    r2 = np.concatenate([rgba, re[:extra]])
    xd2, rd2 = torch.from_numpy(x2).cuda(), torch.from_numpy(r2).cuda()
    torch.cuda.synchronize()
    del xd, rd
    g.add(xd2, rd2, f)
    g.sync()
    o.add(x2[:P], r2[:P], f)
    o.add(x2[P:], r2[P:], f)
    assert_layers_equal(g, o, what="2^22 + 3000 points, chunked")
    st = g.stats()
    assert st["points_in"] == P + extra and st["points_binned"] == binned + extra, st
    assert st["max_points_per_cell"] == 1024, st
