"""gem_tiled_step, the peer-stored tiled add path, on one GPU against the CPU oracle: k_route_peer, k_bin_peer with its
bin_one, the depth-2 and depth-3 step graphs and the five receive buffers reused by step.

Everything runs in one process on cuda:0.  The receive buffers are plain device tensors laid out as TiledElevationMap lays
out its symmetric-memory buffers (records int32 [5, W*cap, 4], intensities float32 [5, W*cap], counts int32 [5, W*nblk]
zeroed, flags int32 [64] zeroed, one set per rank); their addresses go to ElevationMap.tiled_attach.

* World 1: one tile owns the map.  Its bin waits only on its own flag, raised by a route ordered before it, so every
  schedule runs: serial with profiling on, graph at depth 2 and graph at depth 3.
* One rank of a W-rank tiling, the other ranks absent: the foreign words of the rank's own flag array are preset to
  INT32_MAX and the foreign counts stay zero, so its bin never waits.  What the route stored into every owner's buffer
  (slots, counts, flags) is checked record by record against a numpy model of the routing.
* W tile handles on the one device, stepped round-robin under the depth-3 graph schedule, where call j bins step j - 1
  and the draining read bins the last routed step: no bin waits for a rank that has not stepped yet, and every flag word
  a call's bin waits on is checked on the host before the call is made.

A tiled handle never scrolls, so the oracle map stays at its initial position.  Every layer is compared bit for bit on
the tile's slice (NaN == NaN); a difference names the layer, the tile, the step, the number of cells and the first one."""
import numpy as np
import pytest

import gem_b200
from gem_b200 import synth, tiled
from gem_b200._lib import GemError
from oracle_lib import OracleMap

pytestmark = pytest.mark.gpu

LAYERS = ["elevation", "variance", "intensity", "color_r", "color_g", "color_b", "lowest"]
ENV = ("GEM_B200_TILED_DEPTH", "GEM_B200_EXCLUSIVE", "GEM_B200_FOLD_BLOCKS", "GEM_B200_LONG_BLOCKS")
SCHEDULES = {
    "profile": {},                           # gem_profile_enable: every step routed, binned and folded inside its call
    "graph_depth2": {"GEM_B200_TILED_DEPTH": "2"},
    "graph_depth3": {"GEM_B200_TILED_DEPTH": "3"},
}
RES = 0.1
INT32_MAX = 2**31 - 1
MAX_LAUNCH = 1 << 22               # gem_create caps max_points at the fold's 22-bit point index
CAP = 140_032                      # 547 blocks of 256: an HDL-64 frame (about 130k returns) fits
# records per cell that fill one chunk level of the bin and start the next: 8 | 9 (level 1), 40 | 41 (2), 168 | 169 (3),
# 680 | 681 (4), 2729 and 3000 (level 5: a record's walk follows the published pointers of levels 2, 3 and 4)
CHUNK_CELLS = (8, 9, 40, 41, 168, 169, 680, 681, 2729, 3000)
_SCENE = synth.make_scene()
_HDL = {}


def _env(monkeypatch, schedule):
    for k in ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in SCHEDULES[schedule].items():
        monkeypatch.setenv(k, v)                 # gem_create and gem_tiled_attach read the schedule


def _frame(T):
    return gem_b200.make_frame(T, gem_b200.LaserSensorProcessor())


def _pose(x, y, yaw=0.0):
    return synth.pose_matrix(x, y, synth.SENSOR_HEIGHT, yaw)


def _hdl(k):
    if k not in _HDL:
        _HDL[k] = synth.hdl64_frame(k, scene=_SCENE)
    return _HDL[k]


def _cloud(xyzi, rgba, T):
    return {"xyzi": np.ascontiguousarray(xyzi, np.float32), "rgba": None if rgba is None else np.ascontiguousarray(rgba, np.uint8),
            "T": T}


def _hdl_cloud(k, x=None, y=None, n=None, rgba=True, every=1):
    fr = _hdl(k)
    T = fr["T"].copy()
    if x is not None:
        T[0, 3], T[1, 3] = x, y
    xyzi, c = fr["xyzi"][::every], fr["rgba"][::every]
    if n is not None:
        xyzi, c = xyzi[:n], c[:n]
    return _cloud(xyzi, c if rgba else None, T)


def _chunk_level_cloud(seed, ox, oy):
    """one cell per entry of CHUNK_CELLS (a row of cells 0.3 m apart from (ox, oy)), the cells' records shuffled together so
    that every cell's list spans many warps and blocks, heights spread over the gate, 5 % more points above the height
    window, zero intensities and zero colour channels mixed in.  Sensor frame = map frame shifted by the sensor height, so
    a point's cell is the cell of its (x, y)."""
    rng = np.random.default_rng(seed)
    parts = []
    for k, cnt in enumerate(CHUNK_CELLS):
        cx, cy = ox + 0.05 + 0.3 * k, oy + 0.05           # cell centres: cell edges lie on multiples of RES
        m = cnt + cnt // 20
        p = np.stack([cx + rng.uniform(-0.03, 0.03, m), cy + rng.uniform(-0.03, 0.03, m), rng.uniform(-1.83, -1.43, m)], 1)
        p[cnt:, 2] += rng.uniform(2.6, 3.5, m - cnt)         # h > 0.8: rejected by the window
        parts.append(p)
    xyz = np.concatenate(parts)
    n = xyz.shape[0]
    inten = rng.integers(0, 256, n).astype(np.float32)
    inten[rng.uniform(size=n) < 0.1] = 0.0
    rgba = rng.integers(1, 256, (n, 4)).astype(np.uint8)
    zc = rng.uniform(size=n) < 0.1
    rgba[zc, rng.integers(0, 3, int(zc.sum()))] = 0
    order = rng.permutation(n)
    c = _cloud(np.concatenate([xyz, inten[:, None]], 1)[order], rgba[order], _pose(0.0, 0.0))
    c["chunk_cells"] = True
    return c


def _random_cloud(n, seed, ox=0.0, oy=0.0, extent=12.0, rgba=True):
    """uniform points around (ox, oy), some above the height window and some outside a 25.6 m grid, zero intensities and
    zero colour channels mixed in"""
    c = synth.random_cloud(n, seed=seed, extent=extent, zmin=-2.5, zmax=-0.6, zero_colour_frac=0.2)
    xyzi = c["xyzi"].copy()
    xyzi[:, 0] += np.float32(ox)
    xyzi[:, 1] += np.float32(oy)
    xyzi[::7, 3] = 0.0
    return _cloud(xyzi, c["rgba"] if rgba else None, _pose(0.0, 0.0))


def _full_cloud(n, seed):
    """exactly n points: an HDL-64 frame topped up with uniform points"""
    h = _hdl_cloud(9)
    m = n - h["xyzi"].shape[0]
    assert m >= 0, "the HDL-64 frame is larger than the capacity"
    r = synth.random_cloud(m, seed=seed, extent=12.0, zmin=-2.0, zmax=-0.8)
    T = h["T"]
    return _cloud(np.concatenate([h["xyzi"], r["xyzi"]]), np.concatenate([h["rgba"], r["rgba"]]), T)


def _diff(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape:
        return f"shape {a.shape} != {b.shape}"
    if a.dtype.kind == "f":
        a32, b32 = a.astype(np.float32), b.astype(np.float32)
        ok = (a32.view(np.uint32) == b32.view(np.uint32)) | (np.isnan(a32) & np.isnan(b32))
    else:
        ok = a == b
    if ok.all():
        return None
    bad = np.argwhere(~ok)
    i = tuple(int(v) for v in bad[0])
    return f"{bad.shape[0]} cells differ, first at {i}: device={a[i]!r} oracle={b[i]!r}"


def _assert_tile(g, o, rank, world, where):
    r0, nr, c0, nc = tiled.tile_of_rank(rank, world, o.length)
    for name in LAYERS:
        d = _diff(g.get_layer(name), o.get_layer(name)[r0:r0 + nr, c0:c0 + nc])
        assert d is None, f"{where}: layer {name}, tile {rank} of {world} (rows {r0}+{nr}, cols {c0}+{nc}): {d}"


def _oracle_process(o, c):
    """process_points of one cloud on the oracle: (key, var, h) per point"""
    x = c["xyzi"]
    key, var, _, _, zt = o.process_points(x[:, 0], x[:, 1], x[:, 2], _frame(c["T"]))
    return key, var, zt


def _oracle_fuse(o, c, key, var, h):
    x, rgba = c["xyzi"], c["rgba"]
    n = x.shape[0]
    R, G, B = (np.zeros(n, np.int32),) * 3 if rgba is None else (rgba[:, k].astype(np.int32) for k in range(3))
    o.fuse_points(key, R, G, B, x[:, 3], h, var)


def _oracle_add(o, c):
    """one cloud as one step (OracleMap.add for a finite laser cloud); returns the process_points outputs"""
    key, var, h = _oracle_process(o, c)
    _oracle_fuse(o, c, key, var, h)
    if c.get("chunk_cells"):                 # the crafted cloud really has the intended per-cell record counts
        cnt = np.bincount(key[key >= 0])
        assert sorted(cnt[cnt > 0].tolist()) == sorted(CHUNK_CELLS), sorted(cnt[cnt > 0].tolist())
    return key, var, h


def _oracle_frame(o, clouds):
    """one multi-sensor step: the clouds fused in order; `lowest` is the step's per-cell minimum over all of them (first
    point among equals), the ORACLE DEFINITION applied to one call (test_c5_size_8192_frame_and_multi_sensor_vs_oracle)"""
    low0 = o.get_layer("lowest").reshape(-1).copy()
    keys, hs, hvs = [], [], []
    for c in clouds:
        key, var, h = _oracle_process(o, c)
        _oracle_fuse(o, c, key, var, h)
        keys.append(key); hs.append(h); hvs.append(var)
    key, h, hv = np.concatenate(keys), np.concatenate(hs), np.concatenate(hvs)
    ok = key >= 0
    key, h, hv = key[ok], h[ok], hv[ok]
    order = np.lexsort((np.arange(key.size), h, key))
    first = np.ones(key.size, bool)
    first[1:] = key[order][1:] != key[order][:-1]
    ck, cm, cv = key[order][first], h[order][first], hv[order][first]
    expect = low0.copy()
    upd = cm <= low0[ck]
    expect[ck[upd]] = (cm[upd] + np.float32(3.0) * cv[upd]).astype(np.float32)
    o.set_layer("lowest", expect.reshape(o.shape))
    return keys


class PeerBuffers:
    """The receive buffers of a W-rank tiling on cuda:0, one set per rank.

    alias=True (one rank of a large tiling, the other ranks absent): rank r only ever stores into slots
    [b * W * cap + r * cap, + cap) of owner o's buffer b, so the W record and intensity buffers are views into one
    allocation of 6 W cap slots, owner o's starting o * cap slots in.  The ranges rank r writes, (5 buffers x W owners),
    then land at offsets (b * W + r + o) * cap: all distinct.  The own buffer's sub-buckets of other sources overlap
    them, but their counts stay zero and the bin reads no slot past a count."""

    def __init__(self, world, cap, alias=False):
        import torch
        dev = torch.device("cuda", 0)
        assert cap % 256 == 0
        self.world, self.cap, self.nblk = world, cap, cap // 256
        n = world * cap
        if alias:
            rec = torch.empty((6 * n, 4), dtype=torch.int32, device=dev)
            inten = torch.empty((6 * n,), dtype=torch.float32, device=dev)
            self.rec = [rec.as_strided((5, n, 4), (4 * n, 4, 1), 4 * o * cap) for o in range(world)]
            self.inten = [inten.as_strided((5, n), (n, 1), o * cap) for o in range(world)]
            self._keep = (rec, inten)
        else:
            self.rec = [torch.empty((5, n, 4), dtype=torch.int32, device=dev) for _ in range(world)]
            self.inten = [torch.empty((5, n), dtype=torch.float32, device=dev) for _ in range(world)]
        self.cnt = [torch.zeros((5, world * self.nblk), dtype=torch.int32, device=dev) for _ in range(world)]
        self.flag = [torch.zeros(64, dtype=torch.int32, device=dev) for _ in range(world)]
        torch.cuda.synchronize()

    def attach(self, g, rank, bucket_capacity=None):
        tr, tc = tiled.plan_tiles(self.world)
        g.tiled_attach(tr, tc, rank, self.cap if bucket_capacity is None else bucket_capacity,
                       [t.data_ptr() for t in self.rec], [t.data_ptr() for t in self.inten],
                       [t.data_ptr() for t in self.cnt], [t.data_ptr() for t in self.flag])

    def flags(self, owner):
        import torch
        torch.cuda.synchronize()             # device-wide: no library call, so nothing is drained
        return self.flag[owner].cpu().numpy()


def _tile_map(L, rank, world, max_points):
    return gem_b200.ElevationMap(L, RES, compat_box_filter=False, tile=tiled.tile_of_rank(rank, world, L), max_points=max_points)


def _dev(c, keep):
    import torch
    x = torch.from_numpy(c["xyzi"]).cuda()
    r = None if c["rgba"] is None else torch.from_numpy(c["rgba"]).cuda()
    torch.cuda.synchronize()                 # the library works on its own stream
    keep.append((x, r))                      # inputs stay alive while deferred work may still read them
    return x, r


# ---------------------------------------------------------------------------------------------------------------------
# A. world 1
# ---------------------------------------------------------------------------------------------------------------------
def _world1_script():
    """15 steps, so every one of the five receive buffers is reused at least twice; "check" reads stats() and every
    layer (draining the pipeline), "flush" issues what the pipeline deferred without reading"""
    n1 = _hdl(1)["xyzi"].shape[0]
    return [
        ("add", _hdl_cloud(0, 0.0, 0.0)),
        ("add", _chunk_level_cloud(11, -4.0, 2.0)),
        ("add", None),                                           # n = 0
        ("add", _hdl_cloud(1, 1.5, -1.0, n=(n1 // 256) * 256 - 179)),  # n % 256 == 77
        ("add", _hdl_cloud(2, -1.0, 0.5)),
        ("check",),
        ("refuse",),                                             # cap + 1 points: GEM_ERR_INVALID, nothing changes
        ("add", _full_cloud(CAP, 3)),                            # step 6: every sub-bucket of buffer 1 filled
        ("add", _hdl_cloud(3, 0.5, 1.0, rgba=False)),            # rgba = None
        ("add", _random_cloud(20000, 5, extent=15.0)),           # zero intensities / channels, window and grid rejects
        ("flush",),
        ("add", _hdl_cloud(4, -2.0, -2.0)),
        ("add", _hdl_cloud(5, 2.0, 2.0)),
        ("add", _random_cloud(300, 6, ox=-10.0, oy=10.0, extent=1.0)),  # step 11, buffer 1 again: a small cloud elsewhere
        ("check",),
        ("add", _hdl_cloud(6, 0.0, -3.0)),
        ("add", _chunk_level_cloud(12, 3.0, -6.0)),
        ("add", _hdl_cloud(7, -3.0, 0.0)),
        ("add", _random_cloud(CAP - 1, 8, extent=12.0, rgba=False)),
        ("check",),
    ]


@pytest.mark.parametrize("schedule", list(SCHEDULES))
def test_world1_steps_match_oracle(schedule, monkeypatch):
    _env(monkeypatch, schedule)
    import torch
    L = 256
    bufs = PeerBuffers(1, CAP)
    g = _tile_map(L, 0, 1, CAP)
    if schedule == "profile":
        g.profile_enable()
    o = OracleMap(L, RES, compat_box_filter=False)
    keep = []
    step, last_n, last_binned, stats = 0, 0, 0, None
    try:
        bufs.attach(g, 0)
        for item in _world1_script():
            kind = item[0]
            where = f"[{schedule}] step {step}"
            if kind == "add":
                c = item[1]
                step += 1
                where = f"[{schedule}] step {step}"
                if c is None:
                    g.tiled_step(None, None, _frame(_pose(0.0, 0.0)), n=0)
                    last_n, last_binned = 0, 0
                else:
                    x, r = _dev(c, keep)
                    g.tiled_step(x, r, _frame(c["T"]))
                    key, _, _ = _oracle_add(o, c)
                    last_n, last_binned = c["xyzi"].shape[0], int((key >= 0).sum())
                f = bufs.flags(0)
                assert f[0] == step, f"{where}: flag {f[0]}, want the step counter {step}"
            elif kind == "flush":
                g.flush()
            elif kind == "check":
                stats = g.stats()
                assert stats["points_in"] == last_n, f"{where}: stats {stats}: points_in != {last_n}"
                assert stats["points_binned"] == last_binned, f"{where}: stats {stats}: points_binned != oracle {last_binned}"
                _assert_tile(g, o, 0, 1, where)
            elif kind == "refuse":
                big = _random_cloud(CAP + 1, 4)
                x, r = _dev(big, keep)
                with pytest.raises(GemError, match="GEM_ERR_INVALID"):
                    g.tiled_step(x, r, _frame(big["T"]))
                f = bufs.flags(0)
                assert f[0] == step, f"{where}: refused call moved the flag to {f[0]}"
                assert g.stats() == stats, f"{where}: refused call changed stats(): {g.stats()} != {stats}"
                _assert_tile(g, o, 0, 1, where + " after the refused call")
        torch.cuda.synchronize()
    finally:
        g.close()


# ---------------------------------------------------------------------------------------------------------------------
# B. one rank of a W-rank tiling
# ---------------------------------------------------------------------------------------------------------------------
def _preset_absent_peers(bufs, rank):
    import torch
    W, nb = bufs.world, bufs.nblk
    others = [p for p in range(W) if p != rank]
    bufs.flag[rank][others] = INT32_MAX
    torch.cuda.synchronize()
    f = bufs.flags(rank)
    assert (f[others] == INT32_MAX).all() and f[rank] == 0, f"flags of rank {rank} before the first step: {f[:W]}"
    cnt = bufs.cnt[rank].cpu().numpy().reshape(5, W, nb)
    assert not cnt[:, others].any(), f"foreign counts of rank {rank} are not zero"


def _check_routing(bufs, rank, step, L, c, key, var, h, where):
    """owner o's buffer step % 5 holds, at slots [(rank * nblk + b) * 256, + count), exactly the points of source block b
    whose cell lies in tile o, in source order; counts exact (zeros included); flag[o][rank] == step"""
    import torch
    W, cap, nb = bufs.world, bufs.cap, bufs.nblk
    buf = step % 5
    idx = np.flatnonzero(key >= 0)
    gk = key[idx].astype(np.int64)
    own = np.asarray(tiled.owner_of(gk // L, gk % L, W, L), np.int64)
    blk = idx // 256
    grp = blk * W + own
    order = np.argsort(grp, kind="stable")   # idx ascends: stable keeps source order within (block, owner)
    gs = grp[order]
    within = np.empty(idx.size, np.int64)
    within[order] = np.arange(gs.size) - np.searchsorted(gs, gs, side="left")
    want_cnt = np.bincount(grp, minlength=nb * W).reshape(nb, W).T
    torch.cuda.synchronize()
    for o in range(W):
        got = bufs.cnt[o][buf, rank * nb:(rank + 1) * nb].cpu().numpy()
        d = _diff(got, want_cnt[o])
        assert d is None, f"{where}: counts of source {rank} in owner {o}'s buffer {buf} (by source block): {d}"
        fl = int(bufs.flag[o][rank].item())
        assert fl == step, f"{where}: flag[{o}][{rank}] = {fl}, want {step}"
    rec = torch.stack([bufs.rec[o][buf, rank * cap:(rank + 1) * cap] for o in range(W)]).cpu().numpy()
    inten = torch.stack([bufs.inten[o][buf, rank * cap:(rank + 1) * cap] for o in range(W)]).cpu().numpy()
    slot = blk * 256 + within
    got = rec[own, slot]
    rgba = c["rgba"]
    rgb = np.zeros(idx.size, np.int64) if rgba is None else (
        rgba[idx, 0].astype(np.int64) | (rgba[idx, 1].astype(np.int64) << 8) | (rgba[idx, 2].astype(np.int64) << 16))
    want = np.stack([gk, h[idx].view(np.int32), var[idx].view(np.int32), rgb], 1).astype(np.int64).astype(np.int32)
    for k, field in enumerate(("gkey", "h bits", "var bits", "rgb")):
        bad = np.flatnonzero(got[:, k] != want[:, k])
        assert bad.size == 0, (f"{where}: routed {field} differs in {bad.size} of {idx.size} records; first: point {idx[bad[0]]} "
                               f"-> owner {own[bad[0]]} slot {rank * cap + slot[bad[0]]}: device {got[bad[0], k]} model {want[bad[0], k]}")
    gi, wi = inten[own, slot].view(np.uint32), c["xyzi"][idx, 3].view(np.uint32)
    bad = np.flatnonzero(gi != wi)
    assert bad.size == 0, (f"{where}: routed intensity differs in {bad.size} of {idx.size} records; first: point {idx[bad[0]]} "
                           f"-> owner {own[bad[0]]} slot {rank * cap + slot[bad[0]]}")
    return int(idx.size)


def _run_one_rank(world, rank, L, cap, clouds, bufs, where0):
    import torch
    g = _tile_map(L, rank, world, world * cap)
    o = OracleMap(L, RES, compat_box_filter=False)
    keep = []
    try:
        bufs.attach(g, rank)
        _preset_absent_peers(bufs, rank)
        routed = 0
        for step, c in enumerate(clouds, start=1):
            where = f"{where0} step {step}"
            if c is None:
                g.tiled_step(None, None, _frame(_pose(0.0, 0.0)), n=0)
                c = _cloud(np.zeros((0, 4), np.float32), None, _pose(0.0, 0.0))
            else:
                x, r = _dev(c, keep)
                g.tiled_step(x, r, _frame(c["T"]))
            torch.cuda.synchronize()
            key, var, h = _oracle_add(o, c)
            routed += _check_routing(bufs, rank, step, L, c, key, var, h, where)
            _assert_tile(g, o, rank, world, where)
            f = bufs.flags(rank)
            others = [p for p in range(world) if p != rank]
            assert (f[others] == INT32_MAX).all(), f"{where}: a foreign flag of rank {rank} changed: {f[:world]}"
        assert routed > 10000, f"{where0}: only {routed} routed records"
    finally:
        g.close()


@pytest.mark.parametrize("world,rank", [(2, 1), (4, 1), (64, 27)])
def test_one_rank_of_a_tiling_routes_and_folds(world, rank, monkeypatch):
    """rank 27 of 64 owns the interior tile (3, 3) of an 8 x 8 tiling; at world 64 the clouds are thinned to 16k points
    so that all 64 buffer sets (5 x 64 x 16384 records each) fit in 7 GB"""
    _env(monkeypatch, "graph_depth2")
    L = 512
    every, cap = (1, CAP) if world <= 4 else (9, 16384)
    n1 = _hdl(1)["xyzi"].shape[0] // every
    clouds = [
        _hdl_cloud(0, -3.0, 2.0, every=every),
        _hdl_cloud(1, 4.0, -1.0, n=n1 // 3, every=every),
        None,
        _chunk_level_cloud(21, 6.0, 0.1) if world == 64 else _hdl_cloud(2, 0.0, 0.0),
        _hdl_cloud(3, 1.0, 1.0, rgba=False, every=every),
        _random_cloud(500, 22, ox=-12.0, oy=12.0, extent=2.0),       # buffer 1 again, after the full step 1
        _hdl_cloud(4, -5.0, 5.0, every=every),
        _chunk_level_cloud(23, -1.5, 0.0),                           # across the seams at the map centre
    ]
    bufs = PeerBuffers(world, cap)
    _run_one_rank(world, rank, L, cap, clouds, bufs, f"rank {rank} of {world}")


# ---------------------------------------------------------------------------------------------------------------------
# C. several ranks on one GPU, depth 3
# ---------------------------------------------------------------------------------------------------------------------
def _require_flags(bufs, rank, step, where):
    """the flag words rank's bin of `step` waits on must already hold >= step; otherwise the call is not made"""
    f = bufs.flags(rank)[:bufs.world]
    if (f < step).any():
        pytest.fail(f"{where}: rank {rank}'s bin of step {step} would wait on flags {f.tolist()}; call not made")


def _seam_cloud(rank, step, world):
    """rank's sensor near the map centre, where the tile seams meet"""
    k = 10 * step + rank
    return _hdl_cloud(k, -6.0 + 12.0 * (rank % 2) + 0.5 * step, -5.0 + 10.0 * (rank // 2))


@pytest.mark.parametrize("world", [2, 4])
def test_ranks_round_robin_depth3_match_multi_sensor_oracle(world, monkeypatch):
    _env(monkeypatch, "graph_depth3")
    import torch
    L = 512
    bufs = PeerBuffers(world, CAP)
    maps = [_tile_map(L, r, world, world * CAP) for r in range(world)]
    o = OracleMap(L, RES, compat_box_filter=False)
    keep = []
    routed = [None] * world                      # per rank: the step routed and not binned yet
    try:
        for r, g in enumerate(maps):
            bufs.attach(g, r)

        def drain_all(where):
            for r, g in enumerate(maps):
                if routed[r] is not None:
                    _require_flags(bufs, r, routed[r], where)
                g.flush()
                torch.cuda.synchronize()
                routed[r] = None

        def check(where, keys):
            drain_all(where)
            for r, g in enumerate(maps):
                _assert_tile(g, o, r, world, where)
                mine = sum(int((np.asarray(tiled.owner_of(k[k >= 0] // L, k[k >= 0] % L, world, L)) == r).sum()) for k in keys)
                st = g.stats()
                assert st["points_binned"] == mine, f"{where}: rank {r} stats {st}: points_binned != oracle {mine}"

        steps = 8
        for j in range(1, steps + 1):
            clouds = [_seam_cloud(r, j, world) for r in range(world)]
            for r, g in enumerate(maps):
                where = f"[{world} ranks, depth 3] step {j} rank {r}"
                if routed[r] is not None:
                    _require_flags(bufs, r, routed[r], where)
                x, c = _dev(clouds[r], keep)
                g.tiled_step(x, c, _frame(clouds[r]["T"]))
                torch.cuda.synchronize()             # not g.sync(): that would bin step j before the later ranks route it
                routed[r] = j
            keys = _oracle_frame(o, clouds)
            if j in (4, steps):
                check(f"[{world} ranks, depth 3] step {j}", keys)
    finally:
        for g in maps:
            g.close()


# ---------------------------------------------------------------------------------------------------------------------
# the largest tiling attach accepts: world * cap = max_points = 2^22, i.e. 16384 sub-buckets for k_bin_peer (16 per block
# of its 1056-block wave); one block of capacity more is refused
# ---------------------------------------------------------------------------------------------------------------------
def test_boundary_world1_largest_capacity():
    """world 1 at bucket_capacity 2^22 (16384 sub-buckets): two full 4,194,304-point clouds and a small one against the
    oracle.  Device memory: about 4.5 GB of map scratch (max_points 2^22) and 0.4 GB of receive buffers.  One more block
    (2^22 + 1 points of capacity) is refused by gem_tiled_attach."""
    import torch
    L = 256
    g = _tile_map(L, 0, 1, MAX_LAUNCH)
    o = OracleMap(L, RES, compat_box_filter=False)
    keep = []
    try:
        small = PeerBuffers(1, 256)
        with pytest.raises(GemError, match="exceeds max_points"):
            small.attach(g, 0, bucket_capacity=MAX_LAUNCH + 1)
        with pytest.raises(GemError, match="gem_tiled_attach first"):
            g.tiled_step(None, None, _frame(_pose(0.0, 0.0)), n=0)
        bufs = PeerBuffers(1, MAX_LAUNCH)
        bufs.attach(g, 0)
        for step, c in enumerate([_random_cloud(MAX_LAUNCH, 31, extent=13.0), _full_cloud(MAX_LAUNCH, 32),
                                  _random_cloud(1000, 33, ox=5.0, oy=-5.0, extent=1.0)], start=1):
            x, r = _dev(c, keep)
            g.tiled_step(x, r, _frame(c["T"]))
            key, _, _ = _oracle_add(o, c)
            st = g.stats()
            where = f"[world 1, capacity 2^22] step {step}"
            assert st["points_in"] == c["xyzi"].shape[0] and st["points_binned"] == int((key >= 0).sum()), f"{where}: {st}"
            _assert_tile(g, o, 0, 1, where)
        torch.cuda.synchronize()
    finally:
        g.close()


def test_boundary_world64_largest_capacity(monkeypatch):
    """rank 27 of 64 at bucket_capacity 65536 (64 x 256 sub-buckets = 16384): routing and own tile checked as in B on
    clouds of exactly 65536 points.  The 64 record and intensity buffers alias one 0.5 GB allocation (PeerBuffers,
    alias=True) instead of 27 GB; map scratch about 4.5 GB.  65537 (one more block) is refused by gem_tiled_attach."""
    _env(monkeypatch, "graph_depth2")
    world, rank, L, cap = 64, 27, 512, MAX_LAUNCH // 64
    g = _tile_map(L, rank, world, MAX_LAUNCH)
    try:
        bufs = PeerBuffers(world, cap, alias=True)
        with pytest.raises(GemError, match="exceeds max_points"):
            bufs.attach(g, rank, bucket_capacity=cap + 1)
    finally:
        g.close()

    def exactly(c, n, seed):
        m = n - c["xyzi"].shape[0]
        r = synth.random_cloud(m, seed=seed, extent=25.0, zmin=-2.0, zmax=-0.8)
        return _cloud(np.concatenate([c["xyzi"], r["xyzi"]]), np.concatenate([c["rgba"], r["rgba"]]), c["T"])

    clouds = [exactly(_hdl_cloud(0, 0.0, 0.0, every=3), cap, 41), exactly(_chunk_level_cloud(42, 6.0, 0.1), cap, 43),
              _random_cloud(700, 44, ox=-12.0, oy=12.0, extent=2.0)]
    _run_one_rank(world, rank, L, cap, clouds, bufs, f"[rank {rank} of {world}, capacity {cap}]")
