"""The call scripts of tests/sequence_cases.py on the oracle alone: every script runs, the restatement of gem_move's
band arithmetic agrees with the oracle's Move, and every hand-written script reaches the hazard it is named after: every
later reader straight after every hazard kind, and the node's frame loop growing and shrinking what its readers return."""
import numpy as np
import pytest

import sequence_cases as sc

f32 = np.float32
HAND = {s.name: s for s in sc.hand_written()}


@pytest.fixture(scope="module")
def traces():
    return {s.name: (s, sc.run_oracle(s)) for s in sc.all_scripts()}


def _counts(L, keys):
    k = keys[keys >= 0]
    return np.bincount(k, minlength=L * L)


def _previous(trace, i, ops):
    for j in range(i - 1, -1, -1):
        if trace[j][0] in ops:
            return j
    return None


def test_script_names_are_unique_and_sizes_in_range():
    scripts = sc.all_scripts()
    assert len({s.name for s in scripts}) == len(scripts)
    for s in scripts:
        assert 64 <= s.L <= 200, s.name
        for op, a in s.steps:
            if op == "multi":
                assert 2 <= len(a["clouds"]) <= 8
                assert sum(s.clouds[c]["xyzi"].shape[0] for c in a["clouds"]) <= sc.MAX_POINTS, s.name
            elif op in ("add", "process"):
                assert s.clouds[a["cloud"]]["xyzi"].shape[0] <= sc.MAX_POINTS, s.name


def test_generator_is_deterministic():
    for seed in sc.SEEDS:
        a, b = sc.random_script(seed), sc.random_script(seed)
        assert [op for op, _ in a.steps] == [op for op, _ in b.steps]
        for name in a.clouds:
            assert np.array_equal(a.clouds[name]["xyzi"], b.clouds[name]["xyzi"])


@pytest.mark.parametrize("name", sc.SCRIPT_NAMES)
def test_move_model_matches_the_oracle(traces, name):
    """the Python gem_move restatement (bands, centre, start) against orc_move, at every move of every script"""
    s, trace = traces[name]
    centre, start = [f32(0), f32(0)], [0, 0]
    for i, (op, a, out) in enumerate(trace):
        if op == "move":
            centre, start, shift, ops = sc.move_model(s.L, s.res, centre, start, a["pos"])
            oc, ost, osh = out["returned"]
            assert np.array_equal(np.array(centre, f32).view(np.uint32), oc.view(np.uint32)), (name, i)
            assert list(start) == [int(v) for v in ost], (name, i)
            assert np.array_equal(np.array(shift, f32).view(np.uint32), osh.view(np.uint32)), (name, i)
            assert ops == out["ops"]
        elif op in ("opt_move", "closeloop"):
            centre = [f32(c) for c in (sc._opt_move_centre if op == "opt_move" else sc._closeloop_centre)(centre, a["p"], s.res)]
            if op == "opt_move":
                assert np.array_equal(np.array(centre, f32), out["aligned"]), (name, i)


def test_move_model_band_wrap_and_full_shift():
    L = 64
    # from start 0 a positive shift clears the band just below the storage edge, no wrap
    _, start, _, ops = sc.move_model(L, 0.1, [0, 0], [0, 0], (0.3, 0.0, 0.0))
    assert ops == [("rows", L - 3, 3)] and start == [L - 3, 0]
    # then a larger negative shift starts there and wraps past the edge: two ops
    _, _, _, ops = sc.move_model(L, 0.1, [f32(0.3), 0], start, (-0.2, 0.0, 0.0))
    assert ops == [("rows", L - 3, 3), ("rows", 0, 2)]
    for d in (L, -L, L + 5, -L - 1):
        _, _, _, ops = sc.move_model(L, 0.1, [0, 0], [0, 0], (0.0, d * 0.1, 0.0))
        assert ops == [("all",)]


# ---- the hazards of the hand-written scripts ------------------------------------------------------------------------------
def _check_long_clear(s, trace, i):
    j = _previous(trace, i, ("add", "multi"))
    assert j is not None
    counts = _counts(s.L, trace[j][2]["keys"])
    band = sc.band_cells(s.L, trace[i][2]["ops"])
    k = counts[band]
    assert (k > 40).sum() >= 2, f"{s.name} step {i}: the band holds no cell of more than 40 records from step {j}"
    assert ((k > 8) & (k <= 40)).sum() >= 2, f"{s.name} step {i}: the band holds no cell of 9..40 records from step {j}"


def _check_wrap(s, trace, i):
    ops = trace[i][2]["ops"]
    for kind in ("rows", "cols"):
        assert sum(op[0] == kind for op in ops) == 2, f"{s.name} step {i}: the {kind} band does not wrap: {ops}"


def _check_overflow(s, trace, i):
    """the moves up to step i run back to back and queue more than MAX_REGION_OPS ops for the next add; the oldest ones
    clear cells the newest ones do not"""
    n, j, bands = 0, i, []
    while j >= 0 and trace[j][0] == "move":
        n += len(trace[j][2]["ops"])
        bands = list(trace[j][2]["ops"]) + bands
        j -= 1
    assert n > sc.MAX_REGION_OPS, f"{s.name} step {i}: {n} ops pending"
    assert trace[i + 1][0] in ("add", "multi"), s.name
    old = set(sc.band_cells(s.L, bands[:n - sc.MAX_REGION_OPS]).tolist())
    new = set(sc.band_cells(s.L, bands[n - sc.MAX_REGION_OPS:]).tolist())
    k = _counts(s.L, trace[_previous(trace, j + 1, ("add", "multi"))][2]["keys"])
    only_old = np.array(sorted(old - new), np.int64)
    assert only_old.size and (k[only_old] > 0).sum() > 0, f"{s.name} step {i}: the overflowing ops clear nothing of their own"


def _check_full_shift_pending(s, trace, i):
    op = trace[i - 1]
    assert op[0] == "add" and op[1]["variant"] in sc.PIPELINED, f"{s.name} step {i}: no pipelined add right before"
    assert trace[i][2]["ops"] and trace[i][2]["ops"][0] == ("all",), f"{s.name} step {i}: {trace[i][2]['ops']}"
    k = _counts(s.L, op[2]["keys"])
    assert (k > 40).any(), s.name


def _check_boundary(s, trace, i):
    op, a, out = trace[i]
    j = _previous(trace, i, ("move", "opt_move", "closeloop"))       # the centre the move starts from
    if j is None:
        before = np.array([0, 0], f32)
    else:
        assert trace[j][0] == "move", s.name
        before = trace[j][2]["state"][0]
    moved = False
    for ax in range(2):
        p = f32(a["pos"][ax])
        sh = sc.index_shift(float(p), f32(before[ax]), f32(s.res))
        for nb in (np.nextafter(p, f32(np.inf)), np.nextafter(p, f32(-np.inf))):
            moved |= sc.index_shift(float(nb), f32(before[ax]), f32(s.res)) != sh
    assert moved, f"{s.name} step {i}: {a['pos']} is not one ulp from a shift boundary"


def _check_var_below_floor(s, trace, i):
    v = trace[i][2]["variance"]
    assert trace[i][1]["dv"] < 0
    assert ((v < f32(1e-4)) & (v != f32(-10))).sum() > 100, f"{s.name} step {i}: no variance fell below 1e-4"


def _check_set_below_floor(s, trace, i):
    v = trace[i][2]["variance"]
    assert ((v < f32(1e-4)) & (v != f32(-10))).sum() > 100, s.name


def _check_pending_fold_and_clears(s, trace, i):
    assert trace[i - 1][0] == "move" and trace[i - 1][2]["ops"], s.name
    assert trace[i - 2][0] == "add" and trace[i - 2][1]["variant"] in sc.PIPELINED, s.name


def _check_multi_frames(s, trace, i):
    Ts = trace[i][2]["frames"]
    assert len({np.asarray(T).tobytes() for T in Ts}) == len(Ts), f"{s.name} step {i}: segments share a frame"
    j = _previous(trace, i, ("multi",))
    if j is not None:
        prev = {np.asarray(T).tobytes() for T in trace[j][2]["frames"]}
        assert not prev & {np.asarray(T).tobytes() for T in Ts}, f"{s.name} step {i}: frames repeat those of step {j}"


def _check_harvest(s, trace, i):
    assert trace[i][2]["harvest"][1] > 10, f"{s.name} step {i}: the harvest takes {trace[i][2]['harvest'][1]} records"


def _check_reader(s, trace, i):
    assert trace[i][0] in sc.READERS, f"{s.name} step {i}: {trace[i][0]} is not one of the later readers"


def _check_reader_fold_in_flight(s, trace, i):
    """a pipelined add right before the reader, whose fold changes cells the reader reads"""
    _check_reader(s, trace, i)
    op, a, out = trace[i - 1]
    assert op == "add" and a["variant"] in ("stream", "host_async"), f"{s.name} step {i}: no pipelined add right before"
    hit = _counts(s.L, out["keys"])[trace[i][2]["shown"]]
    assert (hit > 0).sum() > 100, f"{s.name} step {i}: the fold in flight touches {(hit > 0).sum()} shown cells"


def _check_reader_queued_clears(s, trace, i):
    """a move right before the reader whose bands wrap the storage edge on both axes or clear the whole map, over cells
    that held heights, with no fusing call since the fill before it"""
    _check_reader(s, trace, i)
    op, _, out = trace[i - 1]
    assert op == "move", f"{s.name} step {i}: no move right before"
    ops = out["ops"]
    assert ("all",) in ops or all(sum(o[0] == k for o in ops) == 2 for k in ("rows", "cols")), f"{s.name} step {i}: {ops}"
    assert out["band_filled"] > 100, f"{s.name} step {i}: the bands clear {out['band_filled']} cells with heights"


def _check_reader_floor_pending(s, trace, i):
    _check_reader(s, trace, i)
    op, a, out = trace[i - 1]
    assert op in ("var_update", "set_variance"), f"{s.name} step {i}: {op} right before"
    v = out["variance"]
    assert ((v < f32(1e-4)) & (v != f32(-10))).sum() > 100, f"{s.name} step {i}: no variance below the floor"
    assert any(op in ("add", "multi", "empty", "fuse") for op, _, _ in trace[i + 1:]), f"{s.name} step {i}: no Fuse follows"


def _check_reader_parked(s, trace, i):
    """gem_process_points right before the reader, its fuse still to come, with the clears of a move parked"""
    _check_reader(s, trace, i)
    assert trace[i - 1][0] == "process" and trace[i - 2][0] == "move" and trace[i - 2][2]["ops"], s.name
    j = next(j for j in range(i + 1, len(trace)) if trace[j][0] in ("add", "multi", "empty", "fuse", "process"))
    assert trace[j][0] == "fuse", f"{s.name} step {i}: the fuse does not follow"


CHECKS = {"harvest": _check_harvest, "long_clear": _check_long_clear, "wrap": _check_wrap, "overflow": _check_overflow,
          "full_shift_pending": _check_full_shift_pending, "boundary": _check_boundary,
          "var_below_floor": _check_var_below_floor, "set_below_floor": _check_set_below_floor,
          "pending_fold_and_clears": _check_pending_fold_and_clears, "multi_frames": _check_multi_frames,
          "reader_fold_in_flight": _check_reader_fold_in_flight, "reader_queued_clears": _check_reader_queued_clears,
          "reader_floor_pending": _check_reader_floor_pending, "reader_parked": _check_reader_parked}


@pytest.mark.parametrize("name", sorted(HAND))
def test_hand_written_script_reaches_its_hazard(traces, name):
    s, trace = traces[name]
    assert s.hazards or name in ("empty_call_flushes", "export_around_raytracing", "host_async_alternating",
                                 "reader_between_pipelined", "node_frame_loop")
    for kind, i in s.hazards:
        CHECKS[kind](s, trace, i)


def test_every_later_reader_follows_every_hazard(traces):
    """across the readers_after_* scripts each reader op sits directly after each hazard kind, and after each way to
    raise it: a stream and a host_async fold, wrapping bands and a full shift, a negative var_update and a set_variance"""
    seen, ways = set(), set()
    for s, trace in traces.values():
        for kind, i in s.hazards:
            if kind in sc.READER_HAZARDS:
                op = trace[i][0]
                seen.add((op, kind))
                prev_op, prev_a, prev_out = trace[i - 1]
                way = prev_a.get("variant") if prev_op == "add" else \
                    ("all" if ("all",) in prev_out.get("ops", []) else "wrap") if prev_op == "move" else prev_op
                ways.add((op, way))
    missing = [(op, kind) for op in sc.READERS for kind in sc.READER_HAZARDS if (op, kind) not in seen]
    assert not missing, missing
    missing = [(op, w) for op in sc.READERS for w in ("stream", "host_async", "wrap", "all", "var_update", "set_variance",
                                                      "process") if (op, w) not in ways]
    assert not missing, missing


def test_readers_after_hazards_read_sources_at_both_kinds_and_cut_both_ways(traces):
    """each readers_after_* script reads the shown map and the snapshot, marks at both costmap sizes (update_origin
    between every two marks), and cuts dense with a local map to densify as well as plain"""
    for name in (n for n in HAND if n.startswith("readers_after_")):
        s, trace = traces[name]
        srcs = {(op, a["src"]) for op, a, _ in trace if "src" in a}
        assert {(op, src) for op in ("grid_cloud", "split", "octrees") for src in ("shown", "snapshot")} <= srcs, name
        assert {a["size"] for op, a, _ in trace if op == "costmap"} == set(sc.COST_SIZES), name
        cuts = [(a["dense"], out["local_taken"]) for op, a, out in trace if op == "cut"]
        assert any(d and n > 100 for d, n in cuts) and any(not d for d, _ in cuts), (name, cuts)
        assert any(out["local"][1] > 100 for op, _, out in trace if op == "local"), name


def _rises_and_falls(v):
    return len(v) >= 3 and max(v) > v[0] and max(v) > v[-1]


def test_node_frame_loop_sizes_rise_and_fall(traces):
    """on one handle the grid cloud, the harvest and the costmap window (and what the costmap marks) grow and later
    shrink, so every shared scratch is reused both larger and smaller than before; cuts are taken dense and plain"""
    s, trace = traces["node_frame_loop"]
    grid = [out["cloud"].shape[0] for op, a, out in trace if op == "grid_cloud"]
    harvest = [out["local"][1] for op, _, out in trace if op == "local"]
    window = [a["size"][0] * a["size"][1] for op, a, _ in trace if op == "costmap"]
    marked = [out["marks"]["marked"] for op, _, out in trace if op == "costmap"]
    for what, v in (("grid cloud", grid), ("harvest", harvest), ("costmap window", window), ("costmap marks", marked)):
        assert _rises_and_falls(v), (what, v)
    assert len(grid) == sc.NODE_FRAMES
    cuts = [(a["dense"], out["local_taken"]) for op, a, out in trace if op == "cut"]
    assert any(d and n > 0 for d, n in cuts) and any(not d and n > 0 for d, n in cuts), cuts


def _same_output(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same_output(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_same_output(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    if isinstance(a, float):
        return np.float64(a).tobytes() == np.float64(b).tobytes()
    return a == b


@pytest.mark.parametrize("name", ["node_frame_loop", "readers_after_stream_fold", "random_103"])
def test_reader_traces_are_deterministic(traces, name):
    """a second oracle run of the script gives the same outputs, bit for bit"""
    s, trace = traces[name]
    again = sc.run_oracle(sc.script_by_name(name))
    assert len(again) == len(trace)
    for i, ((op, _, out), (_, _, out2)) in enumerate(zip(trace, again)):
        assert _same_output(out, out2), (name, i, op)


def test_random_scripts_draw_the_later_readers():
    ops = {op for seed in sc.SEEDS for op, _ in sc.random_script(seed).steps}
    assert len(ops & set(sc.READERS)) >= 5, ops


def test_every_add_variant_and_empty_call_is_scripted():
    seen, empty = set(), set()
    for s in HAND.values():
        for op, a in s.steps:
            if op == "add":
                seen.add(a["variant"])
            elif op == "multi":
                seen.add("multi")
            elif op == "empty":
                empty.add(a["variant"])
    assert seen == set(sc.ADD_VARIANTS) | {"multi"}
    assert empty == set(sc.EMPTY_VARIANTS)


def test_multi_steady_state_runs_five_or_more_calls_back_to_back():
    s = HAND["multi_steady_state"]
    ops = [op for op, _ in s.steps]
    run = best = 0
    for op in ops:
        run = run + 1 if op == "multi" else (run if op == "move" else 0)
        best = max(best, run)
    assert best >= 5


def test_clouds_are_kept_whole_by_the_sensor_filter():
    """the device map receives the raw clouds: nothing in them is dropped by cleanPointCloud"""
    from oracle_lib import OracleMap
    o = OracleMap(64, 0.1, compat_box_filter=False)
    f = sc.frame(np.eye(4))
    for s in list(HAND.values())[:3]:
        for c in s.clouds.values():
            assert o.clean_point_cloud(c["xyzi"], c["rgba"], f)[0].shape[0] == c["xyzi"].shape[0]
    o.close()
