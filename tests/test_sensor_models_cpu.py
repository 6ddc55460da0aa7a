"""Stereo and perfect sensor models on the CPU: the C oracle (tests/orc_sensor_models.c) bit for bit against an
independent restatement in plain Python floats with explicit float32 rounding at each cast, the `lowest` ORACLE
DEFINITION, the twelve shipped sensor configs mapped to models, and the C++ helpers compiling."""
import json
import math
import os
import tempfile

import numpy as np
import pytest

import native
import oracle_lib
import sensor_models_oracle as smo
from gem_b200 import _lib
from gem_b200.elevation_map import (LaserSensorProcessor, PerfectSensorProcessor, StereoSensorProcessor,
                                    StructuredLightSensorProcessor, make_frame)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "sensor_processors.json")
F = np.float32
ASLAM = dict(p_1=0.03287, p_2=-0.0001276, p_3=0.4850, p_4=399.1046, p_5=0.000006735, lateral_factor=0.001376915,
             depth_to_disparity_factor=47.3)
TINY = float(np.float32(1e-45))  # the smallest subnormal float
CRAFTED_Z = [1.5, 0.0, -0.0, TINY, -TINY, -2.0, 3.0e38, 0.25, 7.0]


def _ddiv(a, b):
    """IEEE double division (Python raises on a zero divisor)"""
    with np.errstate(all="ignore"):
        return float(np.float64(a) / np.float64(b))


def _dmul(a, b):
    with np.errstate(all="ignore"):
        return float(np.float64(a) * np.float64(b))


def _dadd(a, b):
    with np.errstate(all="ignore"):
        return float(np.float64(a) + np.float64(b))


def _f(v):
    """(float) cast: round a double to float32"""
    with np.errstate(all="ignore"):
        return F(v)


def restated_variances(s, x, y, z, idx):
    """(vN, vL) of StereoSensorProcessor.cpp:78-90 / PerfectSensorProcessor.cpp:87-88 as include/gem_b200.h defines them"""
    if s.type == _lib.SENSOR_PERFECT:
        return F(0.0), F(0.0)
    w = s.cloud_width
    row, col = (idx // w, idx % w) if w else (0, idx)
    p = list(s.stereo_p)
    dtd = s.depth_to_disparity_factor
    disp = _ddiv(dtd, float(F(z)))
    a = _ddiv(dtd, _dmul(disp, disp))
    sj = _dadd(_dadd(_dmul(p[2], disp), p[3]), -float(col))
    si = float(240 - row)
    with np.errstate(all="ignore"):
        root = float(np.sqrt(np.float64(_dadd(_dmul(sj, sj), _dmul(si, si)))))
    vn = _f(_dmul(_dmul(a, a), _dadd(_dmul(_dadd(_dmul(p[4], disp), p[1]), root), p[0])))
    with np.errstate(all="ignore"):
        x, y, z = F(x), F(y), F(z)
        dist = np.sqrt((x * x + y * y) + z * z)
    l_ = _dmul(s.lateral_factor, float(dist))
    return vn, _f(_dmul(l_, l_))


def restated_point(frame, box, x, y, z, idx):
    """(accepted, h, hv, xt, yt) of the per-point step (gpu.cu:384-431) with the restated variances"""
    T = np.array(frame.T[:], F)
    sJ, rv, cs, pm, bs = (np.array(getattr(frame, k)[:], F) for k in
                          ("sensor_jacobian", "rotation_variance", "C_SB_transpose", "P_mul_C_BM_transpose", "B_r_BS_skew"))
    with np.errstate(all="ignore"):
        x, y, z = F(x), F(y), F(z)
        h = ((T[8] * x + T[9] * y) + T[10] * z) + T[11]
        flag = box and ((-1.5 < x < 1.5 and -1.5 < y < 1.5) or (-1 < y < 1) or y > 0)
        if not (frame.rel_lower < float(h) < frame.rel_upper) or flag:
            return False, F(-1), F(-1), F(-1), F(-1)
        xt = ((T[0] * x + T[1] * y) + T[2] * z) + T[3]
        yt = ((T[4] * x + T[5] * y) + T[6] * z) + T[7]
        vn, vl = restated_variances(frame.sensor, x, y, z, idx)
        q = [(cs[3 * j] * x + cs[3 * j + 1] * y) + cs[3 * j + 2] * z for j in range(3)]
        S = [F(0) + bs[0], -q[2] + bs[1], q[1] + bs[2], q[2] + bs[3], F(0) + bs[4], -q[0] + bs[5], -q[1] + bs[6],
             q[0] + bs[7], F(0) + bs[8]]
        rj = [(pm[0] * S[j] + pm[1] * S[3 + j]) + pm[2] * S[6 + j] for j in range(3)]
        A1 = [(rj[0] * rv[j] + rj[1] * rv[3 + j]) + rj[2] * rv[6 + j] for j in range(3)]
        term1 = (A1[0] * rj[0] + A1[1] * rj[1]) + A1[2] * rj[2]
        SV = [vl, F(0), F(0), F(0), vl, F(0), F(0), F(0), vn]
        B1 = [(sJ[0] * SV[j] + sJ[1] * SV[3 + j]) + sJ[2] * SV[6 + j] for j in range(3)]
        term2 = (B1[0] * sJ[0] + B1[1] * sJ[1]) + B1[2] * sJ[2]
        return True, h, term1 + term2, xt, yt


def frames():
    """stereo (aslam) organised 640 wide, width 1, unorganised, all-zero parameters; perfect; with and without
    rotation variance and a tilted sensor"""
    c, s = math.cos(0.3), math.sin(0.3)
    T = np.array([[c, 0, s, 0.2], [0, 1, 0, -0.1], [-s, 0, c, 0.7], [0, 0, 0, 1]])
    rot = dict(rotation_variance=np.diag([1e-4, 2e-4, 3e-4]), C_SB_transpose=np.eye(3),
               B_r_BS_skew=np.array([[0, -0.3, 0.1], [0.3, 0, -0.2], [-0.1, 0.2, 0]]))
    out = []
    for sensor in (StereoSensorProcessor(**ASLAM, cloud_width=640), StereoSensorProcessor(**ASLAM, cloud_width=1),
                   StereoSensorProcessor(**ASLAM), StereoSensorProcessor(cloud_width=640), PerfectSensorProcessor()):
        out.append(make_frame(np.eye(4), sensor))
        out.append(make_frame(T, sensor, **rot))
    return out


def crafted_points():
    """(x, y, z, idx0): crafted depths at pixel rows 0/239/240/241/479/480/1000 of a 640-wide cloud, plus a run of
    indices just below 2^31"""
    x, y, z = [], [], []
    rows = [0, 239, 240, 241, 479, 480, 1000]
    idx = []
    for r in rows:
        for k, zz in enumerate(CRAFTED_Z):
            idx.append(r * 640 + 37 * k)
    n = idx[-1] + 1
    pts = np.zeros((n, 3), F)
    rng = np.random.default_rng(5)
    pts[:, 0] = rng.uniform(-3, 3, n)
    pts[:, 1] = rng.uniform(-3, 3, n)
    pts[:, 2] = rng.uniform(0.3, 6.0, n)
    for j, i in enumerate(idx):
        pts[i, 2] = CRAFTED_Z[j % len(CRAFTED_Z)]
    return pts


@pytest.mark.parametrize("fi", range(10))
def test_oracle_matches_the_restatement_on_crafted_points(fi):
    frame = frames()[fi]
    pts = crafted_points()
    sel = np.arange(0, pts.shape[0], 97)  # every crafted row is covered by the stride below as well
    sel = np.unique(np.concatenate([sel, np.flatnonzero(np.isin(pts[:, 2], np.array(CRAFTED_Z, F)))]))
    om = oracle_lib.OracleMap(200, 0.05, compat_box_filter=False)
    key, var, xt, yt, zt = smo.process_points(om, pts[:, 0], pts[:, 1], pts[:, 2], frame)
    for i in sel:
        acc, h, hv, x_, y_ = restated_point(frame, False, *pts[i], int(i))
        if not acc:
            assert key[i] == -1
        for a, b in ((h, zt[i]), (hv, var[i]), (x_, xt[i]), (y_, yt[i])):
            assert np.float32(a).tobytes() == np.float32(b).tobytes(), (i, pts[i], a, b)
        if acc:
            g, st = om.points_to_index(x_, y_)
            assert key[i] == st


def test_index_near_2_31_and_width_one():
    """row / col from idx0 + i: indices just below 2^31, for a 640-wide, a 1-wide and an unorganised cloud"""
    n = 9
    pts = np.stack([np.full(n, 0.3, F), np.full(n, -0.2, F), np.array(CRAFTED_Z, F)], 1)
    idx0 = 2 ** 31 - n
    for width in (640, 1, 0, 7):
        frame = make_frame(np.eye(4), StereoSensorProcessor(**ASLAM, cloud_width=width))
        om = oracle_lib.OracleMap(64, 0.1, compat_box_filter=False)
        _, var, _, _, _ = smo.process_points(om, pts[:, 0], pts[:, 1], pts[:, 2], frame, idx0=idx0)
        for i in range(n):
            _, _, hv, _, _ = restated_point(frame, False, *pts[i], idx0 + i)
            assert np.float32(hv).tobytes() == var[i].tobytes(), (width, i)


def test_crafted_depths_give_what_the_expression_gives():
    """z = +-0: infinite disparity, a = 0 and 0 * inf = NaN; a subnormal z underflows to 0; negative z: a finite
    variance; nothing is clamped"""
    model = make_frame(np.eye(4), StereoSensorProcessor(**ASLAM, cloud_width=640)).sensor
    s = smo.sensor_of(make_frame(np.eye(4), StereoSensorProcessor(**ASLAM, cloud_width=640)))
    vn0, _ = smo.variances(s, 0.1, 0.1, 0.0, 5)
    vns, _ = smo.variances(s, 0.1, 0.1, TINY, 5)
    vneg, _ = smo.variances(s, 0.1, 0.1, -2.0, 5)
    assert np.isnan(vn0) and vns == 0 and np.isfinite(vneg)
    for z in (0.0, -0.0, TINY, -TINY, -2.0, 3e38):
        a = smo.variances(s, 0.1, 0.1, z, 1234)
        b = restated_variances(model, 0.1, 0.1, z, 1234)
        assert [np.float32(v).tobytes() for v in a] == [np.float32(v).tobytes() for v in b], z


def test_all_zero_parameters_and_perfect():
    """the node's all-zero stereo defaults: disparity 0, a = 0 / 0 = NaN, so vN is NaN and vL is 0; perfect: both 0"""
    st = smo.sensor_of(make_frame(np.eye(4), StereoSensorProcessor(cloud_width=640)))
    pf = smo.sensor_of(make_frame(np.eye(4), PerfectSensorProcessor()))
    for z in (0.5, 2.0, -1.0):
        vn, vl = smo.variances(st, 0.2, 0.3, z, 1000)
        assert np.isnan(vn) and vl == 0
        assert smo.variances(pf, 0.2, 0.3, z, 1000) == (0, 0)


def test_lowest_oracle_definition():
    """per geographic cell: m = min h, i* the first index attaining it; lowest = m + 3 hv[i*] iff m <= lowest_old"""
    frame = make_frame(np.eye(4), StereoSensorProcessor(**ASLAM, cloud_width=4), base_z=0.0)
    om = oracle_lib.OracleMap(32, 0.1, compat_box_filter=False)
    # four points in one cell: heights 1.0, 0.5, 0.5 (a tie: the first wins), 0.7; one point elsewhere at 200
    pts = np.array([[0.01, 0.01, 1.0], [0.02, 0.02, 0.5], [0.03, 0.03, 0.5], [0.04, 0.04, 0.7], [0.5, 0.5, 200.0]], F)
    om.set_layer("lowest", np.full(32 * 32, 100.0, F))
    key, var, xt, yt, zt = smo.process_points(om, pts[:, 0], pts[:, 1], pts[:, 2], frame)
    low = om.get_layer("lowest").reshape(-1)
    g, _ = om.points_to_index(xt[1], yt[1])
    assert low[g] == F(F(0.5) + F(3) * var[1])
    g2, _ = om.points_to_index(xt[4], yt[4])
    assert low[g2] == F(100.0)  # 200 > lowest_old: unchanged


def _model_of(entry):
    """GEM's node: the processor of sensor_processor/type with the node's defaults for missing keys (Laser.cpp:44-46,
    SL.cpp:40-47, Stereo.cpp:26-32; ignore_points_* SPB.cpp:61-62; Perfect reads nothing)"""
    kind = entry["type"]
    g = lambda k, d=0.0: float(entry.get(k, d))
    win = dict(ignore_points_above=g("ignore_points_above", math.inf), ignore_points_below=g("ignore_points_below", -math.inf))
    if kind == "laser":
        return LaserSensorProcessor(min_radius=g("min_radius"), beam_angle=g("beam_angle"), beam_constant=g("beam_constant"), **win)
    if kind == "structured_light":
        return StructuredLightSensorProcessor(
            normal_factor_a=g("normal_factor_a"), normal_factor_b=g("normal_factor_b"), normal_factor_c=g("normal_factor_c"),
            normal_factor_d=g("normal_factor_d"), normal_factor_e=g("normal_factor_e"), lateral_factor=g("lateral_factor"),
            cutoff_min_depth=g("cutoff_min_depth", 2.2250738585072014e-308), cutoff_max_depth=g("cutoff_max_depth", 1.7976931348623157e308),
            **win)
    if kind == "stereo":
        return StereoSensorProcessor(p_1=g("p_1"), p_2=g("p_2"), p_3=g("p_3"), p_4=g("p_4"), p_5=g("p_5"),
                                     lateral_factor=g("lateral_factor"), depth_to_disparity_factor=g("depth_to_disparity_factor"),
                                     **win)
    assert kind == "perfect"
    return PerfectSensorProcessor()


def shipped_models():
    with open(GOLDEN) as fh:
        return {name: _model_of(e) for name, e in json.load(fh).items()}


def test_the_twelve_shipped_configs_map_to_models():
    with open(GOLDEN) as fh:
        cfg = json.load(fh)
    assert len(cfg) == 12
    models = shipped_models()
    types = {n: models[n].model().type for n in cfg}
    assert types["aslam.yaml"] == _lib.SENSOR_STEREO and types["perfect.yaml"] == _lib.SENSOR_PERFECT
    assert sum(t in (_lib.SENSOR_LASER, _lib.SENSOR_STRUCTURED_LIGHT) for t in types.values()) == 10
    # the datasheet config names its normal factors factor_a/b/c, which the node never reads
    ds = models["primesense_carmine_109_short_range_datasheet.yaml"].model()
    assert "factor_a" in cfg["primesense_carmine_109_short_range_datasheet.yaml"]
    assert (ds.normal_factor_a, ds.normal_factor_b, ds.normal_factor_c, ds.normal_factor_e) == (0.0, 0.0, 0.0, 0.0)
    st = models["aslam.yaml"].model()
    assert list(st.stereo_p) == [0.03287, -0.0001276, 0.4850, 399.1046, 0.000006735] and st.depth_to_disparity_factor == 47.3
    # Perfect ignores the height window whatever is set on it
    f = make_frame(np.eye(4), models["perfect.yaml"], base_z=3.0)
    assert f.rel_lower == -math.inf and f.rel_upper == math.inf


def test_stereo_defaults_are_the_nodes():
    m = StereoSensorProcessor().model()
    assert list(m.stereo_p) == [0.0] * 5 and m.depth_to_disparity_factor == 0.0 and m.lateral_factor == 0.0
    assert m.cloud_width == 0 and m.type == 2


def compile_sensor_models_smoke(outdir):
    return native.facade_program("sensor_models_smoke", outdir, ["-Wextra"])


def test_cxx_helpers_compile():
    with tempfile.TemporaryDirectory() as d:
        assert os.path.exists(compile_sensor_models_smoke(d))
