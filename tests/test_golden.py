"""Golden vectors produced by THE REFERENCE ITSELF (tests/golden/gem_golden_v2.npz, generated on
an H100 by tests/golden/make_golden.py from the reference's gpu_process.cu compiled
unmodified).  CPU: the oracle must reproduce them; GPU: the CUDA path (through the C ABI) must.

  ref_nofma_* : reference compiled with -fmad=false  -> bit-exact
  ref_fma_*   : reference's own flags               -> indices equal, floats within 1e-5 rel

The inputs are the seeded stream golden_inputs() generates, pinned by their digest.  The reference's outputs are stored
as the XOR of their bytes against the oracle's outputs on the same inputs (ref_lib.xor_against), next to the digests of
those oracle outputs: reference() checks that the oracle still produces exactly them (which also pins the oracle) and
rebuilds the reference's outputs bit for bit.
"""
import hashlib
import os

import numpy as np
import pytest

import gem_b200
from gem_b200 import synth
import ref_lib
from oracle_lib import OracleMap
from shim_lib import shim  # noqa: F401  (a fixture)

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gem_golden_v2.npz")
L, RES, NFRAMES, STRIDE = 96, 0.2, 3, 11
EXACT = ("key", "var", "xt", "yt", "zt", "centre", "start", "shift", "feat_elevation", "feat_variance", "feat_intensity",
         "feat_color_r", "feat_color_g", "feat_color_b", "elev_after_ray")
# the reference's outputs the comparisons read, per build: only these are stored
COMPARED = {"ref_nofma": EXACT + ("feat_traver",), "ref_fma": ("key", "zt", "var", "feat_elevation")}


def golden_inputs():
    """a seeded 3-frame HDL-64E-shaped stream (subsampled), reference demo axes (so the hard-coded box filter of
    gpu_process.cu:393 keeps points), for a 96x96 @ 0.2 m map"""
    scene = synth.make_scene()
    out = []
    for k in range(NFRAMES):
        fr = synth.hdl64_frame(k, scene=scene, compat_axes=True, speed=8.0)
        fr["xyzi"] = np.ascontiguousarray(fr["xyzi"][k::STRIDE])
        fr["rgba"] = np.ascontiguousarray(fr["rgba"][k::STRIDE])
        fr["rgba"][::13, 1] = 0          # exercise the "any channel zero -> keep old colour" rule
        out.append(fr)
    return out


def inputs_digest(frames):
    h = hashlib.sha256()
    for fr in frames:
        for name in ("xyzi", "rgba", "T", "position"):
            h.update(ref_lib.digest(np.asarray(fr[name])).encode())
    return h.hexdigest()


def bits(a):
    a = np.asarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


@pytest.fixture(scope="module")
def gold():
    g = np.load(GOLD, allow_pickle=False)
    assert "reference gpu_process.cu" in str(g["generated_by"])
    return g


@pytest.fixture(scope="module")
def frames(gold):
    fr = golden_inputs()
    assert inputs_digest(fr) == str(gold["inputs_sha256"]), "the seeded golden inputs changed"
    return fr


def drive(m, frames):
    out = {}
    for k, fr in enumerate(frames):
        f = gem_b200.make_frame(fr["T"], gem_b200.LaserSensorProcessor())
        xyzi, rgba = fr["xyzi"], fr["rgba"]
        out[f"f{k}_centre"], out[f"f{k}_start"], out[f"f{k}_shift"] = m.move(fr["position"])
        key, var, xt, yt, zt = m.process_points(xyzi[:, 0].copy(), xyzi[:, 1].copy(), xyzi[:, 2].copy(), f)
        R, G, B = (rgba[:, j].astype(np.int32) for j in range(3))
        m.fuse_points(key, R, G, B, xyzi[:, 3], zt, var)
        feat = m.map_feature()
        m.raytracing()
        out[f"f{k}_key"], out[f"f{k}_var"], out[f"f{k}_xt"], out[f"f{k}_yt"], out[f"f{k}_zt"] = key, var, xt, yt, zt
        for name in feat:
            out[f"f{k}_feat_{name}"] = feat[name]
        out[f"f{k}_elev_after_ray"] = m.get_layer("elevation").reshape(-1)
    return out


def reference(g, oracle_out):
    """the reference's outputs (keys ref_nofma_<name>, ref_fma_<name>), rebuilt from the oracle's outputs"""
    ref = {}
    for name, like in oracle_out.items():
        assert str(g[f"oracle_{name}_sha256"]) == ref_lib.digest(like), (
            f"oracle drifted from the output the reference's was recorded against: {name}")
        for tag, names in COMPARED.items():
            if name.split("_", 1)[1] in names:
                ref[f"{tag}_{name}"] = ref_lib.rebuild(like, g[f"{tag}_{name}_xor"])
    return ref


def check_against_reference(out, ref, what):
    for k in range(NFRAMES):
        for name in EXACT:
            a, b = out[f"f{k}_{name}"], ref[f"ref_nofma_f{k}_{name}"]
            assert np.array_equal(bits(np.asarray(a, b.dtype)), bits(b)), f"{what}: frame {k} {name} differs from the reference (-fmad=false build)"
        # traversability: CUDA libm trig in the reference vs the deterministic trig here
        valid = ref[f"ref_nofma_f{k}_feat_elevation"] != -10
        tr_r, tr_o = ref[f"ref_nofma_f{k}_feat_traver"][valid], out[f"f{k}_feat_traver"][valid]
        assert np.array_equal(tr_r == -10, tr_o == -10)
        both = tr_r != -10
        d = np.abs(tr_r[both] - tr_o[both])
        assert np.mean(d[~np.isnan(d)] < 1e-4) > 0.995
        # reference's own flags (FMA contraction): BASELINE tolerance
        kf = ref[f"ref_fma_f{k}_key"]
        assert np.mean(kf == out[f"f{k}_key"]) > 0.9995
        same = (kf == out[f"f{k}_key"]) & (kf >= 0)
        assert np.allclose(ref[f"ref_fma_f{k}_zt"][same], out[f"f{k}_zt"][same], rtol=1e-5, atol=0)
        assert np.allclose(ref[f"ref_fma_f{k}_var"][same], out[f"f{k}_var"][same], rtol=1e-5, atol=0)
        ve = ref[f"ref_fma_f{k}_feat_elevation"]
        ok = np.isclose(ve, out[f"f{k}_feat_elevation"], rtol=1e-5, atol=1e-6)
        assert ok.mean() > 0.999
    assert (ref[f"ref_nofma_f{NFRAMES - 1}_feat_elevation"] != -10).sum() > 500


def test_oracle_reproduces_reference_golden(gold, frames):
    out = drive(OracleMap(L, RES, compat_box_filter=True), frames)
    # reference() also checks that every oracle output is bit for bit the one stored with the golden data
    check_against_reference(out, reference(gold, out), "oracle")


@pytest.mark.gpu
def test_cuda_path_reproduces_reference_golden(gold, frames, shim):
    """through the C ABI and through the drop-in shim's nine entry points (compat/gpu_process_shim.cpp)"""
    oracle_out = drive(OracleMap(L, RES, compat_box_filter=True), frames)
    ref = reference(gold, oracle_out)
    for what, m in (("gem_b200 CUDA path", gem_b200.ElevationMap(L, RES, compat_box_filter=True)),
                    ("the drop-in shim", shim(L, RES))):
        out = drive(m, frames)
        check_against_reference(out, ref, what)
        for k in range(NFRAMES):   # bit-exact vs the oracle incl. the feature layers
            for name in ("feat_traver", "feat_rough", "feat_slope"):
                a, b = out[f"f{k}_{name}"], oracle_out[f"f{k}_{name}"]
                same = (bits(a) == bits(b)) | (np.isnan(a) & np.isnan(b))
                assert same.all(), f"{what}: frame {k} {name}"
