"""ctypes access to the reference's own GPU library built by oracle/build_ref.py
(oracle/_ref/libgpu_ref*.so = the reference's gpu_process.cu compiled unmodified against the
stand-in Eigen header + oracle/ref_harness.cu), and PinnedRef, which replays its recorded outputs
where that library is absent.  TEST INFRASTRUCTURE."""
from __future__ import annotations

import ctypes as C
import hashlib
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")


def available(nofma: bool = True) -> bool:
    return os.path.exists(os.path.join(REF_DIR, "libgpu_ref_nofma.so" if nofma else "libgpu_ref.so"))


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


class RefMap:
    """The reference keeps ONE map per process in __device__ globals (gpu_process.cu:20-56):
    create one RefMap per loaded library at a time."""
    _libs = {}

    def __init__(self, length, resolution, mahalanobis=2.5, obstacle_threshold=0.7, nofma=True):
        name = "libgpu_ref_nofma.so" if nofma else "libgpu_ref.so"
        if name not in RefMap._libs:
            RefMap._libs[name] = C.CDLL(os.path.join(REF_DIR, name))
        self.lib = RefMap._libs[name]
        self.L, self.res = int(length), float(resolution)
        self.lib.ref_init(self.L, C.c_float(self.res), C.c_float(mahalanobis), C.c_float(obstacle_threshold))

    def move(self, pos):
        p = np.asarray(pos, np.float32)
        centre, start, shift = np.zeros(2, np.float32), np.zeros(2, np.int32), np.zeros(2, np.float32)
        self.lib.ref_move(_p(p), _p(centre), _p(start), _p(shift), C.c_float(self.res))
        return centre, start, shift

    def process_points(self, x, y, z, frame):
        x, y, z = (np.array(a, np.float32, copy=True) for a in (x, y, z))
        n = x.shape[0]
        key = np.empty(n, np.int32)
        var, xt, yt, zt = (np.empty(n, np.float32) for _ in range(4))
        arr = lambda v: np.array(v[:], np.float32)
        T, sJ, rv = arr(frame.T), arr(frame.sensor_jacobian), arr(frame.rotation_variance)
        cs, pm, bs = arr(frame.C_SB_transpose), arr(frame.P_mul_C_BM_transpose), arr(frame.B_r_BS_skew)
        s = frame.sensor
        self.lib.ref_process_points(_p(key), _p(x), _p(y), _p(z), _p(var), _p(xt), _p(yt), _p(zt), _p(T), n,
                                    C.c_double(frame.rel_lower), C.c_double(frame.rel_upper), C.c_float(s.min_radius),
                                    C.c_float(s.beam_angle), C.c_float(s.beam_constant), _p(sJ), _p(rv), _p(cs), _p(pm),
                                    _p(bs))
        return key, var, xt, yt, zt

    def fuse_points(self, index, R, G, B, intensity, height, var):
        i32 = lambda a: np.ascontiguousarray(a, np.int32)
        f32 = lambda a: np.ascontiguousarray(a, np.float32)
        index, R, G, B = i32(index), i32(R), i32(G), i32(B)
        intensity, height, var = f32(intensity), f32(height), f32(var)
        self.lib.ref_fuse(index.shape[0], _p(index), _p(R), _p(G), _p(B), _p(intensity), _p(height), _p(var))

    def var_update(self, dv):
        self.lib.ref_var_update(C.c_float(dv))

    def map_feature(self):
        n = self.L * self.L
        out = {k: np.zeros(n, np.float32) for k in ("elevation", "variance", "rough", "slope", "traver", "intensity")}
        out.update({k: np.zeros(n, np.int32) for k in ("color_r", "color_g", "color_b")})
        self.lib.ref_map_feature(_p(out["elevation"]), _p(out["variance"]), _p(out["color_r"]), _p(out["color_g"]),
                                 _p(out["color_b"]), _p(out["rough"]), _p(out["slope"]), _p(out["traver"]),
                                 _p(out["intensity"]))
        return out

    def raytracing(self):
        self.lib.ref_raytracing()

    def opt_move(self, opt_p, height_update):
        """Map_optmove: returns the aligned position it moved the centre to"""
        p = np.array(opt_p, np.float32, copy=True)
        out = np.zeros(2, np.float32)
        self.lib.ref_optmove(_p(p), C.c_float(height_update), C.c_float(self.res), _p(out))
        return out

    def closeloop(self, update_position, height_update):
        p = np.array(update_position, np.float32, copy=True)
        self.lib.ref_closeloop(_p(p), C.c_float(height_update), C.c_float(self.res))

    def state(self):
        """(central_coordinate, start_indice, [sensorZatLowestScan]) as float32[2], int32[2], float32[1]"""
        centre, start, sz = np.zeros(2, np.float32), np.zeros(2, np.int32), np.zeros(1, np.float32)
        self.lib.ref_get_state(_p(centre), _p(start), _p(sz))
        return centre, start, sz

    def get_layer(self, name):
        which, dtype = LAYERS[name]
        out = np.empty(self.L * self.L, dtype)
        self.lib.ref_get_layer(which, _p(out))
        return out.reshape(self.L, self.L)

    def layers(self, names):
        return {n: self.get_layer(n) for n in names}

    def set_layer(self, name, arr):
        which, dtype = LAYERS[name]
        a = np.ascontiguousarray(arr, dtype).reshape(-1)
        assert a.shape[0] == self.L * self.L, (name, a.shape)
        self.lib.ref_set_layer(which, _p(a))


# the reference's device layers the harness reads and writes: name -> (harness index, element type)
LAYERS = {"lowest": (0, np.float32), "traver": (1, np.float32), "elevation": (2, np.float32), "variance": (3, np.float32),
          "intensity": (4, np.float32), "color_r": (5, np.int32), "color_g": (6, np.int32), "color_b": (7, np.int32)}


def _bytes(a):
    return np.frombuffer(np.ascontiguousarray(a).tobytes(), np.uint8)


def digest(a):
    """SHA-256 of an array's dtype, shape and bytes"""
    a = np.ascontiguousarray(a)
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(a.tobytes())
    return h.hexdigest()


def xor_against(out, like):
    """the stored form of the reference's array `out`: its bytes XOR those of the oracle's array `like` for the same
    call on the same inputs (same dtype and shape), all zero where the two agree, so it compresses to almost nothing"""
    out, like = np.ascontiguousarray(out), np.ascontiguousarray(like)
    assert out.dtype == like.dtype and out.shape == like.shape, (out.dtype, out.shape, like.dtype, like.shape)
    return np.bitwise_xor(_bytes(out), _bytes(like))


def rebuild(like, x):
    """the reference's array, bit for bit, from the oracle's array it was stored against and the stored XOR"""
    like = np.ascontiguousarray(like)
    return np.bitwise_xor(_bytes(like), x).view(like.dtype).reshape(like.shape)


def pack(store):
    """a recording as a few arrays instead of two per call: every stored XOR one after the other (`xor`, lengths
    `xor_len`, in the order of `keys`) and the oracle digests as raw bytes (`oracle_sha256`, one row of 32 per key);
    other entries are kept as they are.  Packed(np.load(...)) reads it back with the store's interface."""
    keys = sorted(k[:-4] for k in store if k.endswith("_xor"))
    xs = [np.asarray(store[k + "_xor"], np.uint8) for k in keys]
    out = {k: v for k, v in store.items() if not (k.endswith("_xor") or k.endswith("_oracle_sha256"))}
    out["keys"] = np.array(keys)
    out["xor"] = np.concatenate(xs) if xs else np.zeros(0, np.uint8)
    out["xor_len"] = np.array([x.size for x in xs], np.int64)
    out["oracle_sha256"] = np.array([np.frombuffer(bytes.fromhex(str(store[k + "_oracle_sha256"])), np.uint8)
                                     for k in keys], np.uint8).reshape(len(keys), 32)
    return out


class Packed:
    """the store interface (store[tag_n + "_xor"], store[tag_n + "_oracle_sha256"]) over a packed recording"""

    def __init__(self, npz):
        keys = [str(k) for k in npz["keys"]]
        ends = np.cumsum(npz["xor_len"])
        self._xor = npz["xor"]
        self._at = {k: (int(e - n), int(e)) for k, e, n in zip(keys, ends, npz["xor_len"])}
        self._sha = {k: bytes(row).hex() for k, row in zip(keys, npz["oracle_sha256"])}
        self._other = {k: npz[k] for k in npz.files if k not in ("keys", "xor", "xor_len", "oracle_sha256")}

    def __getitem__(self, key):
        if key.endswith("_xor"):
            a, b = self._at[key[:-4]]
            return self._xor[a:b]
        if key.endswith("_oracle_sha256"):
            return np.array(self._sha[key[:-len("_oracle_sha256")]])
        return self._other[key]


class PinnedRef:
    """RefMap's interface for tests that compare the oracle with the reference, in two modes.

    Record (live=RefMap): calls go to the reference; every array it returns is stored next to the oracle's array for the
    same call on the same inputs (`like`) as the XOR of their bytes (all zero where they agree, so a few KB per frame),
    plus the SHA-256 of the oracle's array.  Replay (live=None): calls that only change the reference's state do
    nothing; a call that returns arrays first checks that the oracle still returns exactly what it returned when they
    were recorded, then rebuilds the reference's arrays bit for bit from `like` and the stored XOR.  So the comparisons
    run unchanged on a machine without the reference or a GPU."""

    def __init__(self, store, tag, live=None):
        self.store, self.tag, self.live, self.n = store, tag, live, 0

    def _pin(self, like, out):
        key = f"{self.tag}_{self.n}"
        self.n += 1
        if self.live is not None:
            self.store[key + "_xor"] = xor_against(out, like)
            self.store[key + "_oracle_sha256"] = np.array(digest(like))
            return np.ascontiguousarray(out)
        assert str(self.store[key + "_oracle_sha256"]) == digest(like), (
            f"{key}: the oracle's output is not the one the reference's output was recorded against "
            "(tests/golden/make_reference_pin.py records it again)")
        return rebuild(like, self.store[key + "_xor"])

    def _pin_all(self, like, out):
        if isinstance(like, dict):
            return {k: self._pin(like[k], None if out is None else out[k]) for k in sorted(like)}
        if isinstance(like, tuple):
            return tuple(self._pin(a, None if out is None else b) for a, b in zip(like, out or (None,) * len(like)))
        return self._pin(like, out)

    def _call(self, like, method, *args, derive=None):
        """derive: a function of the reference's output to pin instead of the output itself (e.g. some cells only,
        where the reference leaves the rest uninitialised); `like` is then the same function of the oracle's output"""
        out = None
        if self.live is not None:
            out = getattr(self.live, method)(*args)
            if derive is not None:
                out = derive(out)
        return self._pin_all(like, out)

    def move(self, pos, like):
        return self._call(like, "move", pos)

    def process_points(self, x, y, z, frame, like):
        return self._call(like, "process_points", x, y, z, frame)

    def map_feature(self, like, derive=None):
        return self._call(like, "map_feature", derive=derive)

    def layers(self, names, like):
        return self._call(like, "layers", names)

    def get_layer(self, name, like, derive=None):
        return self._call(like, "get_layer", name, derive=derive)

    def opt_move(self, opt_p, height_update, like):
        return self._call(like, "opt_move", opt_p, height_update)

    def state(self, like):
        return self._call(like, "state")

    def fuse_points(self, *args):
        if self.live is not None:
            self.live.fuse_points(*args)

    def raytracing(self):
        if self.live is not None:
            self.live.raytracing()

    def var_update(self, dv):
        if self.live is not None:
            self.live.var_update(dv)

    def closeloop(self, update_position, height_update):
        if self.live is not None:
            self.live.closeloop(update_position, height_update)

    def set_layer(self, name, arr):
        if self.live is not None:
            self.live.set_layer(name, arr)
