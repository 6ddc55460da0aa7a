"""Crafted call sequences for the global map's submap stack (gem_global_map_*, DESIGN.md f16).  TEST INFRASTRUCTURE ONLY.

A case is a list of operations run in order on a stack (gem_b200.ElevationMap, global_map_oracle.OracleStack or
PyStack): ("push", records (n, 8) float32, pose 4 x 4), ("update", opt_poses (k, 4, 4), resolution, radius) or
("reset",).  `run` applies them and returns the fused count of every update and the state after every operation."""
from __future__ import annotations

import numpy as np

import refuse_cases as rc

F = np.float32
RES = 0.1


def pose(yaw=0.0, x=0.0, y=0.0, z=0.0, q=None):
    """a row-major 4 x 4 float32 pose from a yaw or a quaternion (w, x, y, z), and a translation"""
    if q is not None:
        w, a, b, c = np.asarray(q, np.float64) / np.linalg.norm(q)
        R = np.array([[1 - 2 * (b * b + c * c), 2 * (a * b - c * w), 2 * (a * c + b * w)],
                      [2 * (a * b + c * w), 1 - 2 * (a * a + c * c), 2 * (b * c - a * w)],
                      [2 * (a * c - b * w), 2 * (b * c + a * w), 1 - 2 * (a * a + b * b)]])
    else:
        R = np.array([[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]])
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = (x, y, z)
    return T.astype(np.float32)


def submap(name, cx, cy, n, var=None, spread=40, res=RES):
    """n records in cells around (cx, cy), some cells repeated"""
    rng = rc._rng(name)
    c = rng.integers(0, max(1, n // 2), n)
    ix = c % spread + int(np.floor(cx / res)) - spread // 2
    iy = c // spread + int(np.floor(cy / res)) - 5
    x, y = rc.in_cell(rng, ix, iy, res)
    if var is None:
        var = rng.choice(np.array([0.2, 0.5, 0.8, 1.0], np.float32), n)
    return rc.records(rng, x, y, var=var)


def chain(name, centres, sizes, poses=None):
    """pushes of submaps around the given keyframe centres: submap s lies around centre s (centre 0 is the origin), and
    keyframe s + 1 is pushed with it"""
    ops = []
    for s, n in enumerate(sizes):
        cx, cy = centres[s]
        nxt = poses[s + 1] if poses is not None else pose(0.0, *centres[s + 1]) if s + 1 < len(centres) else pose(0.0, cx + 1.0, cy)
        ops.append(("push", submap(f"{name}/{s}", cx, cy, n), nxt))
    return ops


def perturbed(kf_poses, seed, k=None, rot=0.004, shift=0.05):
    rng = np.random.default_rng(seed)
    out = []
    for P in kf_poses[: (len(kf_poses) if k is None else k)]:
        d = pose(rng.uniform(-rot, rot), *rng.uniform(-shift, shift, 2))
        out.append((d.astype(np.float64) @ P.astype(np.float64)).astype(np.float32))
    return np.array(out, np.float32).reshape(-1, 4, 4)


def _line(K, step=2.0):
    return [(step * s, 0.3 * (s % 2)) for s in range(K + 1)]


def _kf(centres):
    return [pose(0.0, *c) for c in centres]


def case_gate(K):
    """K submaps all within the radius: K = 0-2 never fuse (not more than two results), K = 3 does"""
    cen = _line(K)
    ops = chain(f"gate{K}", cen, [600, 900, 750][:K])
    return ops + [("update", perturbed(_kf(cen), K, K + 1), RES, 25.0)]


def case_k(k):
    cen = _line(4)
    ops = chain(f"k{k}", cen, [500, 800, 640, 700])
    return ops + [("update", perturbed(_kf(cen), 11, k) if k else np.zeros((0, 4, 4), np.float32), RES, 25.0)]


def case_coincident():
    """keyframes 1 and 2 share a centre: i is not always first in its own list (a tie by distance 0, broken by index)"""
    cen = [(0.0, 0.0), (3.0, 1.0), (3.0, 1.0), (5.0, 0.0), (5.0, 0.0)]
    return chain("coincident", cen, [400, 700, 650, 500]) + [("update", perturbed(_kf(cen), 5), RES, 25.0)]


def case_at_radius():
    """centres exactly at the radius, and one float beyond"""
    r = 4.0
    beyond = float(np.nextafter(F(r), F(10)))
    cen = [(0.0, 0.0), (r, 0.0), (0.0, r), (0.0, -beyond), (r, r)]
    return chain("at_radius", cen, [500, 500, 500, 500]) + [("update", perturbed(_kf(cen), 6), RES, r)]


def case_nan_and_empty():
    """a NaN centre (no neighbours, nobody's neighbour) and empty submaps in the middle of the stack"""
    cen = [(0.0, 0.0), (2.0, 0.0), (float("nan"), 1.0), (4.0, 0.5), (6.0, 0.0), (7.0, 1.0)]
    kf = _kf(cen)
    ops = []
    for s, n in enumerate([600, 0, 700, 800, 0]):
        ops.append(("push", submap(f"nan/{s}", *((3.0, 1.0) if s == 2 else cen[s]), n), kf[s + 1]))
    return ops + [("update", perturbed(kf, 7), RES, 25.0)]


def case_variance():
    """shared cells whose old variance is 0, in (0, 1), 1 and NaN"""
    cen = _line(3, 0.5)
    ops = []
    for s, v in enumerate([F(0.0), F(0.5), F(1.0)]):
        var = np.full(300, v, np.float32)
        var[::7] = rc._bits([0x7fc00000])[0]
        var[1::7] = F(0.3)
        ops.append(("push", submap("variance", 0.0, 0.0, 300, var=var, spread=10), pose(0.0, *cen[s + 1])))
    return ops + [("update", perturbed(_kf(cen), 8), RES, 25.0)]


def case_quaternion_utm():
    """arbitrary quaternion poses at UTM-scale translations"""
    rng = np.random.default_rng(9)
    base = np.array([448_251.3, 5_411_937.6])
    cen = [(0.0, 0.0)] + [tuple(base + rng.uniform(-6, 6, 2)) for _ in range(4)]
    kf = [np.eye(4, dtype=np.float32)] + [pose(x=c[0], y=c[1], z=rng.uniform(-2, 2), q=rng.normal(size=4)) for c in cen[1:]]
    cen = [(float(P[0, 3]), float(P[1, 3])) for P in kf]
    ops = chain("utm", cen, [300, 800, 900, 700], poses=kf + [pose(0.0, *cen[-1])])
    return ops + [("update", perturbed(kf, 10, rot=0.02, shift=0.3), 0.2, 25.0)]


def case_sequence():
    """two updates in a row (the second from the updated trajectory_), pushes after an update, a reset in between"""
    cen = _line(5, 1.5)
    kf = _kf(cen)
    ops = chain("seq", cen[:4], [500, 700, 600])
    ops.append(("update", perturbed(kf, 12, 4), RES, 25.0))
    ops.append(("update", perturbed(kf, 13, 4), RES, 25.0))
    ops += chain("seq2", cen[3:], [650, 550])[:2]
    ops.append(("update", perturbed(kf, 14), RES, 25.0))
    ops.append(("reset",))
    ops += chain("seq3", _line(3), [400, 500, 450])
    ops.append(("update", perturbed(_kf(_line(3)), 15), RES, 25.0))
    return ops


CASES = {
    **{f"gate_K{K}": (lambda K=K: case_gate(K)) for K in range(4)},
    **{f"k_{k}": (lambda k=k: case_k(k)) for k in (0, 2, 4, 6)},
    "coincident": case_coincident,
    "at_radius": case_at_radius,
    "nan_and_empty": case_nan_and_empty,
    "variance": case_variance,
    "quaternion_utm": case_quaternion_utm,
    "sequence": case_sequence,
}


def run(stack, ops, compat=True):
    """apply ops to a stack; returns (fused counts of the updates, state after every op)"""
    fused, states = [], []
    for op in ops:
        if op[0] == "push":
            stack.push(op[1], op[2])
        elif op[0] == "reset":
            stack.reset()
        else:
            fused.append(stack.update(op[1], op[2], op[3], compat))
        states.append(stack.state())
    return fused, states
