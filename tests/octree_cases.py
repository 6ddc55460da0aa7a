"""gem_color_octree test material: an independent Python restatement of the ColorOcTree that pointCloudtoOctomap builds
(a dict per node, octomap's recursive updateNodeRecurs), a decoder of the writeData stream that checks its structure and
O5 on every inner node, and the crafted clouds of DESIGN.md f7.  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import math
import struct

import numpy as np

f32 = np.float32
HIT = f32(math.log(0.7 / 0.3))
MAX = f32(math.log(0.971 / 0.029))
WHITE = (255, 255, 255)


# ---- records --------------------------------------------------------------------------------------------------------
def records(xyz, rgb=None):
    """(n, 8) float32 PointXYZRGBICT records {x, y, z, 1, bgra, covariance, intensity, travers}"""
    xyz = np.asarray(xyz, f32).reshape(-1, 3)
    n = xyz.shape[0]
    rec = np.zeros((n, 8), f32)
    rec[:, :3] = xyz
    rec[:, 3] = 1.0
    rgb = np.full((n, 3), 100, np.uint32) if rgb is None else np.asarray(rgb, np.int64).reshape(-1, 3).astype(np.uint32)
    bgra = (np.uint32(255) << 24) | (rgb[:, 0] << 16) | (rgb[:, 1] << 8) | rgb[:, 2]
    rec.view(np.uint32)[:, 4] = bgra
    rec[:, 5] = 0.01
    rec[:, 6] = 7.0
    rec[:, 7] = 0.5
    return rec


def centres(keys, res):
    """float coordinates of the centres of integer voxel indices s (key - 32768)"""
    return ((np.asarray(keys, np.float64) + 0.5) * res).astype(f32)


# ---- the restatement ------------------------------------------------------------------------------------------------
def _new():
    return {"v": f32(0.0), "c": WHITE, "ch": None}


def _has_children(n):
    return n["ch"] is not None and any(c is not None for c in n["ch"])


def _avg_colour(n):
    s = [c["c"] for c in (n["ch"] or []) if c is not None and c["c"] != WHITE]
    if not s:
        return WHITE
    return tuple(sum(c[i] for c in s) // len(s) for i in range(3))


def _key(rf, c):
    c = float(f32(c))
    if not math.isfinite(c):
        return None
    s = math.floor(rf * c)
    return s + 32768 if -32768 <= s <= 32767 else None


def _pos(k, depth):
    d = 15 - depth
    return ((k[0] >> d) & 1) | (((k[1] >> d) & 1) << 1) | (((k[2] >> d) & 1) << 2)


class PyColorOcTree:
    def __init__(self):
        self.root = None

    def search(self, k):
        n = self.root
        for depth in range(16):
            if n is None or not _has_children(n):
                return n
            n = n["ch"][_pos(k, depth)]
        return n

    def _collapsible(self, n):
        ch = n["ch"]
        if ch is None or any(c is None or _has_children(c) for c in ch):
            return False
        return all(c["v"] == ch[0]["v"] for c in ch)

    def _recurs(self, n, just_created, k, depth):
        if depth == 16:
            v = f32(n["v"] + HIT)
            n["v"] = MAX if v > MAX else v
            return
        pos = _pos(k, depth)
        created = False
        if n["ch"] is None or n["ch"][pos] is None:
            if not _has_children(n) and not just_created:
                n["ch"] = [{"v": n["v"], "c": n["c"], "ch": None} for _ in range(8)]
            else:
                if n["ch"] is None:
                    n["ch"] = [None] * 8
                n["ch"][pos] = _new()
                created = True
        self._recurs(n["ch"][pos], created, k, depth + 1)
        if self._collapsible(n):
            c0 = n["ch"][0]
            n["v"], n["c"] = c0["v"], c0["c"]
            if n["c"] != WHITE:
                n["c"] = _avg_colour(n)
            n["ch"] = None

    def update_node(self, k):
        s = self.search(k)
        if s is not None and s["v"] >= MAX:
            return
        created = self.root is None
        if created:
            self.root = _new()
        self._recurs(self.root, created, k, 0)

    def integrate_colour(self, k, rgb):
        n = self.search(k)
        if n is None:
            return
        if n["c"] == WHITE:
            n["c"] = tuple(rgb)
        else:
            p = 1.0 - 1.0 / (1.0 + math.exp(float(n["v"])))
            n["c"] = tuple(int(pc * p + c * (0.99 - p)) for pc, c in zip(n["c"], rgb))

    def inner(self, n):
        if not _has_children(n):
            return
        for c in n["ch"]:
            if c is not None:
                self.inner(c)
        n["v"] = max(c["v"] for c in n["ch"] if c is not None)
        n["c"] = _avg_colour(n)

    def write(self, n, out):
        bits = 0
        if n["ch"] is not None:
            for i, c in enumerate(n["ch"]):
                if c is not None:
                    bits |= 1 << i
        out += struct.pack("<f", float(n["v"])) + bytes(n["c"]) + bytes([bits])
        if n["ch"] is not None:
            for c in n["ch"]:
                if c is not None:
                    self.write(c, out)


def py_color_octree(rec, resolution):
    """the restatement: (stream uint8 array, inserted, skipped)"""
    rec = np.asarray(rec, f32).reshape(-1, 8)
    rf = 1.0 / resolution
    t = PyColorOcTree()
    ins = 0
    for row in rec:
        k = [_key(rf, c) for c in row[:3]]
        if None in k:
            continue
        bgra = int(row[4:5].view(np.uint32)[0])
        t.update_node(k)
        t.integrate_colour(k, ((bgra >> 16) & 255, (bgra >> 8) & 255, bgra & 255))
        ins += 1
    out = bytearray()
    if t.root is not None:
        t.inner(t.root)
        t.write(t.root, out)
    return np.frombuffer(bytes(out), np.uint8), ins, rec.shape[0] - ins


# ---- the decoder ----------------------------------------------------------------------------------------------------
def decode(stream):
    """walk a ColorOcTree writeData stream: every node 8 bytes, preorder, children 0..7 by the bitset, depth <= 16, the
    stream consumed exactly; O5 checked on every inner node; every value one of the states O2 allows.  Returns
    (nodes, leaves)"""
    b = np.ascontiguousarray(stream, np.uint8).tobytes()
    assert len(b) % 8 == 0
    states = {float(HIT)}
    v = HIT
    while v < MAX:
        v = f32(v + HIT)
        v = MAX if v > MAX else v
        states.add(float(v))
    pos = 0
    counts = [0, 0]

    def node(depth):
        nonlocal pos
        assert pos + 8 <= len(b), "stream ends inside a node"
        val = struct.unpack_from("<f", b, pos)[0]
        rgb = tuple(b[pos + 4:pos + 7])
        bits = b[pos + 7]
        pos += 8
        counts[0] += 1
        assert float(val) in states, val
        if bits == 0:
            counts[1] += 1
            return val, rgb
        assert depth < 16, "an inner node at the leaf level"
        kids = [node(depth + 1) for i in range(8) if bits >> i & 1]
        assert val == max(k[0] for k in kids), (depth, val, kids)
        s = [k[1] for k in kids if k[1] != WHITE]
        want = tuple(sum(c[i] for c in s) // len(s) for i in range(3)) if s else WHITE
        assert rgb == want, (depth, rgb, want)
        return val, rgb

    if b:
        node(0)
    assert pos == len(b), "bytes after the root's subtree"
    return counts[0], counts[1]


# ---- crafted clouds -------------------------------------------------------------------------------------------------
def block_keys(origin, side, order="morton", rng=None):
    """the side^3 voxel indices of an aligned cube at `origin` (multiples of side), in Morton, reverse or random order"""
    g = np.arange(side)
    k = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    code = np.zeros(k.shape[0], np.int64)
    for d in range(8):
        for a in range(3):
            code |= ((k[:, a] >> d) & 1).astype(np.int64) << (3 * d + a)
    k = k[np.argsort(code, kind="stable")] + np.asarray(origin)
    if order == "reverse":
        k = k[::-1]
    elif order == "random":
        k = k[rng.permutation(k.shape[0])]
    return k


def cloud(keys, res, rgb=None):
    return records(centres(keys, res), rgb)


def crafted_cases():
    """(name, records, resolution) of every crafted family"""
    rng = np.random.default_rng(7)
    out = []
    out.append(("empty", records(np.zeros((0, 3))), 0.1))
    out.append(("one_point", records([[0.31, -0.52, 1.17]], [[10, 20, 30]]), 0.1))
    bad = []
    for v in (np.nan, np.inf, -np.inf, 1e18, -1e18, -32769.0, 32768.0):
        for a in range(3):
            p = [0.5, 0.5, 0.5]
            p[a] = v
            bad.append(p)
    out.append(("all_skipped", records(bad), 1.0))
    edge = [[-32768.0, -32768.0, -32768.0], [32767.5, 32767.5, 32767.5], [-32768.0, 32767.0, 0.0],
            [32767.999, -32767.5, -0.5]]
    out.append(("keys_0_and_65535", records(edge + bad[:6], [[1, 2, 3]] * 10), 1.0))
    for res in (0.1, 0.2, 0.05, 0.15):
        c = []
        for k in range(-6, 7):
            b = f32(k * res)
            for v in (np.nextafter(b, f32(-np.inf)), b, np.nextafter(b, f32(np.inf))):
                c.append([v, f32(-k * res), b])
                c.append([f32(0.3), v, np.nextafter(b, f32(np.inf))])
                c.append([v, v, v])
        out.append((f"boundaries_{res}", records(c, rng.integers(0, 256, (len(c), 3))), res))
    # one voxel hit 1..8 times, each voxel far from the others
    cols = [(255, 255, 255), (0, 0, 0), (200, 10, 90), (255, 255, 255), (3, 250, 128), (0, 0, 0), (255, 255, 254),
            (90, 90, 90)]
    pts, rgbs = [], []
    for h in range(1, 9):
        for variant in range(3):
            key = (10 * h, -10 * variant - 3, 5 * h)
            for j in range(h):
                pts.append(key)
                rgbs.append(cols[(j + variant * h) % 8] if variant < 2 else cols[0 if j % 2 else 1])
    out.append(("one_voxel_1_to_8_hits", cloud(pts, 0.1, rgbs), 0.1))
    # 2 x 2 x 2 blocks
    blk = block_keys((0, 0, 0), 2)
    col = rng.integers(0, 255, (64, 3))
    out.append(("block_equal_hits", cloud(np.concatenate([blk, blk[::-1]]), 0.1, col[:16]), 0.1))
    out.append(("block_unequal_hits", cloud(np.concatenate([blk, blk[:5]]), 0.1, col[:13]), 0.1))
    w = col[:8].copy()
    w[0] = 255
    out.append(("block_last_is_child0_white", cloud(blk[::-1], 0.1, w[::-1]), 0.1))
    out.append(("block_last_is_child0_coloured", cloud(blk[::-1], 0.1, col[:8]), 0.1))
    out.append(("block_last_not_child0", cloud(blk[[0, 1, 2, 3, 4, 5, 7, 6]], 0.1, col[:8]), 0.1))
    out.append(("block_all_white", cloud(blk, 0.1, [WHITE] * 8), 0.1))
    after = np.concatenate([blk, blk[[3]], blk[[0, 1, 2, 4, 5, 6, 7]], blk[[5]]])
    out.append(("block_hit_after_prune", cloud(after, 0.1, col[:after.shape[0]]), 0.1))
    sat = np.concatenate([blk] * 7 + [blk[[2, 6]]])
    out.append(("block_saturated", cloud(sat, 0.1, rng.integers(0, 256, (sat.shape[0], 3))), 0.1))
    half = np.concatenate([blk] * 4 + [blk[[0]], blk] + [blk[[1]]] * 3)
    out.append(("block_saturates_unevenly", cloud(half, 0.1, rng.integers(0, 256, (half.shape[0], 3))), 0.1))
    # cascades
    for side in (4, 8):
        for order in ("morton", "reverse", "random"):
            k = block_keys((-side, side, 0), side, order, rng)
            rep = np.concatenate([k, k[rng.permutation(k.shape[0])[: k.shape[0] // 3]]])
            out.append((f"cube{side}_{order}", cloud(rep, 0.1, rng.integers(0, 256, (rep.shape[0], 3))), 0.1))
    k = block_keys((0, 0, 0), 4)
    k = np.concatenate([k, k])
    out.append(("cube4_twice_saturating_order", cloud(np.concatenate([k, k, k]), 0.2, rng.integers(0, 256, (3 * k.shape[0], 3))), 0.2))
    seven = np.concatenate([block_keys((2 * i, 0, 0), 2)[[j for j in range(8) if j != i % 8]] for i in range(8)])
    out.append(("seven_of_eight", cloud(seven, 0.1, rng.integers(0, 256, (seven.shape[0], 3))), 0.1))
    mixed = np.concatenate([block_keys((0, 0, 0), 4, "random", rng), block_keys((4, 0, 0), 2, "random", rng),
                            [[6, 0, 0], [7, 1, 1], [-1, -1, -1], [4, 4, 4], [3, 4, 0]], block_keys((8, 8, 8), 8, "random", rng),
                            block_keys((0, 0, 0), 4, "random", rng)[:20]])
    mixed = mixed[rng.permutation(mixed.shape[0])]
    out.append(("full_subtrees_beside_leaves", cloud(mixed, 0.1, rng.integers(0, 256, (mixed.shape[0], 3))), 0.1))
    # small random clouds with many points per voxel (the restatement is slow; the GPU suite runs large ones)
    for i, (n, box) in enumerate(((3000, 6), (5000, 12), (4000, 3))):
        k = rng.integers(-box, box, (n, 3))
        out.append((f"random_small_{i}", cloud(k, 0.1, rng.integers(0, 256, (n, 3))), 0.1))
    return out


def random_cloud(rng, n, box, voxels, res=0.1):
    """n points drawn among `voxels` random voxel indices in [-box, box)^3 (many points per voxel), jittered inside
    their voxel, random colours"""
    vk = rng.integers(-box, box, (voxels, 3))
    k = vk[rng.integers(0, voxels, n)]
    xyz = ((k + rng.uniform(0.02, 0.98, (n, 3))) * res).astype(f32)
    return records(xyz, rng.integers(0, 256, (n, 3)))
