"""Cases for the gem_ros_* messages (DESIGN.md f15).  CPU only, no GPU or torch imports.

- map states (apply() to gem_b200.ElevationMap and oracle_lib.OracleMap alike, with move / set_layer / opt_move only):
  L in {1, 2, 3, 5, 31, 32, 33, 64, 257}, scrolled starts, the frame after opt_move, crafted layers (-10 cells, NaN
  and negative elevations, -0, colours 0 and 255, intensity bit patterns with NaN payloads);
- headers with frame_id lengths 0-20 and 300 (so that every layer of a grid map meets all 16 byte phases) and output
  base offsets 0-15;
- record clouds: empty, one record, three parts.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

f32 = np.float32
MAP_SIZES = [1, 2, 3, 5, 31, 32, 33, 64, 257]
FRAME_ID_LENGTHS = list(range(21)) + [300]
OFFSETS = list(range(16))
SPECIAL_BITS = np.array([0x7FC00000, 0x7FC00001, 0xFFA00000, 0x7F800001, 0x80000000, 0x00000000, 0x00000001, 0x7F800000,
                         0xFF800000, 0x3F800000], np.uint32)


def frame_id(n: int) -> str:
    return "".join(chr(ord("a") + i % 26) for i in range(n))


@dataclass
class MapCase:
    name: str
    L: int
    res: float
    moves: list          # positions passed to move(), in order
    opt: tuple | None    # (opt_p, height_update) for an opt_move after the layers are set
    seed: int

    def apply(self, m):
        for p in self.moves:
            m.move(np.asarray(p, f32))
        rng = np.random.default_rng(self.seed)
        L = self.L
        elev = rng.normal(0.0, 0.3, (L, L)).astype(f32)
        empty = rng.random((L, L)) < 0.2
        elev[empty] = f32(-10.0)
        flat = elev.reshape(-1)
        k = min(flat.size, 4)
        flat[rng.choice(flat.size, k, replace=False)] = np.array([-0.0, np.nan, -3.0, 5.5], f32)[:k]
        var = rng.uniform(0.0, 0.05, (L, L)).astype(f32)
        inten = rng.integers(0, 1 << 32, (L, L), dtype=np.uint64).astype(np.uint32)
        ib = inten.reshape(-1)
        ib[:min(ib.size, SPECIAL_BITS.size)] = SPECIAL_BITS[:ib.size]
        cols = [rng.choice(np.array([0, 255, 1, 128, 254], np.int32), (L, L)) for _ in range(3)]
        m.set_layer("elevation", elev)
        m.set_layer("variance", var)
        m.set_layer("intensity", inten.view(f32))
        for name, c in zip(("color_r", "color_g", "color_b"), cols):
            m.set_layer(name, c)
        if self.opt is not None:
            m.opt_move(np.asarray(self.opt[0], f32), self.opt[1])


def map_cases() -> list[MapCase]:
    out = []
    for i, L in enumerate(MAP_SIZES):
        res = 0.1 if L < 64 else 0.2
        out.append(MapCase(f"L{L}", L, res, [], None, 100 + i))
        out.append(MapCase(f"L{L}_scrolled", L, res, [(0.0, 0.0, 0.0), (res * (L // 3 + 1.2), -res * (L // 4 + 2.3), 0.0)],
                           None, 200 + i))
    out.append(MapCase("L33_opt_move", 33, 0.1, [(0.0, 0.0, 0.0), (0.75, 0.42, 0.0)], ((1.13, 0.27), 0.25), 301))
    out.append(MapCase("L64_opt_move", 64, 0.2, [(0.0, 0.0, 0.0), (-2.1, 3.3, 0.0)], ((-1.0, 2.05), -0.5), 302))
    return out


def case(name: str) -> MapCase:
    return next(c for c in map_cases() if c.name == name)


def records(n: int, seed: int = 0) -> np.ndarray:
    """n (8,) uint32 PointXYZRGBICT-like records with arbitrary bit patterns (the calls copy bytes)"""
    rng = np.random.default_rng(seed)
    rec = rng.integers(0, 1 << 32, (n, 8), dtype=np.uint64).astype(np.uint32)
    if n:
        rec[0, :min(8, SPECIAL_BITS.size)] = SPECIAL_BITS[:8]
    return rec


def cloud_parts():
    """name -> list of record arrays (the parts of one cloud)"""
    return {"empty": [], "empty_part": [records(0)], "one": [records(1, 1)],
            "three": [records(5, 2), records(0), records(77, 3)], "large": [records(3000, 4), records(1, 5)]}
