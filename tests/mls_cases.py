"""Crafted clouds for gem_mls_upsample (DESIGN.md f10), each named for what it exercises.  TEST INFRASTRUCTURE ONLY.

A case is (name, records, overrides): records an (n, 8) float32 array of PointXYZRGBICT records, overrides the
parameters that differ from GEM's (search radius 0.5, Gauss 0.25, order 5, RANDOM_UNIFORM_DENSITY at 1000)."""
from __future__ import annotations

import numpy as np

NONE = {"upsampling": "none"}


def records(xyz, seed=0):
    """PointXYZRGBICT records of the points: w = 1, a colour, covariance, intensity and travers that differ per point"""
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    n = xyz.shape[0]
    rng = np.random.default_rng(seed + 1000)
    r = np.zeros((n, 8), np.float32)
    r[:, :3] = xyz
    r[:, 3] = 1.0
    bgra = rng.integers(0, 256, (n, 4), dtype=np.uint32)
    r[:, 4] = (bgra[:, 0] | (bgra[:, 1] << 8) | (bgra[:, 2] << 16) | (bgra[:, 3] << 24)).astype(np.uint32).view(np.float32)
    r[:, 5] = rng.random(n, dtype=np.float32)
    r[:, 6] = rng.random(n, dtype=np.float32) * 100
    r[:, 7] = rng.random(n, dtype=np.float32) * 2 - 1
    return r


def lattice(step, half, z=None, rot=None):
    g = np.arange(-half, half + step / 2, step)
    x, y = np.meshgrid(g, g, indexing="ij")
    x, y = x.ravel(), y.ravel()
    zz = np.zeros_like(x) if z is None else z(x, y)
    p = np.stack([x, y, zz], 1)
    return p if rot is None else p @ np.asarray(rot).T


def rot(ax, ay):
    ca, sa, cb, sb = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay)
    rx = np.array([[1, 0, 0], [0, ca, -sa], [0, sa, ca]])
    ry = np.array([[cb, 0, sb], [0, 1, 0], [-sb, 0, cb]])
    return ry @ rx


POLY = {1: lambda x, y: 0.3 * x - 0.2 * y + 0.1,
        2: lambda x, y: 0.3 * x * x - 0.4 * x * y + 0.2 * y,
        3: lambda x, y: 0.5 * x ** 3 - 0.3 * y * y + 0.1 * x * y,
        4: lambda x, y: 0.4 * x ** 4 - 0.3 * x * y ** 3 + 0.2 * y * y,
        5: lambda x, y: 0.6 * x ** 5 - 0.4 * x * x * y ** 3 + 0.2 * y ** 4 - 0.1 * x}


def _cases():
    rng = np.random.default_rng(7)
    c = []
    c.append(("tilted_lattice_plane", records(lattice(0.1, 0.7, rot=rot(0.4, -0.3))), {}))
    c.append(("tilted_lattice_plane_none", records(lattice(0.1, 0.7, rot=rot(0.4, -0.3))), NONE))
    for o in range(1, 6):
        c.append((f"poly_surface_order{o}", records(lattice(0.08, 0.6, z=POLY[o])), {"order": o, "upsampling": "none"}))
        c.append((f"poly_surface_order{o}_sampled", records(lattice(0.1, 0.5, z=POLY[o])), {"order": o, "point_density": 400}))
    c.append(("two_neighbours", records([[0, 0, 0], [0.1, 0, 0], [5, 5, 5], [5.1, 5, 5]]), {}))
    c.append(("three_neighbours", records([[0, 0, 0], [0.1, 0, 0], [0, 0.1, 0.01], [5, 5, 5]]), {}))
    for k in (20, 21, 22):   # one cluster of exactly k points around nr_coeff = 21
        p = rng.normal(0, 0.08, (k, 3)) * [1, 1, 0.2]
        c.append((f"cluster_{k}_neighbours", records(p, k), NONE))
        c.append((f"cluster_{k}_neighbours_sampled", records(p, k), {}))
    # d2 exactly (float)(r r): 0.5^2 = 0.25 is exact, so the points at distance 0.5 on the axes are neighbours; the ones
    # one float step further are not
    e = np.float32(0.5)
    far = np.nextafter(e, np.float32(1))
    c.append(("boundary_exact_radius", records([[0, 0, 0], [e, 0, 0], [0, e, 0], [0, 0, e], [far, 0.0, 0], [0, -far, 0],
                                                [0.1, 0.1, 0]]), NONE))
    # equal d2: a ring of points at the same distance, in shuffled index order
    ang = np.arange(24) * (2 * np.pi / 24)
    ring = np.stack([0.25 * np.cos(ang), 0.25 * np.sin(ang), 0 * ang], 1).astype(np.float32)
    ring = np.concatenate([[[0, 0, 0]], ring[rng.permutation(24)], np.abs(ring[:6])], 0)
    c.append(("equal_d2_ties", records(ring), {"order": 3, "upsampling": "none"}))
    c.append(("equal_d2_ties_sampled", records(ring), {"order": 2}))
    p = lattice(0.1, 0.4, z=POLY[2]).astype(np.float32)
    p[3] = [np.nan, 0, 0]
    p[10] = [0, np.inf, 0]
    p[17] = [0, 0, -np.inf]
    p[25, 2] = np.nan
    c.append(("non_finite_records", records(p), {"order": 2}))
    line = np.stack([np.linspace(-0.4, 0.4, 40), np.linspace(-0.2, 0.2, 40), np.linspace(0, 0.1, 40)], 1)
    c.append(("collinear_singular", records(line), NONE))
    c.append(("collinear_singular_sampled", records(line), {}))
    # eigen33: an exactly planar set has c0 == 0 (computeRoots2); planes facing x, y and z and a random tilt select the
    # three cross products; near-z and near-xy normals take both unitOrthogonal branches
    c.append(("plane_normal_z_roots2", records(lattice(0.1, 0.5)), NONE))
    c.append(("plane_normal_x", records(lattice(0.1, 0.5)[:, [2, 0, 1]]), NONE))
    c.append(("plane_normal_y", records(lattice(0.1, 0.5)[:, [0, 2, 1]]), NONE))
    c.append(("noisy_plane_normal_z", records(lattice(0.1, 0.5) + rng.normal(0, 0.003, (121, 3))), NONE))
    c.append(("noisy_plane_normal_x", records(lattice(0.1, 0.5)[:, [2, 0, 1]] + rng.normal(0, 0.003, (121, 3))), NONE))
    c.append(("noisy_plane_normal_y", records(lattice(0.1, 0.5)[:, [0, 2, 1]] + rng.normal(0, 0.003, (121, 3))), NONE))
    c.append(("noisy_plane_tilted", records(lattice(0.1, 0.5, rot=rot(1.1, 0.7)) + rng.normal(0, 0.003, (121, 3))), {}))
    c.append(("density_zero", records(lattice(0.1, 0.5, z=POLY[3])), {"point_density": 0}))
    c.append(("density_k_hundreds", records([[0, 0, 0], [0.1, 0, 0], [0, 0.1, 0.02], [0.05, 0.05, 0.01]]), {"point_density": 3000}))
    c.append(("density_k_hundreds_fitted", records(lattice(0.2, 0.2, z=POLY[1]) + [0, 0, 0]), {"order": 1, "point_density": 4000}))
    # more than 512 neighbours: the global-memory sort of the long lists
    blob = rng.normal(0, 0.12, (700, 3)) * [1, 1, 0.3]
    c.append(("long_list_over_shared_budget", records(blob), {"order": 2, "point_density": 4000}))
    c.append(("long_list_over_shared_budget_none", records(blob), {"order": 5, "upsampling": "none"}))
    for o in range(1, 6):
        c.append((f"noisy_surface_order{o}", records(lattice(0.07, 0.5, z=POLY[5]) + rng.normal(0, 0.004, (225, 3))), {"order": o}))
    c.append(("no_polynomial_fit", records(lattice(0.1, 0.5, z=POLY[2])), {"polynomial_fit": False}))
    c.append(("no_polynomial_fit_none", records(lattice(0.1, 0.5, z=POLY[2])), {"polynomial_fit": False, "upsampling": "none"}))
    c.append(("small_radius_gauss", records(lattice(0.05, 0.3, z=POLY[2])), {"search_radius": 0.12, "sqr_gauss_param": 0.02,
                                                                            "order": 2}))
    c.append(("far_from_origin", records(lattice(0.1, 0.4, z=POLY[2]) + [1000.0, -2000.0, 50.0]), {"order": 2}))
    c.append(("seeded_draws", records(lattice(0.1, 0.5, z=POLY[2])), {"order": 2, "seed": 0xDEADBEEFCAFEF00D}))
    c.append(("empty", np.zeros((0, 8), np.float32), {}))
    return c


_CACHE = None


def cases():
    global _CACHE
    if _CACHE is None:
        _CACHE = _cases()
    return _CACHE


def case_names():
    return [c[0] for c in cases()]


def case_by_name(name):
    for c in cases():
        if c[0] == name:
            return c
    raise KeyError(name)


def blob(n, sigma, seed=3):
    """a dense 3D blob: thousands of neighbours per point at r = 0.5"""
    rng = np.random.default_rng(seed)
    return records(rng.normal(0, sigma, (n, 3)), seed)


def kitti_like(step=0.2, half=15.0, seed=5):
    """a KITTI-like 0.2 m grid cloud: a gently rolling ground, ~20 neighbours in 0.5 m, no fit, 25 samples per point"""
    rng = np.random.default_rng(seed)
    p = lattice(step, half, z=lambda x, y: 0.2 * np.sin(0.3 * x) + 0.1 * np.cos(0.2 * y))
    p = p[rng.random(p.shape[0]) < 0.9]
    return records(p, seed)
