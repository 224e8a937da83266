"""The product build's walk of the 4-wide quantised tree (dwide.cuh) against an independent answer: seeded closest-hit and occlusion queries on
BASELINE config 3's million-triangle room, every ray against EVERY triangle in float64 (no BVH, no shared code).  Closest hits go through
etxb_debug_trace (k_debug_trace with `wide`), which calls trace_closest_wide as k_trace_closest_wide does; occlusion queries go through
etxb_debug_occluded (k_debug_occluded), which sets its segments up with shadow_segment as k_shadow_resolve does and walks them with wide_step,
the walk of k_shadow_resolve<true>.  Rays include axis-aligned directions and directions with one zero component, where the reciprocal guard
of wide_begin matters; the occlusion queries also run through the BVH2 walks of both builds."""
import ctypes as C

import numpy as np
import pytest

from etx_tracer_b200 import scenes, structs as S

pytestmark = pytest.mark.gpu

RAY_EPSILON = 15.0 / (65504.0 - 1.0)  # dcore.cuh kRayEpsilon


@pytest.fixture(scope="module")
def room():
    sd = scenes.procedural_room(32, 18, env_size=(64, 32))
    sc = sd.scene
    nv, nt = int(sc["vertices"]["count"][0]), int(sc["triangles"]["count"][0])
    verts = np.frombuffer((C.c_char * (nv * S.VERTEX.itemsize)).from_address(int(sc["vertices"]["a"][0])), dtype=S.VERTEX)
    tris = np.frombuffer((C.c_char * (nt * S.TRIANGLE.itemsize)).from_address(int(sc["triangles"]["a"][0])), dtype=S.TRIANGLE)
    pos = verts["pos"].astype(np.float64)
    a, b, c = pos[tris["i"][:, 0]], pos[tris["i"][:, 1]], pos[tris["i"][:, 2]]
    return sd, a, b - a, c - a, pos.min(axis=0), pos.max(axis=0)


def hit_distances(o, d, a, e1, e2):
    """Moeller-Trumbore in float64 of one ray against every triangle: the distance along d, +inf where it misses."""
    pv = np.cross(d, e2)
    det = (e1 * pv).sum(axis=1)
    ok = np.abs(det) > 0
    inv = np.where(ok, 1.0 / np.where(ok, det, 1.0), 0.0)
    tv = o - a
    u = (tv * pv).sum(axis=1) * inv
    qv = np.cross(tv, e1)
    v = (qv * d).sum(axis=1) * inv
    t = (qv * e2).sum(axis=1) * inv
    return np.where(ok & (u >= 0) & (v >= 0) & (u + v <= 1), t, np.inf)


def directions(rng, n):
    d = rng.normal(size=(n, 3))
    d[:24] = 0.0  # axis-aligned, both signs
    d[np.arange(24), np.arange(24) % 3] = np.where(np.arange(24) % 2 == 0, 1.0, -1.0)
    d[np.arange(24, 48), np.arange(24) % 3] = 0.0  # one zero component
    return d / np.linalg.norm(d, axis=1, keepdims=True)


def test_wide_walk_closest_hits_against_float64_brute_force(api_lib, room):
    sd, a, e1, e2, lo, hi = room
    rng = np.random.default_rng(2024)
    n = 192
    rays = np.zeros((n, 8), dtype=np.float32)
    rays[:, 0:3] = lo + (hi - lo) * (0.2 + 0.6 * rng.random((n, 3)))
    rays[:, 4:7] = directions(rng, n)
    rays[:, 3], rays[:, 7] = 1e-4, 3.0e38
    o64, d64 = rays[:, 0:3].astype(np.float64), rays[:, 4:7].astype(np.float64)
    best_t, best_tri = np.full(n, np.inf), np.full(n, -1, dtype=np.int64)
    for k in range(n):
        t = hit_distances(o64[k], d64[k], a, e1, e2)
        t = np.where(t > 1e-4, t, np.inf)
        j = int(t.argmin())
        if np.isfinite(t[j]):
            best_t[k], best_tri[k] = t[j], j
    assert (best_tri >= 0).mean() > 0.5
    g = api_lib.GPUVCM(sd, flavor="fast")
    assert g.debug_select_tree(True), "the room has stochastic BSDFs: the product build must have built the wide tree"
    uvt, tri, _ = g.debug_trace(rays, np.arange(n, dtype=np.uint32) + 11)
    g.close()
    found = tri != S.INVALID
    assert np.array_equal(found, best_tri >= 0)
    np.testing.assert_allclose(uvt[found, 2], best_t[found], rtol=2e-4, atol=1e-5)
    assert (tri[found].astype(np.int64) == best_tri[found]).mean() > 0.97  # edge / coplanar ties may name another triangle at the same distance


def test_wide_walk_occlusion_against_float64_brute_force(api_lib, room):
    sd, a, e1, e2, lo, hi = room
    rng = np.random.default_rng(4048)
    n = 192
    p0 = lo + (hi - lo) * (0.2 + 0.6 * rng.random((n, 3)))
    length = np.linalg.norm(hi - lo) * (0.05 + 0.6 * rng.random(n))
    p1 = p0 + directions(rng, n) * length[:, None]
    segments = np.concatenate([p0, p1], axis=1).astype(np.float32)
    s0, s1 = segments[:, 0:3].astype(np.float64), segments[:, 3:6].astype(np.float64)
    expect, clear_cut = np.zeros(n, dtype=bool), np.ones(n, dtype=bool)
    for k in range(n):
        d = s1[k] - s0[k]
        dist = np.linalg.norm(d)
        t_max = dist - max(RAY_EPSILON, dist * RAY_EPSILON)  # the segment as k_shadow_resolve shortens it
        t = hit_distances(s0[k], d / dist, a, e1, e2)
        expect[k] = ((t > RAY_EPSILON) & (t < t_max)).any()
        # a surface within a hair of either end decides on float rounding: such a segment does not count
        clear_cut[k] = not ((np.abs(t - t_max) < 1e-4 * dist) | (np.abs(t - RAY_EPSILON) < 1e-4)).any()
    assert clear_cut.mean() > 0.9
    assert 0.1 < expect[clear_cut].mean() < 0.9, expect[clear_cut].mean()
    for flavor, wide in (("fast", True), ("fast", False), ("parity", False)):
        g = api_lib.GPUVCM(sd, flavor=flavor)
        assert g.debug_select_tree(wide) or not wide
        got = g.debug_occluded(segments)
        g.close()
        assert np.array_equal(got[clear_cut], expect[clear_cut]), (flavor, wide, np.flatnonzero(got[clear_cut] != expect[clear_cut]))


@pytest.fixture(scope="module")
def api_lib():
    from etx_tracer_b200 import api as m
    return m
