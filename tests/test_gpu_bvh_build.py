"""The device builders (csrc/bvh_build_device.cu) against the host builder they reproduce (csrc/bvh_build.cpp): the BVH2 (nodes, tri_pos,
tri_index, max_depth) and the 4-wide tree (nodes, max_stack) byte for byte, in both library flavours, on the full-size configs, the dumped
reference asset, seeded triangle soups, tiny and degenerate meshes, and special float values; then the trees an upload and an update commit."""
import os

import numpy as np
import pytest

from etx_tracer_b200 import scenes, structs as S

gpu = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FLAVORS = ["fast", "parity"]
WIDE_STACK = 96  # kWideStackSize (csrc/bvh.h)


@pytest.fixture(scope="module")
def api():
    from etx_tracer_b200 import api as m
    return m


@pytest.fixture(scope="module", params=FLAVORS)
def ctx(api, request):
    g = api.GPUVCM(None, flavor=request.param)
    yield g
    g.close()


def _soup(tris):
    """float[T, 3, 3] -> (positions float[3T, 3], indices uint32[T, 3])"""
    tris = np.asarray(tris, dtype=np.float32).reshape(-1, 3, 3)
    return tris.reshape(-1, 3), np.arange(tris.shape[0] * 3, dtype=np.uint32).reshape(-1, 3)


def _mesh(sd):
    return sd.a_vertices["pos"].astype(np.float32), sd.a_triangles["i"].astype(np.uint32)


def _same_trees(g, positions, indices):
    host = g.debug_build_trees(positions, indices, device=False)
    dev = g.debug_build_trees(positions, indices, device=True)
    assert host["max_depth"] == dev["max_depth"]
    assert host["bvh_nodes"].tobytes() == dev["bvh_nodes"].tobytes()
    assert host["tri_pos"].tobytes() == dev["tri_pos"].tobytes()
    assert host["tri_index"].tobytes() == dev["tri_index"].tobytes()
    assert host["max_stack"] == dev["max_stack"]
    assert host["wide_nodes"].tobytes() == dev["wide_nodes"].tobytes()
    return host


# ---- seeded corpora ---------------------------------------------------------------------------------------------------------------------------
def _uniform(n=20000, seed=1):
    r = np.random.default_rng(seed)
    c = r.uniform(-10, 10, (n, 1, 3))
    return _soup(c + r.normal(0, 0.05, (n, 3, 3)))


def _clustered(n=30000, seed=2):
    r = np.random.default_rng(seed)
    centers = r.uniform(-100, 100, (12, 3))
    c = centers[r.integers(0, 12, n)][:, None, :] + r.normal(0, 0.5, (n, 1, 3)) * r.choice([1e-3, 1.0], (n, 1, 1))
    return _soup(c + r.normal(0, 0.01, (n, 3, 3)))


def _long_thin(n=20000, seed=3):
    r = np.random.default_rng(seed)
    a = r.uniform(-50, 50, (n, 1, 3))
    d = r.normal(0, 1, (n, 1, 3))
    d *= r.uniform(5, 40, (n, 1, 1)) / np.linalg.norm(d, axis=2, keepdims=True)
    return _soup(np.concatenate([a, a + d, a + d * 0.5 + r.normal(0, 1e-3, (n, 1, 3))], axis=1))


def _small(n):
    r = np.random.default_rng(100 + n)
    return _soup(r.uniform(-1, 1, (n, 3, 3)))


def _identical(n=300):
    return _soup(np.tile(np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32), (n, 1, 1)))


def _collinear(n=500, seed=4):
    # every centroid on the x axis: the y and z centroid extents are zero
    r = np.random.default_rng(seed)
    x = np.sort(r.uniform(-5, 5, n)).astype(np.float32)
    t = np.zeros((n, 3, 3), np.float32)
    t[:, :, 0] = x[:, None]
    t[:, 1, 1], t[:, 2, 1] = 0.5, -0.5
    t[:, 1, 2], t[:, 2, 2] = -0.25, 0.25
    return _soup(t)


def _coplanar(n=800, seed=5):
    # every centroid in the plane z = 0, some repeated
    r = np.random.default_rng(seed)
    xy = r.integers(0, 20, (n, 2)).astype(np.float32)
    t = np.zeros((n, 3, 3), np.float32)
    t[:, :, :2] = xy[:, None, :]
    t[:, 1, 0] += 0.3
    t[:, 2, 2] = 0.0
    t[:, 1, 2], t[:, 2, 2] = 0.2, -0.2
    return _soup(t)


def _geometric(n=120):
    # triangles at x = 2^k: SAH peels one off per level until the depth limit takes over with median splits
    x = np.ldexp(1.0, np.arange(n) - 60).astype(np.float32)
    w = x * np.float32(0.25)
    t = np.zeros((n, 3, 3), np.float32)
    t[:, 0, 0], t[:, 1, 0], t[:, 2, 0] = x, x + w, x
    t[:, 2, 1] = w
    return _soup(t)


def _nested(levels=50, seed=6):
    # at every level a few wide triangles around a much smaller copy of the rest: SAH peels the levels off one by one into the depth
    # limit's median splits, and the wide tree's stack grows past kWideStackSize
    r = np.random.default_rng(seed)
    out = []
    s = 1.0
    for _ in range(levels):
        c = r.uniform(-1, 1, (6, 1, 3)) * s
        out.append(c + r.uniform(-0.2, 0.2, (6, 3, 3)) * s)
        s *= 0.3
    return _soup(np.concatenate(out))


def _special(seed=7):
    r = np.random.default_rng(seed)
    base = r.uniform(-1, 1, (400, 3, 3)).astype(np.float32)
    v = base.reshape(-1)
    k = len(v)
    idx = r.permutation(k)
    big = np.float32(3.4028235e38)
    v[idx[0:200]] = 0.0
    v[idx[200:400]] = -0.0
    v[idx[400:500]] = np.float32(1e-40) * r.choice([-1, 1], 100)  # denormals
    v[idx[500:560]] = big * r.choice([-1, 1], 60)
    v[idx[560:600]] = np.nextafter(big, 0) * r.choice([-1, 1], 40)
    v[idx[600:610]] = np.inf
    v[idx[610:620]] = -np.inf
    v[idx[620:630]] = np.nan
    return _soup(v.reshape(-1, 3, 3))


def _signed_zeros(seed=8):
    # boxes whose extremes are +0 and -0 in varying order, in bins and in nodes
    r = np.random.default_rng(seed)
    t = r.choice([0.0, -0.0, 1.0, -1.0, 0.5], (600, 3, 3)).astype(np.float32)
    return _soup(t)


CORPUS = {
    "uniform": _uniform, "clustered": _clustered, "long_thin": _long_thin, "identical": _identical, "collinear": _collinear,
    "coplanar": _coplanar, "geometric": _geometric, "nested": _nested, "special": _special, "signed_zeros": _signed_zeros,
    **{f"tris{n}": (lambda n=n: _small(n)) for n in range(6)},
}


@gpu
@pytest.mark.parametrize("name", sorted(CORPUS))
def test_device_trees_equal_host_trees(ctx, name):
    host = _same_trees(ctx, *CORPUS[name]())
    if name == "tris0":
        assert host["bvh_nodes"].shape[0] == 1 and host["tri_index"][0] == 0xFFFFFFFF
    print(f"{name}: {host['bvh_nodes'].shape[0]} nodes, max_depth {host['max_depth']}, max_stack {host['max_stack']}")


@gpu
def test_depth_limit_and_rejected_wide_tree(ctx):
    host = _same_trees(ctx, *_nested())
    assert 56 <= host["max_depth"] < 64  # below kBvhStackSize, through the depth limit's median splits
    assert host["max_stack"] >= WIDE_STACK


@gpu
def test_reference_asset(ctx):
    z = np.load(os.path.join(GOLDEN, "ref_cornell_40.npz"))
    v = np.frombuffer(z["vertices"].tobytes(), dtype=S.VERTEX)
    t = np.frombuffer(z["triangles"].tobytes(), dtype=S.TRIANGLE)
    _same_trees(ctx, v["pos"].astype(np.float32), t["i"].astype(np.uint32))


@gpu
@pytest.mark.parametrize("name", ["C1", "C2", "C3", "C4", "C5"])
def test_full_size_configs(api, name):
    pos, idx = _mesh(scenes.config(name, scale=1.0 / 64))  # the film is shrunk; the geometry is the config's
    for flavor in FLAVORS:
        g = api.GPUVCM(None, flavor=flavor)
        host = _same_trees(g, pos, idx)
        dev = g.debug_build_trees(pos, idx, device=True)
        print(f"{name} {flavor}: {idx.shape[0]} triangles, host {host['seconds'] * 1e3:.1f} ms, device {dev['seconds'] * 1e3:.1f} ms")
        g.close()


# ---- committed trees ------------------------------------------------------------------------------------------------------------------
def _plastic_box():
    return scenes.material_box("plastic", 32, 32, samples=4)


def _moved(sd):
    # one vertex moved along the normal of its wall
    sd.a_vertices["pos"][0] += np.float32(0.01)
    return sd


def _committed(g):
    return (g.buffer(S.BUF_BVH_NODES, np.uint8).tobytes(), g.buffer(S.BUF_BVH_TRIS, np.uint8).tobytes(), g.buffer(S.BUF_WIDE_NODES, np.uint8).tobytes())


def _expected(g, sd, wide):
    host = g.debug_build_trees(*_mesh(sd), device=False)
    return host["bvh_nodes"].tobytes(), host["tri_pos"].tobytes(), host["wide_nodes"].tobytes() if wide else b""


@gpu
@pytest.mark.parametrize("flavor", FLAVORS)
def test_upload_and_update_commit_the_host_trees(api, flavor):
    s1 = _plastic_box()
    a = api.GPUVCM(s1, flavor=flavor)
    wide = a.debug_select_tree(True)
    assert wide == (flavor == "fast")  # plastic is stochastic: the product build walks the 4-wide tree
    assert _committed(a) == _expected(a, s1, wide)
    s2 = _moved(_plastic_box())
    info = a.update_scene(s2)
    assert not (info["kept"] & S.KEPT_GEOMETRY) and info["bvh_seconds"] > 0.0
    assert _committed(a) == _expected(a, s2, wide)
    a.render(1)
    a.close()


@gpu
def test_group_update_commits_the_host_trees(api):
    s1 = _plastic_box()
    g = api.GPUVCMGroup(s1, lanes=2, flavor="fast")
    for lane in g.lanes:
        assert _committed(lane) == _expected(lane, s1, True)
    s2 = _moved(_plastic_box())
    g.update_scene(s2)
    for lane in g.lanes:
        assert _committed(lane) == _expected(lane, s2, True)
    g.close()


@gpu
def test_camera_only_update_builds_nothing(api):
    s1, s2 = _plastic_box(), _plastic_box()
    s2.set_camera([0.2, 1.1, 3.6], [0.0, 0.9, -6.18], [0.0, 1.0, 0.0], s2.width, s2.height, 39.6, clip_near=0.1, clip_far=100.0)
    a = api.GPUVCM(s1, flavor="fast")
    before = _committed(a)
    info = a.update_scene(s2)
    assert info["kept"] & S.KEPT_GEOMETRY and info["bvh_seconds"] == 0.0
    assert _committed(a) == before
    a.close()


@gpu
def test_refused_update_keeps_the_committed_tree(api):
    s1 = _plastic_box()
    a = api.GPUVCM(s1, flavor="fast")
    before = _committed(a)
    bad = _plastic_box()
    bad.a_triangles["i"][0, 0] = 1 << 30
    with pytest.raises(api.EtxbError):
        a.update_scene(bad)
    assert _committed(a) == before
    a.render(1)
    a.close()


@gpu
def test_device_memory_flat_over_geometry_edits(api):
    import torch
    s1, s2 = _plastic_box(), _moved(_plastic_box())
    a = api.GPUVCM(s1, flavor="fast")
    levels = []
    for k in range(20):
        a.update_scene(s2 if k % 2 == 0 else s1)
        torch.cuda.synchronize()
        levels.append(torch.cuda.mem_get_info()[0])
    assert levels[-1] >= levels[2], levels
    a.close()
