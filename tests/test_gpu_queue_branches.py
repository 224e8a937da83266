"""The large-queue branches of the light and camera passes render what the small-queue branches render (product build).

A pass over a long queue takes other code paths than one over a short queue (module.cu, etxb_debug_thresholds): the gather queue is sorted
by its merge keys, the gather gives each warp several queries (and the closure gather mixes their pairs in one shared list), vertex
connections run over a host-sized, material-pair-sorted list, path queues are grouped by material, and the queue size is read back every
bounce.  Within one render these branches differ only in order: the per-pair and per-photon sampler streams are keyed by the light-vertex
ordinal or the photon index, the Lambert gather's lane assignment depends only on the query's own cells, and every query moves its path's
stream on by one draw.  So a small film rendered with every large-queue branch forced on equals the same film with every branch forced off:
integer state and sampler states bit for bit, float-atomic sums (films, gathered camera values) within 1e-6 relative L2.  The forced
branches are proven to have run through etxb_debug_get_branch_counts.  The natural-size cases (C3 at 512x288, C4 at 384x384: 147 456
paths, so the first bounce runs 32 queries per warp on up to 144 SMs) render with the default thresholds against the same film with every
branch forced off."""
import functools

import numpy as np
import pytest

from conftest import bit_equal, rel_l2
from etx_tracer_b200 import scenes, structs as S

gpu = pytest.mark.gpu

FORCED_ON = dict(merge_sort_min_queries=0, merge_min_warps_per_sm=0, tail_queue=0, sort_queue_min=0)
FORCED_OFF = dict(merge_sort_min_queries=S.NEVER, merge_min_warps_per_sm=S.NEVER, tail_queue=S.NEVER, sort_queue_min=S.NEVER, merge_qpw=1)
QPW = (2, 8, 32)  # 32 = what a long queue runs; 2 leaves warps half empty

EXACT_BUFFERS = ((S.BUF_LIGHT_SAMPLER, np.uint32), (S.BUF_CAMERA_SAMPLER, np.uint32), (S.BUF_LIGHT_PATH_COUNT, np.uint32),
                 (S.BUF_LIGHT_PATH_OFFSET, np.uint32), (S.BUF_PHOTON_RECORDS, np.uint32))


def _connect_only():
    o = S.default_vcm_options()
    o["options"] = S.VCM_CONNECT_ONLY
    return o


def _stochastic(sd):
    """the scene has a surface the generic gather and the connection stage handle (module.cu validate_scene: not Lambert, not always delta)"""
    for m in sd.a_materials:
        lambert = int(m["cls"]) == S.MAT_DIFFUSE and int(m["diffuse_variation"]) == 0
        smooth = max(float(m["roughness"]["value"][0]), float(m["roughness"]["value"][1])) <= 1e-4 and int(m["roughness"]["image_index"]) == S.INVALID
        delta = (int(m["cls"]) in (S.MAT_DIELECTRIC, S.MAT_CONDUCTOR) and smooth) or int(m["cls"]) in (S.MAT_THINFILM, S.MAT_MIRROR, S.MAT_VOID)
        if not lambert and not delta:
            return True
    return False


# name -> (scene factory, iterations, options factory or None)
SCENES = {
    "c1_cornell": (lambda: scenes.cornell_box(64, 64, samples=16, spectral=False), 2, None),
    "c2_cornell_sphere": (lambda: scenes.cornell_box(64, 64, samples=256, spectral=True, sphere=True, sphere_segments=32, sphere_rings=17), 2, None),
    "c3_room": (lambda: scenes.procedural_room(64, 36, env_size=(256, 128)), 2, None),
    "c4_dragon": (lambda: scenes.sss_dragon(40, 40), 2, None),
    "c5_cloud": (lambda: scenes.cloud_box(40, 40, grid=64), 3, _connect_only),
    "sky_room": (lambda: scenes.sky_room(48, 48), 2, None),
}
for _kind in scenes.MATERIAL_KINDS:
    for _spectral in (False, True):
        SCENES[f"material_box[{_kind}]" + ("/spectral" if _spectral else "/rgb")] = (
            functools.partial(scenes.material_box, _kind, 48, 48, spectral=_spectral), 2, None)


@functools.lru_cache(maxsize=None)
def _scene(name):
    return SCENES[name][0]()


@pytest.fixture(scope="module")
def api():
    from etx_tracer_b200 import api as m
    return m


def _render(g, thresholds, iterations, options):
    g.debug_thresholds(**thresholds)
    if options is not None:
        g.options[:] = options
    g.render(iterations)
    out = {f"buf{bid}": g.buffer(bid, dt) for bid, dt in EXACT_BUFFERS}
    out["counters"] = {k: v for k, v in g.counters().items() if k != "kernel_launches"}
    out["film_camera"] = g.film(S.FILM_CAMERA)[..., :3]
    out["film_light"] = g.film(S.FILM_LIGHT)[..., :3]
    out["gathered"] = g.buffer(S.BUF_CAMERA_GATHERED, np.float32)
    return out, g.debug_branch_counts()


def _assert_same_render(a, b, label):
    for key in a:
        if key == "counters":
            assert a[key] == b[key], (label, {k: (a[key][k], b[key][k]) for k in a[key] if a[key][k] != b[key][k]})
        elif key in ("film_camera", "film_light", "gathered"):
            assert rel_l2(a[key], b[key]) <= 1e-6, (label, key, rel_l2(a[key], b[key]))
        else:
            assert bit_equal(a[key], b[key]), (label, key)


def _assert_small_branches(counts, merging):
    assert counts["merge_sorts"] == 0 and counts["connect_launches"] == 0 and counts["pair_sorts"] == 0 and counts["queue_sorts"] == 0, counts
    assert all(n == 0 for q, n in counts["merge_qpw"].items() if q != 1), counts
    assert (counts["merge_qpw"][1] > 0) == merging, counts


@gpu
@pytest.mark.parametrize("name", sorted(SCENES))
def test_forced_large_queue_branches_equal_small_ones(api, name):
    sd = _scene(name)
    _, iterations, options = SCENES[name]
    opts = options() if options else None
    merging = options is None
    stochastic = _stochastic(sd)
    g = api.GPUVCM(sd, flavor="fast")
    small, counts = _render(g, FORCED_OFF, iterations, opts)
    _assert_small_branches(counts, merging)
    assert small["counters"]["merge_queries"] > 0 or not merging, small["counters"]
    if merging:
        assert small["counters"]["merge_accepts"] > 0, small["counters"]  # the photon map is queried and found
    for qpw in QPW:
        large, counts = _render(g, dict(FORCED_ON, merge_qpw=qpw), iterations, opts)
        _assert_same_render(large, small, f"qpw {qpw}")
        assert counts["merge_qpw"][qpw] > 0 if merging else counts["merge_qpw"][qpw] == 0, counts
        assert all(n == 0 for q, n in counts["merge_qpw"].items() if q != qpw), counts
        assert (counts["merge_sorts"] > 0) == merging, counts
        # the connection stage, its pair sort and the path-queue sort exist in scenes with stochastic BSDFs
        assert (counts["connect_launches"] > 0) == stochastic, counts
        assert (counts["pair_sorts"] > 0) == stochastic, counts
        assert (counts["queue_sorts"] > 0) == stochastic, counts
    g.close()


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


NATURAL = {
    "c3_room_512x288": lambda: scenes.procedural_room(512, 288, env_size=(256, 128)),
    "c4_dragon_384x384": lambda: scenes.sss_dragon(384, 384),
}


@gpu
@pytest.mark.parametrize("name", sorted(NATURAL))
def test_natural_size_branches_equal_small_ones(api, name):
    """no override: the first bounce of a 147 456-path film fills 32 queries per warp on up to 144 SMs"""
    sd = NATURAL[name]()
    paths = sd.width * sd.height
    sm = _sm_count()
    if paths < 32 * 32 * sm:
        pytest.skip(f"{paths} paths do not fill 32 queries per warp on {sm} SMs")
    g = api.GPUVCM(sd, flavor="fast")
    natural, counts = _render(g, {}, 2, None)
    assert counts["merge_qpw"][32] > 0 and counts["merge_sorts"] > 0, counts
    assert counts["connect_launches"] > 0 and counts["pair_sorts"] > 0 and counts["queue_sorts"] > 0, counts
    small, counts = _render(g, FORCED_OFF, 2, None)
    _assert_small_branches(counts, True)
    _assert_same_render(natural, small, "natural")
    g.close()


@gpu
def test_thresholds_are_checked(api):
    g = api.GPUVCM(scenes.cornell_box(16, 16), flavor="fast")
    with pytest.raises(api.EtxbError):
        g.debug_thresholds(merge_qpw=3)
    with pytest.raises(api.EtxbError):
        g.debug_thresholds(merge_sort_min_queries=0)  # a sorted gather queue needs the exact count, which the tail does not read back
    with pytest.raises(ValueError):
        g.debug_thresholds(no_such_threshold=1)
    g.debug_thresholds()
    g.render(1)
    counts = g.debug_branch_counts()
    assert counts["merge_qpw"][1] > 0 and counts["merge_sorts"] == 0, counts  # 256 paths: one query per warp, no sort
    g.close()
