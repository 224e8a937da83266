"""The photon gather query by query (etxb_debug_merge): the camera pass's own launch code over a one-bounce queue of staged queries, against
a float64 model of the reference's Lambert gather and against the reference's own VCMSpatialGridData::gather (oracle_merge), in both builds.
The render tests compare gathers only through converged images; these pin the plumbing around the BSDF: cell enumeration and hashing
(including the reference's second sweep of a bucket two neighbour cells hash to), the virtual range over the eight cells, the compaction into
the shared list and its 32-at-a-time finish, which photon and which query a pair belongs to, the inclusive radius and bounding-box tests, the
depth cut, the normal test, the MIS and kernel weights and the spectral luminance scale.

  Lambert, RGB (merge_cases.floor_scene and the Cornell box)    per query within 1e-5 (parity) / 1e-4 (product) of the float64 model, zero
                                                                  exactly where the model is; candidate and accept totals exactly the model's
  Lambert, product build, 1 / 4 / 32 queries per warp, sorted     bit-identical sums and counters
  and unsorted queue
  every material kind + the textured sky room, RGB + spectral    parity: bit-exact against the oracle on the same sampler (R = 1), sampler
                                                                  state afterwards included; product: queries whose values do not depend on the
                                                                  sampler within RTOL_FAST of the oracle, the others as means over 256 samplers
                                                                  within 5.5 sigma (+ 1e-5 relative: some outputs vary only at rounding level)
  delta-only floors (smooth conductor / dielectric, thin film,   parity build only: the camera pass never merges at them, so the product build
  mirror, void)                                                   has no gather for them when the scene has nothing else to merge at
Run with -m gpu."""
import numpy as np
import pytest

import merge_cases as mc
from conftest import bit_equal
from etx_tracer_b200 import scenes, structs as S

pytestmark = pytest.mark.gpu

FLAVORS = ("fast", "parity")
RTOL_MODEL = {"parity": 1e-5, "fast": 1e-4}
RTOL_FAST = 1e-3   # the product build's closures differ from the reference by up to 6e-4 relative per evaluation (test_gpu_closures.py)
K_SIGMA = 5.5
REPS = 256
OPTION_SETS = {"epanechnikov": dict(kernel=1, mis=True), "box": dict(kernel=0, mis=True), "no_mis": dict(kernel=1, mis=False)}


@pytest.fixture(scope="module")
def api():
    from etx_tracer_b200 import api as m
    return m


@pytest.fixture(scope="module")
def merge_oracle(oracle_mod):
    if not oracle_mod.has_merge():
        pytest.skip("oracle/_ref predates oracle_merge (rebuild it with oracle/build_oracle.sh where the reference sources exist)")
    return oracle_mod


def _context(api, sd, flavor, opts):
    g = api.GPUVCM(sd, flavor=flavor)
    g.options[:] = opts
    g.run()
    return g


def _kd(sd, material):
    return sd.a_spectra[int(sd.a_materials[material]["scattering"]["spectrum_index"])]["integrated"].astype(np.float64)


def _check_grid(grid, recs, opts):
    radius = np.float32(opts["initial_radius"][0])
    assert grid["photon_count"] == len(recs)
    assert bit_equal(grid["bbox_min"], recs["pos"].min(axis=0)) and bit_equal(grid["bbox_max"], recs["pos"].max(axis=0)), grid
    assert grid["cell_size"] == np.float32(2) * radius and grid["radius_squared"] == radius * radius, grid
    assert grid["hash_table_mask"] == (1 << int(np.ceil(np.log2(len(recs))))) - 1, grid


def _compare_model(out, grid, recs, queries, kd, sd, opts, flavor, label):
    model, counts = mc.lambert_gather(grid, recs, queries, out["pos"], out["nrm"], kd, sd.width * sd.height, opts, int(sd.scene["max_path_length"][0]))
    dev = out["merged"].astype(np.float64)
    scale = np.abs(model).max()
    err = np.abs(dev - model)
    bad = np.flatnonzero((err > RTOL_MODEL[flavor] * np.abs(model) + 1e-7 * scale).any(axis=1))
    assert bad.size == 0, (label, bad[:5].tolist(), dev[bad[:3]].tolist(), model[bad[:3]].tolist())
    assert np.array_equal(dev == 0.0, model == 0.0), (label, np.flatnonzero((dev == 0.0) != (model == 0.0))[:8].tolist())
    inside = np.all((out["pos"] >= grid["bbox_min"]) & (out["pos"] <= grid["bbox_max"]), axis=1)
    assert grid["merge_queries"] == int(inside.sum()), (label, grid["merge_queries"], int(inside.sum()))
    assert (grid["merge_candidates"], grid["merge_accepts"]) == (counts["candidates"], counts["accepts"]), (label, grid, counts)
    nz = model != 0
    return float((err[nz] / np.abs(model[nz])).max()) if nz.any() else 0.0, counts["duplicate_buckets"]


@pytest.mark.parametrize("flavor", FLAVORS)
@pytest.mark.parametrize("option_set", sorted(OPTION_SETS))
def test_lambert_gather_matches_float64_model(api, flavor, option_set):
    opts = mc.options(**OPTION_SETS[option_set])
    sd = mc.floor_scene()
    path_count = sd.width * sd.height
    g = _context(api, sd, flavor, opts)
    wl = mc.light_wavelengths(path_count)
    report = []
    for name, (recs, queries) in sorted(mc.cases(path_count).items()):
        out, grid = g.debug_merge(recs, wl, queries)
        _check_grid(grid, recs, opts)
        if name == "boundary":
            # dyadic barycentrics on dyadic vertices: the staged positions are exact
            tri, u, v = queries["tri"], queries["u"].astype(np.float64), queries["v"].astype(np.float64)
            x = np.where(tri == 0, -4 + 8 * v, -4 + 8 * (u + v))
            z = np.where(tri == 0, -4 + 8 * (u + v), -4 + 8 * u)
            assert bit_equal(out["pos"], np.stack([x, np.zeros_like(x), z], axis=1).astype(np.float32)), out["pos"]
            assert bit_equal(out["nrm"], np.tile(np.float32([0, 1, 0]), (len(queries), 1)))
        rel, dup = _compare_model(out, grid, recs, queries, _kd(sd, 0), sd, opts, flavor, name)
        report.append(f"{name}: {len(queries)} queries, max rel {rel:.2e}, {dup} duplicate buckets, {grid['merge_accepts']} accepts")
    print(f"\n[merge model] {flavor}/{option_set}: " + "; ".join(report))
    g.close()


def _realistic(api, sd, queries_n, seed, radius=None):
    """photons of one light pass of `sd` (parity build) and queries at camera-ray hits: (records, light wavelengths, queries, opts)"""
    g = api.GPUVCM(sd, flavor="parity")
    g.render(1)
    recs = g.buffer(S.BUF_PHOTON_RECORDS, np.uint8).view(S.LIGHT_VERTEX_REC)
    wl = g.buffer(S.BUF_LIGHT_PATH_WAVELENGTH, np.float32)
    rng = np.random.default_rng(seed)
    cam = sd.camera
    origin = np.asarray(cam["position"][0], np.float64)
    fwd = np.asarray(cam["direction"][0], np.float64)
    d = mc._unit(fwd + rng.uniform(-0.45, 0.45, (4 * queries_n, 3)))
    rays = np.zeros((len(d), 8), np.float32)
    rays[:, :3], rays[:, 3], rays[:, 4:7], rays[:, 7] = origin, 0.0, d, 1e30
    uvt, tri, _ = g.debug_trace(rays, np.arange(len(d), dtype=np.uint32))
    g.close()
    hit = np.flatnonzero(tri != S.INVALID)[:queries_n]
    q = np.zeros(len(hit), dtype=S.MERGE_QUERY)
    q["tri"], q["u"], q["v"], q["w_i"] = tri[hit], uvt[hit, 0], uvt[hit, 1], d[hit]
    q["throughput"] = rng.uniform(0.2, 1.5, (len(hit), 3))
    if sd.scene["flags"][0] & S.SCENE_SPECTRAL:
        q["throughput"][:, 1:] = q["throughput"][:, :1]
    q["wavelength"] = rng.uniform(390.0, 830.0, len(hit))
    q["d_vcm"], q["d_vm"] = rng.uniform(0.0, 4.0, len(hit)), rng.uniform(0.0, 4.0, len(hit))
    q["total_path_depth"] = rng.integers(1, 4, len(hit))
    q["seed"] = rng.integers(0, 2**32, len(hit), dtype=np.uint64).astype(np.uint32)
    q["medium"] = S.INVALID
    opts = S.default_vcm_options()
    if radius is not None:
        opts["initial_radius"] = radius
    return recs, wl, q, opts


@pytest.mark.parametrize("flavor", FLAVORS)
def test_lambert_gather_on_a_light_pass_matches_float64_model(api, flavor):
    """the realistic tier: photons of a Cornell-box light pass, queries where camera rays hit, a dyadic radius"""
    sd = scenes.cornell_box(64, 64, samples=16)
    recs, wl, q, opts = _realistic(api, sd, 512, 23, radius=2.0 ** -4)
    g = _context(api, sd, flavor, opts)
    out, grid = g.debug_merge(recs, wl, q)
    g.close()
    _check_grid(grid, recs, opts)
    tri_material = sd.a_triangles["material_index"][q["tri"]]
    kd = np.stack([_kd(sd, m) for m in tri_material])
    rel, dup = _compare_model(out, grid, recs, q, kd, sd, opts, flavor, "cornell")
    assert grid["merge_accepts"] > 1000, grid
    print(f"\n[merge model] {flavor}/cornell light pass: {len(recs)} photons, {len(q)} queries, max rel {rel:.2e}, {dup} duplicate buckets")


def test_lambert_sums_do_not_depend_on_the_queue_order(api):
    """product build: 1, 4 or 32 queries per warp, queue sorted by merge key or not — the lane assignment of the Lambert gather depends only on
    the query's own cells, so every per-query sum and counter is bit-identical"""
    opts = mc.options()
    sd = mc.floor_scene()
    path_count = sd.width * sd.height
    g = _context(api, sd, "fast", opts)
    wl = mc.light_wavelengths(path_count)
    recs, queries = mc.case_random(29, path_count, queries=path_count)
    first = None
    for qpw in (1, 4, 32):
        for sort in (False, True):
            g.debug_thresholds(merge_qpw=qpw, merge_sort_min_queries=0 if sort else S.NEVER, tail_queue=0 if sort else S.NEVER)
            g.run()
            out, grid = g.debug_merge(recs, wl, queries)
            counts = g.debug_branch_counts()
            assert counts["merge_qpw"][qpw] == 1 and (counts["merge_sorts"] == 1) == sort, counts
            got = (out["merged"], [grid[k] for k in ("merge_queries", "merge_candidates", "merge_accepts")])
            if first is None:
                first = got
                assert grid["merge_accepts"] > 10000, grid
            else:
                assert bit_equal(got[0], first[0]) and got[1] == first[1], (qpw, sort, got[1], first[1])
    g.close()


# ---- every material kind against the reference's own gather -------------------------------------------------------------------------------
KINDS = [("floor", k) for k in sorted(scenes.MATERIAL_KINDS)] + [("sky_room", "textured")]


def _material_case(kind, spectral, queries_n):
    sd = mc.floor_scene(spectral=spectral, material=scenes.MATERIAL_KINDS[kind])
    recs, queries = mc.case_random(31, sd.width * sd.height, spectral=spectral, queries=queries_n)
    return sd, recs, mc.light_wavelengths(sd.width * sd.height), queries, mc.options()


def _always_delta(m):
    """module.cu validate_scene: a material no vertex of the camera pass merges at (smooth conductor or dielectric, thin film, mirror, void)"""
    smooth = max(float(m["roughness"]["value"][0]), float(m["roughness"]["value"][1])) <= 1e-4 and int(m["roughness"]["image_index"]) == S.INVALID
    return (int(m["cls"]) in (S.MAT_DIELECTRIC, S.MAT_CONDUCTOR) and smooth) or int(m["cls"]) in (S.MAT_THINFILM, S.MAT_MIRROR, S.MAT_VOID)


def _sampler_states(oracle_mod, seeds, reps):
    """Sampler(seed, r).seed for every query and r: the state the oracle's repetition r starts from, row-major (query, r)"""
    a = np.repeat(np.asarray(seeds, np.uint32), reps)
    b = np.tile(np.arange(reps, dtype=np.uint32), len(seeds))
    return oracle_mod.sampler_kat(a, b, 0)[0][:, 0]


@pytest.mark.parametrize("spectral", [False, True], ids=["rgb", "spectral"])
@pytest.mark.parametrize("where,kind", KINDS, ids=[f"{w}-{k}" for w, k in KINDS])
def test_parity_gather_is_bit_exact_against_the_reference(api, merge_oracle, where, kind, spectral):
    if where == "sky_room":
        sd = scenes.sky_room(48, 48, spectral=spectral)
        recs, wl, queries, opts = _realistic(api, sd, 512, 37)
    else:
        sd, recs, wl, queries, opts = _material_case(kind, spectral, 256)
    o = merge_oracle.Oracle(sd)
    o.set_options(opts)
    o.begin(0)
    ref, ref_grid = o.merge(recs, wl, queries, 1)
    o.close()
    dev_q = queries.copy()
    dev_q["seed"] = _sampler_states(merge_oracle, queries["seed"], 1)
    g = _context(api, sd, "parity", opts)
    out, grid = g.debug_merge(recs, wl, dev_q)
    g.close()
    for k in ("bbox_min", "bbox_max"):
        assert bit_equal(grid[k], ref_grid[k]), (k, grid[k], ref_grid[k])
    assert (grid["cell_size"], grid["radius_squared"], grid["hash_table_mask"]) == (ref_grid["cell_size"], ref_grid["radius_squared"], ref_grid["hash_table_mask"])
    same = (out["merged"].view(np.uint32) == ref[:, :3].astype(np.float32).view(np.uint32)).all(axis=1)
    assert same.all(), (kind, f"{int((~same).sum())} of {len(same)} queries differ", out["merged"][~same][:3].tolist(), ref[~same, :3][:3].tolist())
    assert np.array_equal(out["seed"], ref[:, 6].astype(np.uint32)), kind
    assert grid["merge_candidates"] > 0, grid
    if kind not in ("mirror", "thinfilm", "void"):  # their evaluate() is invalid everywhere (delta lobes only): nothing is gathered, on both sides
        assert grid["merge_accepts"] > 0 and (ref[:, :3] != 0).any(), grid


@pytest.mark.parametrize("spectral", [False, True], ids=["rgb", "spectral"])
@pytest.mark.parametrize("where,kind", KINDS, ids=[f"{w}-{k}" for w, k in KINDS])
def test_product_gather_matches_the_reference(api, merge_oracle, where, kind, spectral):
    if where == "sky_room":
        sd = scenes.sky_room(64, 64, spectral=spectral)
        recs, wl, queries, opts = _realistic(api, sd, 16, 41)
    else:
        sd, recs, wl, queries, opts = _material_case(kind, spectral, 16)
        if _always_delta(sd.a_materials[0]):
            pytest.skip("a delta material: the camera pass never merges at it (the parity build's serial gather is still compared)")
    n = len(queries)
    assert n * REPS <= sd.width * sd.height
    o = merge_oracle.Oracle(sd)
    o.set_options(opts)
    o.begin(0)
    ref, _ = o.merge(recs, wl, queries, REPS)
    o.close()
    dev_q = np.repeat(queries, REPS)
    dev_q["seed"] = _sampler_states(merge_oracle, queries["seed"], REPS)
    g = _context(api, sd, "fast", opts)
    out, grid = g.debug_merge(recs, wl, dev_q)
    g.close()
    v = out["merged"].astype(np.float64).reshape(n, REPS, 3)
    mg, vg = v.mean(axis=1), v.var(axis=1)
    mr, vr = ref[:, :3], ref[:, 3:6]
    det = (vg == 0) & (vr == 0)
    err = np.abs(mg - mr)
    scale = np.abs(mr).max()
    bad_det = np.flatnonzero((det & (err > RTOL_FAST * np.abs(mr) + 1e-6 * scale)).any(axis=1))
    sigma = np.sqrt(vg / REPS + vr / REPS)
    bad_rnd = np.flatnonzero((~det & (err > K_SIGMA * sigma + 1e-5 * np.abs(mr) + 1e-7 * scale)).any(axis=1))
    rel = float((err[det & (mr != 0)] / np.abs(mr[det & (mr != 0)])).max()) if (det & (mr != 0)).any() else 0.0
    z = float((err[~det] / np.maximum(sigma[~det], 1e-30)).max()) if (~det).any() else 0.0
    rnd_nz = ~det & (mr != 0)
    rel_rnd = float((err[rnd_nz] / np.abs(mr[rnd_nz])).max()) if rnd_nz.any() else 0.0
    print(f"\n[merge oracle] {where}-{kind}/{'spectral' if spectral else 'rgb'}/fast: {n} queries x {REPS}, sampler-independent outputs {int(det.sum())} "
          f"(max rel {rel:.2e}), random {int((~det).sum())} (max z {z:.2f}, max rel {rel_rnd:.2e})")
    assert bad_det.size == 0, (kind, bad_det[:4].tolist(), mg[bad_det[:3]].tolist(), mr[bad_det[:3]].tolist())
    assert bad_rnd.size == 0, (kind, bad_rnd[:4].tolist(), mg[bad_rnd[:3]].tolist(), mr[bad_rnd[:3]].tolist(), sigma[bad_rnd[:3]].tolist())
