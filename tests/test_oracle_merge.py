"""oracle_merge (the reference's own VCMSpatialGridData::gather, compiled in place) against the float64 Lambert model of merge_cases, on
every case set in RGB with the three option sets of test_gpu_merge.py: the two references the device gather is held to agree with each
other.  No GPU: the staged positions are computed here (dyadic barycentrics on dyadic vertices are exact in float32)."""
import numpy as np
import pytest

import merge_cases as mc
from etx_tracer_b200 import structs as S

OPTION_SETS = {"epanechnikov": dict(kernel=1, mis=True), "box": dict(kernel=0, mis=True), "no_mis": dict(kernel=1, mis=False)}


@pytest.fixture(scope="module")
def merge_oracle(oracle_mod):
    if not oracle_mod.has_merge():
        pytest.skip("oracle/_ref predates oracle_merge (rebuild it with oracle/build_oracle.sh where the reference sources exist)")
    return oracle_mod


def staged(queries):
    """the floor point of each query, as make_intersection interpolates it (exact for the dyadic sets, within an ulp otherwise)"""
    u, v = queries["u"].astype(np.float32), queries["v"].astype(np.float32)
    w = np.float32(1) - u - v
    a, b, c, d = (np.float32([x, 0, z]) for x, z in ((-4, -4), (4, -4), (4, 4), (-4, 4)))
    t0 = (queries["tri"] == 0)[:, None]
    p = np.where(t0, a * w[:, None] + d * u[:, None] + c * v[:, None], a * w[:, None] + c * u[:, None] + b * v[:, None])
    return p.astype(np.float32), np.tile(np.float32([0, 1, 0]), (len(queries), 1))


@pytest.mark.parametrize("option_set", sorted(OPTION_SETS))
def test_oracle_merge_matches_float64_model(merge_oracle, option_set):
    opts = mc.options(**OPTION_SETS[option_set])
    sd = mc.floor_scene()
    path_count = sd.width * sd.height
    kd = sd.a_spectra[int(sd.a_materials[0]["scattering"]["spectrum_index"])]["integrated"]
    wl = mc.light_wavelengths(path_count)
    o = merge_oracle.Oracle(sd)
    o.set_options(opts)
    o.begin(0)
    duplicates = 0
    for name, (recs, queries) in sorted(mc.cases(path_count).items()):
        ref, grid = o.merge(recs, wl, queries, 1, threads=1)
        assert grid["photon_count"] == len(recs) and grid["hash_table_mask"] == (1 << int(np.ceil(np.log2(len(recs))))) - 1, grid
        assert np.array_equal(grid["bbox_min"], recs["pos"].min(axis=0)) and np.array_equal(grid["bbox_max"], recs["pos"].max(axis=0)), grid
        assert grid["cell_size"] == 2 * mc.RADIUS and grid["radius_squared"] == mc.RADIUS ** 2, grid
        pos, nrm = staged(queries)
        model, counts = mc.lambert_gather(grid, recs, queries, pos, nrm, kd, path_count, opts)
        err = np.abs(ref[:, :3] - model)
        bad = np.flatnonzero((err > 1e-5 * np.abs(model) + 1e-7 * np.abs(model).max()).any(axis=1))
        assert bad.size == 0, (name, bad[:5].tolist(), ref[bad[:3], :3].tolist(), model[bad[:3]].tolist())
        assert np.array_equal(ref[:, :3] == 0.0, model == 0.0), (name, np.flatnonzero((ref[:, :3] == 0.0) != (model == 0.0))[:8].tolist())
        assert (ref[:, 3:6] == 0.0).all()  # one repetition: no variance
        assert counts["accepts"] > 0, name
        duplicates += counts["duplicate_buckets"]
    assert duplicates > 0  # the sparse sets put two neighbour cells in one bucket
    o.close()


def test_oracle_merge_repetitions_restart_the_sampler(merge_oracle):
    """a Lambert gather draws nothing: every repetition returns the same sum and the sampler is untouched (Sampler(seed, 0))"""
    sd = mc.floor_scene()
    path_count = sd.width * sd.height
    recs, queries = mc.case_clusters(3, path_count)
    o = merge_oracle.Oracle(sd)
    o.set_options(mc.options())
    o.begin(0)
    one, _ = o.merge(recs, mc.light_wavelengths(path_count), queries, 1)
    many, _ = o.merge(recs, mc.light_wavelengths(path_count), queries, 8)
    o.close()
    assert np.array_equal(one[:, :3], many[:, :3]) and (many[:, 3:6] == 0.0).all()
    start = merge_oracle.sampler_kat(queries["seed"], np.zeros(len(queries), np.uint32), 0)[0][:, 0]
    assert np.array_equal(one[:, 6].astype(np.uint32), start)
    assert S.MERGE_QUERY.itemsize == 64 and S.LIGHT_VERTEX_REC.itemsize == 96
