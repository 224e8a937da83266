"""Seeded photon sets and merge queries for the gather tests (etxb_debug_merge against a float64 model and the oracle's own gather), and the
float64 model of the reference's Lambert gather (VCMSpatialGridData::gather, vcm_shared.hxx:805-925).

The scene is a flat floor: two triangles spanning x, z in [-4, 4] at y = 0 (normal +y), dyadic vertices, plus a small area light.  A
query is a hit on the floor given by dyadic barycentrics, so its position is exact in any rounding mode; with a dyadic merge radius
(`initial_radius`, iteration 0: the radius scale is exactly 1) the cell size is a power of two and every distance, cell coordinate and
bounding-box test of the boundary cases below is exact on both sides.

Case sets (each returns records and queries; light_wavelengths() gives the wavelength per light path):
  clusters    photons packed into a few tight clusters: one cell holds hundreds of photons, the gather's shared list refills many times
  sparse      1, 2, 3 and 5 photons: a hash table of 1-8 buckets, where two of a query's eight cells often hash to the same bucket (the
              reference then sweeps that bucket twice, and so must the device)
  boundary    photons at exactly distance r (the test is inclusive) and 2^-20 beyond, one whose float32 distance rounds to r (inside
              for the reference too: the model tests distances in float32 as both sides do), photons on cell faces, queries at md = 0.5
              of a cell, on the faces of the photon bounding box (inclusive) and just outside it, photon path lengths at the depth cut
              exactly and one past it, back-facing photon normals, photon directions from below the surface
  random      uniform photons over and above the floor with random directions and normals; the realistic tier of the test draws its
              photons from a light pass instead
"""
import numpy as np

from etx_tracer_b200 import scenes, structs as S

FLOOR = 4.0           # the floor spans [-FLOOR, FLOOR] in x and z
RADIUS = 0.25         # dyadic merge radius: cell size 0.5, radius squared 1/16
MAX_PATH_LENGTH = 12  # small, so that the depth cut is reachable with short photon paths
KD = (0.5, 0.25, 0.75)


def floor_scene(width=64, height=64, spectral=False, material=None):
    """The dyadic floor; `material` = add_material kwargs of the floor (default: Lambert KD)."""
    sd = scenes.SceneData()
    sd.name = "merge_floor" + ("/spectral" if spectral else "/rgb")
    floor = sd.add_material("floor", **(material if material is not None else dict(kd=list(KD), two_sided=1)))
    light = sd.add_material("light", kd=[0.0, 0.0, 0.0], emission=scenes.spd_rgb_luminance([4.0, 4.0, 4.0]), two_sided=1)
    a, b, c, d = (-FLOOR, 0.0, -FLOOR), (FLOOR, 0.0, -FLOOR), (FLOOR, 0.0, FLOOR), (-FLOOR, 0.0, FLOOR)
    sd.add_mesh([a, d, c, a, c, b], [(0.0, 1.0, 0.0)] * 6, [[0, 1, 2], [3, 4, 5]], floor)  # triangle 0 = (a, d, c), triangle 1 = (a, c, b)
    sd.add_quad([-0.5, 3.0, -0.5], [0.5, 3.0, -0.5], [0.5, 3.0, 0.5], [-0.5, 3.0, 0.5], light)
    sd.set_camera([0.0, 3.0, 6.0], [0.0, 0.0, 0.0], [0.0, 1.0, 0.0], width, height, 50.0, clip_near=0.1, clip_far=100.0)
    return sd.finalize(samples=16, spectral=spectral, max_path_length=MAX_PATH_LENGTH)


def options(kernel=1, mis=True):
    o = S.default_vcm_options()
    o["initial_radius"] = RADIUS
    o["kernel"] = kernel
    if not mis:
        o["options"] = int(o["options"][0]) & ~S.VCM_ENABLE_MIS
    return o


def floor_hit(x, z):
    """(triangle, u, v) of the floor point (x, 0, z): triangle 0 = (a, d, c) covers z >= x, triangle 1 = (a, c, b) covers x >= z."""
    x, z = np.asarray(x, np.float64), np.asarray(z, np.float64)
    t0 = z >= x
    v0, u0 = (x + FLOOR) / (2 * FLOOR), (z - x) / (2 * FLOOR)
    u1, v1 = (z + FLOOR) / (2 * FLOOR), (x - z) / (2 * FLOOR)
    return np.where(t0, 0, 1).astype(np.uint32), np.where(t0, u0, u1), np.where(t0, v0, v1)


def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def make_records(pos, nrm=None, w_i=None, path_length=None, rng=None, path_count=4096, spectral=False):
    """Light-vertex records at `pos` (n, 3): normals +y, arriving from above, short paths unless given; seeded throughput and MIS terms."""
    rng = rng or np.random.default_rng(1)
    n = len(pos)
    r = np.zeros(n, dtype=S.LIGHT_VERTEX_REC)
    r["pos"] = pos
    r["nrm"] = (0.0, 1.0, 0.0) if nrm is None else nrm
    r["w_i"] = _unit(np.stack([rng.uniform(-0.6, 0.6, n), -np.ones(n), rng.uniform(-0.6, 0.6, n)], axis=1)) if w_i is None else w_i
    r["path_length"] = rng.integers(1, 4, n) if path_length is None else path_length
    r["throughput"] = rng.uniform(0.2, 2.0, (n, 3))
    if spectral:
        r["throughput"][:, 1:] = r["throughput"][:, :1]
    r["d_vcm"] = rng.uniform(0.0, 4.0, n)
    r["d_vc"] = rng.uniform(0.0, 4.0, n)
    r["d_vm"] = rng.uniform(0.0, 4.0, n)
    r["bc"] = (1.0, 0.0, 0.0)
    r["tri"] = 0
    r["material"] = 0
    r["medium"] = S.INVALID
    r["path_index"] = rng.integers(0, path_count, n)
    r["ordinal"] = np.arange(n)
    return r


def make_queries(x, z, rng, w_i=None, depth=None, spectral=False):
    tri, u, v = floor_hit(x, z)
    n = len(tri)
    q = np.zeros(n, dtype=S.MERGE_QUERY)
    q["tri"], q["u"], q["v"] = tri, u, v
    q["w_i"] = _unit(np.stack([rng.uniform(-0.7, 0.7, n), -np.ones(n), rng.uniform(-0.7, 0.7, n)], axis=1)) if w_i is None else w_i
    q["throughput"] = rng.uniform(0.2, 1.5, (n, 3))
    if spectral:
        q["throughput"][:, 1:] = q["throughput"][:, :1]
    q["wavelength"] = rng.uniform(390.0, 830.0, n)
    q["d_vcm"] = rng.uniform(0.0, 4.0, n)
    q["d_vm"] = rng.uniform(0.0, 4.0, n)
    q["total_path_depth"] = rng.integers(1, 4, n) if depth is None else depth
    q["seed"] = rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32)
    q["medium"] = S.INVALID
    return q


def _dyadic(rng, lo, hi, n, step=1.0 / 64.0):
    return np.round(rng.uniform(lo, hi, n) / step) * step


def case_clusters(seed, path_count=4096, spectral=False):
    rng = np.random.default_rng(seed)
    centers = np.stack([rng.uniform(-3, 3, 6), np.zeros(6), rng.uniform(-3, 3, 6)], axis=1)
    pos = np.concatenate([c + rng.normal(scale=0.06, size=(220, 3)) * (1, 0.2, 1) for c in centers])
    recs = make_records(pos, rng=rng, path_count=path_count, spectral=spectral)
    qc = centers[rng.integers(0, 6, 96)] + np.stack([_dyadic(rng, -0.25, 0.25, 96), np.zeros(96), _dyadic(rng, -0.25, 0.25, 96)], axis=1)
    return recs, make_queries(qc[:, 0], qc[:, 2], rng, spectral=spectral)


def case_sparse(seed, count, path_count=4096, spectral=False):
    """`count` photons near the origin; the queries sit among them and in cells around them"""
    rng = np.random.default_rng(seed)
    pos = np.stack([_dyadic(rng, -0.5, 0.5, count), np.zeros(count), _dyadic(rng, -0.5, 0.5, count)], axis=1)
    recs = make_records(pos, rng=rng, path_count=path_count, spectral=spectral)
    m = 48
    # on the photons (with one photon its point is the whole bounding box), near them, anywhere (mostly outside the small box)
    near = pos[rng.integers(0, count, m // 2)]
    x = np.concatenate([pos[:, 0], near[:, 0] + _dyadic(rng, -0.2, 0.2, m // 2), _dyadic(rng, -0.75, 0.75, m // 2)])
    z = np.concatenate([pos[:, 2], near[:, 2] + _dyadic(rng, -0.2, 0.2, m // 2), _dyadic(rng, -0.75, 0.75, m // 2)])
    return recs, make_queries(x, z, rng, spectral=spectral)


def case_boundary(seed, path_count=4096, spectral=False):
    """Every boundary of the module docstring; dyadic positions around two anchor photons that fix the bounding box."""
    rng = np.random.default_rng(seed)
    r = RADIUS
    ulp = 2.0 ** -20
    qx, qz = np.array([0.5, 0.75, -1.25, 1.0]), np.array([0.5, -1.0, 0.25, 1.5])  # on-grid query centres (md = 0 or 0.5 once bbox_min = -2)
    pos, nrm, w_i, plen = [], [], [], []

    def add(p, n=(0.0, 1.0, 0.0), w=(0.0, -1.0, 0.0), length=1):
        pos.append(p), nrm.append(n), w_i.append(w), plen.append(length)

    add((-2.0, -0.5, -2.0))  # anchor: bbox_min = (-2, -0.5, -2) -> every cell face is at a multiple of 0.5
    add((2.0, 0.5, 2.0))     # bbox_max = (2, 0.5, 2)
    for x, z in zip(qx, qz):
        for d in ((r, 0, 0), (-r, 0, 0), (0, 0, r), (0, 0, -r), (0, r, 0), (0, -r, 0)):
            add((x + d[0], d[1], z + d[2]))                                      # distance exactly r: accepted
        add((x + r + ulp, 0.0, z))                                                # 2^-20 beyond: rejected
        add((x - r + ulp, 0.0, z))                                                # 2^-20 inside (and at a float32 distance of exactly r from the query at (0.25, 0.25))
        add((x + 0.125, 0.0, z), length=MAX_PATH_LENGTH - 2)                      # with depth 1: path_length + depth + 1 = max: accepted
        add((x - 0.125, 0.0, z), length=MAX_PATH_LENGTH - 1)                      # one past the cut: rejected
        add((x, 0.0, z + 0.125), n=(0.0, -1.0, 0.0))                              # back-facing photon normal: rejected
        add((x, 0.0, z - 0.125), w=(0.0, 1.0, 0.0))                               # arriving from below the floor: Lambert rejects it
        add((x, 0.0, z + 0.0625), n=(0.0, 2.0 ** -24, 1.0))                       # normal at the kEpsilon edge of the normal test
    for k in range(-3, 4):                                                        # photons on cell faces (x or z a multiple of 0.5)
        add((0.5 * k, 0.0, 0.5 * k + 0.125))
        add((0.5 * k + 0.125, 0.0, 0.5 * k))
    pos = np.array(pos, np.float64)
    recs = make_records(pos, nrm=np.array(nrm), w_i=np.array(w_i), path_length=np.array(plen), rng=rng, path_count=path_count, spectral=spectral)
    # queries: the centres (md = 0), cell centres (md = 0.5 on every axis), the bbox faces and corners (inclusive) and just outside them
    cx = list(qx) + [0.25, -0.75, 1.25, 2.0, -2.0, 2.0, -2.0, 0.0, 2.0 + 2.0 ** -10, -2.0 - 2.0 ** -10, 0.0]
    cz = list(qz) + [0.25, -1.75, 0.75, 0.0, 0.0, 2.0, -2.0, 2.0, 0.0, 0.0, -2.0 - 2.0 ** -10]
    depth = np.ones(len(cx), np.uint32)
    return recs, make_queries(np.array(cx), np.array(cz), rng, w_i=np.tile([0.0, -1.0, 0.0], (len(cx), 1)), depth=depth, spectral=spectral)


def case_random(seed, path_count=4096, spectral=False, photons=3000, queries=256):
    rng = np.random.default_rng(seed)
    pos = np.stack([rng.uniform(-3.5, 3.5, photons), rng.uniform(-0.3, 0.3, photons), rng.uniform(-3.5, 3.5, photons)], axis=1)
    nrm = _unit(rng.normal(size=(photons, 3)) + (0.0, 2.0, 0.0))
    w = _unit(rng.normal(size=(photons, 3)) + (0.0, -1.5, 0.0))
    recs = make_records(pos, nrm=nrm, w_i=w, rng=rng, path_count=path_count, spectral=spectral)
    return recs, make_queries(rng.uniform(-3.5, 3.5, queries).astype(np.float32), rng.uniform(-3.5, 3.5, queries).astype(np.float32), rng, spectral=spectral)


def cases(path_count=4096, spectral=False):
    """name -> (records, queries) of every set above"""
    out = {"clusters": case_clusters(11, path_count, spectral), "boundary": case_boundary(13, path_count, spectral),
           "random": case_random(17, path_count, spectral)}
    for n in (1, 2, 3, 5):
        out[f"sparse{n}"] = case_sparse(100 + n, n, path_count, spectral)
    return out


def light_wavelengths(path_count, seed=5):
    return np.random.default_rng(seed).uniform(390.0, 830.0, path_count).astype(np.float32)


# ---- float64 model of the reference's Lambert gather ------------------------------------------------------------------------------------
K_EPSILON = 1.192092896e-07
HASH = (73856093, 19349663, 83492791)


def cell_index(mask, x, y, z):
    """VCMSpatialGridData::cell_index: int32 coordinates times unsigned constants, wrapped to 32 bits"""
    h = ((np.asarray(x, np.int64) * HASH[0]) ^ (np.asarray(y, np.int64) * HASH[1]) ^ (np.asarray(z, np.int64) * HASH[2])) & 0xFFFFFFFF
    return (h & mask).astype(np.int64)


def cells_of(pos, bbox_min, cell_size):
    """floor((pos - bbox_min) / cell_size) in float32, as both sides compute it"""
    m = (np.asarray(pos, np.float32) - np.asarray(bbox_min, np.float32)) / np.float32(cell_size)
    return np.floor(m).astype(np.int64), m - np.floor(m)


def lambert_gather(grid, recs, queries, staged_pos, staged_nrm, kd, path_count, opts, max_path_length=MAX_PATH_LENGTH):
    """Per query float64 merged rgb plus the candidate / accept / duplicate-bucket counts, on the grid parameters the hook reports (an RGB
    scene whose queries all sit on untextured Lambert surfaces of reflectance `kd`, one row per query or one for all).  The eight neighbour cells are enumerated as the reference does, so a bucket two
    of them hash to is swept twice."""
    mask, cs, r2 = int(grid["hash_table_mask"]), float(grid["cell_size"]), float(grid["radius_squared"])
    bmin, bmax = np.asarray(grid["bbox_min"], np.float64), np.asarray(grid["bbox_max"], np.float64)
    pc, _ = cells_of(recs["pos"], bmin, cs)
    bucket = cell_index(mask, pc[:, 0], pc[:, 1], pc[:, 2])
    members = [np.flatnonzero(bucket == b) for b in range(mask + 1)]
    radius = float(opts["initial_radius"][0])
    vc_weight = 1.0 / (np.pi * radius * radius * path_count)
    use_mis = bool(int(opts["options"][0]) & S.VCM_ENABLE_MIS)
    epan = int(opts["kernel"][0]) == 1
    kd = np.broadcast_to(np.asarray(kd, np.float64), (len(queries), 3))
    out = np.zeros((len(queries), 3))
    candidates = accepts = duplicates = 0
    for i, q in enumerate(queries):
        p32 = np.asarray(staged_pos[i], np.float32)
        p = p32.astype(np.float64)
        if not (np.all(p >= bmin) and np.all(p <= bmax)):
            continue
        a, md = cells_of(p[None], bmin, cs)
        a, md = a[0], md[0]
        b = a + np.where(md < 0.5, -1, 1)
        idx = [int(cell_index(mask, b[0] if c & 1 else a[0], b[1] if c & 2 else a[1], b[2] if c & 4 else a[2])) for c in range(8)]
        duplicates += 8 - len(set(idx))
        nrm = np.asarray(staged_nrm[i], np.float64)
        w_i = np.asarray(q["w_i"], np.float64)
        fn = nrm if np.dot(nrm, w_i) < 0.0 else -nrm
        rev_cos = np.dot(nrm, -w_i)
        c_value = kd[i] / np.pi * np.asarray(q["throughput"], np.float64)
        w_camera_base = float(q["d_vcm"]) * vc_weight
        total = np.zeros(3)
        for cell in idx:
            for j in members[cell]:
                candidates += 1
                # the distance test is the reference's float32 one: a photon whose float32 distance rounds to r is inside
                d = recs["pos"][j] - p32
                d2 = float((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
                if d2 > r2 or int(recs["path_length"][j]) + int(q["total_path_depth"]) + 1 > max_path_length:
                    continue
                if np.dot(nrm, recs["nrm"][j].astype(np.float64)) <= K_EPSILON:
                    continue
                w_in = recs["w_i"][j].astype(np.float64)
                cos_o = -np.dot(fn, w_in)
                if cos_o <= K_EPSILON:
                    continue
                accepts += 1
                pdf = cos_o / np.pi
                facing = rev_cos if np.dot(nrm, w_in) < 0.0 else -rev_cos
                rev_pdf = 0.0 if facing <= K_EPSILON else facing / np.pi
                w_light = float(recs["d_vcm"][j]) * vc_weight + float(recs["d_vm"][j]) * pdf
                w_camera = w_camera_base + float(q["d_vm"]) * rev_pdf
                weight = 1.0 / (1.0 + w_light + w_camera) if use_mis else 1.0
                kernel = max(2.0 * (1.0 - d2 / r2), 0.0) if epan else 1.0
                total += recs["throughput"][j].astype(np.float64) * (kernel * weight)
        out[i] = c_value * total
    return out, dict(candidates=candidates, accepts=accepts, duplicate_buckets=duplicates)
