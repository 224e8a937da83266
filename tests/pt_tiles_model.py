"""Numpy model of the path tracer's noise estimate over pixel tiles (kernels_pt.cuh: k_film_noise_level, k_film_noise_dilate; module.cu:
pt_estimate_noise_levels) and of the reference's one-frame estimate it must reproduce (film.cxx:233-330).

Every array is in film storage order (row r is film row H - 1 - r, like ETXB_BUF_PIXEL_INFO).  `info` holds the per-pixel history words: sample
count (bits 0-29), converged (bit 30), tmp (bit 31).
"""
import numpy as np

CONVERGED, TMP = np.uint32(1 << 30), np.uint32(1 << 31)
COUNT_MASK = np.uint32((1 << 30) - 1)
EPSILON = np.float32(1.192092896e-07)  # kEpsilon (dcore.cuh)


def tile_rank(width, x, y, world):
    """etxb_set_partition's rule: the 32x32 tile of film pixel (x, y), numbered row by row, belongs to rank tile % world."""
    tiles_x = (width + 31) // 32
    return ((np.asarray(y) // 32) * tiles_x + np.asarray(x) // 32) % world


def owner_map(width, height, world):
    """(H, W) rank of every storage pixel"""
    r, x = np.mgrid[0:height, 0:width]
    return tile_rank(width, x, height - 1 - r, world)


def words_per_row(width):
    return (width + 31) // 32


def error_levels(camera, adaptive):
    """the first pass's error level, in float32 steps as the kernel rounds them (camera / adaptive: (H, W, 4) float32)"""
    c, a = camera.astype(np.float32), adaptive.astype(np.float32)
    diff = np.abs(c[..., 0] - a[..., 0]) + np.abs(c[..., 1] - a[..., 1]) + np.abs(c[..., 2] - a[..., 2])
    norm = np.abs(c[..., 0]) + np.abs(c[..., 1]) + np.abs(c[..., 2])
    den = np.where(norm < np.float32(1.0), np.sqrt(norm), norm).astype(np.float32) + EPSILON
    return (diff / den).astype(np.float32)


def level_pass(camera, adaptive, info, threshold, owned):
    """k_film_noise_level on the owned pixels: (info, error, active, converged count, error sum).  `active` = not converged after the pass."""
    info = info.copy()
    err = np.zeros(info.shape, np.float32)
    ev = owned & ((info & CONVERGED) == 0)
    lv = error_levels(camera, adaptive)
    conv = lv < np.float32(threshold)
    err[ev] = lv[ev]
    info[ev] = (info[ev] & COUNT_MASK) | np.where(conv[ev], CONVERGED | TMP, np.uint32(0)).astype(np.uint32)
    active = ev & ~conv
    return info, err, active, int((ev & conv).sum()), float(lv[ev].astype(np.float64).sum())


def pack_mask(active):
    """the active mask: storage row r holds ceil(W / 32) words, bit x % 32 of word x // 32"""
    h, w = active.shape
    wpr = words_per_row(w)
    padded = np.zeros((h, wpr * 32), bool)
    padded[:, :w] = active
    weights = (np.uint64(1) << np.arange(32, dtype=np.uint64))
    return (padded.reshape(h, wpr, 32).astype(np.uint64) * weights).sum(-1).astype(np.uint32)


def row_windows(mask):
    """noise_row_window for every word: bit x set where a pixel x - 4 .. x + 5 of the row is active (funnel shifts over the neighbouring words)"""
    cur = mask.astype(np.uint64)
    prev = np.zeros_like(cur)
    nxt = np.zeros_like(cur)
    prev[:, 1:] = cur[:, :-1]
    nxt[:, :-1] = cur[:, 1:]
    m32 = np.uint64(0xFFFFFFFF)
    d = cur.copy()
    for s in range(1, 6):
        d |= ((cur | (nxt << np.uint64(32))) >> np.uint64(s)) & m32
    for s in range(1, 5):
        d |= (((cur << np.uint64(32)) | prev) << np.uint64(s)) >> np.uint64(32) & m32
    return d.astype(np.uint32)


def dilate(mask, info, owned):
    """k_film_noise_dilate: clears tmp where the row window holds an active pixel, converged where the row window of any row y - 4 .. y + 5 does"""
    h, w = info.shape
    rows = row_windows(mask)
    box = np.zeros_like(rows)
    for r in range(h):
        box[r] = np.bitwise_or.reduce(rows[max(0, r - 4):min(h - 1, r + 5) + 1], axis=0)
    x = np.arange(w)
    row_bit = ((rows[:, x // 32] >> (x % 32).astype(np.uint32)) & 1).astype(bool)
    box_bit = ((box[:, x // 32] >> (x % 32).astype(np.uint32)) & 1).astype(bool)
    out = info.copy()
    out[owned & row_bit] &= ~TMP
    out[owned & box_bit] &= ~CONVERGED
    return out


def tiled_estimate(camera, adaptive, info, threshold, world, absent=()):
    """The estimate of `world` ranks, each on its own view (zeros outside its tiles), masks summed as the all-reduce sums them; the ranks in
    `absent` contribute no words (a context with a partition and no communicator sees only its own).  Returns the composed (info, error,
    converged count, error sum)."""
    h, w = info.shape
    own = owner_map(w, h, world)
    views, total = [], np.zeros((h, words_per_row(w)), np.uint32)
    conv_count, err_sum = 0, 0.0
    for r in range(world):
        mine = own == r
        cam = np.where(mine[..., None], camera, 0).astype(np.float32)
        ada = np.where(mine[..., None], adaptive, 0).astype(np.float32)
        inf = np.where(mine, info, 0).astype(np.uint32)
        inf, err, active, n, e = level_pass(cam, ada, inf, threshold, mine)
        views.append((mine, inf, err))
        if r not in absent:
            total += pack_mask(active)
            conv_count += n
            err_sum += e
    out_info, out_err = np.zeros_like(info), np.zeros(info.shape, np.float32)
    for mine, inf, err in views:
        d = dilate(total, inf, mine)
        out_info[mine], out_err[mine] = d[mine], err[mine]
    return out_info, out_err, conv_count, err_sum


def reference_estimate(camera, adaptive, info, threshold):
    """Film::estimate_noise_levels on the whole film in its scatter form (film.cxx:233-330): the first pass, then every active pixel clears tmp
    of x - 5 .. x + 4 of its row, then every pixel without tmp clears converged of y - 5 .. y + 4 of its column."""
    h, w = info.shape
    info, err, active, n, e = level_pass(camera, adaptive, info, threshold, np.ones(info.shape, bool))
    tmp = (info & TMP) != 0
    for y, x in zip(*np.nonzero(active)):
        tmp[y, max(0, x - 5):min(w, x + 5)] = False
    conv = (info & CONVERGED) != 0
    for y, x in zip(*np.nonzero(~tmp)):
        conv[max(0, y - 5):min(h, y + 5), x] = False
    out = (info & COUNT_MASK) | np.where(conv, CONVERGED, np.uint32(0)) | np.where(tmp, TMP, np.uint32(0))
    return out.astype(np.uint32), err, n, e


def random_film(rng, h, w):
    """(camera, adaptive) float32 (H, W, 4): the adaptive layer is close to the camera layer inside a random disk (the estimate converges there,
    up to a few scattered noisy pixels that keep their surroundings open) and far from it outside"""
    cam = rng.uniform(0.0, 2.0, (h, w, 4)).astype(np.float32)
    y, x = np.mgrid[0:h, 0:w]
    cy, cx, radius = rng.uniform(0, h), rng.uniform(0, w), rng.uniform(0.3, 0.8) * max(h, w)
    amp = np.where((y - cy) ** 2 + (x - cx) ** 2 < radius ** 2, 0.01, 0.6)
    amp = np.where(rng.random((h, w)) < 0.01, 0.6, amp)
    ada = (cam * (1.0 + amp[..., None] * rng.uniform(-1.0, 1.0, (h, w, 4)))).astype(np.float32)
    return cam, ada


def left_lit_scene(samples=64, spectral=False):
    """96 x 32 pixels, so three pixel tiles side by side (ranks 0, 1, 0 of two): a lit diffuse wall fills the left ~17 pixel columns and the
    rest of the frame sees nothing.  The black pixels converge at the first estimate (error level 0), more than five pixels away from any
    noisy one, so rank 1 of two has converged completely after iteration 32 while rank 0 goes on."""
    from etx_tracer_b200 import scenes
    from etx_tracer_b200.scenes import SceneData
    sd = SceneData()
    sd.name = "left-lit wall"
    white = sd.add_material("white", kd=[0.8, 0.8, 0.8], two_sided=1)
    light = sd.add_material("light", kd=[0.0, 0.0, 0.0], emission=scenes.spd_rgb_luminance([10.0, 8.0, 6.0]), two_sided=1)
    # the camera's 40 degrees are the horizontal field of view: x = -1.82 .. 1.82 at the wall, pixel column 16 at x = -1.2; the lamp is above the view
    sd.add_quad([-10, -3, 0], [-1.2, -3, 0], [-1.2, 3, 0], [-10, 3, 0], white)
    sd.add_quad([-3, 1.5, 0.3], [-1.5, 1.5, 0.3], [-1.5, 1.5, 1.3], [-3, 1.5, 1.3], light)
    sd.set_camera([0.0, 0.0, 5.0], [0.0, 0.0, 0.0], [0.0, 1.0, 0.0], 96, 32, 40.0, clip_near=0.1, clip_far=100.0)
    return sd.finalize(samples=samples, spectral=spectral)
