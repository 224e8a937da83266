"""The path tracer's noise estimate over pixel tiles, on the CPU: the tile rule gives every word of the active mask one owner, the mask -> dilation
form equals the reference's scatter passes, and summing the ranks' masks reproduces the one-frame estimate (tests/pt_tiles_model.py; the device
kernels are held to the same model in test_gpu_pt_tiles.py)."""
import numpy as np
import pytest

import pt_tiles_model as M


@pytest.mark.parametrize("width", [1, 31, 32, 33, 95, 1920])
@pytest.mark.parametrize("height", [1, 31, 33, 97])
def test_every_mask_word_has_one_owner(width, height):
    """Tiles are 32 pixels wide and start at multiples of 32, and a storage row is one film row: the 32 pixels of a mask word (those inside the
    film) belong to one rank, for any world and with partial tiles at the right and top edges."""
    for world in range(1, 9):
        own = M.owner_map(width, height, world)
        wpr = M.words_per_row(width)
        padded = np.full((height, wpr * 32), -1)
        padded[:, :width] = own
        words = padded.reshape(height, wpr, 32)
        for r in range(height):
            for k in range(wpr):
                ranks = set(words[r, k][words[r, k] >= 0].tolist())
                assert len(ranks) == 1, (width, height, world, r, k, ranks)
        assert set(np.unique(own).tolist()) <= set(range(world))


def _history(rng, h, w, rounds):
    """a reachable history: `rounds` reference estimates on random films (counts made up), then a fresh random film"""
    info = rng.integers(32, 64, (h, w)).astype(np.uint32)
    for _ in range(rounds):
        cam, ada = M.random_film(rng, h, w)
        info = M.reference_estimate(cam, ada, info, 0.3)[0]
    return info


SIZES = [(1, 1), (7, 5), (31, 33), (36, 40), (70, 95), (1, 200), (64, 3), (40, 64)]


@pytest.mark.parametrize("h,w", SIZES)
@pytest.mark.parametrize("rounds", [0, 1, 2])
def test_mask_dilation_equals_the_reference_scatter_form(h, w, rounds):
    """One rank owning the whole film: pack the mask, dilate it with the funnel-shift row windows, and get the reference's info words — also
    when earlier estimates left converged pixels, which read as converged in the mask and may be reopened near an active pixel."""
    rng = np.random.default_rng(1000 * h + w + rounds)
    info = _history(rng, h, w, rounds)
    cam, ada = M.random_film(rng, h, w)
    for thr in (0.05, 0.3, 0.9):
        want, err_want, n_want, e_want = M.reference_estimate(cam, ada, info, thr)
        got, err, n, e = M.tiled_estimate(cam, ada, info, thr, 1)
        assert np.array_equal(got, want), (h, w, rounds, thr)
        assert np.array_equal(err, err_want) and n == n_want and e == pytest.approx(e_want, rel=1e-12)


@pytest.mark.parametrize("h,w", SIZES)
@pytest.mark.parametrize("world", [2, 3, 5, 8])
def test_summed_masks_give_the_one_frame_estimate(h, w, world):
    """Each rank's view holds zeros outside its tiles; the summed masks are the one-frame mask, so the composed info words and error levels
    are the one-frame ones, and the counts add up."""
    rng = np.random.default_rng(7 * h + w + world)
    info = _history(rng, h, w, 1)
    cam, ada = M.random_film(rng, h, w)
    want, err_want, n_want, e_want = M.reference_estimate(cam, ada, info, 0.3)
    got, err, n, e = M.tiled_estimate(cam, ada, info, 0.3, world)
    assert np.array_equal(got, want) and np.array_equal(err, err_want)
    assert n == n_want and e == pytest.approx(e_want, rel=1e-12)


def _old_partition_estimate(cam, ada, info, thr, rank, world):
    """What a context with a partition and no communicator ran before the mask: the whole-film passes over a film that is zero outside its tiles
    (a zero pixel has error level 0, so it converges at the first estimate)"""
    mine = M.owner_map(info.shape[1], info.shape[0], world) == rank
    return M.reference_estimate(np.where(mine[..., None], cam, 0).astype(np.float32), np.where(mine[..., None], ada, 0).astype(np.float32),
                                np.where(mine, info, 0).astype(np.uint32), thr)


@pytest.mark.parametrize("h,w", [(36, 40), (70, 95), (96, 80)])
@pytest.mark.parametrize("world", [2, 3])
def test_absent_ranks_read_as_converged(h, w, world):
    """A partition without a communicator sums no other rank's words: zero words read as converged, so its own pixels get the history they got
    when the estimate ran over the whole (zero elsewhere) film — over several estimates.  Only the counts change: they are its own pixels'."""
    rng = np.random.default_rng(h + w + world)
    own = M.owner_map(w, h, world)
    for rank in range(world):
        mine = own == rank
        old = np.zeros((h, w), np.uint32)
        new = old.copy()
        for _ in range(3):
            cam, ada = M.random_film(rng, h, w)
            old, err_old, _, _ = _old_partition_estimate(cam, ada, old, 0.3, rank, world)
            absent = [r for r in range(world) if r != rank]
            new_all, err_new, n, _ = M.tiled_estimate(cam, ada, new, 0.3, world, absent=absent)
            new = np.where(mine, new_all, 0).astype(np.uint32)
            assert np.array_equal(new[mine], old[mine]) and np.array_equal(err_new[mine], err_old[mine])
            assert n <= int(mine.sum())
