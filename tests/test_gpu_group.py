"""etxb_group's mode changes are checked once, before any NCCL call: pixel tiles refuse a reserved split lane, and a group that has a
communicator refuses a second one of either kind.  Every rank makes the same calls, so every rank refuses alike and none is left waiting in a
collective; the refused group keeps rendering in the mode it had.  One GPU."""
import ctypes

import numpy as np
import pytest

from etx_tracer_b200 import scenes

gpu = pytest.mark.gpu


def _lane_worlds(g):
    worlds = []
    for lane in g.lanes:
        world, rank = ctypes.c_uint32(0), ctypes.c_uint32(0)
        g._check(g.lib.etxb_comm_world(lane.h, ctypes.byref(world), ctypes.byref(rank)))
        worlds.append(world.value)
    return worlds


def _renders(g, iterations):
    st = g.render(iterations)
    assert st["completed_iterations"] == iterations and st["overflow"] == 0
    film = g.film()[..., :3]
    assert np.all(np.isfinite(film)) and film.sum() > 0


@gpu
def test_tiles_refuse_a_split_lane():
    """World 2 with one process: were the refusal not made before the lanes' communicators, this call would wait for a rank that never comes."""
    from etx_tracer_b200 import api
    g = api.GPUVCMGroup(scenes.cornell_box(48, 40, samples=4), lanes=2)
    try:
        g._check(g.lib.etxb_group_reserve_split_lane(g.h))
        with pytest.raises(api.EtxbError) as e:
            g.comm_init(2, 0, np.zeros(3 * api.COMM_ID_BYTES, dtype=np.uint8))
        assert e.value.code == -1 and "split lane" in str(e.value)
        assert _lane_worlds(g) == [1, 1]
        _renders(g, 3)
    finally:
        g.close()


@gpu
@pytest.mark.parametrize("second", ["tiles", "replicas"])
def test_a_second_communicator_is_refused(second):
    """A world-1 etxb_group_comm_init_replicas leaves the group in its one-GPU mode but gives it a communicator: a second init of either kind
    is refused (it would overwrite, and leak, that communicator), and the group renders and is destroyed as before."""
    import torch  # noqa: F401  (loads torch's bundled libnccl, which the module shares)
    from etx_tracer_b200 import api
    try:
        ids = api.comm_unique_ids(3)
    except api.EtxbError:
        pytest.skip("libnccl cannot be loaded")
    g = api.GPUVCMGroup(scenes.cornell_box(48, 40, samples=4), lanes=2)
    try:
        g.comm_init_replicas(1, 0, ids[:api.COMM_ID_BYTES])
        with pytest.raises(api.EtxbError) as e:
            if second == "tiles":
                g.comm_init(1, 0, ids)
            else:
                g.comm_init_replicas(1, 0, ids[api.COMM_ID_BYTES:2 * api.COMM_ID_BYTES])
        assert e.value.code == -1 and "already has a communicator" in str(e.value)
        assert _lane_worlds(g) == [1, 1]
        _renders(g, 4)
        assert np.array_equal(g.comm_reduce_film(), g.film())
    finally:
        g.close()
