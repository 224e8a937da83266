"""World-size-2 run of the host's part in the module's multi-GPU path (etx_tracer_b200/multigpu.py) on CPU tensors over gloo."""
import os
import socket

import numpy as np
import torch.distributed as dist
import torch.multiprocessing as mp

from etx_tracer_b200 import multigpu


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _ids_worker(rank, world, port, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        calls = []

        def make_ids(count):  # stands in for api.comm_unique_ids (ncclGetUniqueId inside the module): only rank 0 may be asked
            calls.append(count)
            return (np.arange(count * 128) % 251).astype(np.uint8)

        ids = multigpu.distribute_comm_ids(dist, rank, 3, make_ids, device="cpu")
        np.savez(os.path.join(out_dir, f"ids{rank}.npz"), ids=ids, calls=np.array(calls))
    finally:
        dist.destroy_process_group()


def test_comm_ids_reach_every_rank_over_gloo(tmp_path):
    """The host's whole part in the module's own multi-GPU path (etxb_group_comm_init): rank 0's NCCL ids, byte for byte, on every rank."""
    world = 2
    mp.spawn(_ids_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    r = [np.load(tmp_path / f"ids{k}.npz") for k in range(world)]
    want = (np.arange(3 * 128) % 251).astype(np.uint8)
    assert np.array_equal(r[0]["ids"], want) and np.array_equal(r[1]["ids"], want)
    assert r[0]["calls"].tolist() == [3] and r[1]["calls"].size == 0
