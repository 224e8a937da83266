"""The host's part in a multi-GPU render (one process per GPU).

The module runs every multi-GPU exchange itself, over NCCL: the pixel-tile exchange inside etxb_enqueue_iteration (etxb_comm_init,
etxb_group_comm_init) and the frame reduce of whole-frame replicas (etxb_group_comm_init_replicas).  All the host does is hand the same NCCL
unique ids to every rank, over whatever process group the launcher set up.
"""
from . import structs as S

# bytes of one ETXB_BUF_PHOTON_RECORDS record; kept at this import path for code written against the earlier host-driven exchange
RECORD_BYTES = S.LIGHT_VERTEX_REC.itemsize


def distribute_comm_ids(dist, rank, count, make_ids, device="cuda"):
    """Rank 0 asks the module for `count` NCCL unique ids (make_ids(count) -> uint8[count * 128]) and every rank receives the same bytes (one
    broadcast over `dist`'s default process group)."""
    import numpy as np
    import torch
    n = count * 128
    buf = torch.zeros(n, dtype=torch.uint8, device=device)
    if rank == 0:
        ids = np.ascontiguousarray(make_ids(count), dtype=np.uint8)
        assert ids.size == n
        buf.copy_(torch.from_numpy(ids))
    dist.broadcast(buf, src=0)
    return buf.cpu().numpy()
