"""Multi-GPU plumbing: one process per GPU, reads sharded by contiguous
read-id ranges, index image broadcast once, SAM chunks gathered in rank order.

The reference's only parallelism is `-p N` threads pulling reads from one
input (hisat2.cpp:3657-3696) with `--reorder` restoring input order
(outq.cpp:51-99).  Reads are independent under --no-spliced-alignment, so the
GPU equivalent shards reads across ranks with NO data-path collective: the
only collective is the start-up broadcast of the packed index image (NCCL over
NVLink/NVSwitch when the backend is nccl, gloo in the CPU tests).
"""
import numpy as np


def shard_range(n_units, rank, world):
    """Contiguous [lo, hi) range of read (pair) ids for `rank`; sizes differ by
    at most one and concatenating the shards in rank order restores input order."""
    base, rem = divmod(n_units, world)
    lo = rank * base + min(rank, rem)
    hi = lo + base + (1 if rank < rem else 0)
    return lo, hi


def broadcast_image(image, rank, device=None, src=0):
    """Broadcast the packed index image (uint8) from rank `src`.

    image: numpy uint8 array on the source rank (ignored elsewhere).
    Returns a torch uint8 tensor (on `device` if given) holding the image on
    every rank.  With backend nccl the destination is device memory that
    ht2gpu_open_device_image can adopt without another copy.
    """
    import torch
    import torch.distributed as dist
    dev = device if device is not None else "cpu"
    n = torch.zeros(1, dtype=torch.int64, device=dev)
    if rank == src:
        n[0] = int(image.nbytes)
    dist.broadcast(n, src=src)
    if rank == src:
        buf = torch.from_numpy(np.ascontiguousarray(image)).to(dev)
    else:
        buf = torch.empty(int(n.item()), dtype=torch.uint8, device=dev)
    dist.broadcast(buf, src=src)
    return buf


def gather_bytes(chunk, rank, world, dst=0):
    """Gather one bytes object per rank to `dst`; returns the list (rank order)
    on dst and None elsewhere -- the host-side equivalent of --reorder."""
    import torch.distributed as dist
    out = [None] * world if rank == dst else None
    dist.gather_object(chunk, out, dst=dst)
    return out
