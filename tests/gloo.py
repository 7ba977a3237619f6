"""Ranks as processes for the multi-process tests: a free local port, the process-group setup of every
rank and the spawn wrapper around them."""
import os
import socket

import torch.distributed as dist
import torch.multiprocessing as mp


def free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _main(rank, world, port, backend, fn, args, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group(backend, rank=rank, world_size=world)
    try:
        ret[rank] = fn(rank, world, *args)
    finally:
        dist.destroy_process_group()


def spawn(world, fn, *args, backend="gloo"):
    """{rank: fn(rank, world, *args)} from ``world`` processes joined in one process group of ``backend``;
    ``fn`` is a module-level function with a picklable result.  An exception in a rank fails the call."""
    with mp.Manager() as mgr:
        ret = mgr.dict()
        mp.spawn(_main, args=(world, free_port(), backend, fn, args, ret), nprocs=world, join=True)
        return dict(ret)
