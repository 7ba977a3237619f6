"""W emulated ranks on one device: one thread per rank, with the torch.distributed collectives the
sharded paths use (all_reduce with SUM, all_gather) replaced by an in-process exchange between the
threads of a ``ThreadGroup``.  Each thread runs the real sharded code -- shard objects, engine
functions, evaluators -- with ``group=`` its ThreadGroup; collectives on any other group go to
torch.distributed as usual."""
import threading

import torch
import torch.distributed as dist

_me = threading.local()


class ThreadGroup:
    def __init__(self, world):
        self.world = world
        self.barrier = threading.Barrier(world, timeout=300)
        self.slots = [None] * world
        self.calls = [0] * world      # collectives each rank joined

    def exchange(self, t):
        """Every rank's ``t`` (a copy), in rank order."""
        rank = _me.rank
        self.calls[rank] += 1
        self.slots[rank] = t.clone()
        self.barrier.wait()
        everyone = list(self.slots)
        self.barrier.wait()           # nobody overwrites a slot before all have read it
        return everyone


def thread_collectives(monkeypatch):
    """Routes dist.all_reduce / dist.all_gather on a ThreadGroup to the threads."""
    all_reduce, all_gather = dist.all_reduce, dist.all_gather

    def reduce_(t, op=dist.ReduceOp.SUM, group=None, async_op=False):
        if not isinstance(group, ThreadGroup):
            return all_reduce(t, op=op, group=group, async_op=async_op)
        assert op == dist.ReduceOp.SUM
        everyone = group.exchange(t)
        acc = everyone[0]
        for x in everyone[1:]:        # rank order
            acc = acc + x
        t.copy_(acc)

    def gather_(out, t, group=None, async_op=False):
        if not isinstance(group, ThreadGroup):
            return all_gather(out, t, group=group, async_op=async_op)
        for dst, x in zip(out, group.exchange(t)):
            dst.copy_(x)

    monkeypatch.setattr(dist, "all_reduce", reduce_)
    monkeypatch.setattr(dist, "all_gather", gather_)


def run_ranks(world, fn, group=None):
    """[fn(rank, group) for every rank], run concurrently, one thread per rank; the first exception
    of any rank is re-raised (the others then fail at the broken barrier instead of waiting)."""
    group = group or ThreadGroup(world)
    out, errors = [None] * world, []

    def body(rank):
        _me.rank = rank
        try:
            with torch.no_grad():
                out[rank] = fn(rank, group)
        except BaseException as e:    # noqa: B902 -- reported by the caller
            errors.append((rank, e))
            group.barrier.abort()

    threads = [threading.Thread(target=body, args=(rank,)) for rank in range(world)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    first = [e for e in errors if not isinstance(e[1], threading.BrokenBarrierError)] or errors
    if first:
        raise first[0][1]
    return out
