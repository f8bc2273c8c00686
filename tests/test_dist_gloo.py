"""N>1 host logic on CPU: world_size-2 gloo run of the batch sharding + all-gather plumbing
(SURVEY.md §8e). The per-shard 'forward' is a deterministic CPU stand-in; the kernels are not
involved (they are covered by the -m gpu tests)."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, total, q):
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "so-net_b200"))
    from sonet_b200 import dist as sdist
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world),
                      MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    sdist.init_from_env(backend="gloo")
    g = torch.Generator().manual_seed(0)
    inputs = {"pc": torch.randn(total, 3, 16, generator=g)}

    def fwd(shard):   # any per-cloud function: shard-invariant by construction
        return torch.stack([shard["pc"].sum(dim=(1, 2)), shard["pc"].amax(dim=(1, 2))], dim=1)

    out = sdist.ShardedForward(fwd)(inputs, total)
    if rank == 0:
        # by value: a tensor would cross the queue as a file descriptor that its sender hands out
        # on request, and this process may have exited before the parent asks for it
        q.put(out.numpy())
    dist.barrier()
    dist.destroy_process_group()


def _run(total):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, total, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = torch.from_numpy(q.get(timeout=120))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    g = torch.Generator().manual_seed(0)
    pc = torch.randn(total, 3, 16, generator=g)
    want = torch.stack([pc.sum(dim=(1, 2)), pc.amax(dim=(1, 2))], dim=1)
    assert torch.equal(out, want)   # bit-exact vs the unsharded run


def test_gloo_world2_even_shards():
    _run(8)


def test_gloo_world2_ragged_shards():
    _run(7)
