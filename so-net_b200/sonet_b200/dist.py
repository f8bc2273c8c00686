"""Batch-sharded multi-GPU forward (SURVEY.md §8e): one process per GPU, weights replicated,
the global batch split contiguously over ranks, and ONE all-gather per forward of the per-shard
logits (or per-cloud losses) over NCCL/NVLink. Every op of the eval forward is per-cloud, so there
is no exchange step inside the path and the gathered result is bit-identical to a 1-GPU run.

DataParallelTraining (below) trains over the ranks with synchronised BatchNorm and rank-ordered
gradient sums: the semantics of one process over the global batch.

The same code runs on CPU with the gloo backend (tests/test_dist_gloo.py, world_size 2) — only the
collective plumbing is exercised there, never the kernels.
"""
import os

import torch
import torch.distributed as dist
import torch.optim.optimizer as _optimizer
from torch.nn.modules.batchnorm import _BatchNorm


def env_world():
    return (int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0")),
            int(os.environ.get("WORLD_SIZE", "1")))


def init_from_env(backend=None):
    """Initialise torch.distributed from torchrun's environment. Returns (rank, local_rank, world).
    With WORLD_SIZE=1 no process group is created."""
    rank, local_rank, world = env_world()
    if torch.cuda.is_available():
        torch.cuda.set_device(local_rank % max(torch.cuda.device_count(), 1))
    if world > 1 and not dist.is_initialized():
        backend = backend or ("nccl" if torch.cuda.is_available() else "gloo")
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        kw = {}
        if backend == "nccl":
            kw["device_id"] = torch.device("cuda", torch.cuda.current_device())
        dist.init_process_group(backend=backend, rank=rank, world_size=world, **kw)
    return rank, local_rank, world


def shard_bounds(total, rank, world):
    """Contiguous split of `total` clouds: the first (total % world) ranks get one extra."""
    base, rem = divmod(total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def all_gather_rows(local, total_rows=None, out=None):
    """Gather [rows_r, ...] shards from every rank into [sum rows, ...] in rank order.
    Equal shards use one all_gather_into_tensor (into `out` when given: a persistent buffer avoids
    a caching-allocator round trip per step); ragged shards pad to the largest."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return local
    world = dist.get_world_size()
    local = local.contiguous()
    if total_rows is None or total_rows % world == 0:
        if out is None:
            out = local.new_empty((local.shape[0] * world,) + tuple(local.shape[1:]))
        dist.all_gather_into_tensor(out, local)
        return out
    sizes = [shard_bounds(total_rows, r, world) for r in range(world)]
    rows = max(hi - lo for lo, hi in sizes)
    padded = local.new_zeros((rows,) + tuple(local.shape[1:]))
    padded[:local.shape[0]] = local
    out = local.new_empty((rows * world,) + tuple(local.shape[1:]))
    dist.all_gather_into_tensor(out, padded)
    return torch.cat([out[r * rows:r * rows + (hi - lo)] for r, (lo, hi) in enumerate(sizes)])


class ShardedForward:
    """Runs `forward_fn(shard_inputs) -> [rows, ...]` on this rank's contiguous slice of a global
    batch and all-gathers the rows. `forward_fn` is e.g. a classifier.Model's set_input+test_model."""

    def __init__(self, forward_fn):
        self.forward_fn = forward_fn
        self.rank, _, self.world = env_world()

    def __call__(self, global_inputs, total_rows):
        lo, hi = shard_bounds(total_rows, self.rank, self.world)
        shard = {k: v[lo:hi] for k, v in global_inputs.items()}
        return all_gather_rows(self.forward_fn(shard), total_rows)


class SonetComm:
    """The C-ABI collective (sonet_comm_init / sonet_allgather, csrc/comm.cu): an NCCL communicator
    created through libsonet_b200 on the current device. torch.distributed must be initialised
    (any backend): its process group is only the transport of the 128-byte unique id."""

    def __init__(self):
        import ctypes
        from . import _C
        self._C = _C
        rank, world = dist.get_rank(), dist.get_world_size()
        dev = torch.device("cuda", torch.cuda.current_device())
        idt = torch.zeros(128, dtype=torch.uint8)
        if rank == 0:
            _C.check(_C.lib().sonet_comm_unique_id(idt.data_ptr()), "sonet_comm_unique_id")
        idt = idt.to(dev) if dist.get_backend() == "nccl" else idt
        dist.broadcast(idt, src=0)
        idt = idt.cpu().contiguous()
        handle = ctypes.c_void_p()
        _C.check(_C.lib().sonet_comm_init(idt.data_ptr(), rank, world, ctypes.byref(handle)),
                 "sonet_comm_init")
        self.handle, self.rank, self.world = handle, rank, world

    def all_gather(self, local, out, stream=None):
        """out [world*rows, ...] <- every rank's local [rows, ...]; asynchronous on `stream`
        (default: the current stream); CUDA-graph capturable."""
        local = local.contiguous()
        st = (stream or torch.cuda.current_stream(local.device)).cuda_stream
        self._C.check(self._C.lib().sonet_allgather(self.handle, local.data_ptr(), out.data_ptr(),
                                                    local.numel() * local.element_size(), st),
                      "sonet_allgather")
        return out

    def destroy(self):
        if self.handle:
            self._C.check(self._C.lib().sonet_comm_destroy(self.handle), "sonet_comm_destroy")
            self.handle = None


class AsyncGather:
    """Per-step all-gather of result rows that completes under the NEXT step's forward.

    launch(i, rows): stage the rows (a graph's static output buffer is overwritten by the next
    replay) and start the gather of step i; wait_prev(i): make the current stream wait for the
    gather of step i-1 — called at the end of step i, so every gather ends inside a step.
    impl 'torch': torch.distributed.all_gather_into_tensor(async_op=True) (NCCL's own stream);
    impl 'sonet': sonet_allgather on a side stream ordered by events."""

    def __init__(self, world, rows_shape, dev, impl="torch"):
        self.world, self.impl, self.dev = world, impl, dev
        self.stage = [torch.empty(rows_shape, dtype=torch.float32, device=dev) for _ in range(2)]
        full = (rows_shape[0] * world,) + tuple(rows_shape[1:])
        self.out = [torch.empty(full, dtype=torch.float32, device=dev) for _ in range(2)]
        self.pending = [None, None]
        if impl == "sonet":
            self.comm = SonetComm()
            self.side = torch.cuda.Stream(device=dev)
            self.ev_fwd = [torch.cuda.Event(), torch.cuda.Event()]
            self.ev_done = [torch.cuda.Event(), torch.cuda.Event()]

    def launch(self, i, rows):
        j = i & 1
        self.stage[j].copy_(rows)
        if self.impl == "torch":
            self.pending[j] = dist.all_gather_into_tensor(self.out[j], self.stage[j], async_op=True)
        else:
            cur = torch.cuda.current_stream(self.dev)
            self.ev_fwd[j].record(cur)
            self.side.wait_event(self.ev_fwd[j])
            self.comm.all_gather(self.stage[j], self.out[j], stream=self.side)
            self.ev_done[j].record(self.side)
            self.pending[j] = self.ev_done[j]
        return self.out[j]

    def _wait(self, j):
        p = self.pending[j]
        if p is None:
            return
        if self.impl == "torch":
            p.wait()
        else:
            torch.cuda.current_stream(self.dev).wait_event(p)
        self.pending[j] = None

    def wait_prev(self, i):
        self._wait((i - 1) & 1)

    def drain(self):
        self._wait(0)
        self._wait(1)


# ---- data-parallel training ----------------------------------------------------------------------
def _process_group():
    """(rank, world) of the initialised process group; (0, 1) without one."""
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def gather_shards(local, counts):
    """Every rank's rows, concatenated in rank order: rank r contributes counts[r] rows of the same
    trailing shape. NCCL: one all_gather_into_tensor of the shards, padded to the largest when they
    are ragged (as all_gather_rows). gloo, which offers CUDA tensors all_reduce only: an all_reduce
    of a zero-filled [sum counts, ...] buffer in which each rank filled its own rows. Adding zeros
    is exact, so both give the same bits. Without a process group: `local` itself."""
    rank, world = _process_group()
    if world == 1:
        return local
    local = local.contiguous()
    if local.shape[0] != counts[rank]:
        raise RuntimeError("gather_shards: rank %d holds %d rows, expected %d"
                           % (rank, local.shape[0], counts[rank]))
    rest = tuple(local.shape[1:])
    if dist.get_backend() == "gloo":
        out = local.new_zeros((sum(counts),) + rest)
        lo = sum(counts[:rank])
        out[lo:lo + counts[rank]] = local
        dist.all_reduce(out)
        return out
    rows = max(counts)
    if all(c == rows for c in counts):
        out = local.new_empty((rows * world,) + rest)
        dist.all_gather_into_tensor(out, local)
        return out
    padded = local.new_zeros((rows,) + rest)
    padded[:local.shape[0]] = local
    out = local.new_empty((rows * world,) + rest)
    dist.all_gather_into_tensor(out, padded)
    return torch.cat([out[r * rows:r * rows + c] for r, c in enumerate(counts)])


class _Exchange:
    """train_ops.EXCHANGE of a DataParallelTraining: the BatchNorm records' gather along the cloud
    axis. Optionally times every gather with CUDA events (kind 'bn' or 'grad')."""

    def __init__(self, global_batch, rank, world):
        self.global_batch, self.rank, self.world = global_batch, rank, world
        self.counts = [hi - lo for lo, hi in (shard_bounds(global_batch, r, world)
                                              for r in range(world))]
        self.events = None          # {kind: [(start, end), ...]} while timing

    def global_rows(self, B):
        if B != self.counts[self.rank]:
            raise RuntimeError("DataParallelTraining: rank %d ran a train step on %d clouds; its "
                               "shard of the global batch of %d is %d clouds (shard_bounds)"
                               % (self.rank, B, self.global_batch, self.counts[self.rank]))
        return self.global_batch

    def gather(self, rec, counts=None, kind="bn"):
        if self.events is None or not rec.is_cuda:
            return gather_shards(rec, counts or self.counts)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = gather_shards(rec, counts or self.counts)
        e1.record()
        self.events.setdefault(kind, []).append((e0, e1))
        return out


def check_sync_batchnorm(modules):
    """Raise unless every BatchNorm below `modules` runs on train_ops.norm_act_train in a train step:
    the norm of a MyLinear / MyConv2d / EquivariantLayer with a kernel activation (relu, elu, none),
    with the train kernels enabled. Instance norm is per cloud and needs no exchange."""
    from . import layers, train_ops
    if not train_ops.ENABLED:
        raise RuntimeError("DataParallelTraining needs the train kernels (train_ops.ENABLED = True): "
                           "only their BatchNorm synchronises over the ranks")
    owners = (layers.MyLinear, layers.MyConv2d, layers.EquivariantLayer)
    for root in modules:
        for name, m in root.named_modules():
            for cname, child in m.named_children():
                if not isinstance(child, _BatchNorm):
                    continue
                if not (isinstance(m, owners) and child is getattr(m, "norm", None)
                        and m.normalization == "batch"
                        and m.activation in layers.KERNEL_ACTIVATIONS):
                    where = "%s.%s" % (name, cname) if name else cname
                    raise RuntimeError(
                        "DataParallelTraining: the BatchNorm %s (%s in %s, activation %r) does not "
                        "run on the train kernels, so its statistics would not be synchronised"
                        % (where, type(child).__name__, type(m).__name__,
                           getattr(m, "activation", None)))


class DataParallelTraining:
    """Data-parallel training of a Model (classifier, segmenter or auto-encoder: the reference's
    models/*.py under install(), or this package's wrappers) over the ranks of the initialised
    process group, with the semantics of one process over the global batch:

      * every BatchNorm normalises by the statistics of the whole global batch and updates its
        running statistics with the global count. Each rank writes the train-mode BatchNorm's one
        fp64 record per (cloud, channel) (sonet_bn_cloud_partials_f32), as a single process does;
        the records are gathered along the cloud axis and folded in ascending cloud order
        (sonet_bn_sync_forward_f32 / _backward_f32). The records depend only on their cloud, so
        mean, var, y, dx, dgamma and dbeta are bit-identical at every world size and sharding, and
        to those of one process over the global batch;
      * before every step of an optimizer over the model's parameters, its gradients are scaled
        by B_r / Bg (every loss of the reference is a batch mean), gathered and summed in
        ascending rank order: every rank steps on the same gradient of the global-batch loss.
        The BatchNorms' gamma and beta are left alone: the exchange already made their
        gradients those of the global-batch loss, identical on every rank;
      * parameters and buffers are broadcast from rank 0 once, here.

    Each rank calls set_input with its shard, rows shard_bounds(global_batch, rank, world) of the
    global batch (DeviceDataset.batch(..., shard=(rank, world))). The host RNGs (`random`,
    `np.random`: the point dropout of the reference's optimize(), the per-cloud augmentation
    scalars) must be seeded identically on every rank; nn.Dropout masks differ per rank, as they
    do between two single-GPU runs. Without a process group the exchange is the identity: a
    one-process run is the reference for a run over G ranks.

    The optimizers are hooked through torch.optim's global step pre-hook, restricted to those
    that step a parameter of the model, so optimizers the Model creates lazily in its first
    optimize() are covered too. close() removes the exchange and the hook."""

    def __init__(self, model, global_batch):
        from . import layers, train_ops
        self.rank, self.world = _process_group()
        self.global_batch = int(global_batch)
        if not self.world <= self.global_batch <= 65535:
            raise ValueError("DataParallelTraining: the global batch (%d) must hold at least one "
                             "cloud per rank (%d ranks) and at most 65535"
                             % (self.global_batch, self.world))
        self.modules = ([model] if isinstance(model, torch.nn.Module) else
                        [v for v in vars(model).values() if isinstance(v, torch.nn.Module)])
        check_sync_batchnorm(self.modules)
        if train_ops.EXCHANGE is not None:
            raise RuntimeError("DataParallelTraining: another instance is installed; close() it")
        state = {}
        for m in self.modules:
            for t in list(m.parameters()) + list(m.buffers()):
                state[id(t)] = t
        self._param_ids = {id(p) for m in self.modules for p in m.parameters()}
        # the BatchNorms' gamma and beta: their gradients leave the exchange as the global ones
        self._bn_ids = {id(p) for m in self.modules for mm in m.modules()
                        if isinstance(mm, _BatchNorm) for p in mm.parameters()}
        if self.world > 1:
            with torch.no_grad():
                for t in state.values():
                    dist.broadcast(t.data, src=0)
            for m in self.modules:
                layers.invalidate(m)       # the broadcast writes bypass the version counters
        lo, hi = shard_bounds(self.global_batch, self.rank, self.world)
        self.local_batch = hi - lo
        self.exchange = _Exchange(self.global_batch, self.rank, self.world)
        self._hook = _optimizer.register_optimizer_step_pre_hook(self._reduce_grads)
        train_ops.EXCHANGE = self.exchange

    def _reduce_grads(self, optimizer, args, kwargs):
        params = [p for g in optimizer.param_groups for p in g["params"] if p.grad is not None]
        if self.world == 1 or not any(id(p) in self._param_ids for p in params):
            return
        params = [p for p in params if id(p) not in self._bn_ids]
        if not params:
            return
        flat = torch.cat([p.grad.reshape(-1) for p in params])
        flat.mul_(self.local_batch / self.global_batch)
        rows = self.exchange.gather(flat.unsqueeze(0), [1] * self.world, kind="grad")
        total = rows[0].clone()
        for r in range(1, self.world):          # ascending rank order: the same bits everywhere
            total += rows[r]
        o = 0
        for p in params:
            n = p.grad.numel()
            p.grad.copy_(total[o:o + n].view_as(p.grad))
            o += n

    def shard(self):
        """(lo, hi): this rank's rows of the global batch."""
        return shard_bounds(self.global_batch, self.rank, self.world)

    def start_timing(self):
        """Time every exchange with CUDA events from now on (see exchange_ms)."""
        self.exchange.events = {}

    def exchange_ms(self):
        """{kind: (count, total ms)} of the exchanges timed since start_timing(); synchronises."""
        torch.cuda.synchronize()
        return {k: (len(v), sum(a.elapsed_time(b) for a, b in v))
                for k, v in (self.exchange.events or {}).items()}

    def close(self):
        """Remove the BatchNorm exchange and the optimizer hook: train steps are single-process
        steps again. Their BatchNorms give the bits they gave under the exchange at world 1, except
        those of the decoder's 3x3 convolutions below UPCONV_MIN_HW, which return to PyTorch's
        BatchNorm."""
        from . import train_ops
        if self._hook is not None:
            self._hook.remove()
            self._hook = None
        if train_ops.EXCHANGE is self.exchange:
            train_ops.EXCHANGE = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
