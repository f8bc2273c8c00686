"""Shared plumbing of the three caller-facing Model wrappers (classifier / segmenter /
autoencoder): double-buffered asynchronous set_input and CUDA-graph replay of the eval forward.

set_input copies into the input buffer set that the in-flight forward is NOT reading, on a
dedicated copy stream, and the next forward makes the compute stream wait for exactly that copy.
The reference call order (set_input, then forward / test_model — models/classifier.py:64-105) is
unchanged; a serving loop that wants the host-to-device copy hidden simply issues
set_input(batch i+1) before it reads the results of batch i.

enable_cuda_graph(True) replays test_model() as ONE CUDA graph per input buffer set: every C-ABI
entry point is allocation- and synchronisation-free, so the ~15-40 Python/ctypes op calls of a step
become one graph launch. Outputs then live in per-graph static buffers; the attributes that other
code reads after a forward (model.score, encoder.som_node, chamfer_criteria.loss_array, ...) are
re-bound to the replayed graph's buffers on every replay.

enable_train_graph(True) does the same for optimize(): one graph per input buffer set holds the
forward, the losses, zero_grad, the backward and both optimizers' step(). See enable_train_graph
for what re-captures, what stays eager and how the weight caches see a replay.
"""
import torch

from . import layers, ops, train_ops


class _InputSet:
    def __init__(self, spec, dev):
        self.t = {name: fn(dev) for name, fn in spec}
        self.ready = torch.cuda.Event() if dev.type == "cuda" else None      # copy finished
        self.consumed = torch.cuda.Event() if dev.type == "cuda" else None   # last forward finished


class GraphedModel:
    # subclasses: ordered (attribute name, allocator(dev)) of the set_input arguments
    _INPUT_SPEC = ()
    # objects (attribute paths on self, "" = self) -> attribute names to snapshot per graph
    _SNAPSHOT = {}

    def _init_io(self, dev):
        self._dev = dev
        self._sets = [_InputSet(self._INPUT_SPEC, dev) for _ in range(2)]
        self._cur = 0
        self._copy_stream = torch.cuda.Stream(device=dev) if dev.type == "cuda" else None
        self._use_graph = False
        self._graphs = {}
        self._graph_stream = None
        self._use_train_graph = False
        self._train_graphs = {}
        self._optim = None
        self._bind(self._sets[0])

    # ---- inputs --------------------------------------------------------------------------------------
    def _bind(self, s):
        for name, _ in self._INPUT_SPEC:
            setattr(self, name, s.t[name])
        self._after_bind(s)

    def _after_bind(self, s):
        pass

    def _set_input(self, *srcs):
        """Copy one batch (host or device tensors) into the idle device buffer set. Pinned host
        tensors are copied asynchronously on the copy stream; the next forward waits for this copy
        only."""
        self._cur ^= 1
        s = self._sets[self._cur]
        dsts = [s.t[name] for name, _ in self._INPUT_SPEC]
        if self._copy_stream is None:
            for d, t in zip(dsts, srcs):
                d.resize_(t.size()).copy_(t)
        else:
            cur = torch.cuda.current_stream(self._dev)
            cs = self._copy_stream
            cs.wait_event(s.consumed)        # the forward that last read this set is done
            if any(t.is_cuda for t in srcs):
                cs.wait_stream(cur)          # device-side sources produced on the caller's stream
            with torch.cuda.stream(cs):
                for d, t in zip(dsts, srcs):
                    if d.size() != t.size():
                        d.resize_(t.size())
                    d.copy_(t, non_blocking=True)
                    if t.is_cuda:
                        t.record_stream(cs)
                s.ready.record(cs)
        self._bind(s)

    def _wait_inputs(self):
        s = self._sets[self._cur]
        if s.ready is not None:
            torch.cuda.current_stream(self._dev).wait_event(s.ready)
        return s

    def _mark_consumed(self, s):
        if s.consumed is not None:
            s.consumed.record(torch.cuda.current_stream(self._dev))

    # ---- CUDA-graph replay of the eval forward ---------------------------------------------------------
    def enable_cuda_graph(self, flag=True):
        """Replay test_model() as one CUDA graph per input buffer set. Graphs are re-captured when
        an input shape or any parameter/buffer version changes."""
        self._use_graph = bool(flag) and self._dev.type == "cuda"
        self._graphs = {}
        if self._use_graph and self._graph_stream is None:
            self._graph_stream = torch.cuda.Stream(device=self._dev)

    def enable_train_graph(self, flag=True):
        """Replay optimize() as one CUDA graph per input buffer set: forward, losses, zero_grad,
        backward and both optimizers' step(). N calls make exactly N updates: the first call for a
        new key is an eager step on the capture stream (it warms the weight packs, the scratch
        buffers and the optimizers' state), the next one captures the graph and replays it once,
        and later ones replay it. The model's attributes (score, loss, predicted_pc, the encoder's
        cached tensors, ...) and every p.grad are re-bound to the graph's static tensors after
        each replay.

        A graph is re-captured when its key changes: the input shapes, SONET_TRAIN_TC,
        train_ops.ENABLED and WGRAD_TC, a layer's activation, a BatchNorm's momentum at this
        epoch, a param group's lr / betas / eps / weight_decay, which parameters require grad,
        opt.dropout, a parameter's storage, or an optimizer's state dict (load_state_dict).
        Tensor versions are not part of the key; instead every replay bumps the versions of the
        parameters and buffers it updated in place, so the BatchNorm folds, the wgmma packs
        derived from them and the eval graph's key see the update as they see an eager step.

        The optimizers become capturable (torch.optim.Adam(capturable=True)) at the first step
        that takes the graph path; state from earlier eager steps carries over (`step` moves to
        the device). enable_train_graph(False) turns them back into ordinary Adams (`step` back on
        the host), so later eager steps run exactly as in a model that never enabled the graph.
        Steps stay eager while opt.random_pc_dropout_lower_limit < 0.99 (the reference's
        optimize() then draws the point count on the host, so N changes from step to step), while
        a DataParallelTraining is installed (train_ops.EXCHANGE), and on non-CUDA devices; such a
        step runs the optimizers in whichever mode they are in (capturable once a graphed step has
        run: the same update, which may round differently). nn.Dropout masks come from PyTorch's
        graph-safe generator: each replay draws new ones, and torch.manual_seed reproduces them.

        Each input buffer set holds one graph, and set_input alternates the sets, so a training
        loop holds two graphs (two private memory pools). A batch of another size (an epoch's
        short last batch) re-keys its set, and the next full batch on that set re-keys it back:
        each costs one eager step and one capture."""
        self._use_train_graph = bool(flag) and self._dev.type == "cuda"
        self._train_graphs = {}
        if self._use_train_graph and self._graph_stream is None:
            self._graph_stream = torch.cuda.Stream(device=self._dev)
        if not self._use_train_graph and self._optim is not None:
            self._make_capturable(False)

    def invalidate(self):
        """Forget folded/packed weights and captured graphs (call after editing parameters
        through `.data`, which does not bump tensor versions — see layers.invalidate)."""
        for m in self._state_modules():
            layers.invalidate(m)
        self._graphs = {}
        self._train_graphs = {}

    def _state_modules(self):
        raise NotImplementedError

    def _eval_forward(self):
        raise NotImplementedError

    def _state_key(self, s):
        if not hasattr(self, "_state_tensors"):
            self._state_tensors = [t for m in self._state_modules()
                                   for t in list(m.parameters()) + list(m.buffers())]
        if not hasattr(self, "_act_modules"):
            self._act_modules = [m for sm in self._state_modules() for m in sm.modules()
                                 if hasattr(m, "activation")]
        ver = 0
        for t in self._state_tensors:
            ver += t._version
        # the precision mode and the layers' activations pick the kernels a forward launches: a
        # graph captured for one must not replay for another (activation is a plain attribute)
        return (tuple(tuple(t.shape) for t in s.t.values()), ver,
                getattr(self.encoder, "fuse_pool", None), getattr(self.encoder, "_fpo_demand", None),
                layers.tc_mode(), tuple(m.activation for m in self._act_modules))

    def _resolve(self, path):
        obj = self
        for part in [p for p in path.split(".") if p]:
            obj = getattr(obj, part)
        return obj

    def _test_model_graph(self):
        s = self._sets[self._cur]
        cur = torch.cuda.current_stream(self._dev)
        cur.wait_event(s.ready)
        key = self._state_key(s)
        g = self._graphs.get(self._cur)
        with torch.no_grad():
            if g is None or g["key"] != key:
                # warm-up AND capture run on the model's capture stream, so per-stream scratch
                # (the pool keys) is created and left clean before the capture starts
                gs = self._graph_stream
                gs.wait_stream(cur)
                with torch.cuda.stream(gs):
                    for _ in range(2):           # warm every host-side cache (folded/packed weights)
                        self._eval_forward()
                torch.cuda.synchronize(self._dev)
                key = self._state_key(s)         # the warm-up may have switched encoder paths
                graph = torch.cuda.CUDAGraph()
                k0, c0 = ops.KERNEL_LAUNCHES, ops.LAUNCHES
                with torch.cuda.graph(graph, stream=gs):
                    self._eval_forward()
                g = dict(key=key, graph=graph, kernels=ops.KERNEL_LAUNCHES - k0,
                         calls=ops.LAUNCHES - c0, snap=self._snapshot())
                self._graphs[self._cur] = g
            g["graph"].replay()
        ops.KERNEL_LAUNCHES += g["kernels"]      # the replay launches the captured kernels
        ops.LAUNCHES += g["calls"]
        # cached attributes point at THIS graph's static buffers again (two input sets = two
        # graphs = two buffer sets); attributes that were still lazy (None) at capture time become
        # lazy again and are recomputed from the replayed buffers on demand
        self._rebind(g["snap"])
        s.consumed.record(cur)

    def _snapshot(self):
        snap = {}
        for path, names in self._SNAPSHOT.items():
            obj = self._resolve(path)
            snap[path] = {n: getattr(obj, n) for n in names if hasattr(obj, n)}
        return snap

    def _rebind(self, snap):
        for path, vals in snap.items():
            obj = self._resolve(path)
            for n, v in vals.items():
                setattr(obj, n, v)

    # ---- training step, eager or as a CUDA graph -------------------------------------------------------
    def _make_optimizers(self):
        raise NotImplementedError

    def _train_step(self, epoch, forward):
        raise NotImplementedError

    def optimize(self, epoch=None):
        """One training step of the reference's Model.optimize() on the differentiable PyTorch
        path, or with enable_train_graph(True) on its CUDA graph."""
        if self._optim is None:
            self._optim = self._make_optimizers()
        if self._train_graph_applies():
            return self._optimize_graph(epoch)
        self._train_step(epoch, self.forward)

    def _train_graph_applies(self):
        """enable_train_graph is on and none of its eager cases holds: a random point dropout
        (the point count varies per step), an installed DataParallelTraining, a non-CUDA device."""
        return (self._use_train_graph and train_ops.EXCHANGE is None
                and not self.opt.random_pc_dropout_lower_limit < 0.99)

    def _train_state(self):
        if not hasattr(self, "_train_lists"):
            mods = [m for sm in self._state_modules() for m in sm.modules()]
            self._train_lists = (
                [p for sm in self._state_modules() for p in sm.parameters()],
                [b for sm in self._state_modules() for b in sm.buffers()],
                [m for m in mods if hasattr(m, "activation")],
                [m for m in mods if isinstance(m, layers._MomentumDecayBatchNorm)])
        return self._train_lists

    def _train_key(self, s, epoch):
        params, _, acts, bns = self._train_state()
        return (tuple(tuple(t.shape) for t in s.t.values()), train_ops.train_f16(),
                train_ops.ENABLED, train_ops.WGRAD_TC, tuple(m.activation for m in acts),
                tuple(m.momentum_at(epoch) for m in bns),
                tuple((g["lr"], g["betas"], g["eps"], g["weight_decay"])
                      for o in self._optim for g in o.param_groups),
                tuple(p.requires_grad for p in params), tuple(p.data_ptr() for p in params),
                tuple(t.data_ptr() for t in s.t.values()), tuple(id(o.state) for o in self._optim),
                self.opt.dropout)

    def _make_capturable(self, flag=True):
        """Adam's capturable mode: `step` lives on the parameter's device (as load_state_dict
        places it for a capturable group) and the update reads no host value. flag=False: the
        ordinary mode, `step` a host scalar as Adam creates it."""
        for o in self._optim:
            if all(g.get("capturable", False) == flag for g in o.param_groups):
                continue
            o.defaults["capturable"] = flag
            for g in o.param_groups:
                g["capturable"] = flag
            for p, st in o.state.items():
                if "step" in st:
                    st["step"] = st["step"].to(dtype=torch.float32,
                                               device=p.device if flag else "cpu")

    def _optimize_graph(self, epoch):
        self._make_capturable()
        s = self._sets[self._cur]
        cur = torch.cuda.current_stream(self._dev)
        cur.wait_event(s.ready)
        key = self._train_key(s, epoch)
        g = self._train_graphs.get(self._cur)
        gs = self._graph_stream
        if g is None or g["key"] != key:
            # a new key: this step runs eagerly on the capture stream, so that every host-side
            # cache, per-stream library workspace and the optimizers' state exist before capture
            self._train_graphs.pop(self._cur, None)
            gs.wait_stream(cur)
            with torch.cuda.stream(gs):
                self._train_step(epoch, self._forward)
            cur.wait_stream(gs)
            self._train_graphs[self._cur] = dict(key=key, graph=None)
            s.consumed.record(cur)
            return
        if g["graph"] is None:
            graph = torch.cuda.CUDAGraph()
            pre = self._snapshot()
            k0, c0 = ops.KERNEL_LAUNCHES, ops.LAUNCHES
            gs.wait_stream(cur)
            with torch.cuda.graph(graph, stream=gs):
                self._train_step(epoch, self._forward)
            # the captured calls are counted when the graph replays
            g.update(graph=graph, kernels=ops.KERNEL_LAUNCHES - k0, calls=ops.LAUNCHES - c0)
            ops.KERNEL_LAUNCHES, ops.LAUNCHES = k0, c0
            # re-bind what the step assigns (the segmenter's step leaves `loss` alone); an
            # attribute left None stays None after a replay, as after an eager step
            g["snap"] = {path: {n: v for n, v in vals.items() if v is None or v is not pre[path].get(n)}
                         for path, vals in self._snapshot().items()}
            g["grads"] = [(p, p.grad) for p in self._train_state()[0]]
            # the graph reads and writes these: a later step must not free them under it
            g["keep"] = (train_ops.scratch_buffers(), [o.state for o in self._optim])
        g["graph"].replay()
        ops.KERNEL_LAUNCHES += g["kernels"]
        ops.LAUNCHES += g["calls"]
        self._rebind(g["snap"])
        for m in self._state_modules():
            m.train()
        for p, grad in g["grads"]:
            if p.grad is not grad:
                p.grad = grad
        # the replay updated parameters and running statistics in place, unseen by autograd
        params, bufs, _, _ = self._train_state()
        torch.autograd.graph.increment_version(params + bufs)
        s.consumed.record(cur)


ENCODER_SNAPSHOT = ("som_node", "first_pn_out_masked_max", "knn_center_1", "knn_feature_1",
                    "final_pn_out", "feature", "_assign", "_lazy_src",
                    "_mask", "_centers", "_x_aug", "_first_pn_out")
