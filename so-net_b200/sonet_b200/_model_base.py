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
"""
import torch

from . import layers, ops


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

    def invalidate(self):
        """Forget folded/packed weights and captured graphs (call after editing parameters
        through `.data`, which does not bump tensor versions — see layers.invalidate)."""
        for m in self._state_modules():
            layers.invalidate(m)
        self._graphs = {}

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
                snap = {}
                for path, names in self._SNAPSHOT.items():
                    obj = self._resolve(path)
                    snap[path] = {n: getattr(obj, n) for n in names if hasattr(obj, n)}
                g = dict(key=key, graph=graph, kernels=ops.KERNEL_LAUNCHES - k0,
                         calls=ops.LAUNCHES - c0, snap=snap)
                self._graphs[self._cur] = g
            g["graph"].replay()
        ops.KERNEL_LAUNCHES += g["kernels"]      # the replay launches the captured kernels
        ops.LAUNCHES += g["calls"]
        # cached attributes point at THIS graph's static buffers again (two input sets = two
        # graphs = two buffer sets); attributes that were still lazy (None) at capture time become
        # lazy again and are recomputed from the replayed buffers on demand
        for path, vals in g["snap"].items():
            obj = self._resolve(path)
            for n, v in vals.items():
                setattr(obj, n, v)
        s.consumed.record(cur)


ENCODER_SNAPSHOT = ("som_node", "first_pn_out_masked_max", "knn_center_1", "knn_feature_1",
                    "final_pn_out", "feature", "_assign", "_lazy_src",
                    "_mask", "_centers", "_x_aug", "_first_pn_out")
