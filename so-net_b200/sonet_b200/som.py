"""BatchSOM — util/som.py:176-366 on the sm_90a kernels: the node buffer, query_topk / query
(the assignment half the per-batch forward uses) and batch-SOM training (batch_update /
optimize, SURVEY.md §8f-4) as ONE kernel launch for all iterations of all clouds
(csrc/som_train.cu). The potential-field node initialisation (util/potential_field.py) is
host-side numpy, as in the reference, computed once per (node_num, dim) and cached.
"""
import itertools
import math

import numpy as np
import torch

from . import ops

_PF_CACHE = {}


def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _fma_sq(a, c):
    """RN(a*a + c), one rounding, for float64 arrays with c >= 0: the exact square (Dekker's
    product), the exact sum with c, and the low parts folded in with round-to-odd so that the last
    addition rounds once (Boldo & Melquiond: no cancellation, the high part dominates)."""
    p = a * a
    t = a * 134217729.0                                    # Veltkamp split, 2^27 + 1
    ah = t - (t - a)
    al = a - ah
    e = ((ah * ah - p) + 2.0 * ah * al) + al * al          # a*a = p + e exactly
    s, ts = _two_sum(p, c)
    w, werr = _two_sum(ts, e)
    odd = (w.view(np.int64) & 1) == 1
    w = np.where((werr != 0) & ~odd, np.nextafter(w, np.where(werr > 0, np.inf, -np.inf)), w)
    return s + w


def _row_norm(f):
    """np.linalg.norm of every row of f [n, dim] (dim < 16), bit for bit: for a 1-D float64
    vector it is sqrt(x.dot(x)), and a dot that short is BLAS ddot's scalar tail, an FMA chain
    dot = fma(x[i], x[i], dot). A plain ((x*x + y*y) + z*z) differs in the last bit for about 10 %
    of 3-vectors, and the potential field amplifies that: at 121 nodes its output moved by 5e-5,
    at 256 nodes it converged to a different arrangement."""
    acc = f[:, 0] * f[:, 0]
    for i in range(1, f.shape[1]):
        acc = _fma_sq(f[:, i], acc)
    return np.sqrt(acc)


def potential_field_nodes(node_num, dim=3):
    """Initial SOM nodes [node_num, dim] float64: PotentialField(node_num, dim).optimize()
    (util/potential_field.py:11-87) — 100 Jacobi steps of pairwise repulsion + wall attraction
    from the seed-2017 uniform start, then the row-major grid reorder. Vectorised over the
    destination node; the source loop keeps the reference's accumulation order (wall force first,
    then sources k = 0..n-1) and its scalar arithmetic (the norm of _row_norm; f_norm ** 2 of a
    numpy scalar is libm's pow(), which differs from the rounded product for about 0.1 % of the
    inputs), so the trajectory is the reference's bit for bit."""
    key = (node_num, dim)
    if key in _PF_CACHE:
        return _PF_CACHE[key].copy()
    rs = np.random.RandomState(2017)                       # potential_field.py:15-17
    node = rs.rand(node_num, dim) * 2 - 1
    lr = 0.01
    for _ in range(100):                                   # :55-70
        wall = np.where(np.abs(node) < 0.01, 0.0, -1 * node * node_num / 1.5)   # :29-41
        force = np.zeros((node_num, dim)) + wall
        f = node[:, None, :] - node[None, :, :]            # [dst, src k]: force from k (:22-27)
        f_norm = _row_norm(f.reshape(-1, dim)) + 0.00001
        sq = np.fromiter(map(math.pow, f_norm.tolist(), itertools.repeat(2.0)), np.float64,
                         count=f_norm.size)
        contrib = (f.reshape(-1, dim) / f_norm[:, None] / sq[:, None]).reshape(f.shape)
        for k in range(node_num):
            force += contrib[:, k]
        node = node + force * lr
    # reorder (:72-87): sort by x, cut into rows, sort each row by y
    node = node[node[:, 0].argsort()]
    rows = int(math.sqrt(node_num))
    grid = node.reshape((rows, rows, dim))
    for i in range(rows):
        grid[i] = grid[i][grid[i][:, 1].argsort()]
    node = grid.reshape((node_num, dim))
    _PF_CACHE[key] = node.copy()
    return node


class BatchSOM():
    def __init__(self, rows=4, cols=4, dim=3, gpu_id=None, batch_size=10):
        self.rows = rows
        self.cols = cols
        self.dim = dim
        self.node_num = rows * cols

        self.sigma = 0.4                 # util/som.py:183-185
        self.learning_rate = 0.5
        self.max_iteration = 60

        self.gpu_id = gpu_id
        assert gpu_id is not None and gpu_id >= 0
        self.device = torch.device("cuda:%d" % gpu_id if torch.cuda.is_available() else "cpu")
        self.batch_size = batch_size
        # node: BxCx(rows*cols)
        self.node = torch.zeros(batch_size, dim, self.node_num, dtype=torch.float32,
                                device=self.device)
        self.node_idx_list = torch.arange(self.node_num, dtype=torch.int64, device=self.device)
        self.last_assignment = None  # dict from ops.som_assign for the most recent query
        self._init_w = None          # lazily built: only SOM training needs them
        self._node_init_value = None
        self._schedule = None

    # ---- training-side state (util/som.py:195-235), built on first use ---------------------------
    @property
    def init_weighting_matrix(self):
        """[node_num, rows, cols]: Gaussian of width self.sigma around every grid cell
        (util/som.py:214-229), computed with the reference's numpy expressions."""
        if self._init_w is None:
            d = 2 * np.pi * self.sigma * self.sigma
            w = torch.empty(self.node_num, self.rows, self.cols, dtype=torch.float32)
            for idx in range(self.node_num):
                i, j = self.idx2multi(idx)
                ax = np.exp(-np.power(np.arange(self.rows) - i, 2) / d)
                ay = np.exp(-np.power(np.arange(self.cols) - j, 2) / d)
                w[idx] = torch.from_numpy(np.outer(ax, ay).astype(np.float32))
            self._init_w = w             # kept on the host: schedules are tabulated there once
        return self._init_w

    @property
    def node_init_value(self):
        """[dim, node_num] float32 potential-field start (util/som.py:203-206)."""
        if self._node_init_value is None:
            pf = potential_field_nodes(self.node_num, self.dim)
            self._node_init_value = torch.from_numpy(pf.transpose().astype(np.float32)).contiguous()
        return self._node_init_value

    def node_init(self, batch_size):
        self.batch_size = batch_size
        self.node = self.node_init_value.to(self.device).unsqueeze(0).expand(
            batch_size, self.dim, self.node_num).contiguous()

    def idx2multi(self, i):
        return (i // self.cols, i % self.cols)

    def get_weighting_matrix(self, sigma):
        """util/som.py:231-235 (host tensor [node_num, rows, cols])."""
        scale = 1.0 / ((sigma / self.sigma) ** 2)
        return torch.exp(torch.log(self.init_weighting_matrix) * scale)

    def _weights_lr(self, schedule):
        """Tabulate (weights [T,M,M], lr [T]) on the device for a list of (learning_rate, sigma)."""
        W = torch.stack([self.get_weighting_matrix(sg).view(self.node_num, self.node_num)
                         for _, sg in schedule]).contiguous()
        lr = torch.tensor([l for l, _ in schedule], dtype=torch.float32)
        return W.to(self.device), lr.to(self.device)

    def batch_update(self, x, learning_rate, sigma):
        """One assign-and-update iteration on the current nodes (util/som.py:295-347)."""
        assert x.size()[1] == self.dim and x.size()[0] == self.batch_size
        W, lr = self._weights_lr([(learning_rate, sigma)])
        self.node = ops.som_train(x.detach().contiguous(), self.node.contiguous(), W, lr)

    def optimize(self, x):
        """util/som.py:352-366: potential-field start, max_iteration/3 iterations at the initial
        rate, then max_iteration iterations with decaying rate and neighbourhood width — all
        80 iterations of every cloud in ONE kernel launch."""
        if not x.is_cuda:
            raise RuntimeError("sonet_b200.BatchSOM.optimize runs on CUDA tensors only")
        self.batch_size = x.size()[0]
        if self._schedule is None:
            sched = [(self.learning_rate, self.sigma)] * int(self.max_iteration / 3)
            for it in range(self.max_iteration):
                sched.append((self.learning_rate / (1 + 2 * it / self.max_iteration),
                              self.sigma / (1 + 2 * it / self.max_iteration)))
            self._schedule = self._weights_lr(sched)
        W, lr = self._schedule
        self.node = ops.som_train(x.detach().contiguous(),
                                  self.node_init_value.to(x.device), W, lr)

    # ---- assignment (the per-batch forward) -------------------------------------------------------
    def query_topk(self, x, k):
        """x [B,3,N] -> (mask [B,kN,M] int32, mask_row_max [B,M] int32, min_idx [B,kN] int64),
        util/som.py:237-269. Slot order: ascending distance (the reference's is unspecified)."""
        node = self.node
        if node.shape[0] != x.shape[0]:
            node = node.expand(x.shape[0], node.shape[1], node.shape[2])
        mask, row_max, idx64, idx32 = ops.som_query_topk(x.detach().contiguous(), node.contiguous(), k)
        self.last_assignment = dict(min_idx_i32=idx32, min_idx_i64=idx64, row_max=row_max,
                                    count=None, cluster_mean=None)
        return mask, row_max, idx64

    def query(self, x):
        """k=1 variant (util/som.py:271-293): (mask [B,N,M] float, mask_row_max [B,M] float)."""
        M = self.rows * self.cols
        a = ops.som_assign(x.detach().contiguous(), self.node.contiguous(), 1, want_stats=False)
        self.last_assignment = a
        return ops.som_mask(a["min_idx_i32"], M).float(), a["row_max"].float()


class SOM():
    """The single-cloud SOM of util/som.py:17-173, the one data/build_som/save_som.ipynb trains per
    shape: node [dim, M], node_init(), query(x), batch_update(x, iteration) and optimize(x) for a
    cloud x [dim, N]. It is a BatchSOM with one cloud, so every call runs the sm_90a SOM kernels
    and optimize() equals BatchSOM.optimize of the same cloud bit for bit. The nodes live on
    cuda:gpu_id; gpu_id < 0 (the reference's CPU mode) or a bool (the notebook passes True) selects
    the current CUDA device, since there is no CPU path. Only dim = 3 has kernels."""

    def __init__(self, rows=4, cols=4, dim=3, gpu_id=-1):
        if dim != 3:
            raise RuntimeError("sonet_b200.SOM: dim=%d has no kernel (3 only)" % dim)
        if isinstance(gpu_id, bool) or gpu_id is None or gpu_id < 0:
            gpu_id = torch.cuda.current_device() if torch.cuda.is_available() else 0
        self._batch = BatchSOM(rows, cols, dim, gpu_id, 1)
        self.rows, self.cols, self.dim, self.node_num = rows, cols, dim, rows * cols
        self.sigma = self._batch.sigma
        self.learning_rate = self._batch.learning_rate
        self.max_iteration = self._batch.max_iteration
        self.gpu_id = gpu_id
        self.device = self._batch.device
        self.node_idx_list = torch.arange(self.node_num, dtype=torch.float32, device=self.device)
        self.node_init()

    @property
    def node(self):
        """[dim, M] float32 (a view of the one cloud's nodes)."""
        return self._batch.node[0]

    @property
    def node_init_value(self):
        return self._batch.node_init_value

    @property
    def init_weighting_matrix(self):
        return self._batch.init_weighting_matrix

    def node_init(self):
        self._batch.node_init(1)

    def get_weighting_matrix(self, sigma):
        return self._batch.get_weighting_matrix(sigma)

    def idx2multi(self, i):
        return self._batch.idx2multi(i)

    def _cloud(self, x):
        if x.dim() != 2 or x.size(0) != self.dim:
            raise RuntimeError("sonet_b200.SOM: x must be [%d, N], got %s" % (self.dim, tuple(x.shape)))
        return x.to(self.device, torch.float32).unsqueeze(0)

    def query(self, x):
        """util/som.py:78-100: (mask [N, M] float, mask_row_max [M] float)."""
        mask, row_max = self._batch.query(self._cloud(x))
        return mask[0], row_max[0]

    def batch_update(self, x, iteration):
        """One iteration at the rates of util/som.py:102-110."""
        decay = 1 + 2 * iteration / self.max_iteration
        self._batch.batch_size = 1
        self._batch.batch_update(self._cloud(x), self.learning_rate / decay, self.sigma / decay)

    def optimize(self, x):
        """util/som.py:168-173: potential-field start, max_iteration/3 iterations at the initial
        rates, then max_iteration decaying ones, in one kernel launch."""
        self._batch.optimize(self._cloud(x))
