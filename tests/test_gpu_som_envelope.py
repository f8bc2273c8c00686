"""-m gpu: the SOM kernels across the library's whole node-count envelope (M = 1 .. 256, k = 1 .. 4;
node_knn up to 4096 nodes), at the shapes where their code paths change, against plain
high-precision references:

  som_train       vs the exact-sum numpy emulation of tests/som_emu.py, bit for bit (see there
                  why bit equality is the expected result), and vs the reference's own BatchSOM
                  fixtures at 3x3, 11x11 and 16x16 grids;
  query_topk / som_mask / som_assign / som_group_decenter / som_sort_decenter / pool_finalize /
  node_knn        vs the oracle's C restatement, one-hot / fp64 references and property checks."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import som_emu
from helpers import assert_close, golden

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


# ---- fixtures and references -----------------------------------------------------------------------
def _grid(M):
    """rows x cols of a BatchSOM with M nodes (rows the largest divisor <= sqrt(M))."""
    r = int(np.sqrt(M))
    while M % r:
        r -= 1
    return r, M // r


def _som(M, B=1):
    from sonet_b200 import som
    r, c = _grid(M)
    return som.BatchSOM(r, c, 3, 0, B)


def _W(s, sigma):
    M = s.node_num
    return s.get_weighting_matrix(sigma).view(1, M, M).contiguous()


def _cloud(rs, B, N, scale=1.0):
    from oracle.make_golden import som_cloud
    return som_cloud(rs, B, N) * np.float32(scale)


def _train_limits(M):
    """(N_x, N_max) of sonet_som_train on this device: the largest N whose cloud is resident in
    shared memory, and the largest N it accepts — the launcher's byte formula (csrc/som_train.cu)
    against the opt-in shared memory per block."""
    cap = torch.cuda.get_device_properties(DEV).shared_memory_per_block_optin
    w = 4 * M * M if 4 * M * M <= 64 * 1024 else 0
    fixed = 16 * M + 4 * 4 * M + 8 * 3 * ((M + 1) // 2) + w
    return (cap - fixed - 16) // 13, cap - fixed - 16


def _train(x, node0, W, lr, want_idx=True):
    from sonet_b200 import ops
    return ops.som_train(torch.from_numpy(np.ascontiguousarray(x)).to(DEV),
                         torch.from_numpy(np.ascontiguousarray(node0)).to(DEV),
                         W.to(DEV), lr.to(DEV), want_idx=want_idx)


def _assert_train_exact(x, node0, W, lr, what):
    """Kernel vs emulation: nodes and the last assignment bit for bit."""
    node, idx = _train(x, node0, W, lr)
    margin = som_emu.Margin()
    want, want_idx = som_emu.train(x, node0, W.numpy(), lr.numpy(), margin)
    got = node.cpu().numpy()
    ulp = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64)).max()
    assert np.array_equal(idx.cpu().numpy(), want_idx), "%s: assignment differs (%r)" % (what, margin)
    assert np.array_equal(got, want), "%s: nodes differ by up to %d ulp (%r)" % (what, ulp, margin)
    return got, idx


# ---- som_train: one step across the envelope -----------------------------------------------------
TRAIN_M = [1, 2, 9, 25, 64, 121, 128, 129, 144, 256]
TRAIN_N = ["resident", "resident+1", "n%4=1", "n%4=2", "n%4=3", "n<4", "n<M"]


def _train_n(M, kind):
    n_x, _ = _train_limits(M)
    return {"resident": n_x, "resident+1": n_x + 1, "n%4=1": 1001, "n%4=2": 1002, "n%4=3": 1003,
            "n<4": 3, "n<M": max(1, M // 3)}[kind]


@pytest.mark.parametrize("kind", TRAIN_N)
@pytest.mark.parametrize("M", TRAIN_M)
def test_som_train_one_step_bit_exact(M, kind):
    """Odd M (packed node pairs, the duplicate skipped); W in shared memory up to M = 128 and read
    from global memory from 129; the cloud resident in shared memory up to N_x points and read
    from global memory at N_x + 1; the N % 4 tail of the per-node scan; mostly empty nodes; node
    id 255 in the uint8 assignment table and 768 update threads at M = 256. Both node_init forms:
    [3,M] shared by the clouds, and [B,3,M] with a different start per cloud."""
    N = _train_n(M, kind)
    B = 1 if kind.startswith("resident") else 2
    rs = np.random.RandomState(M * 7 + N)
    x = _cloud(rs, B, N)
    node0 = rs.uniform(-0.8, 0.8, size=(3, M)).astype(np.float32)
    s = _som(M)
    W, lr = _W(s, 0.3), torch.tensor([0.5])
    _assert_train_exact(x, node0, W, lr, "M=%d N=%d shared start" % (M, N))
    nodeb = np.stack([node0 + np.float32(0.05) * b for b in range(B)]).astype(np.float32)
    _assert_train_exact(x, nodeb, W, lr, "M=%d N=%d batched start" % (M, N))


@pytest.mark.parametrize("M", [9, 25, 64, 121])
def test_som_train_sparse_update_sums_round_once(M):
    """Clouds of 3 .. 7 points: each node update sums a few comparable terms, which often add up
    exactly to an fp32 midpoint, plus Gaussian-tail terms (W down to ~1e-21) that decide the
    side. An fp64 running sum drops those tails and rounds the midpoint to even; the kernel
    carries the sum exactly (TwoSum) and rounds once, as the emulation does. (Before it did,
    about one node coordinate in 5000 of such clouds was one ulp off.)"""
    s = _som(M)
    W, lr = _W(s, 0.3), torch.tensor([0.5])
    for seed in range(8):
        rs = np.random.RandomState(seed)
        N = 3 + seed % 5
        x = _cloud(rs, 8, N)
        node0 = rs.uniform(-0.8, 0.8, size=(3, M)).astype(np.float32)
        _assert_train_exact(x, node0, W, lr, "M=%d N=%d seed %d" % (M, N, seed))


# ---- som_train: adversarial inputs ------------------------------------------------------------------
def _lattice(side, step=0.25, z=False):
    """Nodes on an exactly representable grid: [3, side*side] (z = 0), or [3, side^3] with z."""
    a = (np.arange(side) - (side - 1) / 2.0) * step
    if z:
        g = np.stack(np.meshgrid(a, a, a, indexing="ij"), 0).reshape(3, -1)
    else:
        g = np.stack(np.meshgrid(a, a, indexing="ij"), 0).reshape(2, -1)
        g = np.concatenate([g, np.zeros((1, g.shape[1]))], 0)
    return g.astype(np.float32)


def test_som_train_ties_duplicates_and_points_on_nodes():
    """Duplicate nodes, points equidistant from two or four nodes and points exactly on a node:
    every tie goes to the lowest node index (torch.min's first minimum), so the higher duplicate
    of a pair never receives a point."""
    M = 25
    node0 = _lattice(5)
    dup = [(3, 1), (20, 12), (24, 0)]
    for hi, lo in dup:
        node0[:, hi] = node0[:, lo]
    rs = np.random.RandomState(11)
    on = node0[:, rs.randint(0, M, size=300)]                       # exactly on nodes
    mid = (node0[:, :-1] + node0[:, 1:]) / 2                        # between neighbours
    cell = node0[:, :M - 6] + np.float32(0.125) * np.array([[1], [1], [0]], np.float32)
    x = np.concatenate([on, mid, cell, rs.uniform(-0.6, 0.6, size=(3, 401)).astype(np.float32)], 1)
    x = np.stack([x, x[:, ::-1]]).astype(np.float32)                # B = 2, N % 4 = 1
    s = _som(M)
    _, idx = _assert_train_exact(x, node0, _W(s, 0.4), torch.tensor([0.5]), "ties")
    idx = idx.cpu().numpy()
    for hi, lo in dup:
        assert not (idx == hi).any(), "a point went to the higher duplicate %d of %d" % (hi, lo)
    d = som_emu.distances(x, np.broadcast_to(node0, (2, 3, M)))
    assert (d.min(axis=2) == 0).sum() >= 600                       # the on-node points are exact
    ties = (d == d.min(axis=2, keepdims=True)).sum(axis=2) > 1
    assert ties.sum() > 300                                         # many exact ties exercised


def test_som_train_large_offset_rounding_decides():
    """Coordinates offset by 1e3: the distances are dominated by float32 rounding of (x - n)^2, so
    the assignment is decided by exactly the kernel's rounding order."""
    M = 64
    rs = np.random.RandomState(12)
    x = _cloud(rs, 2, 2001, 0.002) + np.float32(1000.0)      # ~30 float32 steps per axis
    node0 = (rs.uniform(-0.002, 0.002, size=(3, M)) + 1000.0).astype(np.float32)
    margin = som_emu.Margin()
    som_emu.train(x, node0, [], [], margin)
    assert margin.gap == 0.0                                        # rounding creates exact ties
    s = _som(M)
    _assert_train_exact(x, node0, _W(s, 0.4), torch.tensor([0.5]), "offset 1e3")


def test_som_train_asymmetric_weights():
    """An asymmetric W straight into ops.som_train: delta[j] = sum_m (...)[m] * W[m][j] * lr. The
    Gaussian W is symmetric, so only this pins the W[m][j] convention (node m's mean pulls node j
    with weight W[m][j])."""
    rs = np.random.RandomState(13)
    for M in (9, 121, 256):                       # W in shared memory, in shared memory, in global
        W = torch.from_numpy(rs.uniform(0, 1, size=(2, M, M)).astype(np.float32))
        W[:, 0, :] = 0.0                          # node 0's mean pulls nobody ...
        W[:, :, 1] *= 3.0                         # ... node 1 is pulled harder by every mean
        assert not torch.equal(W[0], W[0].t())
        x = _cloud(rs, 2, 1500)
        node0 = rs.uniform(-0.7, 0.7, size=(3, M)).astype(np.float32)
        _assert_train_exact(x, node0, W, torch.tensor([0.3, 0.2]), "asymmetric W, M=%d" % M)


@pytest.mark.parametrize("M,N", [(9, 1003), (256, 5), (121, 20000)])
def test_som_train_zero_iterations(M, N):
    """T = 0: the nodes pass through unchanged and the last assignment is the assignment against
    the initial nodes (the arithmetic of iteration 1), for both node_init forms."""
    rs = np.random.RandomState(M + N)
    x = _cloud(rs, 2, N)
    node0 = rs.uniform(-0.8, 0.8, size=(3, M)).astype(np.float32)
    W, lr = torch.zeros(0, M, M), torch.zeros(0)
    for start in (node0, np.stack([node0, node0[:, ::-1]]).astype(np.float32)):
        node, idx = _train(x, start, W, lr)
        assert np.array_equal(node.cpu().numpy(), np.broadcast_to(start, (2, 3, M)))
        want_node, want_idx = som_emu.train(x, start, [], [])
        assert np.array_equal(idx.cpu().numpy(), want_idx)
        assert idx.dtype == torch.int32 and int(idx.min()) >= 0 and int(idx.max()) < M
    assert not (want_idx == 0).all()


# ---- som_train: BatchSOM.optimize at 3x3, 11x11 and 16x16 ---------------------------------------
def _oracle_trajectory(oracle_mod, g, r, sched):
    """The reference's node after every step (oracle.som_batch_update is pinned bit for bit to the
    reference by oracle/make_golden.py)."""
    init_w = oracle_mod.som_init_weighting_matrix(r, r)
    x = torch.from_numpy(g["x"])
    node = torch.from_numpy(g["node_init_value"]).unsqueeze(0).expand(x.shape[0], -1, -1).contiguous()
    out = []
    for lr, sigma in sched:
        node, _ = oracle_mod.som_batch_update(node, x, init_w, lr, sigma)
        out.append(node.numpy())
    return out


@pytest.mark.parametrize("name,r", [("som_train_m9", 3), ("som_train_m121", 11),
                                    ("som_train_m256", 16)])
def test_som_optimize_vs_emulation_and_reference_golden(oracle_mod, name, r):
    """The 80-iteration schedule of BatchSOM.optimize: bit-exact against the emulation iterated
    80 times; within 1e-4 of the reference's own optimize() (two single batch_update steps within
    1e-6); independent of the batch composition. On a golden mismatch the message names the
    first iteration and point whose assignment flips, and its distance gap."""
    from sonet_b200 import ops
    g = golden(name)
    x = torch.from_numpy(g["x"]).to(DEV)
    B, M = x.shape[0], r * r
    s = _som(M, B)
    s.node_init(B)
    assert np.array_equal(s.node[0].cpu().numpy(), g["node_init_value"])
    s.batch_update(x, 0.5, 0.4)
    assert_close(s.node, g["node_after_1"], "batch_update 1", 1e-6)
    s.batch_update(x, 0.31, 0.22)
    assert_close(s.node, g["node_after_2"], "batch_update 2", 1e-6)
    s.optimize(x)
    full = s.node.clone()
    W, lr = s._schedule
    assert W.shape == (80, M, M)
    node, idx = ops.som_train(x, s.node_init_value.to(DEV), W, lr, want_idx=True)
    assert torch.equal(node, full)
    margin = som_emu.Margin()
    want, want_idx = som_emu.train(g["x"], g["node_init_value"], W.cpu().numpy(), lr.cpu().numpy(),
                                   margin)
    got = full.cpu().numpy()
    ulp = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64)).max()
    print("%s: max ulp kernel vs emulation %d, %r" % (name, ulp, margin))
    assert np.array_equal(idx.cpu().numpy(), want_idx)
    assert ulp == 0
    err = np.abs(got - g["node_optimized"]).max()
    print("%s: max |kernel - reference| %.3g" % (name, err))
    if err > 1e-4 * max(1.0, float(np.abs(g["node_optimized"]).max())):
        traj = _oracle_trajectory(oracle_mod, g, r, _schedule(s))
        flip = som_emu.first_divergence(g["x"], g["node_init_value"], W.cpu().numpy(),
                                        lr.cpu().numpy(), traj)
        pytest.fail("%s: kernel vs reference %.3g; first assignment flip (iteration, cloud, point, "
                    "gap): %s" % (name, err, flip))
    # shard invariance
    s.optimize(x[1:].contiguous())
    assert torch.equal(s.node, full[1:])


def _schedule(s):
    """BatchSOM.optimize's (learning rate, sigma) list."""
    sched = [(s.learning_rate, s.sigma)] * int(s.max_iteration / 3)
    for it in range(s.max_iteration):
        sched.append((s.learning_rate / (1 + 2 * it / s.max_iteration),
                      s.sigma / (1 + 2 * it / s.max_iteration)))
    return sched


# ---- query_topk: every mask-store variant ----------------------------------------------------------
QT_M = [1, 4, 16, 32, 36, 64, 96, 100, 121, 128, 160, 256]


@pytest.mark.parametrize("k", [1, 2, 3, 4])
@pytest.mark.parametrize("M", QT_M)
def test_query_topk_mask_paths(oracle_mod, M, k):
    """M = 64 (16-byte stores), M % 32 == 0 (int2 stores at 64, scalar stores otherwise), and
    M % 32 != 0 (som_mask after the assignment); N not a multiple of 32, and N < 32."""
    from sonet_b200 import ops
    if k > M:
        pytest.skip("k <= M")
    rs = np.random.RandomState(M * 5 + k)
    for N in (77, 19):
        x = torch.from_numpy(rs.uniform(-1, 1, size=(2, 3, N)).astype(np.float32))
        node = torch.from_numpy(rs.uniform(-1, 1, size=(2, 3, M)).astype(np.float32))
        mask, row_max, idx64, idx32 = ops.som_query_topk(x.to(DEV), node.to(DEV), k)
        want_idx, _ = oracle_mod.som_topk(x, node, k)
        assert torch.equal(idx32.cpu(), want_idx)
        assert torch.equal(idx64.cpu(), want_idx.long())
        assert torch.equal(mask.cpu(), F.one_hot(idx32.cpu().long(), M).int())
        _, want_row_max, _ = oracle_mod.query_topk(x, node, k)
        assert torch.equal(row_max.cpu(), want_row_max)


def _c_query_topk(x, node, k, mask_view):
    from sonet_b200 import _C
    B, _, N = x.shape
    M = node.shape[2]
    row_max = torch.empty((B, M), dtype=torch.int32, device=DEV)
    idx64 = torch.empty((B, k * N), dtype=torch.int64, device=DEV)
    idx32 = torch.empty((B, k * N), dtype=torch.int32, device=DEV)
    _C.check(_C.lib().sonet_som_query_topk(_C.ptr(x), _C.ptr(node), B, N, M, k, _C.ptr(mask_view),
                                           _C.ptr(row_max), _C.ptr(idx64), _C.ptr(idx32), None),
             "sonet_som_query_topk")
    return row_max, idx32


@pytest.mark.parametrize("M,off", [(64, 1), (64, 2), (64, 3), (128, 1), (36, 2), (121, 1)])
def test_query_topk_and_mask_misaligned(oracle_mod, M, off):
    """The alignment fallbacks, through the C-ABI with a mask pointer `off` ints into a larger
    buffer: at M = 64 an offset of 1 (or 3) int takes the som_mask fallback (and its scalar kernel),
    an offset of 2 ints (8- but not 16-byte aligned) the fused int2 store. The ints around the
    mask stay untouched."""
    from sonet_b200 import _C
    B, N, k = 2, 45, 3
    rs = np.random.RandomState(M + off)
    x = torch.from_numpy(rs.uniform(-1, 1, size=(B, 3, N)).astype(np.float32)).to(DEV)
    node = torch.from_numpy(rs.uniform(-1, 1, size=(B, 3, M)).astype(np.float32)).to(DEV)
    total = B * k * N * M
    buf = torch.full((total + 8,), 7, dtype=torch.int32, device=DEV)
    view = buf[off:off + total].view(B, k * N, M)
    row_max, idx32 = _c_query_topk(x, node, k, view)
    want_idx, _ = oracle_mod.som_topk(x.cpu(), node.cpu(), k)
    assert torch.equal(idx32.cpu(), want_idx)
    assert torch.equal(view.cpu(), F.one_hot(want_idx.long(), M).int())
    assert bool((buf[:off] == 7).all()) and bool((buf[off + total:] == 7).all())
    assert torch.equal(row_max.cpu(), oracle_mod.query_topk(x.cpu(), node.cpu(), k)[1])
    # sonet_som_mask on its own at the same offset (M % 4 != 0 or unaligned: the scalar kernel)
    buf.fill_(7)
    _C.check(_C.lib().sonet_som_mask(_C.ptr(idx32), B, k * N, M, _C.ptr(view), None), "sonet_som_mask")
    assert torch.equal(view.cpu(), F.one_hot(want_idx.long(), M).int())
    assert bool((buf[:off] == 7).all()) and bool((buf[off + total:] == 7).all())


@pytest.mark.parametrize("M", [9, 64, 121])
def test_batchsom_query_float_mask(oracle_mod, M):
    """BatchSOM.query (util/som.py:271-293): the k = 1 float one-hot mask and row max."""
    rs = np.random.RandomState(M)
    B, N = 2, 333
    x = torch.from_numpy(rs.uniform(-1, 1, size=(B, 3, N)).astype(np.float32))
    node = torch.from_numpy(rs.uniform(-1, 1, size=(B, 3, M)).astype(np.float32))
    s = _som(M, B)
    s.node = node.to(DEV)
    mask, row_max = s.query(x.to(DEV))
    assert mask.dtype == torch.float32 and mask.shape == (B, N, M)
    want_idx, _ = oracle_mod.som_topk(x, node, 1)
    want = F.one_hot(want_idx.long(), M).float()
    assert torch.equal(mask.cpu(), want)
    assert torch.equal(row_max.cpu(), want.max(dim=1)[0])


# ---- som_assign at k = 4 and large M, with exact ties -------------------------------------------------
def _tie_cloud(node, rs, N):
    """Points on nodes, halfway between grid neighbours and at cell centres (exact 2- and 4-way
    distance ties on a lattice), plus random points; [1, 3, N]."""
    M = node.shape[1]
    on = node[:, rs.randint(0, M, size=N // 4)]
    mid = (node[:, rs.randint(0, M - 1, size=N // 4)] + np.float32(0.125) *
           np.array([[1], [0], [0]], np.float32))
    cell = (node[:, rs.randint(0, M, size=N // 4)] + np.float32(0.125) *
            np.array([[1], [1], [0]], np.float32))
    rnd = rs.uniform(-2, 2, size=(3, N - 3 * (N // 4))).astype(np.float32)
    return np.concatenate([on, mid, cell, rnd], 1)[None].astype(np.float32)


@pytest.mark.parametrize("M", [121, 256])
def test_som_assign_k4_ties(oracle_mod, M):
    from sonet_b200 import ops
    side = int(round(np.sqrt(M)))
    rs = np.random.RandomState(M)
    node = _lattice(side)[None]
    x = _tie_cloud(node[0], rs, 3001)
    x = np.concatenate([x, x[:, :, ::-1]]).astype(np.float32)
    node = np.concatenate([node, node[:, :, ::-1]]).astype(np.float32)        # B = 2
    xt, nt = torch.from_numpy(x), torch.from_numpy(node)
    a = ops.som_assign(xt.to(DEV), nt.to(DEV), 4, want_i64=True)
    want_idx, _ = oracle_mod.som_topk(xt, nt, 4)
    assert torch.equal(a["min_idx_i32"].cpu(), want_idx)                    # indices + slot order
    assert torch.equal(a["min_idx_i64"].cpu(), want_idx.long())
    cnt = torch.stack([torch.bincount(want_idx[b].long(), minlength=M) for b in range(2)])
    assert torch.equal(a["count"].cpu().long(), cnt)
    assert torch.equal(a["row_max"].cpu().long(), (cnt > 0).long())
    # cluster_mean: within fp32 summation error of the fp64 mean
    N = x.shape[2]
    xs = np.concatenate([x] * 4, axis=2).astype(np.float64)                  # stacked copies
    idx = want_idx.numpy()
    c = cnt.numpy().astype(np.float64)
    den = (c.astype(np.float32) + np.float32(1e-5)).astype(np.float64)
    got = a["cluster_mean"].cpu().numpy().astype(np.float64)
    for b in range(2):
        for ch in range(3):
            s64 = np.bincount(idx[b], weights=xs[b, ch], minlength=M)
            a64 = np.bincount(idx[b], weights=np.abs(xs[b, ch]), minlength=M)
            want = s64 / den[b]
            bar = ((c[b] + 2) * a64 / den[b] + np.abs(want)) * 2.0 ** -24
            assert (np.abs(got[b, ch] - want) <= bar).all(), (b, ch)
    d = som_emu.distances(x, node)
    srt = np.sort(d, axis=2)
    assert (srt[:, :, :5][:, :, 1:] == srt[:, :, :5][:, :, :-1]).any(axis=2).sum() > N // 2


def test_som_assign_nan_point_stays_in_range():
    """A NaN point compares false against every distance, so every node is a NaN one and its k
    slots take nodes 0..k-1 in index order: in range for everything downstream."""
    from sonet_b200 import ops
    M, k, N = 121, 4, 200
    rs = np.random.RandomState(5)
    x = rs.uniform(-1, 1, size=(1, 3, N)).astype(np.float32)
    x[0, :, 17] = np.nan
    x[0, 1, 40] = np.nan
    node = torch.from_numpy(_lattice(11)[None])
    a = ops.som_assign(torch.from_numpy(x).to(DEV), node.to(DEV), k)
    idx = a["min_idx_i32"].cpu().view(k, N)
    for n in (17, 40):
        assert idx[:, n].tolist() == list(range(k))
    assert int(idx.min()) >= 0 and int(idx.max()) < M
    assert int(a["count"].sum()) == k * N


# ---- som_group_decenter / som_sort_decenter at M in {121, 256}, k = 4 --------------------------------
def _group_limit_staged(M, k, with_sn):
    from sonet_b200 import ops
    lo, hi = 1, 1 << 20
    assert ops.som_group_mode(lo, M, k, with_sn, DEV) == ops.SOM_GROUP_STAGED
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if ops.som_group_mode(mid, M, k, with_sn, DEV) == ops.SOM_GROUP_STAGED \
            else (lo, mid)
    return lo


@pytest.mark.parametrize("M", [121, 256])
@pytest.mark.parametrize("use_sn", [True, False])
@pytest.mark.parametrize("where", ["staged", "staged+1", "cached", "cached+1"])
def test_som_group_and_sort_decenter_k4(M, use_sn, where):
    """k = 4: the cached (k*N <= 16384) and uncached node-id passes, staged and unstaged, with and
    without normals. som_group_decenter as test_som_group_decenter_matches_two_kernel_path checks
    it; som_sort_decenter (arbitrary order inside a node) by properties. (At k = 4 and these M
    the staging limit lies above N = 4096, so a cached launch is always staged.)"""
    from sonet_b200 import ops
    k = 4
    n_s = _group_limit_staged(M, k, use_sn)
    N = {"staged": n_s, "staged+1": n_s + 1, "cached": 4096, "cached+1": 4097}[where]
    mode = ops.som_group_mode(N, M, k, use_sn, DEV)
    assert mode != ops.SOM_GROUP_NONE
    assert (mode == ops.SOM_GROUP_STAGED) == (N <= n_s)
    assert (where == "staged+1") == (mode == ops.SOM_GROUP_UNSTAGED)
    print("M=%d sn=%s N=%d: %s, %s" % (M, use_sn, N, "staged" if mode == ops.SOM_GROUP_STAGED
                                       else "unstaged", "cached" if k * N <= 16384 else "uncached"))
    rs = np.random.RandomState(M + N)
    B = 2
    x = torch.from_numpy(rs.uniform(-1.2, 1.2, size=(B, 3, N)).astype(np.float32)).to(DEV)
    sn = torch.from_numpy(rs.normal(size=(B, 3, N)).astype(np.float32)).to(DEV) if use_sn else None
    side = int(round(np.sqrt(M)))
    node = torch.from_numpy(_lattice(side, step=2.0 / side)[None].repeat(B, 0)).to(DEV)
    node[1, :, 3:9] += 40.0                                          # empty nodes
    a = ops.som_assign(x, node, k)
    idx = a["min_idx_i32"]
    xs, ns, p0, count, cmean = ops.som_group_decenter(x, sn, idx, M, k)
    again = ops.som_group_decenter(x, sn, idx, M, k)
    for u, v in zip((xs, ns, p0, count, cmean), again):
        assert torch.equal(u, v)
    assert torch.equal(count, a["count"])
    assert_close(cmean, a["cluster_mean"], "cluster_mean", tol=1e-5)
    order = torch.argsort(idx.long(), dim=1, stable=True)
    assert torch.equal(ns.long(), torch.gather(idx.long(), 1, order))
    n_of = order % N
    x_g = torch.gather(x, 2, n_of.unsqueeze(1).expand(-1, 3, -1))
    ctr = torch.gather(cmean, 2, ns.long().unsqueeze(1).expand(-1, 3, -1))
    assert torch.equal(xs[:, 0:3], x_g - ctr)
    if use_sn:
        assert torch.equal(xs[:, 3:6], torch.gather(sn, 2, n_of.unsqueeze(1).expand(-1, 3, -1)))
    assert torch.equal(p0.long(), (order == 0).long().argmax(dim=1))

    # som_sort_decenter on the assignment's own statistics
    cm2 = a["cluster_mean"]
    xs2, ns2, p02 = ops.som_sort_decenter(x, sn, cm2, idx, a["count"], k)
    assert bool((ns2[:, 1:] >= ns2[:, :-1]).all())                          # grouped by node
    assert torch.equal(ns2, ns)                                              # same node runs
    xst = torch.cat([x] * k, dim=2)
    snt = torch.cat([sn] * k, dim=2) if use_sn else None
    for b in range(B):
        # each row is (x - cluster_mean[node]) of one stacked copy of that node, exactly
        rows = xs2[b]
        want = torch.cat([xst[b] - torch.gather(cm2[b], 1, idx[b].long().unsqueeze(0).expand(3, -1))]
                         + ([snt[b]] if use_sn else []), 0)
        want_sorted = want[:, order[b]]                                      # stable-sort reference
        for m in torch.unique(ns2[b]).tolist():
            sel = (ns2[b] == m).nonzero().squeeze(1)
            lo, hi = int(sel[0]), int(sel[-1]) + 1
            got_rows = rows[:, lo:hi].t().contiguous()
            want_rows = want_sorted[:, lo:hi].t().contiguous()
            assert torch.equal(_sort_rows(got_rows), _sort_rows(want_rows)), (b, m)
        # pos0: the sorted position of stacked copy 0 holds copy 0's row
        assert int(ns2[b, p02[b]]) == int(idx[b, 0])
        assert torch.equal(rows[:, p02[b]], want[:, 0])


def _sort_rows(t):
    """Rows of t [R, C] in lexicographic order (a canonical form of a multiset of rows)."""
    for c in reversed(range(t.shape[1])):
        t = t[torch.argsort(t[:, c], stable=True)]
    return t


# ---- pool_finalize: the scalar kernel -------------------------------------------------------------
@pytest.mark.parametrize("M", [1, 121, 64])
def test_pool_finalize_semantics(M):
    """Ordered-int keys -> values: a never-written key (INT_MIN) and a value <= -1000 give the
    copy-0 feature p0; the keys are reset to INT_MIN. M in {1, 121} runs the scalar kernel, M = 64
    the vector kernel with the same semantics."""
    from sonet_b200 import ops
    B, C = 3, 37
    g = torch.Generator().manual_seed(M)
    vals = torch.randn(B, C, M, generator=g) * 3
    vals[0, :, 0] = -2000.0
    vals[2, 5, -1] = -1000.0
    bits = vals.view(torch.int32)
    keys = (bits ^ ((bits >> 31) & 0x7fffffff))
    keys[1, :, M // 2] = -2 ** 31
    keys[2, 3, 0] = -2 ** 31
    p0 = torch.randn(B, C, generator=g)
    kd = keys.to(DEV)
    out = ops.pool_finalize(kd, p0.to(DEV)).cpu()
    written = keys != -2 ** 31
    want = torch.where(written & (vals > -1000.0), vals, p0.unsqueeze(2).expand(-1, -1, M))
    assert torch.equal(out, want)
    assert bool((kd == -2 ** 31).all())


# ---- node_knn ---------------------------------------------------------------------------------------
def _knn_nodes(M):
    if M == 4096:
        return _lattice(16, z=True)
    side = int(round(np.sqrt(M)))
    return _lattice(side)


@pytest.mark.parametrize("M,K", [(1, 1), (9, 1), (9, 9), (121, 1), (121, 9), (121, 121),
                                 (256, 1), (256, 9), (256, 256), (4096, 1), (4096, 7),
                                 (4096, 9)])
def test_node_knn_ties(oracle_mod, M, K):
    """Grid nodes, so most neighbour distances tie exactly: the result is the (distance, index)
    order — the documented rule — bit for bit against a float32 emulation; against the
    reference's topk (tie order unspecified) as sets wherever no tie straddles position K."""
    from sonet_b200 import ops
    c = _knn_nodes(M)
    coord = np.stack([c, c[:, ::-1]] if M < 4096 else [c]).astype(np.float32)
    B = coord.shape[0]
    got = ops.node_knn(torch.from_numpy(coord).to(DEV), K).cpu().numpy()
    assert got.shape == (B, M, K)
    dx, dy, dz = (coord[:, i, :, None] - coord[:, i, None, :] for i in range(3))   # [B,m,q]
    d = (dx * dx + dy * dy) + dz * dz
    order = np.argsort(d, axis=2, kind="stable")[:, :, :K]                 # ties: lower index
    assert np.array_equal(got, order)
    if M > 1:
        assert (np.sort(d, axis=2)[:, :, 1:] == np.sort(d, axis=2)[:, :, :-1]).any()
    ref = oracle_mod.node_knn(torch.from_numpy(coord), K).numpy()
    ds = np.sort(d, axis=2)
    clean = np.ones(d.shape[:2], bool) if K == M else ds[:, :, K - 1] != ds[:, :, K]
    # (on the 16^3 lattice every node's 9th neighbour sits inside a 12-way tie: nothing to compare)
    assert clean.any() or (M, K) == (4096, 9)
    assert np.array_equal(np.sort(got, axis=2)[clean], np.sort(ref, axis=2)[clean])
