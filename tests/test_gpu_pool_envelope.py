"""-m gpu: the per-node max pool on both of its routes, at every dispatch edge, at the -1000
sentinel and on non-finite values, against one plain reference of the rule.

The rule (the reference's index_max extension plus the masked gather of models/networks.py:181-185):
for every node, scan its points in ascending order with a strict `>` against a running maximum
that starts at float32(-1000); the node's feature is the value at the point that won, or the value
at point 0 (stacked copy 0) when no point beat the sentinel. pool_ref() below is that loop. It
defines the non-finite behaviour by construction: NaN never wins, +inf wins at its first
occurrence, -inf never wins.

Routes under test:
- sonet_index_max_f32 (csrc/index_max.cu): the TMA-staged vector path and the scalar path, the
  uint16_t / int32_t arg-max tables, the warp count per CTA. im_route() mirrors launch_index_max;
  one test checks that the case table reaches every branch and that each case launches the kernel,
  grid and block the mirror names.
- the fused route: the POOL variant of csrc/pointmlp_tc.cu, read back through sonet_pool_finalize
  and through sonet_knn_assemble_pool_f32. Its oracle is pool_ref() on the plain variant's output.
- train_ops.IndexMaxGather and sonet_index_max_backward_f32.

Everything here is selection, not arithmetic: results are compared bit for bit (int32 views, so
NaN payloads and signed zeros count). The one exception is the fp64 autograd check of the backward,
which states its bound.
"""
import contextlib
import json
import os
import re
import tempfile

import numpy as np
import pytest
import torch

DEV = "cuda:0"
gpu = pytest.mark.gpu
SENTINEL = np.float32(-1000.0)
INT_MIN = -2 ** 31
# the H100's limits, for the host-side check that the tables reach every branch
H100_SMS, H100_OPTIN = 132, 227 * 1024


# ---- 0. the reference rule ----------------------------------------------------------------------------
def pool_ref(data, index, K, point0=None):
    """data [B,C,N] f32, index [B,N] int (values in [0,K)) -> (idx int32 [B,C,K], val f32 [B,C,K]).
    point0 [B]: the point an unbeaten node falls back to (default 0, as index_max; the fused route
    passes pos0). N == 0: zeros, as sonet_index_max_f32 defines it."""
    data = np.ascontiguousarray(data, dtype=np.float32)
    index = np.asarray(index)
    B, C, N = data.shape
    idx = np.zeros((B, C, K), np.int32)
    val = np.zeros((B, C, K), np.float32)
    if N == 0:
        return idx, val
    for b in range(B):
        rows = np.ascontiguousarray(data[b].T)                  # [N,C]: one point's channels
        fall = 0 if point0 is None else int(point0[b])
        order = np.argsort(index[b], kind="stable")            # points of a node, ascending
        edge = np.searchsorted(index[b][order], np.arange(K + 1))
        for k in range(K):
            best = np.full(C, SENTINEL, np.float32)
            arg = np.full(C, fall, np.int64)
            for n in order[edge[k]:edge[k + 1]]:
                upd = rows[n] > best
                if upd.any():
                    best[upd] = rows[n][upd]
                    arg[upd] = n
            idx[b, :, k] = arg
            val[b, :, k] = rows[arg, np.arange(C)]
    return idx, val


def clamp_ids(index, K):
    """What the kernel reads an id as: min(uint32(id), K-1)."""
    return np.minimum(np.asarray(index).astype(np.int32).view(np.uint32), np.uint32(K - 1)).astype(np.int64)


def bits(t):
    if isinstance(t, np.ndarray):
        t = torch.from_numpy(np.ascontiguousarray(t))
    return t.detach().cpu().contiguous().view(torch.int32)


def assert_bits(got, want, what):
    g, w = bits(got), bits(want)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    assert torch.equal(g, w), "%s: %d of %d entries differ" % (what, int((g != w).sum()), g.numel())


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def offset_copy(t, off=1):
    """t's values in a contiguous view that starts `off` elements into a fresh buffer (4-byte
    aligned only)."""
    base = torch.zeros(t.numel() + off, dtype=t.dtype, device=DEV)
    v = base[off:].view(t.shape)
    v.copy_(t)
    return v


# ---- 1. sonet_index_max_f32: the dispatch mirror ------------------------------------------------------
IM_CHUNK, IM_STAGES, IM_MAX_WARPS, IM_HDR_BYTES = 2048, 3, 16, 128
IM_GROUP = 32 * 4 * 4       # points of one load group: 32 lanes x IM_UNROLL float4


def im_route(B, C, N, K, mis, sms, optin):
    """launch_index_max: mis is None, "data" or "index" (that tensor only 4-byte aligned)."""
    wide = N > 65536
    per_warp = K * 32 * (4 + (4 if wide else 2))
    vec = N % 4 == 0 and mis is None
    fixed = IM_HDR_BYTES + IM_STAGES * IM_CHUNK * 4 if vec else 0
    NW = min((optin - fixed) // per_warp, IM_MAX_WARPS, max(C, 1))
    r = dict(vec=vec, wide=wide, NW=NW)
    if vec:
        groups = -(-C // NW)
        r.update(groups=groups, items=B * groups, grid=min(B * groups, sms), nch=-(-N // IM_CHUNK),
                 block=(NW + 1) * 32)
    else:
        items = -(-B * C // NW)
        r.update(groups=None, items=items, grid=min(items, sms), nch=None, block=NW * 32)
    return r


# (B, C, N, K, mis)
IM_CASES = [
    # one load group and its neighbours; NW == C < 16; C == 1
    (2, 3, 508, 8, None), (2, 3, 512, 8, None), (2, 3, 516, 8, None), (3, 1, 512, 5, None),
    # chunk edges, NW == 16 and C % NW != 0 (idle consumer warps keep the barrier protocol)
    (2, 20, 2044, 16, None), (2, 20, 2048, 16, None), (2, 20, 2052, 16, None), (2, 17, 4096, 67, None),
    (1, 33, 6144, 40, None), (1, 16, 6148, 64, None), (2, 5, 8192, 3, None),
    # scalar path: N % 4, data alignment, index alignment
    (2, 20, 510, 16, None), (2, 9, 2047, 64, None), (2, 9, 2048, 64, "data"), (2, 9, 2048, 64, "index"),
    (1, 1, 1023, 5, None), (4, 140, 1027, 256, None),
    # 1 < NW < 16 from K
    (2, 9, 1028, 128, None), (2, 9, 1028, 256, None), (1, 6, 2048, 100, None),
    # the table type x the path
    (1, 3, 65532, 8, None), (1, 3, 65535, 8, None), (1, 3, 65536, 8, None), (1, 3, 65537, 8, None),
    (1, 3, 65540, 8, None), (1, 5, 65540, 256, None), (1, 5, 65538, 256, None), (1, 3, 65540, 8, "data"),
    # several work items per CTA: the stage ring and its phase bit carried across items
    (6, 352, 2048, 256, None), (3, 352, 4092, 256, None), (3, 352, 6144, 256, None),
    (3, 352, 8188, 256, None), (3, 352, 10240, 256, None), (40, 64, 4100, 8, None),
]


def im_id(c):
    return "B%d-C%d-N%d-K%d%s" % (c[0], c[1], c[2], c[3], "-" + c[4] if c[4] else "")


def im_coverage(sms, optin):
    """Every branch of the mirror the table must reach, as name -> reached."""
    R = [(c, im_route(*c, sms, optin)) for c in IM_CASES]
    ring = {r["nch"] for c, r in R if r["vec"] and r["items"] > r["grid"]}
    want_N = {508, 512, 516, 2044, 2048, 2052, 4096, 6144, 6148, 8192, 65532, 65535, 65536, 65537, 65540}
    cov = {
        "vec": any(r["vec"] for _, r in R),
        "scalar: N % 4": any(not r["vec"] and c[2] % 4 for c, r in R),
        "scalar: data alignment": any(c[4] == "data" and c[2] % 4 == 0 for c, r in R),
        "scalar: index alignment": any(c[4] == "index" and c[2] % 4 == 0 for c, r in R),
        "N edges": want_N <= {c[2] for c, _ in R},
        "one load group": {IM_GROUP - 4, IM_GROUP, IM_GROUP + 4} <= {c[2] for c, r in R if r["vec"]},
        "NW == 16": any(r["NW"] == 16 for _, r in R),
        "NW == C < 16": any(r["NW"] == c[1] < 16 and c[1] > 1 for c, r in R),
        "C == 1": any(c[1] == 1 and r["vec"] for c, r in R) and any(c[1] == 1 and not r["vec"] for c, r in R),
        "C % NW != 0 (vec)": any(r["vec"] and c[1] % r["NW"] for c, r in R),
        "four work items per CTA at nch == 1 (the ring wraps across items)":
            any(r["vec"] and r["items"] >= 4 * r["grid"] and r["nch"] == 1 for _, r in R),
        "items > grid on the scalar path": any(not r["vec"] and r["items"] > r["grid"] for _, r in R),
    }
    for n in (1, 2, 3, 4, 5):
        cov["items > grid, nch == %d" % n] = n in ring
    for wide in (False, True):
        for vec in (False, True):
            cov["table %s x %s" % ("int32" if wide else "uint16", "vec" if vec else "scalar")] = any(
                r["wide"] == wide and r["vec"] == vec for _, r in R)
        cov["1 < NW < 16 from K, %s table" % ("int32" if wide else "uint16")] = any(
            r["wide"] == wide and 1 < r["NW"] < min(16, c[1]) for c, r in R)
    return cov


# ---- 2. the fused route: case table -------------------------------------------------------------------
TILE, SLAB = 128, 16
ORDERS = ("asc", "desc", "perm", "alt1", "alt8", "run16", "run16+1", "own", "single")
# (P, M, order, pos0 per cloud)
FUSED_CASES = [
    (1, 1, "single", (0, 0)), (15, 2, "alt1", (14, 3)), (16, 3, "perm", (0, 15)),
    (17, 5, "asc", (16, 9)), (63, 2, "alt8", (62, 0)), (64, 3, "desc", (63, 40)),
    (65, 5, "run16+1", (64, 60)), (127, 255, "perm", (126, 1)), (128, 256, "asc", (127, 64)),
    (129, 129, "own", (128, 5)), (129, 2, "alt1", (0, 128)), (200, 200, "own", (199, 13)),
    (1000, 256, "perm", (896, 905)), (1000, 5, "run16", (999, 0)), (1000, 255, "asc", (512, 999)),
    (1000, 1, "single", (77, 900)), (1000, 2, "alt8", (904, 3)), (1000, 3, "run16+1", (1, 998)),
    (1000, 64, "desc", (0, 0)), (1000, 16, "perm", (960, 970)),
]
# the cases that also run in elu and in the one-product fp16 mode
FUSED_CORE = [FUSED_CASES[i] for i in (3, 6, 9, 12, 16)]
MODES = [("relu", False), ("relu", True), ("elu", False), ("elu", True)]


def fused_id(c):
    return "P%d-M%d-%s" % (c[0], c[1], c[2])


def mode_id(m):
    return "%s-%s" % (m[0], "f16" if m[1] else "3xf16")


def node_rows(order, B, P, M, g):
    """Node id of every row [B,P]; every pattern is one the run loop must take as it comes."""
    r = torch.arange(P)
    if order in ("asc", "desc"):
        n = torch.sort(torch.randint(0, M, (B, P), generator=g), dim=1, descending=order == "desc")[0]
    elif order == "perm":
        n = torch.randint(0, M, (B, P), generator=g)
    elif order == "alt1":                       # two nodes, alternating row by row
        n = torch.where(r % 2 == 0, 0, M - 1).expand(B, P)
    elif order == "alt8":                       # rows r0 and r0 + 8 of a thread always differ
        n = torch.where((r // 8) % 2 == 0, M - 1, 0).expand(B, P)
    elif order == "run16":                      # runs of 16, aligned to the warps' slabs
        n = ((r // SLAB) % M).expand(B, P)
    elif order == "run16+1":                    # the same runs shifted by one row
        n = (((r + SLAB - 1) // SLAB) % M).expand(B, P)
    elif order == "own":                        # every row its own node
        assert M == P
        n = torch.stack([torch.randperm(P, generator=g) for _ in range(B)])
    else:
        n = torch.full((B, P), M // 2)
    return n.int().contiguous()


def fused_coverage():
    last = [(P, p) for P, _, _, pos in FUSED_CASES for p in pos if P % TILE and p >= P // TILE * TILE]
    return {
        "P": {1, 15, 16, 17, 63, 64, 65, 127, 128, 129, 1000} <= {c[0] for c in FUSED_CASES},
        "M": {1, 2, 3, 5, 255, 256} <= {c[1] for c in FUSED_CASES},
        "vector and scalar finalize": {True, False} == {c[1] % 4 == 0 for c in FUSED_CASES},
        "orders": set(ORDERS) == {c[2] for c in FUSED_CASES},
        "pos0 == 0": any(0 in c[3] for c in FUSED_CASES),
        "pos0 == P - 1": any(c[0] - 1 in c[3] for c in FUSED_CASES),
        "pos0 in the r0 half of the last partial tile": any(p % SLAB < 8 for _, p in last),
        "pos0 in the r0 + 8 half of the last partial tile": any(p % SLAB >= 8 for _, p in last),
        "pos0 differs per cloud": any(len(set(c[3])) > 1 for c in FUSED_CASES),
        "core cases in the table": all(c in FUSED_CASES for c in FUSED_CORE),
    }


def test_case_tables_reach_every_branch_on_h100():
    """Host side: with the H100's 132 SMs and 227 KB opt-in limit as constants, so a table edit that
    loses a branch fails without a GPU too."""
    for name, ok in {**im_coverage(H100_SMS, H100_OPTIN), **fused_coverage()}.items():
        assert ok, "no case reaches: " + name
    # the warp counts the ring cases rely on
    assert im_route(6, 352, 2048, 256, None, H100_SMS, H100_OPTIN)["NW"] == 4
    assert im_route(1, 5, 65540, 256, None, H100_SMS, H100_OPTIN)["NW"] == 3


def test_pool_ref_is_the_sequential_rule():
    """Host side: pool_ref on a hand-checked example (ties, sentinel, NaN, inf, an empty node)."""
    nan, inf = float("nan"), float("inf")
    #               n: 0     1     2      3     4    5     6     7
    data = np.array([[[2.0, 5.0, 5.0, -1000.0, nan, inf, inf, -inf],
                      [nan, 1.0, nan, -1001.0, 3.0, 3.0, nan, 9.0]]], np.float32)
    index = np.array([[0, 0, 0, 1, 2, 2, 2, 1]])
    idx, val = pool_ref(data, index, 4)
    assert idx.tolist() == [[[1, 0, 5, 0], [1, 7, 4, 0]]]
    assert val[0, 0].tolist() == [5.0, 2.0, inf, 2.0]
    assert val[0, 1, :3].tolist() == [1.0, 9.0, 3.0] and np.isnan(val[0, 1, 3])
    assert pool_ref(data, index, 4, point0=[3])[1][0, 0].tolist() == [5.0, -1000.0, inf, -1000.0]


# ---- 1. sonet_index_max_f32: the tests ----------------------------------------------------------------
def mixed_rows(B, C, N, g):
    """Channel c % 4: 0 random multiples of 1/8 (many exact ties), 1 ascending, 2 descending,
    3 constant."""
    d = (torch.randn(B, C, N, generator=g) * 8).round() / 8
    ramp = torch.arange(N, dtype=torch.float32) / 8 - 500
    d[:, 1::4] = ramp
    d[:, 2::4] = -ramp
    d[:, 3::4] = 0.25
    return d.float().contiguous()


def run_index_max(data, index, K, mis=None):
    """-> (idx, val) of the with-values call; the index-only call must give the same idx."""
    from sonet_b200 import ops
    d = offset_copy(data) if mis == "data" else data.to(DEV)
    i = offset_copy(index) if mis == "index" else index.to(DEV)
    assert (d.data_ptr() % 16 == 0) == (mis != "data") and (i.data_ptr() % 16 == 0) == (mis != "index")
    idx, val = ops.index_max(d, i, K, with_values=True)
    assert torch.equal(ops.index_max(d, i, K), idx)
    return idx, val


def check_index_max(data, index, K, what, mis=None, ref_index=None):
    idx, val = run_index_max(data, index, K, mis)
    widx, wval = pool_ref(data.numpy(), index.numpy() if ref_index is None else ref_index, K)
    assert torch.equal(idx.cpu(), torch.from_numpy(widx)), "%s: %d arg-max differ" % (
        what, int((idx.cpu() != torch.from_numpy(widx)).sum()))
    assert_bits(val, wval, what + " values")
    return widx, wval


_KERNEL = re.compile(r"sonet::(index_max_vec_kernel|index_max_scalar_kernel)<([^>]*)>")


@contextlib.contextmanager
def index_max_launches():
    """The index_max kernels launched inside the block, in order: (kernel, IdxT, grid.x, block.x)."""
    from torch.profiler import ProfilerActivity, profile
    out = []
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        yield out
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    evs = sorted((e for e in trace["traceEvents"] if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    for e in evs:
        m = _KERNEL.search(e["name"])
        if m:
            out.append((m.group(1), m.group(2).strip(), e["args"]["grid"][0], e["args"]["block"][0]))


@gpu
def test_index_max_cases_reach_every_branch_and_launch_what_the_mirror_names():
    from sonet_b200 import ops
    p = torch.cuda.get_device_properties(0)
    sms, optin = p.multi_processor_count, p.shared_memory_per_block_optin
    for name, ok in im_coverage(sms, optin).items():
        assert ok, "no case reaches: " + name
    tensors = []
    for B, C, N, K, mis in IM_CASES:
        d = torch.zeros(B, C, N)
        i = torch.zeros(B, N, dtype=torch.int32)
        tensors.append((offset_copy(d) if mis == "data" else d.to(DEV),
                        offset_copy(i) if mis == "index" else i.to(DEV), K))
    with index_max_launches() as seen:
        for _ in range(2):      # a profiler can miss the first launches after it starts: read the last pass
            for d, i, K in tensors:
                ops.index_max(d, i, K)
    want = []
    for c in IM_CASES:
        r = im_route(*c, sms, optin)
        want.append(("index_max_vec_kernel" if r["vec"] else "index_max_scalar_kernel",
                     "int" if r["wide"] else "unsigned short", r["grid"], r["block"]))
    assert len(want) <= len(seen) <= 2 * len(want), (len(seen), len(want))
    for c, s, w in zip(IM_CASES, seen[-len(want):], want):
        assert s == w, (im_id(c), s, w)


@gpu
@pytest.mark.parametrize("case", IM_CASES, ids=im_id)
def test_index_max_shape_sweep(oracle_mod, case):
    """Ties, ascending, descending and constant rows at every dispatch edge; the reference binary
    pins pool_ref on these finite inputs."""
    B, C, N, K, mis = case
    g = _gen(N * 31 + K)
    data = mixed_rows(B, C, N, g)
    index = torch.randint(0, K, (B, N), generator=g, dtype=torch.int32)
    if K > 2:
        index[index == K // 2] = 0                         # an empty node
    widx, _ = check_index_max(data, index, K, im_id(case), mis)
    assert torch.equal(oracle_mod.index_max(data, index, K), torch.from_numpy(widx))


def quad_case(N):
    """K = 4, one float4 per lane and 128 points: cloud b, lane l holds node assignment
    a = 32 b + l of the 256 (four base-4 digits), channel c the value order c of the 81 over
    {-1, 0, 1}: every same-node pattern of im_update4 meets every tie pattern. N = 256 gives each
    lane a second quad (other assignment, other values) that finds the table already written."""
    B, C = 8, 81
    data = torch.empty(B, C, N)
    index = torch.empty(B, N, dtype=torch.int32)
    for q in range(N // 128):
        for b in range(B):
            for lane in range(32):
                a = (32 * b + lane + 97 * q) % 256
                for j in range(4):
                    index[b, 128 * q + 4 * lane + j] = (a >> (2 * j)) & 3
        for c in range(C):
            v = (c + 40 * q) % 81
            vals = torch.tensor([(v // 3 ** j) % 3 - 1 for j in range(4)], dtype=torch.float32)
            data[:, c, 128 * q:128 * (q + 1)] = vals.repeat(32)
    return data, index


@gpu
@pytest.mark.parametrize("N", [128, 256])
def test_index_max_exhaustive_quad(oracle_mod, N):
    data, index = quad_case(N)
    first = index[:, :128].reshape(-1, 4)
    assert len({tuple(r) for r in first.tolist()}) == 256
    widx, _ = check_index_max(data, index, 4, "quad")
    assert torch.equal(oracle_mod.index_max(data, index, 4), torch.from_numpy(widx))
    check_index_max(data, index, 4, "quad, scalar path", mis="data")


@gpu
@pytest.mark.parametrize("dist", ["one node", "last node only", "K=1", "K=256", "all empty but one"])
def test_index_max_node_distributions(oracle_mod, dist):
    B, C, N = 2, 5, 1028
    g = _gen(len(dist))
    K = {"K=1": 1, "K=256": 256}.get(dist, 24)
    data = mixed_rows(B, C, N, g)
    if dist == "one node":
        index = torch.full((B, N), 7, dtype=torch.int32)
    elif dist in ("last node only", "all empty but one"):
        index = torch.full((B, N), K - 1 if dist == "last node only" else 11, dtype=torch.int32)
    else:
        index = torch.randint(0, K, (B, N), generator=g, dtype=torch.int32)
    for mis in (None, "index"):
        widx, _ = check_index_max(data, index, K, dist, mis)
    assert torch.equal(oracle_mod.index_max(data, index, K), torch.from_numpy(widx))


def special_case():
    """One cloud, 16 nodes, one scenario per channel, all about node 5 unless said otherwise.
    Point 0 belongs to node 0; nodes 12-15 are empty. -> data, index, {scenario: channel}."""
    N, K = 516, 16
    g = _gen(77)
    index = torch.randint(0, 12, (1, N), generator=g, dtype=torch.int32)
    index[0, 0] = 0
    names = ["max == -1000", "max just above -1000", "max just below -1000", "all -inf",
             "NaN before and after the maximum", "NaN only", "NaN at point 0", "+inf twice",
             "+inf and NaN", "-0 then +0", "+0 then -0"]
    ch = {n: c for c, n in enumerate(names)}
    data = (torch.randn(1, len(names), N, generator=g) * 8).round() / 8
    data[0, :, 0] = 7.5
    pts = torch.nonzero(index[0] == 5).flatten()
    assert len(pts) >= 8
    nan, inf = float("nan"), float("inf")
    above = float(np.nextafter(SENTINEL, np.float32(0)))
    below = float(np.nextafter(SENTINEL, np.float32(-np.inf)))

    def node5(name, fill, **at):
        data[0, ch[name], pts] = fill
        for k, v in at.items():
            data[0, ch[name], pts[int(k[1:])]] = v
    node5("max == -1000", -2000.0, p2=-1000.0, p4=-1000.0)
    node5("max just above -1000", -2000.0, p1=-1000.0, p3=above, p5=above)
    node5("max just below -1000", -2000.0, p3=below)
    node5("all -inf", -inf)
    node5("NaN before and after the maximum", -3.0, p0=nan, p2=4.0, p3=nan, p5=4.0, p6=nan)
    node5("NaN only", nan)
    data[0, ch["NaN at point 0"], 0] = nan
    node5("+inf twice", 1.0, p1=inf, p4=inf)
    node5("+inf and NaN", 1.0, p0=nan, p2=inf, p3=nan, p5=inf)
    node5("-0 then +0", -5.0, p1=-0.0, p3=0.0)
    node5("+0 then -0", -5.0, p1=0.0, p3=-0.0)
    data = data.float().contiguous()
    # a NaN with a payload: the gather must preserve its bits
    data.view(torch.int32)[0, ch["NaN at point 0"], 0] = 0x7FC12345
    return data, index, K, ch, pts


@gpu
@pytest.mark.parametrize("mis", [None, "data"], ids=["vec", "scalar"])
def test_index_max_sentinel_and_non_finite(mis):
    data, index, K, ch, pts = special_case()
    widx, wval = check_index_max(data, index, K, "special", mis)
    # what the rule gives, stated: the expectations the kernel was just compared with
    p = pts.tolist()
    for name in ("max == -1000", "max just below -1000", "all -inf", "NaN only"):
        assert widx[0, ch[name], 5] == 0 and wval[0, ch[name], 5] == 7.5, name   # point 0, of node 0
    assert widx[0, ch["max just above -1000"], 5] == p[3]
    assert widx[0, ch["NaN before and after the maximum"], 5] == p[2]
    assert widx[0, ch["+inf twice"], 5] == p[1] and widx[0, ch["+inf and NaN"], 5] == p[2]
    assert widx[0, ch["-0 then +0"], 5] == p[1] and widx[0, ch["+0 then -0"], 5] == p[1]
    c = ch["NaN at point 0"]
    assert widx[0, c, 0] != 0                                         # node 0: the NaN never wins
    assert bits(wval)[0, c, 12:].tolist() == [0x7FC12345] * 4         # empty nodes read point 0


@gpu
@pytest.mark.parametrize("mis", [None, "data"], ids=["vec", "scalar"])
def test_index_max_ids_outside_the_node_range_are_clamped(mis):
    """Every shared-memory access of both paths goes through min(unsigned(id), K-1) (im_update,
    im_update4; im_reduce_row and the table reset loop over k < K), so an id outside [0,K) counts
    as node K-1."""
    B, C, N, K = 2, 7, 1032, 10
    g = _gen(3)
    data = mixed_rows(B, C, N, g)
    index = torch.randint(0, K, (B, N), generator=g, dtype=torch.int32)
    bad = torch.tensor([-1, -5, K, K + 100, INT_MIN, 2 ** 31 - 1, 256, 65536], dtype=torch.int32)
    where = torch.randperm(N, generator=g)[:64]
    index[:, where] = bad.repeat(8)
    index[0, 4:8] = torch.tensor([-1, K, 3, -1], dtype=torch.int32)       # inside one float4
    check_index_max(data, index, K, "clamped ids", mis, ref_index=clamp_ids(index.numpy(), K))


@gpu
def test_index_max_degenerate_shapes():
    from sonet_b200 import ops
    idx, val = ops.index_max(torch.empty(2, 3, 0, device=DEV), torch.empty(2, 0, dtype=torch.int32, device=DEV),
                             5, with_values=True)
    assert idx.shape == val.shape == (2, 3, 5)
    assert not bool(idx.any()) and torch.equal(bits(val), torch.zeros(2, 3, 5, dtype=torch.int32))
    for B, C in ((0, 3), (2, 0)):
        idx, val = ops.index_max(torch.empty(B, C, 64, device=DEV),
                                 torch.zeros(B, 64, dtype=torch.int32, device=DEV), 5, with_values=True)
        assert idx.shape == val.shape == (B, C, 5)
    d, i = torch.zeros(1, 2, 64, device=DEV), torch.zeros(1, 64, dtype=torch.int32, device=DEV)
    for K in (0, 257):
        with pytest.raises(RuntimeError, match="out of range"):
            ops.index_max(d, i, K)
    torch.cuda.synchronize()


# ---- 2. the fused route: the tests --------------------------------------------------------------------
def fused_net(seed, sentinel=False, cin=6):
    """Folded weights and shifts of a first PointResNet, packed for the kernel. sentinel: the last
    layer's channels meet the -1000 rule:
      channel 0: zero weights, shift -1000: every row equals the sentinel;
      channel 1: -1000 - act0[0], where act0[0] = act(x0 - 10) is relu's exact 0 on ordinary rows:
                 maxima of exactly -1000 next to a copy-0 row made different (x0 = 12 -> -1002);
      channels 2, 5, 8, ...: shifts from -998 down to -1006, so per-node maxima straddle -1000."""
    from sonet_b200 import ops
    g = _gen(seed)
    dims = [(64, cin), (128, 64), (256, 128), (384, 320)]
    W = [torch.randn(o, i, generator=g) * (2.0 / i) ** 0.5 for o, i in dims]
    S = [torch.randn(o, generator=g) * 0.1 for o, _ in dims]
    if sentinel:
        W[0][0] = 0
        W[0][0, 0] = 1
        S[0][0] = -10
        W[3][0] = 0
        S[3][0] = -1000
        W[3][1] = 0
        W[3][1, 0] = -1
        S[3][1] = -1000
        c = torch.arange(2, 384, 3)
        S[3][c] = -1000 - torch.linspace(-2, 6, len(c))
    blob, fpar = ops.pointresnet_tc_pack(W, S, cin)
    return blob.to(DEV), fpar.to(DEV)


def run_fused(x, blob, fpar, node, pos0, M, act, f16, what):
    """The plain kernel's rows `full`, and pool_ref on them; the pool kernel read back three ways
    must give those bits, the copy-0 features must be full's pos0 rows, and every key must be back
    at INT_MIN. -> (full [B,384,P] on the host, want [B,384,M])."""
    from sonet_b200 import ops
    B, _, P = x.shape
    g = _gen(P * 1000 + M)
    full = ops.pointresnet_tc(x, blob, fpar, f16=f16, act=act)
    fh = full.cpu()
    want = pool_ref(fh.numpy(), node.cpu().numpy(), M, point0=pos0.cpu().numpy())[1]
    coord = torch.randn(B, 3, M, generator=g).to(DEV)

    def pool():
        keys, p0 = ops.pointresnet_tc_pool(x, blob, fpar, node, pos0, M, finalize=False, f16=f16, act=act)
        assert_bits(p0, fh[torch.arange(B), :, pos0.cpu().long()], what + ": copy-0 features")
        return keys, p0

    def keys_reset(keys):
        assert bool((keys == INT_MIN).all()), what + ": keys not reset"
    keys, p0 = pool()
    assert_bits(ops.pool_finalize(keys, p0), want, what + ": pool_finalize")
    keys_reset(keys)
    for Kn, ctype, aug in ((3, "center", True), (4, "avg", False)):
        nbr = torch.randint(0, M, (B, M, Kn), generator=g).to(DEV)
        keys, p0 = pool()
        _, x_aug, mm = ops.knn_assemble_pool(coord, keys, p0, nbr, Kn, ctype, want_x_aug=aug)
        assert_bits(mm, want, what + ": knn_assemble_pool(K=%d)" % Kn)
        keys_reset(keys)
        if aug:
            feat = mm.gather(2, nbr.view(B, 1, M * Kn).expand(B, 384, M * Kn))
            assert_bits(x_aug[:, 3:], feat, what + ": x_aug features")
        else:
            assert x_aug is None
    return fh, want


def fused_inputs(case, seed, B=2):
    P, M, order, pos0 = case
    g = _gen(seed)
    x = torch.randn(B, 6, P, generator=g).clamp(-3.5, 3.5)
    node = node_rows(order, B, P, M, g)
    return x, node, torch.tensor(pos0[:B], dtype=torch.int32)


@gpu
@pytest.mark.parametrize("case", FUSED_CASES, ids=fused_id)
def test_fused_pool_row_orders_and_shapes(case):
    x, node, pos0 = fused_inputs(case, seed=case[0] * 7 + case[1])
    blob, fpar = fused_net(1)
    run_fused(x.to(DEV), blob, fpar, node.to(DEV), pos0.to(DEV), case[1], "relu", False, fused_id(case))


@gpu
@pytest.mark.parametrize("mode", MODES, ids=mode_id)
@pytest.mark.parametrize("case", FUSED_CORE, ids=fused_id)
def test_fused_pool_core_cases_in_every_mode(case, mode):
    x, node, pos0 = fused_inputs(case, seed=case[0] + case[1])
    blob, fpar = fused_net(2)
    run_fused(x.to(DEV), blob, fpar, node.to(DEV), pos0.to(DEV), case[1], *mode, fused_id(case))


@gpu
def test_fused_pool_does_not_depend_on_the_row_order():
    """The same rows in node-sorted and in shuffled order give the same per-node bits."""
    from sonet_b200 import ops
    B, P, M = 2, 1000, 37
    g = _gen(5)
    x = torch.randn(B, 6, P, generator=g).clamp(-3.5, 3.5)
    node = node_rows("asc", B, P, M, g)
    blob, fpar = fused_net(3)
    pos0 = torch.tensor([17, 801], dtype=torch.int32)
    a = ops.pointresnet_tc_pool(x.to(DEV), blob, fpar, node.to(DEV), pos0.to(DEV), M)
    perm = torch.stack([torch.randperm(P, generator=g) for _ in range(B)])
    xs = x.gather(2, perm[:, None, :].expand(B, 6, P)).contiguous()
    ns = node.gather(1, perm).contiguous()
    inv = torch.argsort(perm, dim=1)
    ps = inv.gather(1, pos0.long()[:, None])[:, 0].int()
    b = ops.pointresnet_tc_pool(xs.to(DEV), blob, fpar, ns.to(DEV), ps.to(DEV), M)
    assert_bits(a, b, "sorted vs shuffled rows")


@gpu
@pytest.mark.parametrize("mode", MODES, ids=mode_id)
def test_fused_pool_sentinel_through_the_kernel(mode):
    B, P, M = 2, 1000, 64
    g = _gen(11)
    x = torch.randn(B, 6, P, generator=g).clamp(-3.5, 3.5)
    node = node_rows("asc", B, P, M, g)
    node[node == 9] = 10                                       # an empty node
    pos0 = torch.tensor([300, 905], dtype=torch.int32)
    x[torch.arange(B), 0, pos0.long()] = 12.0
    blob, fpar = fused_net(4, sentinel=True)
    full, want = run_fused(x.to(DEV), blob, fpar, node.to(DEV), pos0.to(DEV), M, *mode, "sentinel " + mode_id(mode))
    seg = torch.full((B, 384, M), float("-inf")).scatter_reduce(
        2, node.long()[:, None, :].expand(B, 384, P), full, "amax")
    used = torch.zeros(B, M, dtype=torch.bool).scatter_(1, node.long(), True)[:, None, :].expand(B, 384, M)
    straddle = torch.arange(2, 384, 3)
    fell, held = used & (seg <= -1000), used & (seg > -1000)
    assert bool(fell[:, straddle].any()) and bool(held[:, straddle].any())     # both outcomes occur
    assert bool((full[:, 0] == -1000).all())
    if mode[0] == "relu":
        # maxima of exactly -1000 whose fallback differs: `>` and `>=` are told apart
        assert bool((seg[:, 1][used[:, 1]] == -1000).all())
        assert bool((full[torch.arange(B), 1, pos0.long()] == -1002).all())
        assert bool((torch.from_numpy(want)[:, 1] == -1002).all())


NONFINITE = {"nan": float("nan"), "+inf": float("inf"), "-inf": float("-inf")}


def nonfinite_case(kind):
    """P = 400, M = 8. Node 0: rows 0-47 and 128-143, of which the slab 16-31 is non-finite (a
    complete, slab-aligned run next to finite rows in other slabs and another tile); node 1:
    rows 48-79 with the single non-finite row 50; node 2: rows 80-111, all non-finite; the rest
    random over nodes 3-6; node 7 empty. pos0 is the non-finite row 50 in cloud 0 and a finite row
    in cloud 1. A NaN row has all six coordinates NaN, an inf row its first."""
    B, P, M = 2, 400, 8
    g = _gen(23)
    x = torch.randn(B, 6, P, generator=g).clamp(-3.5, 3.5)
    node = torch.randint(3, 7, (B, P), generator=g).int()
    node[:, 0:48] = 0
    node[:, 128:144] = 0
    node[:, 48:80] = 1
    node[:, 80:112] = 2
    bad = torch.zeros(P, dtype=torch.bool)
    bad[16:32] = bad[50] = bad[80:112] = True
    if kind == "nan":
        x[:, :, bad] = NONFINITE[kind]
    else:
        x[:, 0, bad] = NONFINITE[kind]
    return x, node, torch.tensor([50, 5], dtype=torch.int32), M, bad


@gpu
@pytest.mark.parametrize("mode", MODES, ids=mode_id)
@pytest.mark.parametrize("kind", list(NONFINITE))
def test_fused_pool_non_finite_rows(kind, mode):
    x, node, pos0, M, bad = nonfinite_case(kind)
    blob, fpar = fused_net(6)
    full, want = run_fused(x.to(DEV), blob, fpar, node.to(DEV), pos0.to(DEV), M, *mode,
                           "%s rows, %s" % (kind, mode_id(mode)))
    assert bool(torch.isfinite(full[:, :, ~bad]).all())
    if kind == "nan":
        if mode[0] == "elu":
            # ELU keeps NaN and so do the saturating fp16 conversions: the rows reach the pool as NaN
            assert bool(torch.isnan(full[:, :, bad]).all())
            w = torch.from_numpy(want)
            assert bool(torch.isfinite(w[:, :, 0]).all())            # the finite rows of node 0 win
            assert bool(torch.isnan(w[0, :, 2]).all())               # NaN-only node: copy 0, a NaN row
            assert bool(torch.isfinite(w[1, :, 2]).all())            # ... or a finite one
        else:
            assert bool(torch.isfinite(full).all())                  # fmaxf(NaN, 0) = 0 in layer 0


# ---- 3. IndexMaxGather and sonet_index_max_backward_f32 -----------------------------------------------
def backward_ref(go, idx, N):
    """grad_data[r, idx[r,k]] += go[r,k] in fp32, k ascending: the kernel's documented order."""
    R, K = go.shape
    g = np.zeros((R, N), np.float32)
    rows = np.arange(R)
    for k in range(K):
        g[rows, idx[:, k]] += go[:, k]
    return g


# (B, C, N, K, nodes used)
BWD_CASES = [(1, 1, 64, 8, None), (1, 127, 33, 16, None), (2, 64, 100, 64, None), (3, 43, 257, 5, None),
             (2, 9, 300, 256, (3,)), (2, 5, 50, 1, None), (2, 6, 1, 4, (2,)), (1, 3, 65540, 12, None)]


@gpu
@pytest.mark.parametrize("case", BWD_CASES, ids=lambda c: "BC%d-N%d-K%d%s" % (c[0] * c[1], c[2], c[3],
                                                                             "-sparse" if c[4] else ""))
def test_index_max_gather_forward_and_backward(case):
    from sonet_b200 import train_ops
    B, C, N, K, used = case
    g = _gen(B * C + N + K)
    data = mixed_rows(B, C, N, g)
    if used is None:
        index = torch.randint(0, K, (B, N), generator=g, dtype=torch.int32)
    else:                                  # every node empty but these: K-1 gradients meet on point 0
        index = torch.tensor(used, dtype=torch.int32)[torch.randint(0, len(used), (B, N), generator=g)]
    if N > 65536:
        data[:, :, -3:] += 2000            # arg-max beyond the uint16 range
    w = torch.randn(B, C, K, generator=g)
    widx, wval = pool_ref(data.numpy(), index.numpy(), K)
    dirty = torch.full((B, C, N), float("nan"), device=DEV)     # the allocator hands this block out again
    del dirty
    grads = []
    for _ in range(2):
        d = data.to(DEV).requires_grad_(True)
        out = train_ops.IndexMaxGather.apply(d, index.to(DEV), K)
        assert_bits(out, wval, "forward value")
        (out * w.to(DEV)).sum().backward()
        grads.append(d.grad)
    assert_bits(grads[0], grads[1], "two runs")
    want = backward_ref(w.numpy().reshape(B * C, K), widx.reshape(B * C, K), N).reshape(B, C, N)
    assert_bits(grads[0], want, "backward, sequential fp32 order")
    # fp64 autograd of data.gather(2, idx): recursive summation of at most K terms per point, so
    # |error| <= gamma(K - 1) * sum |terms|, gamma(n) = n u / (1 - n u), u = 2^-24
    d64 = data.double().requires_grad_(True)
    (d64.gather(2, torch.from_numpy(widx).long()) * w.double()).sum().backward()
    mag = torch.zeros(B, C, N, dtype=torch.float64).scatter_add_(2, torch.from_numpy(widx).long(), w.double().abs())
    u = 2.0 ** -24
    bound = (K - 1) * u / (1 - (K - 1) * u) * mag
    assert bool(((grads[0].cpu().double() - d64.grad).abs() <= bound).all())
