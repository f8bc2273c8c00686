"""SOM training without a GPU: the host-side pieces (potential-field start, neighbourhood weights)
against the reference's own fixtures at 3x3 .. 16x16 grids, and the exact-sum numpy emulation
(tests/som_emu.py) that the GPU envelope tests hold csrc/som_train.cu to, checked against the
oracle restatement and the reference goldens."""
import fractions

import numpy as np
import pytest
import torch

import som_emu
from helpers import golden

# golden file, grid side
GRIDS = [("som_train_m9", 3), ("som_train", 8), ("som_train_m121", 11), ("som_train_m256", 16)]


def _som(r, B=1):
    from sonet_b200 import som
    return som.BatchSOM(r, r, 3, 0, B)


def _W(s, sigma):
    M = s.node_num
    return s.get_weighting_matrix(sigma).view(M, M).numpy()


def _schedule(s):
    """BatchSOM.optimize's (learning rate, sigma) list: max_iteration / 3 + max_iteration steps."""
    sched = [(s.learning_rate, s.sigma)] * int(s.max_iteration / 3)
    for it in range(s.max_iteration):
        sched.append((s.learning_rate / (1 + 2 * it / s.max_iteration),
                      s.sigma / (1 + 2 * it / s.max_iteration)))
    return sched


@pytest.mark.parametrize("name,r", GRIDS)
def test_potential_field_start_is_the_references(name, r):
    """som.potential_field_nodes is the reference's PotentialField bit for bit. The field is
    chaotic (at 256 nodes a last-bit change in one norm ends in a different arrangement), so this
    pins the scalar arithmetic, not just the algorithm."""
    from sonet_b200 import som
    g = golden(name)
    pf = som.potential_field_nodes(r * r)
    assert pf.dtype == np.float64 and pf.shape == (r * r, 3)
    assert np.array_equal(pf.T.astype(np.float32), g["node_init_value"])
    assert np.array_equal(_som(r).node_init_value.numpy(), g["node_init_value"])


def test_row_norm_is_numpys_norm():
    """The potential field's norm: np.linalg.norm of a 3-vector, row by row, bit for bit (it is
    BLAS ddot's FMA chain, which a plain sum of squares misses in about 10 % of the rows)."""
    from sonet_b200 import som
    rs = np.random.RandomState(3)
    f = rs.normal(size=(20000, 3)) * np.exp(rs.uniform(-8, 4, size=(20000, 1)))
    f[:50, 1:] = 0.0
    want = np.array([np.linalg.norm(v) for v in f])
    assert np.array_equal(som._row_norm(f), want)


@pytest.mark.parametrize("r", [1, 3, 8, 11, 16])
def test_init_weighting_matrix_matches_oracle(oracle_mod, r):
    assert torch.equal(_som(r).init_weighting_matrix, oracle_mod.som_init_weighting_matrix(r, r))


def test_exact_sum_rounding():
    """The emulation's sums are exact: a float64 sum that lands on a float32 midpoint is resolved
    by the exact value, on both sides, and ties go to even."""
    one, h = 1.0, 2.0 ** -24                       # h: half an ulp of float32 at 1
    recomputed = 0
    for terms in ([one, h, 2.0 ** -80], [one, h, -2.0 ** -80], [one, h], [one + 2 * h, h],
                  [3.0, -1.0, 2 * h, 2.0 ** -70, -2.0 ** -71]):
        exact = sum(fractions.Fraction(t) for t in terms)
        want = np.float32(float(exact))             # exact -> float64 is exact for these sums
        if fractions.Fraction(float(exact)) != exact:
            lo = np.float32(float(exact))
            cands = [lo, np.nextafter(lo, np.float32(np.inf)), np.nextafter(lo, np.float32(-np.inf))]
            want = min(cands, key=lambda c: (abs(fractions.Fraction(float(c)) - exact),
                                             int(np.array(c).view(np.int32)) & 1))
        s64 = np.array([sum(terms)])
        a64 = np.array([sum(abs(t) for t in terms)])
        got, n_exact = som_emu.round_sums(s64, a64, np.array([len(terms)]), lambda i: list(terms))
        assert got[0] == want, (terms, got[0], want)
        assert som_emu.f32_exact_sum(terms) == want
        recomputed += n_exact
    assert recomputed == 5                           # every one of them sits on a midpoint


@pytest.mark.parametrize("name,r", GRIDS)
def test_emulation_matches_oracle_batch_update(oracle_mod, name, r):
    """One emulated step against oracle.som_batch_update (the reference's ATen ops) on the golden
    clouds: same assignment, nodes within 1e-6 — they differ only in how the sums are taken."""
    g = golden(name)
    s = _som(r)
    x = g["x"]
    B, M = x.shape[0], r * r
    node = np.ascontiguousarray(np.broadcast_to(g["node_init_value"], (B, 3, M)))
    init_w = oracle_mod.som_init_weighting_matrix(r, r)
    for lr, sigma in ((0.5, 0.4), (0.31, 0.22), (0.2, 0.1)):
        got, idx = som_emu.step(x, node, _W(s, sigma), lr)
        want, want_idx = oracle_mod.som_batch_update(torch.from_numpy(node), torch.from_numpy(x),
                                                     init_w, lr, sigma)
        assert np.array_equal(idx, want_idx.numpy())
        err = np.abs(got - want.numpy()).max()
        assert err <= 1e-6, (lr, sigma, err)
        node = got


@pytest.mark.parametrize("name,r", GRIDS)
def test_emulated_optimize_vs_reference_golden(name, r):
    """The emulation iterated over BatchSOM.optimize's 80-step schedule against the reference's
    own 80 steps: the two-step fixtures within 1e-6, the optimised nodes within 1e-4. The
    smallest best-vs-second distance gap met (printed) says how close an assignment came to
    flipping between the exact and the reference's cascade sums."""
    g = golden(name)
    s = _som(r)
    x = g["x"]
    n1, _ = som_emu.train(x, g["node_init_value"], [_W(s, 0.4)], [0.5])
    assert np.abs(n1 - g["node_after_1"]).max() <= 1e-6
    n2, _ = som_emu.train(x, n1, [_W(s, 0.22)], [0.31])
    assert np.abs(n2 - g["node_after_2"]).max() <= 1e-6
    sched = _schedule(s)
    margin = som_emu.Margin()
    node, _ = som_emu.train(x, g["node_init_value"], [_W(s, sg) for _, sg in sched],
                            [lr for lr, _ in sched], margin)
    err = np.abs(node - g["node_optimized"]).max()
    print("%s: max |emulation - reference| after 80 steps %.3g, %r" % (name, err, margin))
    assert err <= 1e-4 * max(1.0, float(np.abs(g["node_optimized"]).max()))
