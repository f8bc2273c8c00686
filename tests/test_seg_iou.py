"""Part-segmentation IoU on the host: sonet_b200.losses.compute_iou_np_array / compute_iou and the
library's host entry sonet_seg_iou_cpu_f32 against the reference's own outputs
(tests/golden/seg_iou.npz, written by oracle/seg_iou_golden.py)."""
import numpy as np
import pytest
import torch

from helpers import golden

G = golden("seg_iou")
CASES = [str(c) for c in G["cases"]]


def case(tag):
    return (torch.from_numpy(G[tag + "_score"]), torch.from_numpy(G[tag + "_seg"]),
            torch.from_numpy(G[tag + "_label"]))


@pytest.mark.parametrize("tag", CASES)
def test_host_entry_reproduces_the_reference(tag):
    from sonet_b200 import losses
    score, seg, label = case(tag)
    per_shape = losses.compute_iou_np_array(score, seg, label, None, None, None)
    assert per_shape.dtype == np.float64
    assert np.array_equal(per_shape, G[tag + "_iou"])
    assert losses.compute_iou(score, seg, label, None, None, None) == G[tag + "_miou"]


@pytest.mark.parametrize("threads", [1, 3, 64])
def test_thread_count_does_not_change_the_result(threads):
    from sonet_b200 import losses
    score, seg, label = case("random")
    prev = torch.get_num_threads()
    torch.set_num_threads(threads)
    try:
        got = losses.compute_iou_np_array(score, seg, label, None, None, None)
    finally:
        torch.set_num_threads(prev)
    assert np.array_equal(got, G["random_iou"])


def test_partsegiou_on_host_tensors():
    from sonet_b200 import losses
    meter = losses.PartSegIoU()
    ious, labels, correct, points = [], [], 0, 0
    for tag in ("random", "ties", "odd_n"):
        score, seg, label = case(tag)
        meter.update(score, seg, label)
        ious.append(G[tag + "_iou"])
        labels.append(G[tag + "_label"])
        correct += int((torch.max(score, 1)[1] == seg).sum())
        points += seg.numel()
    r = meter.compute()
    iou, lab = np.concatenate(ious), np.concatenate(labels)
    assert r["instance_miou"] == iou.mean()
    cats = sorted(set(lab.tolist()))
    assert list(r["category_miou"]) == cats
    for c in cats:
        assert r["category_miou"][c] == iou[lab == c].mean()
    assert r["class_miou"] == np.asarray([iou[lab == c].mean() for c in cats]).mean()
    assert r["accuracy"] == correct / points


def test_labels_outside_the_table_raise():
    from sonet_b200 import losses
    score, seg, label = case("b1")
    for bad in (16, -1, 1 << 40):
        with pytest.raises(RuntimeError, match="outside the part table"):
            losses.compute_iou(score, seg, torch.tensor([bad]), None, None, None)


def test_host_entry_rejects_bad_arguments(lib_built):
    from sonet_b200 import _C, ops
    lib = _C.lib()
    score, seg, label = case("b1")
    B, C, N = score.shape
    off, ids, K = ops.part_table_csr(None, C, "cpu")
    iou = torch.empty(B, dtype=torch.float64)
    args = [score.data_ptr(), seg.data_ptr(), label.data_ptr(), B, C, N, off.data_ptr(),
            ids.data_ptr(), K, iou.data_ptr(), None, None, 1]

    def rc(**change):
        a = list(args)
        for i, v in change.items():
            a[int(i[1:])] = v
        return lib.sonet_seg_iou_cpu_f32(*a)

    assert rc() == 0 and iou[0].item() == G["b1_iou"][0]
    assert rc(a4=0) == -1 and "bad dimension" in _C.last_error()          # C = 0
    assert rc(a5=-1) == -1                                                 # N < 0
    assert rc(a8=0) == -1                                                  # no category
    assert rc(a12=0) == -1 and "thread_num" in _C.last_error()
    for i in (0, 1, 2, 6, 7, 9):
        assert rc(**{"a%d" % i: None}) == -1 and "null" in _C.last_error()
    assert rc(a4=40) == -1 and "part id" in _C.last_error()               # ids 40..49 >= C
    bad = torch.tensor([16], dtype=torch.int64)
    assert rc(a2=bad.data_ptr()) == -1 and "outside the part table" in _C.last_error()
    bad_off = off.clone()
    bad_off[1] = 0                                                         # category 0 empty
    assert rc(a6=bad_off.data_ptr()) == -1 and "parts" in _C.last_error()
    assert rc(a3=0) == 0                                                   # empty batch: no-op
    with pytest.raises(RuntimeError):
        _C.check(rc(a2=bad.data_ptr()), "sonet_seg_iou_cpu_f32")
    # the device entry checks its host-side arguments before any CUDA call
    assert lib.sonet_seg_iou_f32(None, None, None, 2, 50, 64, None, None, 16, None, None, None,
                                 None) == -1
    assert "null" in _C.last_error()
    assert lib.sonet_seg_iou_f32(None, None, None, 2, 0, 64, None, None, 16, None, None, None,
                                 None) == -1


def test_table_validation_and_shape_errors():
    from sonet_b200 import losses, ops
    score, seg, label = case("b1")
    with pytest.raises(RuntimeError, match="part id"):
        ops.part_table_csr([[0, 1], [2, 50]], 50, "cpu")
    with pytest.raises(RuntimeError, match="parts"):
        ops.part_table_csr([[0, 1], []], 50, "cpu")
    with pytest.raises(RuntimeError, match="no category"):
        ops.part_table_csr([], 50, "cpu")
    with pytest.raises(RuntimeError, match="expected score"):
        losses.compute_iou(score, seg[:, :-1], label, None, None, None)
    with pytest.raises(RuntimeError, match="float32"):
        losses.compute_iou(score.double(), seg, label, None, None, None)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.seg_iou(score, seg, label)


def test_custom_table_with_a_repeated_part():
    """A part listed twice counts twice in the mean, as the reference's loop would."""
    from sonet_b200 import losses
    score, seg, label = case("random")
    table = [[0, 1, 1, 2]] + [list(p) for p in losses.SHAPENET_PART_TABLE[1:]]
    meter = losses.PartSegIoU(table)
    meter.update(score[:1], seg[:1], label[:1])
    pred = torch.max(score[0], 0)[1]
    ious = []
    for p in table[0]:
        g, q = seg[0] == p, pred == p
        i, u = int((g & q).sum()), int((g | q).sum())
        ious.append(1.0 if u == 0 else i / (u + 0.0001))
    assert meter.compute()["instance_miou"] == np.asarray(ious).mean()


def test_every_public_callable_of_the_reference_module_exists():
    from sonet_b200 import losses
    names = [str(n) for n in G["ref_public_callables"]]
    assert {"compute_iou", "compute_iou_np_array", "visualize_pc_seg"} <= set(names)
    for n in names:
        assert callable(getattr(losses, n, None)), n


def test_visualize_pc_seg_colours(tmp_path):
    from sonet_b200 import losses
    rs = np.random.RandomState(3)
    cmap = rs.uniform(0, 1, size=(50, 3))
    (tmp_path / "part_color_mapping.json").write_text(__import__("json").dumps(cmap.tolist()))
    score = torch.from_numpy(rs.normal(size=(50, 20)).astype(np.float32))
    seg = torch.from_numpy(rs.randint(0, 50, size=20))
    seg[:3] = 49
    pc = torch.from_numpy(rs.normal(size=(3, 20)).astype(np.float32))
    shown = []

    class Vis:
        def display_current_results(self, d, epoch, i):
            shown.append((d, epoch, i))

    opt = type("Opt", (), {"dataroot": str(tmp_path)})()
    losses.visualize_pc_seg(score, seg, torch.tensor(0), Vis(), opt, pc, 0)
    (d, epoch, i), = shown
    assert (epoch, i) == (1, 1) and list(d) == ["pc_colored_predicted", "pc_colored_gt"]
    colors = np.fabs(cmap * 255).astype(int)
    xyz, pcol = d["pc_colored_predicted"]
    _, gcol = d["pc_colored_gt"]
    assert np.array_equal(xyz, pc.numpy().T)
    assert np.array_equal(pcol, colors[torch.max(score, 0)[1].numpy()])
    want = colors[seg.numpy()]
    want[:3] = 1
    assert np.array_equal(gcol, want)
