"""CUDA-event times of the encoder's final PointNet (515 -> 768 -> 1024 over B*M = 4096 node rows)
and the max over nodes that follows it, at the cfg-2 shapes (B=64, N=5000, k=3, 8x8 SOM, som_k=9)
and on the tensors a cfg-2 forward feeds it (knn_center_1, knn_feature_1). Times the generic wgmma
layer (`ops.pointwise_layer_tc`, one launch per layer), `ops.rowmax`, and the node-level route the
encoder takes (`ops.nodegemm_pointnet`: split-pack + two bulk-copy-fed GEMMs), whole and launch by
launch. Cases alternate within each repetition, so all see the same clocks; the L2 is flushed
before every timed launch.

    python tools/final_pointnet_time.py [--reps 25] [--json out.json]     (on a GPU box)
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "so-net_b200")):
    sys.path.insert(0, p)
import torch  # noqa: E402

from sonet_b200 import _C, classifier, networks, ops, synth  # noqa: E402

DEV = "cuda"
B, N = 64, 5000


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def _encoder():
    """A cfg-2 classifier after one forward: its encoder holds the final PointNet's inputs."""
    opt = synth.make_opt("classifier", batch_size=B, input_pc_num=N, device="cuda:0")
    cpu = synth.make_opt("classifier", batch_size=B, input_pc_num=N)
    inp = synth.synth_inputs(B, N, seed=0)
    m = classifier.Model(opt)
    m.encoder.load_state_dict(synth.synth_state_dict(networks.Encoder(cpu), seed=1))
    m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
    m.test_model()
    torch.cuda.synchronize()
    return m.encoder


def _cases(enc):
    """name -> (launch(), executed FLOPs per launch in the hi/lo split, or 0)."""
    pn = enc.final_pointnet
    x0, x1 = enc.knn_center_1.contiguous(), enc.knn_feature_1.contiguous()
    l1, l2 = pn.layers
    b1, inv1, s1 = l1._tc_params()
    b2, inv2, s2 = l2._tc_params()
    c1, c2 = l1.conv.out_channels, l2.conv.out_channels
    cin = x0.shape[1] + x1.shape[1]
    rows = x0.shape[0] * x0.shape[2]
    h = ops.pointwise_layer_tc(x0, b1, inv1, s1, c1, l1.activation, x1=x1)
    out = ops.pointwise_layer_tc(h, b2, inv2, s2, c2, None)
    f1, f2 = 3 * 2.0 * rows * cin * c1, 3 * 2.0 * rows * c1 * c2

    def old1():
        ops.pointwise_layer_tc(x0, b1, inv1, s1, c1, l1.activation, x1=x1)

    def old2():
        ops.pointwise_layer_tc(h, b2, inv2, s2, c2, None)

    def old_chain():
        ops.pointwise_layer_tc(ops.pointwise_layer_tc(x0, b1, inv1, s1, c1, l1.activation, x1=x1),
                               b2, inv2, s2, c2, None)

    lib = _C.lib()
    st = ops._stream(x0)
    img0 = torch.empty(lib.sonet_nodegemm_image_bytes(rows, cin, 0), dtype=torch.uint8, device=DEV)
    img1 = torch.empty(lib.sonet_nodegemm_image_bytes(rows, c1, 0), dtype=torch.uint8, device=DEV)
    Bc, C0, P = x0.shape
    a1 = ops.act_code(l1.activation)

    def pack():
        ops._call("sonet_nodegemm_split_pack", _C.ptr(x0), C0, _C.ptr(x1), cin - C0, Bc, P, 0,
                  _C.ptr(img0), st)

    def new1():
        ops._call("sonet_nodegemm_tc_forward", _C.ptr(img0), cin, Bc, P, _C.ptr(b1), float(inv1),
                  _C.ptr(s1), c1, a1, 0, _C.ptr(img1), None, st)

    def new2():
        ops._call("sonet_nodegemm_tc_forward", _C.ptr(img1), c1, Bc, P, _C.ptr(b2), float(inv2),
                  _C.ptr(s2), c2, ops.ACT_NONE, 0, None, _C.ptr(out), st)

    def new_chain():
        ops.nodegemm_pointnet(x0, x1, (b1, inv1, s1), c1, l1.activation, (b2, inv2, s2), c2)

    pack(), new1()
    assert torch.equal(ops.nodegemm_pointnet(x0, x1, (b1, inv1, s1), c1, l1.activation,
                                             (b2, inv2, s2), c2), out), "routes differ"
    return {
        "nodegemm split-pack %d channels" % cin: (pack, 0),
        "nodegemm %d->%d, images out" % (cin, c1): (new1, f1),
        "nodegemm %d->%d, tensor out" % (c1, c2): (new2, f2),
        "node-level chain, pack + both layers": (new_chain, f1 + f2),
        "pointwise_tc %d->%d (%d rows)" % (cin, c1, rows): (old1, f1),
        "pointwise_tc %d->%d (%d rows)" % (c1, c2, rows): (old2, f2),
        "rowmax [%d,%d,%d]" % tuple(out.shape): (lambda: ops.rowmax(out), 0),
        "generic chain, both layers": (old_chain, f1 + f2),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=25)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    card = _card()
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=DEV)
    with torch.no_grad():
        cases = _cases(_encoder())
        for fn, _ in cases.values():      # warm-up: module load, smem attribute
            fn()
        torch.cuda.synchronize()
        ms = {name: [] for name in cases}
        for _ in range(args.reps):
            for name, (fn, _) in cases.items():
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                ms[name].append(e0.elapsed_time(e1))
    res = {}
    for name, (_, flops) in cases.items():
        t = sorted(ms[name])
        med = t[len(t) // 2]
        res[name] = dict(median_ms=med, min_ms=t[0], max_ms=t[-1],
                         executed_tflops=flops / med / 1e9)
        print("%-44s %.4f ms (min %.4f, max %.4f)%s"
              % (name, med, t[0], t[-1],
                 "  %.0f TFLOP/s executed" % res[name]["executed_tflops"] if flops else ""))
    print("card:", card, "| medians of %d alternated launches, L2 flushed" % args.reps)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card, reps=args.reps, kernels=res), f, indent=1)


if __name__ == "__main__":
    main()
