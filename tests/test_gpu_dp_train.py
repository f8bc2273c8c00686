"""-m gpu: DataParallelTraining end to end (tests/_dp_train_run.py). Two ranks train the classifier
(a ragged global batch of 5), the segmenter and the auto-encoder for 3 optimize() steps:

  * over gloo, both ranks on one GPU (torch.distributed.run --nproc-per-node 2), and over NCCL
    on two GPUs (skipped with fewer);
  * after the steps every parameter, gradient and BatchNorm buffer is bit-identical on the ranks;
  * the global-batch loss (the shard losses weighted by B_r / Bg), the running statistics and the
    parameters agree with a one-process DataParallelTraining run over the global batch.

Whole-model bit-identity with the one-process run is not expected: the convolution, linear and
loss gradients are sums over each shard's clouds before the ranks' sums are added, and cuDNN's
first layer is not even run-to-run reproducible (test_gpu_fp16_mode.py:
test_train_step_ignores_fp16_mode). The bars below are 2.5x the largest error measured on one H100
80GB HBM3 (700 W power limit), relative to each tensor's largest magnitude; the run prints how many
tensors match bit for bit."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUN = os.path.join(ROOT, "tests", "_dp_train_run.py")
TASKS = ("classifier", "segmenter", "autoencoder")

# 2.5x the largest error measured over two runs (see the module docstring), per task and quantity.
# Three Adam steps of lr 1e-3 move every parameter with a near-zero gradient by up to 3e-3 either
# way, so a parameter tensor's error is that of the steps' signs, not of the exchange; the decoder's
# first up-convolution sees 2x2 maps, whose running means are small against their largest value.
BAR = {"classifier": {"loss": 3.9e-3, "running": 1.0e-2, "param": 0.126},
       "segmenter": {"loss": 2.1e-3, "running": 1.65e-2, "param": 8.9e-2},
       "autoencoder": {"loss": 8.8e-2, "running": 0.72, "param": 0.176}}


def _env():
    env = dict(os.environ)
    for k in ("RANK", "LOCAL_RANK", "WORLD_SIZE", "LOCAL_WORLD_SIZE", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    return env


def _run(out_dir, backend, nproc, port):
    if nproc == 1:
        cmd = [sys.executable, RUN, out_dir, backend]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node",
               str(nproc), "--master-addr", "127.0.0.1", "--master-port", str(port), RUN, out_dir,
               backend]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=_env())
    assert r.returncode == 0 and r.stdout.count("DP_TRAIN_OK") == nproc, \
        r.stdout[-2000:] + r.stderr[-4000:]


def _load(out_dir, task, world, rank):
    return torch.load(os.path.join(out_dir, "%s_w%d_r%d.pt" % (task, world, rank)))


def _compare(out_dir):
    report = {}
    for task in TASKS:
        r0, r1, ref = (_load(out_dir, task, 2, 0), _load(out_dir, task, 2, 1),
                       _load(out_dir, task, 1, 0))
        assert set(r0) == set(r1) == set(ref), task
        for k in r0:
            if k in ("losses", "rows"):
                continue
            assert torch.equal(r0[k], r1[k]), "%s: %s differs between the ranks" % (task, k)
        Bg = r0["rows"] + r1["rows"]
        worst = dict.fromkeys(BAR[task], (0.0, ""))
        for s, (a, b) in enumerate(zip(r0["losses"], r1["losses"])):
            glob = (r0["rows"] * a + r1["rows"] * b) / Bg
            err = abs(glob - ref["losses"][s]) / abs(ref["losses"][s])
            worst["loss"] = max(worst["loss"], (err, "step %d" % s))
        same = total = 0
        for k, want in ref.items():
            if not k.startswith("state.") or k.endswith("num_batches_tracked"):
                if k.endswith("num_batches_tracked"):
                    assert torch.equal(r0[k], want), k
                continue
            got = r0[k]
            total += 1
            same += int(torch.equal(got, want))
            err = float((got.double() - want.double()).abs().max()
                        / want.double().abs().max().clamp(min=1e-30))
            kind = "running" if k.endswith(("running_mean", "running_var")) else "param"
            worst[kind] = max(worst[kind], (err, k))
        report[task] = worst
        print("\n[dp-train] %s: %d of %d state tensors bit-identical to the one-process run; worst "
              "relative errors: %s" % (task, same, total,
                                       ", ".join("%s %.3g (%s)" % (q, e, w) for q, (e, w) in worst.items())))
    for task, worst in report.items():
        for q, (e, w) in worst.items():
            assert e <= BAR[task][q], "%s: %s error %.3g > %.3g at %s" % (task, q, e, BAR[task][q], w)


def test_gloo_two_ranks_on_one_gpu_match_one_process(tmp_path):
    _run(str(tmp_path), "gloo", 1, None)
    _run(str(tmp_path), "gloo", 2, 29541)
    _compare(str(tmp_path))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_nccl_two_gpus_match_one_process(tmp_path):
    _run(str(tmp_path), "nccl", 1, None)
    _run(str(tmp_path), "nccl", 2, 29543)
    _compare(str(tmp_path))
