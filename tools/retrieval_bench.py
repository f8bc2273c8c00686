"""Time the SHREC'16 retrieval ranking (shrec16/test.py:64-99) at the test split's size, Q = 10,265
shapes with D = 55 scores, with Zipf-like predicted classes and with one class:

  reference   the script's per-query loop restated on CUDA tensors: eq mask, nonzero, gather,
              torch.norm, torch.sort and the two .cpu() copies (file writing excluded), host clock
  rank        ops.retrieval_rank, k = 1000: `call` = eager call, `graph` = the same call replayed
              from a CUDA graph; CUDA events
  host        ops.retrieval_rank on host tensors (C++ host entry), torch's thread count
  savetxt     np.savetxt of the reference's rows, one file per query, over the first --savetxt-files
              queries (per-file time, and that times Q)
  native      RetrievalResult.write(): copy to the host, native formatter and every file write

    python tools/retrieval_bench.py [--out results.jsonl]

Prints one JSON line per class layout with medians in ms, and the GPU's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "so-net_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from sonet_b200 import ops, retrieval  # noqa: E402

Q, D, K = 10265, 55, 1000


def host_ms(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def event_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def reference_loop(feature_map, predicted_labels, model_name_ids, queries):
    """The script's loop body (test.py:65-88) on CUDA tensors, without the file write."""
    out = []
    for i in queries:
        feature = feature_map[i]
        same = torch.nonzero(torch.eq(predicted_labels, predicted_labels[i])).squeeze(1)
        distance = torch.norm(feature.unsqueeze(0) - feature_map[same], p=2, dim=1)
        dsorted, order = torch.sort(distance)
        out.append((model_name_ids[same][order].cpu().numpy(), dsorted.cpu().numpy()))
    return out


def layout(kind, rs):
    if kind == "single":
        lab = np.zeros(Q, dtype=np.int64)
    else:
        p = 1.0 / np.arange(1, D + 1) ** 1.2
        lab = rs.choice(D, size=Q, p=p / p.sum())
    score = (rs.normal(size=(Q, D)) * 0.5).astype(np.float32)
    score[np.arange(Q), lab] += 4.0
    return score


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--savetxt-files", type=int, default=1000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("retrieval_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    rs = np.random.RandomState(2016)
    ids_h = torch.from_numpy(rs.choice(10 ** 6, size=Q, replace=False).astype(np.int64))
    rows = []
    for kind in ("zipf", "single"):
        score_h = torch.from_numpy(layout(kind, rs))
        score = score_h.to(dev)
        ids = ids_h.to(dev)
        pred = torch.max(score, 1)[1]
        r = dict(kind=kind, Q=Q, D=D, k=K, largest_class=int(torch.bincount(pred).max()),
                 gpu=gpu_info(), cpu_threads=torch.get_num_threads())
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ref = reference_loop(score, pred, ids, range(Q))
        torch.cuda.synchronize()
        r["reference_loop_ms"] = (time.perf_counter() - t0) * 1e3
        call = lambda: ops.retrieval_rank(score, k=K)           # noqa: E731
        r["rank_call_ms"] = event_ms(call, a.reps)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            call()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = call()
        r["rank_graph_ms"] = event_ms(graph.replay, a.reps)
        torch.cuda.synchronize()
        # the same distances as the reference loop (within 4 ulp), and the same count
        idx, dist, count = (t.cpu() for t in out[:3])
        worst = 0
        for i in range(0, Q, 97):
            n = min(len(ref[i][1]), K)
            assert int(count[i]) == n
            a32, b32 = dist[i, :n].numpy().view(np.int32), ref[i][1][:n].view(np.int32)
            worst = max(worst, int(np.abs(a32.astype(np.int64) - b32).max()))
        r["max_ulp_vs_reference_loop_sampled"] = worst      # the loop sums in fp32 on the device
        r["host_ms"] = host_ms(lambda: ops.retrieval_rank(score_h, k=K), max(2, a.reps // 5))
        res = retrieval.rank_same_label(score, ids, max_results=K)
        with tempfile.TemporaryDirectory() as tmp:
            n_files = min(a.savetxt_files, Q)
            t0 = time.perf_counter()
            for i in range(n_files):
                nn_result = np.transpose(np.vstack(ref[i]))
                np.savetxt(os.path.join(tmp, "%06d" % int(ids_h[i])), nn_result[0:K, :],
                           fmt="%06d %f", delimiter=" ")
            per_file = (time.perf_counter() - t0) * 1e3 / n_files
            r["savetxt_ms_per_file"] = per_file
            r["savetxt_ms_all_files_scaled"] = per_file * Q
            def native():
                res._host = None                             # include the copy to the host
                res.write(tmp)
            r["native_write_ms"] = host_ms(native, max(2, a.reps // 5))
        rows.append(r)
        print(json.dumps(r), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
