"""make_golden_som_single.py — generates ONLY tests/golden/som_single.npz from the REFERENCE ITSELF:
the single-cloud SOM class of util/som.py:17-173 (the one data/build_som/save_som.ipynb trains per
shape), run on the CPU (gpu_id=-1) on a seeded cloud, by the recipe of oracle/make_golden.py's SOM
fixtures. What sonet_b200.som.SOM must match.

Run in the build container only (needs the reference checkout):

    python tools/make_golden_som_single.py [--force]

Stored: x [3,N], node_init_value [3,M], the nodes after batch_update(x, 0) and then
batch_update(x, 7), the nodes after optimize(x), and query(x)'s mask row maxima for those nodes.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "so-net_b200"))

from oracle import ref_shims  # noqa: E402
from oracle.make_golden import GOLDEN, som_cloud  # noqa: E402

ROWS, N, SEED = 8, 900, 31


def main():
    torch.set_num_threads(4)
    ref = ref_shims.install(use_ref_plugin=False)
    x = torch.from_numpy(som_cloud(np.random.RandomState(SEED), 1, N)[0])      # [3, N]
    som = ref.som.SOM(ROWS, ROWS, 3, -1)
    out = dict(x=x.numpy(), rows=np.int64(ROWS), node_init_value=som.node_init_value.numpy().copy())
    som.node_init()
    som.batch_update(x, 0)
    out["node_after_1"] = som.node.numpy().copy()
    som.batch_update(x, 7)
    out["node_after_2"] = som.node.numpy().copy()
    som.optimize(x)
    out["node_optimized"] = som.node.numpy().copy()
    mask, row_max = som.query(x)
    out["query_row_max"] = row_max.numpy().copy()
    out["query_argmax"] = mask.argmax(dim=1).numpy().astype(np.int64)
    path = os.path.join(GOLDEN, "som_single.npz")
    assert not os.path.exists(path) or "--force" in sys.argv, "%s exists (--force rewrites)" % path
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
