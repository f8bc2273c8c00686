"""sonet_b200 — H100-native (sm_90a) implementation of SO-Net's per-batch forward hot path.

Host side = Python/PyTorch mirroring the reference's module API (lijx10/SO-Net: util/som.py,
models/{operations,layers,networks,losses,classifier,segmenter,autoencoder}.py and the `index_max`
plugin); device side = hand-written CUDA in libsonet_b200.so behind the C-ABI of
include/sonet_b200.h. See README.md and INTEGRATION.md at the repository root.
"""
from . import _C  # noqa: F401  (does not load the library until first use)

__version__ = "0.2.0"
