"""Drop-in installation into a checkout of the reference (lijx10/SO-Net).

    import sonet_b200.install; sonet_b200.install.install("/path/to/SO-Net")
    from models import classifier          # the reference's file, byte-identical
    model = classifier.Model(opt)          # now built from the H100 networks

Registers this package's modules under the names the reference imports
(models/networks.py:10-17, models/losses.py:9): `index_max`, `util.som`, `models.operations`,
`models.layers`, `models.networks`, `models.losses` — so models/{classifier,segmenter,
autoencoder}.py and the train/test scripts run unchanged. `faiss`, `matplotlib` are no longer
needed by the hot path (stubs are registered only if the real packages are missing, because
models/networks.py imports matplotlib unconditionally).
"""
import importlib
import os
import sys
import types


def install(reference_root=None, stub_plotting=True):
    from . import index_max, layers, losses, networks, operations, som

    sys.modules["index_max"] = index_max
    if reference_root is not None and reference_root not in sys.path:
        sys.path.insert(0, reference_root)

    if stub_plotting:
        for name in ("matplotlib", "matplotlib.pyplot", "mpl_toolkits", "mpl_toolkits.mplot3d"):
            try:
                importlib.import_module(name)
            except Exception:
                sys.modules[name] = types.ModuleType(name)
        m3d = sys.modules["mpl_toolkits.mplot3d"]
        if not hasattr(m3d, "Axes3D"):
            m3d.Axes3D = object

    # `util` and `models` stay the reference's packages (visualizer, train loops, Model classes);
    # only the hot-path modules inside them are replaced.
    for pkg_name in ("util", "models"):
        if pkg_name not in sys.modules:
            pkg = types.ModuleType(pkg_name)
            root = os.path.join(reference_root or "", pkg_name)
            pkg.__path__ = [root] if os.path.isdir(root) else []
            sys.modules[pkg_name] = pkg
    sys.modules["util.som"] = som
    sys.modules["util"].som = som
    for name, mod in (("operations", operations), ("layers", layers), ("networks", networks),
                      ("losses", losses)):
        sys.modules["models." + name] = mod
        setattr(sys.modules["models"], name, mod)
    return sys.modules["models"]
