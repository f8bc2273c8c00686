"""Drop-in boundary: the reference's own models/{classifier,segmenter,autoencoder}.py (unmodified,
as the bytecode build product oracle/_ref/pyref that __graft_entry__.build() makes from the
reference tree) run on top of sonet_b200's networks — construction on CPU, and full
set_input()/test_model() forwards on CUDA against the reference's own golden outputs."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(ROOT, "tests", "_dropin_run.py")


def _roots():
    sys.path.insert(0, ROOT)
    from oracle import build as obuild
    out = []
    if obuild.pyref_root():
        out.append(obuild.pyref_root())
    return out


def _run(root, device):
    r = subprocess.run([sys.executable, SCRIPT, root, device], capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and "DROPIN_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def test_reference_model_files_construct_on_our_networks():
    roots = _roots()
    if not roots:
        pytest.skip("no reference tree / bytecode here")
    for root in roots:                       # the sourceless .pyc build product
        _run(root, "cpu")


@pytest.mark.gpu
def test_reference_model_files_forward_on_cuda():
    """models/classifier.py:64-105, models/segmenter.py:66-135, models/autoencoder.py:56-126 run
    unchanged on the CUDA path and reproduce the goldens the reference produced on CPU."""
    roots = _roots()
    if not roots:
        pytest.fail("oracle/_ref/pyref missing: run __graft_entry__.build() where the reference "
                    "tree is available")
    out = _run(roots[-1], "cuda:0")
    assert "classifier.Model ok" in out and "segmenter.Model ok" in out \
        and "autoencoder.Model ok" in out
