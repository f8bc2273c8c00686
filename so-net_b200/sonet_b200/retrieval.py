"""SHREC'16 retrieval ranking of shrec16/test.py:41-99 on the project's kernels.

The script collects the classifier's scores, predicted labels and model ids of the whole test split
(test.py:41-61), then for every shape ranks the shapes of the same predicted label by the L2
distance of their scores and writes one text file per shape, named by its `%06d` model id, with at
most 1000 rows `id distance` (np.savetxt fmt='%06d %f'). Here the ranking is one device call
(ops.retrieval_rank) and the files come from a native formatter:

    bank = RetrievalBank()
    for batch in loader:
        model.forward()
        bank.update(model.score, model_ids)         # stays on the device
    bank.rank().write(output_folder)                 # same names, same bytes

or, from collected tensors, rank_same_label(feature, model_ids).write(output_folder).
"""
import os

import torch

from . import ops


class RetrievalResult:
    """A ranking of every item: idx [Q,k] (positions), dist [Q,k], count [Q], label [Q], and the
    items' model ids [Q], all on the device they were computed on. Reading it on the host
    (`host()`, `files()`, `write()`) synchronises and raises if a label was outside the range."""

    def __init__(self, idx, dist, count, label, model_ids):
        self.idx, self.dist, self.count, self.label, self.model_ids = idx, dist, count, label, model_ids
        self._host = None

    def host(self):
        """(idx, dist, count, label, model_ids) as CPU tensors, checked."""
        if self._host is None:
            h = tuple(t.cpu() for t in (self.idx, self.dist, self.count, self.label, self.model_ids))
            bad = torch.nonzero(h[2] < 0).flatten()
            if bad.numel():
                q = int(bad[0])
                raise RuntimeError("retrieval: label %d of item %d is outside [0, num_labels) (%d "
                                   "such items)" % (int(h[3][q]), q, bad.numel()))
            self._host = h
        return self._host

    def files(self, threads=None):
        """{file name: bytes} of the script's output. A model id that repeats names one file, and
        the last item with that id wins, as the script's successive writes do."""
        idx, dist, count, _, ids = self.host()
        text, offsets = ops.retrieval_format(ids, idx, dist, count, threads=threads)
        offsets = offsets.tolist()
        out = {}
        for q, mid in enumerate(ids.tolist()):
            out["%06d" % mid] = text[offsets[q]:offsets[q + 1]]
        return out

    def write(self, output_folder, threads=None):
        """Write one file per model id into output_folder (which must exist, as for the script)."""
        for name, data in self.files(threads).items():
            with open(os.path.join(output_folder, name), "wb") as f:
                f.write(data)


def rank_same_label(feature, model_ids, label=None, max_results=1000, num_labels=None):
    """Rank every item against the items of its label (shrec16/test.py:64-99): feature [Q,D] f32,
    model_ids [Q] (any integer dtype, any device), label [Q] int64 or None for the row argmax.
    Returns a RetrievalResult; nothing is synchronised until it is read on the host."""
    feature = feature.detach().to(torch.float32).contiguous()
    if label is not None:
        label = label.detach().to(device=feature.device, dtype=torch.int64).contiguous()
    ids = model_ids.detach().to(device=feature.device, dtype=torch.int64).contiguous()
    if tuple(ids.shape) != (feature.shape[0],):
        raise RuntimeError("rank_same_label: model_ids must have shape [Q=%d], got %s"
                           % (feature.shape[0], tuple(ids.shape)))
    idx, dist, count, lab = ops.retrieval_rank(feature, label, num_labels, max_results)
    return RetrievalResult(idx, dist, count, lab, ids)


class RetrievalBank:
    """Collects scores and model ids batch by batch (shrec16/test.py:41-61) on the scores' device;
    rank() ranks the whole collection with the predicted label (argmax of the scores)."""

    def __init__(self):
        self._scores, self._ids = [], []

    def update(self, score, model_ids):
        score = score.detach()
        if score.dim() != 2:
            raise RuntimeError("RetrievalBank.update: score must be [B,D], got %s" % (tuple(score.shape),))
        if self._scores and score.shape[1] != self._scores[0].shape[1]:
            raise RuntimeError("RetrievalBank.update: score width %d differs from %d"
                               % (score.shape[1], self._scores[0].shape[1]))
        ids = model_ids.detach().reshape(-1).to(device=score.device, dtype=torch.int64)
        if ids.numel() != score.shape[0]:
            raise RuntimeError("RetrievalBank.update: %d model ids for %d scores"
                               % (ids.numel(), score.shape[0]))
        self._scores.append(score.to(torch.float32, copy=True))
        self._ids.append(ids.clone())

    def __len__(self):
        return sum(s.shape[0] for s in self._scores)

    def rank(self, max_results=1000):
        if not self._scores:
            raise RuntimeError("RetrievalBank.rank: no scores collected")
        return rank_same_label(torch.cat(self._scores), torch.cat(self._ids),
                               max_results=max_results)
