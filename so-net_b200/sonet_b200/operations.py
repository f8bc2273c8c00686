"""kNN gathers on SOM nodes — same names and contracts as models/operations.py:19-54.

CUDA float32 inputs outside autograd run the sm_90a gather kernel; anything else (training, CPU
tensors handed in by data loaders) composes the equivalent differentiable torch.gather.
"""
import torch

from . import ops


def knn_gather_by_indexing(som_node, som_node_knn_I):
    """som_node [B,C,N], som_node_knn_I [B,N,K] int64 -> [B,C,N,K] (operations.py:38-54)."""
    B, C, N = som_node.size()
    K = som_node_knn_I.size()[2]
    if (som_node.is_cuda and som_node.dtype == torch.float32 and som_node_knn_I.is_cuda
            and not (torch.is_grad_enabled() and som_node.requires_grad)):
        return ops.knn_gather(som_node.detach().contiguous(),
                              som_node_knn_I.to(torch.int64).contiguous())
    idx = som_node_knn_I.unsqueeze(1).expand(B, C, N, K).contiguous().view(B, C, N * K)
    return torch.gather(som_node, dim=2, index=idx).view(B, C, N, K)


def knn_gather_wrapper(som_node, som_node_knn_I):
    """som_node [B,3,N] (or 2 channels), som_node_knn_I [B,N,K] -> [B,3,N,K] (operations.py:19-35)."""
    C = som_node.size()[1]
    assert C == 3 or C == 2
    return knn_gather_by_indexing(som_node, som_node_knn_I)
