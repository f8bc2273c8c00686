"""Drop-in for the reference's pybind11 plugin module `index_max`
(models/index_max_ext/index_max.cpp:154-159): same four callables, same tensor contracts.

    forward_cuda(data f32 [B,C,N] cuda contiguous, index i32 [B,N] cuda contiguous, K) -> i32 [B,C,K]
    forward_cuda_shared_mem(...)            same result (the reference's smem variant)
    forward_cpu(data, index, K)             host tensors, single thread
    forward_multi_thread_cpu(data, index, K, thread_num)

The CUDA entry points run the sm_90a kernel of libsonet_b200 (csrc/index_max.cu) and raise
RuntimeError on non-CUDA / non-contiguous inputs like the reference's CHECK_INPUT
(index_max.cpp:119-121). The host entry points are the plugin's own CPU API (C++ in the same
library); they are never used as a fallback for the CUDA path.
"""
import torch

from . import _C, ops


def forward_cuda(data, index, K):
    return ops.index_max(data, index, K)


def forward_cuda_shared_mem(data, index, K):
    return ops.index_max(data, index, K)


def forward_cuda_with_values(data, index, K):
    """Extension: also returns data gathered at the arg-max (the fused models/networks.py:185)."""
    return ops.index_max(data, index, K, with_values=True)


def _cpu(data, index, K, threads):
    if data.is_cuda or index.is_cuda:
        raise RuntimeError("forward_cpu expects host tensors")
    if data.dtype != torch.float32 or index.dtype != torch.int32:
        raise RuntimeError("forward_cpu expects float32 data and int32 index")
    data = data.contiguous()
    index = index.contiguous()
    B, C, N = data.shape
    out = torch.zeros((B, C, K), dtype=torch.int32)
    _C.check(_C.lib().sonet_index_max_cpu_f32(data.data_ptr(), index.data_ptr(), B, C, N, int(K),
                                              out.data_ptr(), int(threads)),
             "sonet_index_max_cpu_f32")
    return out


def forward_cpu(data, index, K):
    return _cpu(data, index, K, 1)


def forward_multi_thread_cpu(data, index, K, thread_num):
    return _cpu(data, index, K, thread_num)
