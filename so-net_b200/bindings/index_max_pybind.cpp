// index_max_pybind.cpp — the pybind11/ATen binding a maintainer of lijx10/SO-Net would compile in
// place of models/index_max_ext/index_max.cpp (:114-159): the same module name and the same four
// callables, implemented over the C-ABI of libsonet_b200 (include/sonet_b200.h). The repository's
// own product path uses the equivalent ctypes binding (sonet_b200/_C.py); this file exists so that
// the INTEGRATION.md recipe is compiled and exercised by tests/test_pybind_binding.py.
//
//   forward_cuda(data f32 [B,C,N] cuda contiguous, index i32 [B,N] cuda contiguous, K) -> i32 [B,C,K]
//   forward_cuda_shared_mem(...)      same kernel (the reference's smem variant is a tuning variant)
//   forward_cpu(data, index, K), forward_multi_thread_cpu(data, index, K, thread_num)   host tensors
#include <c10/cuda/CUDAStream.h>
#include <torch/extension.h>

#include "sonet_b200.h"

namespace {

void check_inputs(const torch::Tensor& data, const torch::Tensor& index, bool cuda) {
  TORCH_CHECK(data.is_cuda() == cuda && index.is_cuda() == cuda,
              cuda ? "data/index must be CUDA tensors" : "data/index must be host tensors");
  TORCH_CHECK(data.is_contiguous() && index.is_contiguous(), "data/index must be contiguous");
  TORCH_CHECK(data.scalar_type() == torch::kFloat32 && index.scalar_type() == torch::kInt32,
              "data must be float32 and index int32");
  TORCH_CHECK(data.dim() == 3 && index.dim() == 2 && index.size(0) == data.size(0) &&
                  index.size(1) == data.size(2),
              "expected data [B,C,N] and index [B,N]");
}

torch::Tensor forward_cuda(const torch::Tensor data, const torch::Tensor index, const int K) {
  check_inputs(data, index, true);
  auto out = torch::empty({data.size(0), data.size(1), K}, data.options().dtype(torch::kInt32));
  const int rc = sonet_index_max_f32(
      data.data_ptr<float>(), index.data_ptr<int>(), static_cast<int>(data.size(0)),
      static_cast<int>(data.size(1)), static_cast<int>(data.size(2)), K, out.data_ptr<int>(),
      /*out_val=*/nullptr, c10::cuda::getCurrentCUDAStream(data.get_device()).stream());
  TORCH_CHECK(rc == 0, sonet_last_error_string());
  return out;
}

torch::Tensor forward_multi_thread_cpu(const torch::Tensor data, const torch::Tensor index, const int K,
                                       const int thread_num) {
  check_inputs(data, index, false);
  auto out = torch::zeros({data.size(0), data.size(1), K}, data.options().dtype(torch::kInt32));
  const int rc = sonet_index_max_cpu_f32(data.data_ptr<float>(), index.data_ptr<int>(),
                                         static_cast<int>(data.size(0)), static_cast<int>(data.size(1)),
                                         static_cast<int>(data.size(2)), K, out.data_ptr<int>(),
                                         thread_num);
  TORCH_CHECK(rc == 0, sonet_last_error_string());
  return out;
}

torch::Tensor forward_cpu(const torch::Tensor data, const torch::Tensor index, const int K) {
  return forward_multi_thread_cpu(data, index, K, 1);
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("forward_cpu", &forward_cpu, "index_max forward (host, single thread)");
  m.def("forward_multi_thread_cpu", &forward_multi_thread_cpu, "index_max forward (host, threads)");
  m.def("forward_cuda", &forward_cuda, "index_max forward (sm_90a kernel of libsonet_b200)");
  m.def("forward_cuda_shared_mem", &forward_cuda, "same kernel");
}
