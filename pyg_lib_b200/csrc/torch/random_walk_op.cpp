// torch.ops.pyg.random_walk on CUDA tensors — schema verbatim from pyg_lib/csrc/sampler/random_walk.cpp:29-33, result
// equal to the reference's CUDA kernel (sampler/cuda/random_walk_kernel.cu:53-85) under the same CUDA generator state.
// The draws come from at::rand with the reference's shape, dtype, device and stream, so the values and the generator's
// advance are ATen's own (also under CUDA-graph capture); pygb200_random_walk then walks on them and writes the
// [S, walk_length + 1] result directly.
#include "common.h"

namespace pyg {
namespace sampler {
namespace {

at::Tensor random_walk_cuda(const at::Tensor& rowptr, const at::Tensor& col, const at::Tensor& seed, int64_t walk_length, double p,
                            double q) {
  TORCH_CHECK(rowptr.defined() && col.defined() && seed.defined(), "random_walk: 'rowptr', 'col' and 'seed' must be defined");
  TORCH_CHECK(rowptr.is_cuda() && col.is_cuda() && seed.is_cuda(), "pyg_lib_b200: random_walk expects CUDA tensors (no CPU fallback)");
  const auto st = seed.scalar_type();
  // at::checkAllSameType of the reference's wrapper (random_walk.cpp:19-21) + what the kernel assumes
  TORCH_CHECK(rowptr.scalar_type() == st && col.scalar_type() == st, "random_walk: expected 'rowptr' (", rowptr.scalar_type(),
              "), 'col' (", col.scalar_type(), ") and 'seed' (", st, ") to have the same dtype");
  TORCH_CHECK(st == at::kLong || st == at::kInt, "random_walk: index tensors must be int64 or int32, got ", st);
  TORCH_CHECK(rowptr.device() == seed.device() && col.device() == seed.device(), "random_walk: tensors must live on one device");
  TORCH_CHECK(rowptr.dim() == 1 && col.dim() == 1 && seed.dim() == 1, "random_walk: expected one-dimensional tensors");
  TORCH_CHECK(rowptr.is_contiguous() && col.is_contiguous() && seed.is_contiguous(), "random_walk: expected contiguous tensors");
  TORCH_CHECK(rowptr.numel() >= 1, "random_walk: 'rowptr' must have at least one element");
  TORCH_CHECK(p == 1 && q == 1, "Uniform sampling required for now");
  TORCH_CHECK(walk_length >= 0, "random_walk: 'walk_length' must be non-negative, got ", walk_length);

  c10::cuda::CUDAGuard guard(seed.device());
  cudaStream_t stream = at::cuda::getCurrentCUDAStream();
  const int64_t S = seed.size(0);
  // drawn even when S == 0 (the reference draws before its launch fails), so the generator advances as there
  const at::Tensor rand = at::rand({walk_length, S}, seed.options().dtype(at::kFloat));
  at::Tensor out = rowptr.new_empty({S, walk_length + 1});
  PYGB_TORCH_CALL(pygb200_random_walk(rowptr.data_ptr(), col.data_ptr(), rowptr.numel() - 1, col.numel(), seed.data_ptr(), S,
                                      walk_length, rand.data_ptr<float>(), out.data_ptr(), st == at::kInt, stream));
  return out;
}

}  // namespace

TORCH_LIBRARY_FRAGMENT(pyg, m) {
  m.def(TORCH_SELECTIVE_SCHEMA(
      "pyg::random_walk(Tensor rowptr, Tensor col, Tensor seed, int "
      "walk_length, float p, float q) -> Tensor"));
}

TORCH_LIBRARY_IMPL(pyg, CUDA, m) {
  m.impl(TORCH_SELECTIVE_NAME("pyg::random_walk"), TORCH_FN(random_walk_cuda));
}

}  // namespace sampler
}  // namespace pyg
