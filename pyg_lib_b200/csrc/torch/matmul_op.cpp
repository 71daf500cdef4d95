// torch.ops.pyg.segment_matmul / grouped_matmul on CUDA tensors + the Autograd kernel for
// segment_matmul.  Schemas verbatim from pyg_lib/csrc/ops/matmul.cpp:63-68; dispatch keys as
// pyg_lib/csrc/ops/cuda/matmul_kernel.cu:323-328 (CUDA) and ops/autograd/matmul_kernel.cpp:121-124.
#include <torch/autograd.h>

#include "common.h"

namespace pyg {
namespace ops {
namespace {

int dtype_code(at::ScalarType t) {
  switch (t) {
    case at::kFloat: return PYGB200_F32;
    case at::kBFloat16: return PYGB200_BF16;
    case at::kHalf: return PYGB200_F16;
    default: TORCH_CHECK(false, "pyg_lib_b200: matmul supports float32, bfloat16 and float16, got ", t);
  }
}

unsigned mm_flags() {
  // fp32 inputs follow torch.set_float32_matmul_precision like the reference (matmul_kernel.cu:159-165)
  return at::globalContext().float32MatmulPrecision() != at::Float32MatmulPrecision::HIGHEST ? PYGB200_MM_ALLOW_TF32 : 0u;
}

// `ptr` must be a segment pointer over the rows of the input: ptr[0] == 0, non-decreasing, ptr[-1] == N (the reference
// raises through split_with_sizes on the host sizes, matmul_kernel.cu:307-313).  A host ptr is checked here; a device ptr
// is checked by the kernels while they read it and reported by the next matmul call (no sync on the way).
at::Tensor ptr_on_device(const at::Tensor& ptr, const at::Device& dev, int64_t N) {
  // int64 only, like the reference ("expected scalar type Long", matmul_kernel.cu:308-309)
  TORCH_CHECK(ptr.scalar_type() == at::kLong, "expected scalar type Long but found ", ptr.scalar_type());
  if (ptr.device().is_cpu() && ptr.numel() > 0) {
    const at::Tensor pc = ptr.contiguous();
    const int64_t* v = pc.data_ptr<int64_t>();
    bool ok = v[0] == 0 && v[pc.numel() - 1] == N;
    for (int64_t i = 1; i < pc.numel() && ok; ++i) ok = v[i] >= v[i - 1];
    TORCH_CHECK(ok, "segment_matmul: 'ptr' must start at 0, be non-decreasing and end at input.size(0) = ", N);
  }
  return ptr.device() == dev ? ptr.contiguous() : ptr.contiguous().to(dev, /*non_blocking=*/true);
}

at::Tensor segment_matmul_cuda(const at::Tensor& input, const at::Tensor& ptr, const at::Tensor& other) {
  TORCH_CHECK(input.is_cuda() && other.is_cuda(), "pyg_lib_b200: segment_matmul expects CUDA tensors");
  TORCH_CHECK(input.dim() == 2 && ptr.dim() == 1 && other.dim() == 3, "segment_matmul: expected 2-D input, 1-D ptr, 3-D other");
  TORCH_CHECK(input.scalar_type() == other.scalar_type(), "segment_matmul: input and other must have the same dtype");
  TORCH_CHECK(other.size(1) == input.size(1), "segment_matmul: other.size(1) must equal input.size(-1)");
  TORCH_CHECK(ptr.numel() == other.size(0) + 1, "segment_matmul: ptr.numel() must equal other.size(0) + 1");
  c10::cuda::CUDAGuard guard(input.device());
  const at::Tensor x = input.contiguous(), w = other.contiguous();
  const at::Tensor p = ptr_on_device(ptr, input.device(), input.size(0));
  at::Tensor out = input.new_empty({x.size(0), w.size(2)});
  PYGB_TORCH_CALL(pygb200_segment_matmul(x.data_ptr(), p.data_ptr<int64_t>(), w.data_ptr(), nullptr, out.data_ptr(),
                                         x.size(0), x.size(1), w.size(2), w.size(0), dtype_code(x.scalar_type()),
                                         mm_flags(), at::cuda::getCurrentCUDAStream().stream()));
  return out;
}

// fused-bias variant (not in the reference): out[seg b] = x[seg b] @ w[b] + bias[b]
at::Tensor segment_matmul_bias_cuda(const at::Tensor& input, const at::Tensor& ptr, const at::Tensor& other,
                                    const at::Tensor& bias) {
  TORCH_CHECK(input.is_cuda() && other.is_cuda() && bias.is_cuda(), "pyg_lib_b200: segment_matmul_bias expects CUDA tensors");
  TORCH_CHECK(input.dim() == 2 && ptr.dim() == 1 && other.dim() == 3 && bias.dim() == 2, "segment_matmul_bias: bad ranks");
  TORCH_CHECK(input.scalar_type() == other.scalar_type() && bias.scalar_type() == other.scalar_type(),
              "segment_matmul_bias: dtype mismatch");
  TORCH_CHECK(other.size(1) == input.size(1) && ptr.numel() == other.size(0) + 1 && bias.size(0) == other.size(0) &&
                  bias.size(1) == other.size(2), "segment_matmul_bias: shape mismatch");
  c10::cuda::CUDAGuard guard(input.device());
  const at::Tensor x = input.contiguous(), w = other.contiguous(), b = bias.contiguous();
  const at::Tensor p = ptr_on_device(ptr, input.device(), input.size(0));
  at::Tensor out = input.new_empty({x.size(0), w.size(2)});
  PYGB_TORCH_CALL(pygb200_segment_matmul(x.data_ptr(), p.data_ptr<int64_t>(), w.data_ptr(), b.data_ptr(), out.data_ptr(),
                                         x.size(0), x.size(1), w.size(2), w.size(0), dtype_code(x.scalar_type()),
                                         mm_flags(), at::cuda::getCurrentCUDAStream().stream()));
  return out;
}

// dW[b] = X_b^T dY_b as one grouped launch (reference: B torch::matmul calls + at::stack)
at::Tensor segment_matmul_wgrad_cuda(const at::Tensor& input, const at::Tensor& ptr, const at::Tensor& grad_out) {
  TORCH_CHECK(input.is_cuda() && grad_out.is_cuda(), "pyg_lib_b200: segment_matmul_wgrad expects CUDA tensors");
  TORCH_CHECK(input.dim() == 2 && grad_out.dim() == 2 && input.size(0) == grad_out.size(0), "segment_matmul_wgrad: bad shapes");
  TORCH_CHECK(input.scalar_type() == grad_out.scalar_type(), "segment_matmul_wgrad: dtype mismatch");
  c10::cuda::CUDAGuard guard(input.device());
  const at::Tensor x = input.contiguous(), dy = grad_out.contiguous();
  const at::Tensor p = ptr_on_device(ptr, input.device(), input.size(0));
  const int64_t B = ptr.numel() - 1;
  at::Tensor dw = input.new_empty({B, x.size(1), dy.size(1)});
  PYGB_TORCH_CALL(pygb200_segment_matmul_wgrad(x.data_ptr(), p.data_ptr<int64_t>(), dy.data_ptr(), dw.data_ptr(),
                                               x.size(0), x.size(1), dy.size(1), B, dtype_code(x.scalar_type()),
                                               mm_flags(), at::cuda::getCurrentCUDAStream().stream()));
  return dw;
}

std::vector<at::Tensor> grouped_matmul_cuda(const at::TensorList input, const at::TensorList other) {
  TORCH_CHECK(input.size() == other.size(), "Number of 'input' tensors must match number of 'other' tensors");
  std::vector<at::Tensor> outs;
  if (input.empty()) return outs;
  TORCH_CHECK(input[0].is_cuda(), "pyg_lib_b200: grouped_matmul expects CUDA tensors");
  c10::cuda::CUDAGuard guard(input[0].device());
  const int dt = dtype_code(input[0].scalar_type());
  std::vector<pygb200_gemm_problem> ps(input.size());
  std::vector<at::Tensor> keep;  // contiguous copies of operands whose strides the kernel cannot express
  auto describe = [&](const at::Tensor& t, const void** ptr, int64_t* ld, int32_t* colmajor) {
    at::Tensor u = t;
    const bool row_ok = u.stride(1) == 1 || u.size(1) <= 1;
    const bool col_ok = u.stride(0) == 1 || u.size(0) <= 1;
    if (!row_ok && !col_ok) { u = t.contiguous(); keep.push_back(u); }
    if (u.stride(1) == 1 || u.size(1) <= 1) { *colmajor = 0; *ld = u.size(0) > 1 ? u.stride(0) : std::max<int64_t>(u.size(1), 1); }
    else { *colmajor = 1; *ld = u.size(1) > 1 ? u.stride(1) : std::max<int64_t>(u.size(0), 1); }
    *ptr = u.data_ptr();
  };
  for (size_t i = 0; i < input.size(); ++i) {
    const at::Tensor& a = input[i];
    const at::Tensor& b = other[i];
    TORCH_CHECK(a.dim() == 2 && b.dim() == 2, "grouped_matmul: operands must be 2-D");
    TORCH_CHECK(a.size(1) == b.size(0), "grouped_matmul: inner dimensions of pair ", i, " do not match");
    TORCH_CHECK(a.scalar_type() == input[0].scalar_type() && b.scalar_type() == input[0].scalar_type(),
                "grouped_matmul: all tensors must share one dtype");
    TORCH_CHECK(a.device() == input[0].device() && b.device() == input[0].device(), "grouped_matmul: device mismatch");
    at::Tensor c = a.new_empty({a.size(0), b.size(1)});
    outs.push_back(c);
    auto& p = ps[i];
    describe(a, &p.a, &p.lda, &p.a_colmajor);
    describe(b, &p.b, &p.ldb, &p.b_colmajor);
    p.c = c.data_ptr(); p.ldc = std::max<int64_t>(b.size(1), 1);
    p.n = a.size(0); p.k = a.size(1); p.m = b.size(1);
  }
  PYGB_TORCH_CALL(pygb200_grouped_matmul(ps.data(), (int64_t)ps.size(), dt, mm_flags(),
                                         at::cuda::getCurrentCUDAStream().stream()));
  return outs;
}

// ---- autograd for segment_matmul (reference: ops/autograd/matmul_kernel.cpp:68-117)
using torch::autograd::variable_list;

at::Tensor call_segment_matmul(const at::Tensor& input, const at::Tensor& ptr, const at::Tensor& other) {
  static auto op = c10::Dispatcher::singleton().findSchemaOrThrow("pyg::segment_matmul", "")
                       .typed<at::Tensor(const at::Tensor&, const at::Tensor&, const at::Tensor&)>();
  return op.call(input, ptr, other);
}

class SegmentMatmul : public torch::autograd::Function<SegmentMatmul> {
 public:
  static variable_list forward(torch::autograd::AutogradContext* ctx, const at::Tensor& input, const at::Tensor& ptr,
                               const at::Tensor& other) {
    at::AutoDispatchBelowADInplaceOrView g;
    at::Tensor out = call_segment_matmul(input, ptr, other);
    ctx->save_for_backward({input, ptr, other});
    return {out};
  }
  static variable_list backward(torch::autograd::AutogradContext* ctx, variable_list grad_outs) {
    auto grad_out = grad_outs[0];
    auto saved = ctx->get_saved_variables();
    auto input = saved[0], ptr = saved[1], other = saved[2];
    at::Tensor input_grad, other_grad;
    if (torch::autograd::any_variable_requires_grad({input}))  // dX = dY @ W^T per segment
      input_grad = call_segment_matmul(grad_out, ptr, other.transpose(-2, -1));
    if (torch::autograd::any_variable_requires_grad({other}))  // dW[b] = X_b^T @ dY_b, one grouped launch
      other_grad = segment_matmul_wgrad_cuda(input, ptr, grad_out);
    return {input_grad, at::Tensor(), other_grad};
  }
};

at::Tensor segment_matmul_autograd(const at::Tensor& input, const at::Tensor& ptr, const at::Tensor& other) {
  return SegmentMatmul::apply(input, ptr, other)[0];
}

}  // namespace

TORCH_LIBRARY_FRAGMENT(pyg, m) {
  m.def(TORCH_SELECTIVE_SCHEMA("pyg::grouped_matmul(Tensor[] input, Tensor[] other) -> Tensor[]"));
  m.def(TORCH_SELECTIVE_SCHEMA("pyg::segment_matmul(Tensor input, Tensor ptr, Tensor other) -> Tensor"));
  // Additions of this package (not in the reference): fused bias epilogue and the weight-gradient kernel
  m.def(TORCH_SELECTIVE_SCHEMA("pyg::segment_matmul_bias(Tensor input, Tensor ptr, Tensor other, Tensor bias) -> Tensor"));
  m.def(TORCH_SELECTIVE_SCHEMA("pyg::segment_matmul_wgrad(Tensor input, Tensor ptr, Tensor grad_out) -> Tensor"));
}

TORCH_LIBRARY_IMPL(pyg, CUDA, m) {
  m.impl(TORCH_SELECTIVE_NAME("pyg::grouped_matmul"), TORCH_FN(grouped_matmul_cuda));
  m.impl(TORCH_SELECTIVE_NAME("pyg::segment_matmul"), TORCH_FN(segment_matmul_cuda));
  m.impl(TORCH_SELECTIVE_NAME("pyg::segment_matmul_bias"), TORCH_FN(segment_matmul_bias_cuda));
  m.impl(TORCH_SELECTIVE_NAME("pyg::segment_matmul_wgrad"), TORCH_FN(segment_matmul_wgrad_cuda));
}

TORCH_LIBRARY_IMPL(pyg, Autograd, m) {
  m.impl(TORCH_SELECTIVE_NAME("pyg::segment_matmul"), TORCH_FN(segment_matmul_autograd));
}

}  // namespace ops
}  // namespace pyg
