// `pyg::cuda_version` — same schema as the reference (pyg_lib/csrc/library.cpp:19-29).
#include "common.h"

namespace pyg {

int64_t cuda_version() { return pygb200_cuda_version(); }

// process-wide count of kernels launched by libpyg_b200.so (bench.py's `gpu_launches`)
int64_t b200_kernel_launches() { return pygb200_kernel_launches(); }

TORCH_LIBRARY_FRAGMENT(pyg, m) {
  m.def("cuda_version", &cuda_version);
  m.def("b200_kernel_launches", &b200_kernel_launches);
}

// CPU tensors: the reference registers CPU kernels for every op (e.g. sampler/cpu/neighbor_kernel.cpp:980-983,
// ops/cpu/matmul_kernel.cpp:255-262); this library is the CUDA path only (north_star: no CPU fallback).  Instead of the
// dispatcher's generic "could not run ... with arguments from the 'CPU' backend", every pyg:: op called with CPU
// tensors raises one clear message that says what to do.
static void cpu_not_supported(const c10::OperatorHandle& op, c10::DispatchKeySet, torch::jit::Stack*) {
  TORCH_CHECK(false, "pyg_lib_b200: '", op.schema().name(), "' was called with CPU tensors. This build implements the CUDA "
              "(sm_90a) path only and has no CPU fallback: move the graph / feature tensors to a CUDA device, or use the "
              "stock pyg-lib package for CPU sampling (set PYG_LIB_B200_NO_ALIAS=1 to keep `import pyg_lib` from "
              "resolving to this package).");
}

TORCH_LIBRARY_IMPL(pyg, CPU, m) {   // (the dispatcher has no per-namespace fallback: one registration per CUDA-key op)
  for (const char* name : {"pyg::segment_matmul", "pyg::segment_matmul_bias", "pyg::segment_matmul_wgrad", "pyg::grouped_matmul",
                           "pyg::neighbor_sample", "pyg::dist_neighbor_sample", "pyg::subgraph", "pyg::relabel_neighborhood",
                           "pyg::random_walk"})
    m.impl(name, torch::CppFunction::makeFromBoxedFunction<&cpu_not_supported>());
}

}  // namespace pyg
