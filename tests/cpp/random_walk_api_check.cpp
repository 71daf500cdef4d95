// C++ caller of pyg::sampler::random_walk (pyg_lib_b200/csrc/torch/api.h): argument checks raise c10::Error before any
// kernel is reached; CPU tensors reach the dispatcher's "no CPU fallback" error.  With `--gpu SEED` it also walks the
// 10-node cycle graph from every node (twice each, walk_length 12) on cuda:0 after torch::manual_seed(SEED) and prints
// the result, which tests/test_random_walk.py compares with the Python op under the same seed.
#include <torch/torch.h>

#include <cstdlib>
#include <cstring>
#include <iostream>

#include "api.h"

template <typename F>
static bool throws(F f, const char* needle) {
  try { f(); } catch (const c10::Error& e) { return std::strstr(e.what(), needle) != nullptr; }
  return false;
}

int main(int argc, char** argv) {
  const bool gpu = argc > 2 && std::strcmp(argv[1], "--gpu") == 0;
  int bad = 0;
  auto rowptr = torch::arange(0, 21, 2, torch::kLong);
  auto col = torch::stack({torch::arange(-1, 9, torch::kLong).remainder(10), torch::arange(1, 11, torch::kLong).remainder(10)}, 1).flatten();
  auto seed = torch::arange(10, torch::kLong).repeat({2});
  bad += !throws([&] { pyg::sampler::random_walk(rowptr, col, seed.to(torch::kInt), 3); }, "same dtype");
  bad += !throws([&] { pyg::sampler::random_walk(rowptr, col.to(torch::kInt), seed, 3); }, "same dtype");
  bad += !throws([&] { pyg::sampler::random_walk(rowptr, at::Tensor(), seed, 3); }, "undefined");
  bad += !throws([&] { pyg::sampler::random_walk(at::Tensor(), col, seed, 3); }, "undefined");
  if (!gpu) {
    bad += !throws([&] { pyg::sampler::random_walk(rowptr, col, seed, 3); }, "no CPU fallback");
  } else {
    auto dev = torch::Device(torch::kCUDA, 0);
    bad += !throws([&] { pyg::sampler::random_walk(rowptr.to(dev), col.to(dev), seed.to(dev), 3, 2.0, 1.0); },
                   "Uniform sampling required for now");
    torch::manual_seed(std::atoll(argv[2]));
    auto out = pyg::sampler::random_walk(rowptr.to(dev), col.to(dev), seed.to(dev), 12).cpu();
    bad += !(out.size(0) == 20 && out.size(1) == 13);
    std::cout << "WALK";
    auto a = out.accessor<int64_t, 2>();
    for (int64_t i = 0; i < out.size(0); ++i)
      for (int64_t j = 0; j < out.size(1); ++j) std::cout << ' ' << a[i][j];
    std::cout << std::endl;
  }
  std::cout << (bad ? "CPP_API_FAIL " : "CPP_API_OK ") << bad << std::endl;
  return bad ? 1 : 0;
}
