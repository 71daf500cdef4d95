// C++ callers' entry points of libpyg.so — the functions a C++ program (or another extension) links against instead of
// going through Python: same names, namespaces, argument meaning and argument checks as the reference's PYG_API functions
// (pyg_lib/csrc/ops/matmul.h:10-21 + matmul.cpp:12-60, pyg_lib/csrc/sampler/neighbor.h + neighbor.cpp:11-127).  Each one
// validates its arguments and then calls the dispatcher operator of the same name (looked up once), so autograd and the
// CUDA / BackendSelect kernels behind it are exactly what Python reaches through torch.ops.pyg.*.
#pragma once
#include <ATen/ATen.h>

#include <optional>
#include <string>
#include <tuple>
#include <vector>

#define PYGB200_API __attribute__((visibility("default")))

namespace pyg {
namespace ops {

// outs[i] = input[i] @ other[i]; all tensors defined, 2-D, one dtype, inner sizes matching.
PYGB200_API std::vector<at::Tensor> grouped_matmul(const at::TensorList input, const at::TensorList other);

// out[ptr[i]:ptr[i+1]] = input[ptr[i]:ptr[i+1]] @ other[i]; input 2-D, ptr 1-D with other.size(0) + 1 entries, other 3-D.
PYGB200_API at::Tensor segment_matmul(const at::Tensor& input, const at::Tensor& ptr, const at::Tensor& other);

}  // namespace ops

namespace sampler {

typedef std::string node_type;
typedef std::string rel_type;
typedef std::tuple<std::string, std::string, std::string> edge_type;

PYGB200_API std::tuple<at::Tensor, at::Tensor, at::Tensor, std::optional<at::Tensor>, std::vector<int64_t>, std::vector<int64_t>>
neighbor_sample(const at::Tensor& rowptr, const at::Tensor& col, const at::Tensor& seed, const std::vector<int64_t>& num_neighbors,
                const std::optional<at::Tensor>& node_time = std::nullopt, const std::optional<at::Tensor>& edge_time = std::nullopt,
                const std::optional<at::Tensor>& seed_time = std::nullopt, const std::optional<at::Tensor>& edge_weight = std::nullopt,
                bool csc = false, bool replace = false, bool directed = true, bool disjoint = false,
                std::string temporal_strategy = "uniform", bool return_edge_id = true);

PYGB200_API std::tuple<c10::Dict<rel_type, at::Tensor>, c10::Dict<rel_type, at::Tensor>, c10::Dict<node_type, at::Tensor>,
                       std::optional<c10::Dict<rel_type, at::Tensor>>, c10::Dict<node_type, std::vector<int64_t>>,
                       c10::Dict<rel_type, std::vector<int64_t>>>
hetero_neighbor_sample(const std::vector<node_type>& node_types, const std::vector<edge_type>& edge_types,
                       const c10::Dict<rel_type, at::Tensor>& rowptr_dict, const c10::Dict<rel_type, at::Tensor>& col_dict,
                       const c10::Dict<node_type, at::Tensor>& seed_dict,
                       const c10::Dict<rel_type, std::vector<int64_t>>& num_neighbors_dict,
                       const std::optional<c10::Dict<node_type, at::Tensor>>& node_time_dict = std::nullopt,
                       const std::optional<c10::Dict<rel_type, at::Tensor>>& edge_time_dict = std::nullopt,
                       const std::optional<c10::Dict<node_type, at::Tensor>>& seed_time_dict = std::nullopt,
                       const std::optional<c10::Dict<rel_type, at::Tensor>>& edge_weight_dict = std::nullopt, bool csc = false,
                       bool replace = false, bool directed = true, bool disjoint = false,
                       std::string temporal_strategy = "uniform", bool return_edge_id = true);

PYGB200_API std::tuple<at::Tensor, at::Tensor, std::vector<int64_t>>
dist_neighbor_sample(const at::Tensor& rowptr, const at::Tensor& col, const at::Tensor& seed, int64_t num_neighbors,
                     const std::optional<at::Tensor>& node_time = std::nullopt, const std::optional<at::Tensor>& edge_time = std::nullopt,
                     const std::optional<at::Tensor>& seed_time = std::nullopt, const std::optional<at::Tensor>& edge_weight = std::nullopt,
                     bool csc = false, bool replace = false, bool directed = true, bool disjoint = false,
                     std::string temporal_strategy = "uniform");

// [seed.size(0), walk_length + 1] uniform random walks from `seed` (pyg_lib/csrc/sampler/random_walk.h:10-18); CUDA only,
// p == q == 1.
PYGB200_API at::Tensor random_walk(const at::Tensor& rowptr, const at::Tensor& col, const at::Tensor& seed, int64_t walk_length,
                                   double p = 1.0, double q = 1.0);

}  // namespace sampler
}  // namespace pyg
