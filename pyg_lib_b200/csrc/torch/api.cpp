// C++ callers' entry points (api.h): argument validation, then the dispatcher operator of the same name.
// Reference behaviour mirrored: pyg_lib/csrc/ops/matmul.cpp:12-60, pyg_lib/csrc/sampler/neighbor.cpp:11-127 — every
// tensor defined, operands of one call of one dtype, ranks and inner sizes consistent; violations raise c10::Error
// (RuntimeError in Python) before any kernel is reached.  Python goes straight to torch.ops.pyg.* and skips these
// wrappers, which is why the kernels repeat the checks that matter to them.
#include "api.h"

#include <ATen/core/dispatch/Dispatcher.h>

#include "common.h"

namespace pyg {
namespace {

void require_defined(const at::Tensor& t, const char* fn, const char* name) {
  TORCH_CHECK(t.defined(), fn, ": argument '", name, "' is an undefined tensor");
}
void require_same_dtype(const at::Tensor& a, const char* an, const at::Tensor& b, const char* bn, const char* fn) {
  TORCH_CHECK(a.scalar_type() == b.scalar_type(), fn, ": expected '", an, "' (", a.scalar_type(), ") and '", bn, "' (",
              b.scalar_type(), ") to have the same dtype");
}
void require_dim(const at::Tensor& t, int64_t dim, const char* fn, const char* name) {
  TORCH_CHECK(t.dim() == dim, fn, ": expected '", name, "' to be ", dim, "-dimensional, got ", t.dim(), " dimension(s)");
}

}  // namespace

namespace ops {

std::vector<at::Tensor> grouped_matmul(const at::TensorList input, const at::TensorList other) {
  const char* fn = "grouped_matmul";
  TORCH_CHECK(input.size() == other.size(), "Number of 'input' tensors must match number of 'other' tensors");
  for (size_t i = 0; i < input.size(); ++i) {
    require_defined(input[i], fn, "input"); require_defined(other[i], fn, "other");
    require_same_dtype(input[i], "input", input[0], "input[0]", fn);
    require_same_dtype(other[i], "other", input[0], "input[0]", fn);
    require_dim(input[i], 2, fn, "input"); require_dim(other[i], 2, fn, "other");
    TORCH_CHECK(other[i].size(0) == input[i].size(-1), fn, ": expected other[", i, "].size(0) == input[", i, "].size(-1) = ",
                input[i].size(-1), ", got ", other[i].size(0));
  }
  static auto op = c10::Dispatcher::singleton().findSchemaOrThrow("pyg::grouped_matmul", "").typed<decltype(grouped_matmul)>();
  return op.call(input, other);
}

at::Tensor segment_matmul(const at::Tensor& input, const at::Tensor& ptr, const at::Tensor& other) {
  const char* fn = "segment_matmul";
  require_defined(input, fn, "input"); require_defined(ptr, fn, "ptr"); require_defined(other, fn, "other");
  require_same_dtype(input, "input", other, "other", fn);
  require_dim(input, 2, fn, "input"); require_dim(ptr, 1, fn, "ptr"); require_dim(other, 3, fn, "other");
  TORCH_CHECK(other.size(1) == input.size(-1), fn, ": expected other.size(1) == input.size(-1) = ", input.size(-1), ", got ", other.size(1));
  TORCH_CHECK(ptr.numel() == other.size(0) + 1, fn, ": expected ptr.numel() == other.size(0) + 1 = ", other.size(0) + 1, ", got ", ptr.numel());
  static auto op = c10::Dispatcher::singleton().findSchemaOrThrow("pyg::segment_matmul", "").typed<decltype(segment_matmul)>();
  return op.call(input, ptr, other);
}

}  // namespace ops

namespace sampler {

std::tuple<at::Tensor, at::Tensor, at::Tensor, std::optional<at::Tensor>, std::vector<int64_t>, std::vector<int64_t>>
neighbor_sample(const at::Tensor& rowptr, const at::Tensor& col, const at::Tensor& seed, const std::vector<int64_t>& num_neighbors,
                const std::optional<at::Tensor>& node_time, const std::optional<at::Tensor>& edge_time,
                const std::optional<at::Tensor>& seed_time, const std::optional<at::Tensor>& edge_weight, bool csc, bool replace,
                bool directed, bool disjoint, std::string temporal_strategy, bool return_edge_id) {
  const char* fn = "neighbor_sample";
  require_defined(rowptr, fn, "rowptr"); require_defined(col, fn, "col"); require_defined(seed, fn, "seed");
  require_same_dtype(rowptr, "rowptr", col, "col", fn); require_same_dtype(rowptr, "rowptr", seed, "seed", fn);
  static auto op = c10::Dispatcher::singleton().findSchemaOrThrow("pyg::neighbor_sample", "").typed<decltype(neighbor_sample)>();
  return op.call(rowptr, col, seed, num_neighbors, node_time, edge_time, seed_time, edge_weight, csc, replace, directed, disjoint,
                 temporal_strategy, return_edge_id);
}

std::tuple<c10::Dict<rel_type, at::Tensor>, c10::Dict<rel_type, at::Tensor>, c10::Dict<node_type, at::Tensor>,
           std::optional<c10::Dict<rel_type, at::Tensor>>, c10::Dict<node_type, std::vector<int64_t>>,
           c10::Dict<rel_type, std::vector<int64_t>>>
hetero_neighbor_sample(const std::vector<node_type>& node_types, const std::vector<edge_type>& edge_types,
                       const c10::Dict<rel_type, at::Tensor>& rowptr_dict, const c10::Dict<rel_type, at::Tensor>& col_dict,
                       const c10::Dict<node_type, at::Tensor>& seed_dict,
                       const c10::Dict<rel_type, std::vector<int64_t>>& num_neighbors_dict,
                       const std::optional<c10::Dict<node_type, at::Tensor>>& node_time_dict,
                       const std::optional<c10::Dict<rel_type, at::Tensor>>& edge_time_dict,
                       const std::optional<c10::Dict<node_type, at::Tensor>>& seed_time_dict,
                       const std::optional<c10::Dict<rel_type, at::Tensor>>& edge_weight_dict, bool csc, bool replace, bool directed,
                       bool disjoint, std::string temporal_strategy, bool return_edge_id) {
  const char* fn = "hetero_neighbor_sample";
  TORCH_CHECK(rowptr_dict.size() == col_dict.size(), "Number of edge types in 'rowptr_dict' and 'col_dict' must match");
  TORCH_CHECK(rowptr_dict.size() > 0 && seed_dict.size() > 0, fn, ": 'rowptr_dict' and 'seed_dict' must not be empty");
  const at::Tensor& first = rowptr_dict.begin()->value();
  for (const auto& kv : rowptr_dict) { require_defined(kv.value(), fn, "rowptr_dict"); require_same_dtype(kv.value(), "rowptr_dict", first, "rowptr_dict", fn); }
  for (const auto& kv : col_dict) { require_defined(kv.value(), fn, "col_dict"); require_same_dtype(kv.value(), "col_dict", first, "rowptr_dict", fn); }
  for (const auto& kv : seed_dict) { require_defined(kv.value(), fn, "seed_dict"); require_same_dtype(kv.value(), "seed_dict", first, "rowptr_dict", fn); }
  static auto op = c10::Dispatcher::singleton().findSchemaOrThrow("pyg::hetero_neighbor_sample", "").typed<decltype(hetero_neighbor_sample)>();
  return op.call(node_types, edge_types, rowptr_dict, col_dict, seed_dict, num_neighbors_dict, node_time_dict, edge_time_dict,
                 seed_time_dict, edge_weight_dict, csc, replace, directed, disjoint, temporal_strategy, return_edge_id);
}

std::tuple<at::Tensor, at::Tensor, std::vector<int64_t>>
dist_neighbor_sample(const at::Tensor& rowptr, const at::Tensor& col, const at::Tensor& seed, int64_t num_neighbors,
                     const std::optional<at::Tensor>& node_time, const std::optional<at::Tensor>& edge_time,
                     const std::optional<at::Tensor>& seed_time, const std::optional<at::Tensor>& edge_weight, bool csc, bool replace,
                     bool directed, bool disjoint, std::string temporal_strategy) {
  const char* fn = "dist_neighbor_sample";
  require_defined(rowptr, fn, "rowptr"); require_defined(col, fn, "col"); require_defined(seed, fn, "seed");
  require_same_dtype(rowptr, "rowptr", col, "col", fn); require_same_dtype(rowptr, "rowptr", seed, "seed", fn);
  static auto op = c10::Dispatcher::singleton().findSchemaOrThrow("pyg::dist_neighbor_sample", "").typed<decltype(dist_neighbor_sample)>();
  return op.call(rowptr, col, seed, num_neighbors, node_time, edge_time, seed_time, edge_weight, csc, replace, directed, disjoint,
                 temporal_strategy);
}

at::Tensor random_walk(const at::Tensor& rowptr, const at::Tensor& col, const at::Tensor& seed, int64_t walk_length, double p,
                       double q) {
  const char* fn = "random_walk";   // sampler/random_walk.cpp:15-21
  require_defined(rowptr, fn, "rowptr"); require_defined(col, fn, "col"); require_defined(seed, fn, "seed");
  require_same_dtype(rowptr, "rowptr", col, "col", fn); require_same_dtype(rowptr, "rowptr", seed, "seed", fn);
  static auto op = c10::Dispatcher::singleton().findSchemaOrThrow("pyg::random_walk", "").typed<decltype(random_walk)>();
  return op.call(rowptr, col, seed, walk_length, p, q);
}

}  // namespace sampler
}  // namespace pyg
