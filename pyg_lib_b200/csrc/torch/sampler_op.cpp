// torch.ops.pyg.neighbor_sample / hetero_neighbor_sample on CUDA tensors.
//
// Schemas are the reference's, verbatim (pyg_lib/csrc/sampler/neighbor.cpp:129-147); PyG feature-
// detects optional arguments by inspecting them.  Dispatch keys follow SURVEY.md 8(b):
//   pyg::neighbor_sample         -> CUDA key   (reference: CPU only, neighbor_kernel.cpp:980-983)
//   pyg::hetero_neighbor_sample  -> BackendSelect (dict arguments carry no backend key,
//                                   neighbor_kernel.cpp:985-991); the kernel checks devices itself.
// There is no CPU kernel: CPU tensors raise.
#include <ATen/CPUGeneratorImpl.h>

#include <algorithm>
#include <map>
#include <memory>
#include <mutex>

#include "common.h"

namespace pyg {
namespace sampler {
namespace {

typedef std::string node_type;
typedef std::string rel_type;
typedef std::tuple<std::string, std::string, std::string> edge_type;

inline rel_type to_rel_type(const edge_type& k) {  // pyg_lib/csrc/utils/types.h:10-12
  return std::get<0>(k) + "__" + std::get<1>(k) + "__" + std::get<2>(k);
}

// one persistent workspace per (device, stream).  An op binds outputs, runs and exports in separate ABI calls, and torch
// drops the GIL inside ops: `op_mu` is held across the whole op body so that two host threads sampling on the same
// stream cannot interleave (the reference op is reentrant; ADVICE r1).
struct SamplerSlot { pygb200_sampler* s = nullptr; std::mutex op_mu; };
SamplerSlot& get_slot(int device, cudaStream_t stream) {
  static std::mutex mu;
  static std::map<std::pair<int, cudaStream_t>, std::unique_ptr<SamplerSlot>> cache;
  std::lock_guard<std::mutex> lock(mu);
  auto key = std::make_pair(device, stream);
  auto it = cache.find(key);
  if (it != cache.end()) return *it->second;
  auto slot = std::make_unique<SamplerSlot>();
  PYGB_TORCH_CALL(pygb200_sampler_create(&slot->s));
  auto& ref = *slot;
  cache[key] = std::move(slot);
  return ref;
}

// RAII view of torch's default CPU generator as the ABI's engine struct.  The reference draws its
// random words from exactly this generator (rand_engine.h:80-92), so it is read before and written
// back after the run, under the generator's mutex.
struct CpuEngine {
  at::CPUGeneratorImpl* gen;
  std::unique_lock<std::mutex> lock;
  pygb200_mt19937 mt;
  CpuEngine()
      : gen(at::get_generator_or_default<at::CPUGeneratorImpl>(std::nullopt, at::detail::getDefaultCPUGenerator())),
        lock(gen->mutex_) {
    const at::mt19937_data_pod pod = gen->engine().data();
    for (int i = 0; i < 624; ++i) mt.state[i] = pod.state_[i];
    mt.left = pod.left_;
    mt.next = (int32_t)pod.next_;
  }
  void commit() {
    at::mt19937 eng = gen->engine();
    at::mt19937_data_pod pod = eng.data();
    for (int i = 0; i < 624; ++i) pod.state_[i] = mt.state[i];
    pod.left_ = mt.left;
    pod.next_ = (uint32_t)mt.next;
    eng.set_data(pod);
    gen->set_engine(eng);
  }
};

// Results of at most this many worst-case bytes are written in place (views of bound-sized tensors are returned,
// so a caller that keeps a result keeps the bound alive: C2 returns 76 % of its bound, a sparse hetero graph may
// return 7 %).  PYGB200_DIRECT_OUTPUT_MB overrides the 256 MiB default (0 = always export into exact-size tensors).
static const int64_t kDirectOutputBytes = [] {
  const char* e = getenv("PYGB200_DIRECT_OUTPUT_MB");
  return (e ? (int64_t)atoll(e) : 256ll) << 20;
}();
// ... and a view is only handed out when the result fills at least this fraction of its bound-sized buffer (default
// 0.5); emptier results are copied into exact-size tensors so that a caller who queues batches (or pickles one: a
// view serialises its whole storage) never holds more than 2x the payload.  PYGB200_DIRECT_MIN_FILL overrides.
static const double kDirectMinFill = [] {
  const char* e = getenv("PYGB200_DIRECT_MIN_FILL");
  return e ? atof(e) : 0.5;
}();

void check_index_tensor(const at::Tensor& t, const char* name, at::ScalarType st, const at::Device& dev) {
  TORCH_CHECK(t.is_contiguous(), "Non-contiguous '", name, "'");  // neighbor_kernel.cpp:361-363
  TORCH_CHECK(t.scalar_type() == st, "'", name, "' must have the same dtype as the seed tensor");
  TORCH_CHECK(t.device() == dev, "'", name, "' must live on ", dev, " (pyg_lib_b200 has no CPU fallback)");
  TORCH_CHECK(t.dim() == 1, "'", name, "' must be one-dimensional");
}

void check_arguments(bool has_node_time, bool has_edge_time, bool has_seed_time, bool has_weight, bool disjoint) {
  // reference argument checks (neighbor_kernel.cpp:354-380), then what this path does not do
  TORCH_CHECK(!has_node_time || disjoint, "Temporal sampling needs to create disjoint subgraphs");
  TORCH_CHECK(!has_edge_time || disjoint, "Temporal sampling needs to create disjoint subgraphs");
  TORCH_CHECK(!(has_node_time && has_edge_time), "Only one of node-level or edge-level sampling is supported ");
  TORCH_CHECK(!has_edge_time || has_seed_time, "Seed time needs to be specified");
  TORCH_CHECK(!(has_node_time && has_weight), "Biased node temporal sampling not yet supported");   // neighbor_kernel.cpp:377-380
  TORCH_CHECK(!(has_edge_time && has_weight), "Biased edge temporal sampling not yet supported");
}

// edge weights of one relation for the biased path: float32, one per edge, on the sampler's device
const void* weight_ptr(const at::Tensor& w, const at::Tensor& col, const at::Device& dev) {
  TORCH_CHECK(w.device() == dev, "'edge_weight' must live on ", dev, " (pyg_lib_b200 has no CPU fallback)");
  TORCH_CHECK(w.scalar_type() == at::kFloat,
              "pyg_lib_b200: biased sampling takes float32 edge weights (the reference's random stream and key arithmetic "
              "depend on the weight dtype; only float32 is reproduced), got ", w.scalar_type());
  TORCH_CHECK(w.is_contiguous() && w.dim() == 1, "'edge_weight' must be a contiguous one-dimensional tensor");
  TORCH_CHECK(w.numel() == col.numel(), "'edge_weight' must have one entry per edge");
  return w.data_ptr();
}

const int64_t* time_ptr(const at::Tensor& t, const char* name, const at::Device& dev) {
  TORCH_CHECK(t.is_contiguous(), "Non-contiguous '", name, "'");
  TORCH_CHECK(t.scalar_type() == at::kLong, "'", name, "' must be int64 (the reference reads temporal_t = int64_t)");
  TORCH_CHECK(t.device() == dev, "'", name, "' must live on ", dev);
  return t.data_ptr<int64_t>();
}

std::tuple<at::Tensor, at::Tensor, at::Tensor, std::optional<at::Tensor>, std::vector<int64_t>, std::vector<int64_t>>
neighbor_sample_cuda(const at::Tensor& rowptr, const at::Tensor& col, const at::Tensor& seed,
                     const std::vector<int64_t>& num_neighbors, const std::optional<at::Tensor>& node_time,
                     const std::optional<at::Tensor>& edge_time, const std::optional<at::Tensor>& seed_time,
                     const std::optional<at::Tensor>& edge_weight, bool csc, bool replace, bool directed,
                     bool disjoint, std::string temporal_strategy, bool return_edge_id) {
  TORCH_CHECK(temporal_strategy == "uniform" || temporal_strategy == "last", "No valid temporal strategy found");
  check_arguments(node_time.has_value(), edge_time.has_value(), seed_time.has_value(), edge_weight.has_value(), disjoint);
  TORCH_CHECK(seed.is_cuda(), "pyg_lib_b200: neighbor_sample expects CUDA tensors (no CPU fallback)");
  const auto st = seed.scalar_type();
  TORCH_CHECK(st == at::kLong || st == at::kInt, "neighbor_sample: index tensors must be int64 or int32");
  check_index_tensor(rowptr, "rowptr", st, seed.device());
  check_index_tensor(col, "col", st, seed.device());
  check_index_tensor(seed, "seed", st, seed.device());
  TORCH_CHECK(rowptr.numel() >= 1, "'rowptr' must have at least one element");

  c10::cuda::CUDAGuard guard(seed.device());
  cudaStream_t stream = at::cuda::getCurrentCUDAStream();
  SamplerSlot& slot = get_slot(seed.device().index(), stream);
  std::lock_guard<std::mutex> op_lock(slot.op_mu);
  pygb200_sampler* s = slot.s;
  const int L = (int)num_neighbors.size();
  const bool idx32 = st == at::kInt;
  unsigned flags = (replace ? PYGB200_S_REPLACE : 0u) | (disjoint ? PYGB200_S_DISJOINT : 0u) | (idx32 ? PYGB200_S_INDEX32 : 0u) |
                   PYGB200_S_DEFER_CLEANUP;   // export_all below resets the table in the same launch
  std::vector<int64_t> nph(L + 1, 0), eph(L, 0);
  int64_t n_nodes = 0, n_edges = 0;
  const auto opt = seed.options();
  at::Tensor row, colv, node, direct_buf;
  int64_t direct_ecap = 0;
  std::optional<at::Tensor> eid = std::nullopt;
  {
    const int64_t* nt = node_time.has_value() ? time_ptr(*node_time, "node_time", seed.device()) : nullptr;
    const int64_t* et = edge_time.has_value() ? time_ptr(*edge_time, "edge_time", seed.device()) : nullptr;
    const int64_t* stt = seed_time.has_value() ? time_ptr(*seed_time, "seed_time", seed.device()) : nullptr;
    if (stt) TORCH_CHECK(seed_time->numel() == seed.numel(), "'seed_time' must have one entry per seed");
    if (et) TORCH_CHECK(edge_time->numel() == col.numel(), "'edge_time' must have one entry per edge");
    pygb200_temporal tmp{&nt, &et, &stt, temporal_strategy == "last" ? 1 : 0};
    pygb200_relation rel{rowptr.data_ptr(), col.data_ptr(), rowptr.numel() - 1, col.numel(), 0, 0};
    const void* seeds[1] = {seed.data_ptr()};
    const int64_t n_seed = seed.numel();
    // Latency path: result tensors sized by the static bounds and written by the sampling kernels themselves
    // (no export launch, no second host round trip); the caller gets views of their first n entries.
    int64_t ncap = 0, ecap = 0;
    if (!idx32 && !disjoint && L > 0 &&
        pygb200_sampler_bounds(1, 1, L, &rel, &n_seed, num_neighbors.data(), &ncap, &ecap) == PYGB200_OK && ecap > 0 &&
        (3 * ecap + ncap) * 8 <= kDirectOutputBytes) {
      // ONE allocation for the four results (row | col | edge_id | node_id): one allocator call per sampling call
      // (views are only made once, after the run, with the final sizes: every narrow() is a dispatcher call)
      direct_buf = at::empty({(return_edge_id ? 3 : 2) * ecap + ncap}, opt);
      direct_ecap = ecap;
      int64_t* base = direct_buf.data_ptr<int64_t>();
      void* rp = base; void* cp = base + ecap; void* ep = return_edge_id ? base + 2 * ecap : nullptr;
      void* np = base + (return_edge_id ? 3 : 2) * ecap;
      PYGB_TORCH_CALL(pygb200_sampler_bind_outputs(s, 1, 1, &rp, &cp, &ep, &np, &ecap, &ncap));
    }
    // biased sampling; with only "all neighbours" fan-outs the weights are never looked at (neighbor_kernel.cpp:259-265)
    const void* wp = nullptr;
    if (edge_weight.has_value() && std::any_of(num_neighbors.begin(), num_neighbors.end(), [](int64_t k) { return k >= 0; }))
      wp = weight_ptr(*edge_weight, col, seed.device());
    CpuEngine eng;
    if (wp) {
      PYGB_TORCH_CALL(pygb200_sampler_run_weighted(s, 1, 1, L, &rel, seeds, &n_seed, num_neighbors.data(), flags, &eng.mt,
                                                   nph.data(), eph.data(), &n_nodes, &n_edges, stream, &wp, PYGB200_F32));
    } else
    PYGB_TORCH_CALL(pygb200_sampler_run_temporal(s, 1, 1, L, &rel, seeds, &n_seed, num_neighbors.data(), flags, &eng.mt,
                                                 nph.data(), eph.data(), &n_nodes, &n_edges, stream,
                                                 (nt || et) ? &tmp : nullptr));
    eng.commit();
  }
  TORCH_CHECK(directed, "Undirected subgraphs not yet supported");  // raised after sampling, neighbor_kernel.cpp:501
  if (pygb200_sampler_outputs_direct(s)) {
    row = direct_buf.narrow(0, 0, n_edges); colv = direct_buf.narrow(0, direct_ecap, n_edges);
    if (return_edge_id) eid = direct_buf.narrow(0, 2 * direct_ecap, n_edges);
    node = direct_buf.narrow(0, (return_edge_id ? 3 : 2) * direct_ecap, n_nodes);
    const int64_t cap_total = direct_buf.numel(), used = (return_edge_id ? 3 : 2) * n_edges + n_nodes;
    if ((double)used < kDirectMinFill * (double)cap_total) {   // sparse result: do not pin the bound-sized storage
      row = row.clone(); colv = colv.clone(); node = node.clone();
      if (return_edge_id) eid = eid->clone();
    }
  } else {
    row = at::empty({n_edges}, opt); colv = at::empty({n_edges}, opt);
    node = disjoint ? at::empty({n_nodes, 2}, opt) : at::empty({n_nodes}, opt);
    eid = std::nullopt;
    if (return_edge_id) eid = at::empty({n_edges}, opt);
    PYGB_TORCH_CALL(pygb200_sampler_export_all(s, 0, row.data_ptr(), colv.data_ptr(), return_edge_id ? eid->data_ptr() : nullptr, 0,
                                               node.data_ptr(), idx32, stream));
  }
  if (csc) std::swap(row, colv);  // neighbor_kernel.cpp:155-159
  return std::make_tuple(row, colv, node, eid, nph, eph);
}

// pyg::dist_neighbor_sample (dist_neighbor_sample_kernel, neighbor_kernel.cpp:957-978): ONE hop from `seed` with the
// same draws as neighbor_sample, but nothing is mapped: node ids = the seeds followed by every sampled neighbour's
// GLOBAL id in emission order ((batch, node) pairs if disjoint), their edge ids, and cumsum_neighbors_per_node.
std::tuple<at::Tensor, at::Tensor, std::vector<int64_t>>
dist_neighbor_sample_cuda(const at::Tensor& rowptr, const at::Tensor& col, const at::Tensor& seed, int64_t num_neighbors,
                          const std::optional<at::Tensor>& node_time, const std::optional<at::Tensor>& edge_time,
                          const std::optional<at::Tensor>& seed_time, const std::optional<at::Tensor>& edge_weight, bool csc,
                          bool replace, bool directed, bool disjoint, std::string temporal_strategy) {
  TORCH_CHECK(temporal_strategy == "uniform" || temporal_strategy == "last", "No valid temporal strategy found");
  check_arguments(node_time.has_value(), edge_time.has_value(), seed_time.has_value(), edge_weight.has_value(), disjoint);
  TORCH_CHECK(seed.is_cuda(), "pyg_lib_b200: dist_neighbor_sample expects CUDA tensors (no CPU fallback)");
  const auto st = seed.scalar_type();
  TORCH_CHECK(st == at::kLong || st == at::kInt, "dist_neighbor_sample: index tensors must be int64 or int32");
  check_index_tensor(rowptr, "rowptr", st, seed.device());
  check_index_tensor(col, "col", st, seed.device());
  check_index_tensor(seed, "seed", st, seed.device());
  TORCH_CHECK(rowptr.numel() >= 1, "'rowptr' must have at least one element");
  (void)csc;  // no (row, col) pair is returned

  c10::cuda::CUDAGuard guard(seed.device());
  cudaStream_t stream = at::cuda::getCurrentCUDAStream();
  SamplerSlot& slot = get_slot(seed.device().index(), stream);
  std::lock_guard<std::mutex> op_lock(slot.op_mu);
  pygb200_sampler* s = slot.s;
  const bool idx32 = st == at::kInt;
  const unsigned flags = (replace ? PYGB200_S_REPLACE : 0u) | (disjoint ? PYGB200_S_DISJOINT : 0u) | (idx32 ? PYGB200_S_INDEX32 : 0u) |
                         PYGB200_S_NO_DEDUP;
  const int64_t S = seed.numel();
  int64_t nph[2] = {0, 0}, eph[1] = {0}, n_nodes = 0, n_edges = 0;
  {
    const int64_t* nt = node_time.has_value() ? time_ptr(*node_time, "node_time", seed.device()) : nullptr;
    const int64_t* et = edge_time.has_value() ? time_ptr(*edge_time, "edge_time", seed.device()) : nullptr;
    const int64_t* stt = seed_time.has_value() ? time_ptr(*seed_time, "seed_time", seed.device()) : nullptr;
    if (stt) TORCH_CHECK(seed_time->numel() == S, "'seed_time' must have one entry per seed");
    if (et) TORCH_CHECK(edge_time->numel() == col.numel(), "'edge_time' must have one entry per edge");
    pygb200_temporal tmp{&nt, &et, &stt, temporal_strategy == "last" ? 1 : 0};
    pygb200_relation rel{rowptr.data_ptr(), col.data_ptr(), rowptr.numel() - 1, col.numel(), 0, 0};
    const void* seeds[1] = {seed.data_ptr()};
    const void* wp = (edge_weight.has_value() && num_neighbors >= 0) ? weight_ptr(*edge_weight, col, seed.device()) : nullptr;
    CpuEngine eng;
    if (wp)
      PYGB_TORCH_CALL(pygb200_sampler_run_weighted(s, 1, 1, 1, &rel, seeds, &S, &num_neighbors, flags, &eng.mt, nph, eph, &n_nodes,
                                                   &n_edges, stream, &wp, PYGB200_F32));
    else
    PYGB_TORCH_CALL(pygb200_sampler_run_temporal(s, 1, 1, 1, &rel, seeds, &S, &num_neighbors, flags, &eng.mt, nph, eph, &n_nodes,
                                                 &n_edges, stream, (nt || et) ? &tmp : nullptr));
    eng.commit();
  }
  TORCH_CHECK(directed, "Undirected subgraphs not yet supported");  // neighbor_kernel.cpp:501
  const auto opt = seed.options();
  at::Tensor eid = at::empty({n_edges}, opt);
  at::Tensor cum = at::empty({S + 1}, opt.dtype(at::kLong));
  at::Tensor node;
  if (!disjoint) {
    node = at::empty({S + n_edges}, opt);
    node.narrow(0, 0, S).copy_(seed);
    PYGB_TORCH_CALL(pygb200_sampler_export_edges(s, 0, nullptr, node.narrow(0, S, n_edges).data_ptr(), eid.data_ptr(), idx32, stream));
  } else {   // (batch, node): a seed is its own batch; a neighbour inherits the batch (= index) of the seed it came from
    at::Tensor row = at::empty({n_edges}, opt), dst = at::empty({n_edges}, opt);
    PYGB_TORCH_CALL(pygb200_sampler_export_edges(s, 0, row.data_ptr(), dst.data_ptr(), eid.data_ptr(), idx32, stream));
    node = at::stack({at::cat({at::arange(S, opt), row}), at::cat({seed, dst})}, 1);
  }
  PYGB_TORCH_CALL(pygb200_sampler_export_cumsum(s, cum.data_ptr<int64_t>(), stream));
  const at::Tensor cum_host = cum.cpu();   // the API returns a host list (one more sync, as many values as seeds + 1)
  const int64_t* cp = cum_host.data_ptr<int64_t>();
  return std::make_tuple(node, eid, std::vector<int64_t>(cp, cp + S + 1));
}

std::tuple<c10::Dict<rel_type, at::Tensor>, c10::Dict<rel_type, at::Tensor>, c10::Dict<node_type, at::Tensor>,
           std::optional<c10::Dict<rel_type, at::Tensor>>, c10::Dict<node_type, std::vector<int64_t>>,
           c10::Dict<rel_type, std::vector<int64_t>>>
hetero_neighbor_sample_cuda(const std::vector<node_type>& node_types, const std::vector<edge_type>& edge_types,
                            const c10::Dict<rel_type, at::Tensor>& rowptr_dict,
                            const c10::Dict<rel_type, at::Tensor>& col_dict,
                            const c10::Dict<node_type, at::Tensor>& seed_dict,
                            const c10::Dict<rel_type, std::vector<int64_t>>& num_neighbors_dict,
                            const std::optional<c10::Dict<node_type, at::Tensor>>& node_time_dict,
                            const std::optional<c10::Dict<rel_type, at::Tensor>>& edge_time_dict,
                            const std::optional<c10::Dict<node_type, at::Tensor>>& seed_time_dict,
                            const std::optional<c10::Dict<rel_type, at::Tensor>>& edge_weight_dict, bool csc,
                            bool replace, bool directed, bool disjoint, std::string temporal_strategy,
                            bool return_edge_id) {
  TORCH_CHECK(temporal_strategy == "uniform" || temporal_strategy == "last", "No valid temporal strategy found");
  check_arguments(node_time_dict.has_value(), edge_time_dict.has_value(), seed_time_dict.has_value(),
                  edge_weight_dict.has_value(), disjoint);
  TORCH_CHECK(seed_dict.size() > 0, "hetero_neighbor_sample: empty 'seed_dict'");
  const at::Tensor& first_seed = seed_dict.begin()->value();
  TORCH_CHECK(first_seed.is_cuda(), "pyg_lib_b200: hetero_neighbor_sample expects CUDA tensors (no CPU fallback)");
  const auto st = first_seed.scalar_type();
  const auto dev = first_seed.device();
  TORCH_CHECK(st == at::kLong || st == at::kInt, "hetero_neighbor_sample: index tensors must be int64 or int32");
  const bool idx32 = st == at::kInt;

  // node type indices: seed_dict order first (disjoint batch ids follow it, neighbor_kernel.cpp:669-684)
  std::vector<node_type> types;
  std::map<node_type, int> tix;
  auto add_type = [&](const node_type& t) { if (!tix.count(t)) { tix[t] = (int)types.size(); types.push_back(t); } };
  for (const auto& kv : seed_dict) {
    TORCH_CHECK(std::find(node_types.begin(), node_types.end(), kv.key()) != node_types.end(),
                "seed node type '", kv.key(), "' is not in 'node_types'");
    add_type(kv.key());
  }
  for (const auto& t : node_types) add_type(t);
  const int T = (int)types.size(), R = (int)edge_types.size();

  size_t L = 0;
  for (const auto& k : edge_types) L = std::max(L, num_neighbors_dict.at(to_rel_type(k)).size());
  std::vector<pygb200_relation> rels(R);
  std::vector<int64_t> nn((size_t)R * std::max<size_t>(L, 1), 0);
  for (int r = 0; r < R; ++r) {
    const auto& k = edge_types[r];
    const rel_type rk = to_rel_type(k);
    const at::Tensor& rowptr = rowptr_dict.at(rk);
    const at::Tensor& col = col_dict.at(rk);
    check_index_tensor(rowptr, "rowptr", st, dev);
    check_index_tensor(col, "col", st, dev);
    const node_type& src = !csc ? std::get<0>(k) : std::get<2>(k);  // roles swap for csc (neighbor_kernel.cpp:718-719)
    const node_type& dst = !csc ? std::get<2>(k) : std::get<0>(k);
    TORCH_CHECK(tix.count(src) && tix.count(dst), "edge type '", rk, "' uses a node type missing from 'node_types'");
    rels[r].rowptr = rowptr.data_ptr(); rels[r].col = col.data_ptr();
    rels[r].num_src_nodes = rowptr.numel() - 1; rels[r].num_edges = col.numel();
    rels[r].src_type = tix[src]; rels[r].dst_type = tix[dst];
    const auto& v = num_neighbors_dict.at(rk);
    TORCH_CHECK(v.size() == L, "all entries of 'num_neighbors_dict' must have the same number of hops");
    for (size_t h = 0; h < L; ++h) nn[(size_t)r * L + h] = v[h];
  }
  std::vector<const void*> seeds(T, nullptr);
  std::vector<int64_t> n_seeds(T, 0);
  for (const auto& kv : seed_dict) {
    check_index_tensor(kv.value(), "seed", st, dev);
    seeds[tix[kv.key()]] = kv.value().data_ptr();
    n_seeds[tix[kv.key()]] = kv.value().numel();
  }

  c10::cuda::CUDAGuard guard(dev);
  cudaStream_t stream = at::cuda::getCurrentCUDAStream();
  SamplerSlot& slot = get_slot(dev.index(), stream);
  std::lock_guard<std::mutex> op_lock(slot.op_mu);
  pygb200_sampler* s = slot.s;
  unsigned flags = (replace ? PYGB200_S_REPLACE : 0u) | (disjoint ? PYGB200_S_DISJOINT : 0u) | (idx32 ? PYGB200_S_INDEX32 : 0u);
  std::vector<int64_t> nph((size_t)T * (L + 1), 0), eph((size_t)R * std::max<size_t>(L, 1), 0), n_nodes(T, 0), n_edges(std::max(R, 1), 0);
  std::vector<at::Tensor> d_row, d_col, d_eid, d_node;   // bound-sized results (latency path)
  {
    std::vector<const int64_t*> nt(T, nullptr), et(std::max(R, 1), nullptr), stt(T, nullptr);
    bool any = false;
    if (node_time_dict.has_value())
      for (const auto& kv : *node_time_dict)
        if (tix.count(kv.key())) { nt[tix[kv.key()]] = time_ptr(kv.value(), "node_time", dev); any = true; }
    if (edge_time_dict.has_value())
      for (int r = 0; r < R; ++r) {
        const rel_type rk = to_rel_type(edge_types[r]);
        if (edge_time_dict->contains(rk)) { et[r] = time_ptr(edge_time_dict->at(rk), "edge_time", dev); any = true; }
      }
    if (seed_time_dict.has_value())
      for (const auto& kv : *seed_time_dict)
        if (tix.count(kv.key())) stt[tix[kv.key()]] = time_ptr(kv.value(), "seed_time", dev);
    pygb200_temporal tmp{nt.data(), et.data(), stt.data(), temporal_strategy == "last" ? 1 : 0};
    // Latency path (as in neighbor_sample_cuda): bound-sized result tensors the sampling kernels write themselves
    std::vector<int64_t> ncap(T, 0), ecap(R, 0);
    if (!idx32 && !disjoint && L > 0 && R > 0 &&
        pygb200_sampler_bounds(T, R, (int)L, rels.data(), n_seeds.data(), nn.data(), ncap.data(), ecap.data()) == PYGB200_OK) {
      int64_t total = 0;
      bool ok = true;
      for (int t = 0; t < T; ++t) { total += ncap[t]; ok = ok && ncap[t] > 0; }
      for (int r = 0; r < R; ++r) { total += 3 * ecap[r]; ok = ok && ecap[r] > 0; }
      if (ok && total * 8 <= kDirectOutputBytes) {
        const auto opt0 = first_seed.options();
        std::vector<void*> rp(R), cp(R), ep(R, nullptr), np(T);
        d_row.resize(R); d_col.resize(R); d_eid.resize(R); d_node.resize(T);
        for (int t = 0; t < T; ++t) { d_node[t] = at::empty({ncap[t]}, opt0); np[t] = d_node[t].data_ptr(); }
        for (int r = 0; r < R; ++r) {
          d_row[r] = at::empty({ecap[r]}, opt0); d_col[r] = at::empty({ecap[r]}, opt0);
          rp[r] = d_row[r].data_ptr(); cp[r] = d_col[r].data_ptr();
          if (return_edge_id) { d_eid[r] = at::empty({ecap[r]}, opt0); ep[r] = d_eid[r].data_ptr(); }
        }
        PYGB_TORCH_CALL(pygb200_sampler_bind_outputs(s, T, R, rp.data(), cp.data(), ep.data(), np.data(), ecap.data(), ncap.data()));
      }
    }
    // biased sampling: relations that come with weights (neighbor_kernel.cpp:732-745); the others keep drawing uniformly
    std::vector<const void*> wp(std::max(R, 1), nullptr);
    bool biased = false;
    if (edge_weight_dict.has_value() && edge_weight_dict->size() > 0)
      for (int r = 0; r < R; ++r) {
        const rel_type rk = to_rel_type(edge_types[r]);
        const auto& v = num_neighbors_dict.at(rk);
        if (!edge_weight_dict->contains(rk) || std::none_of(v.begin(), v.end(), [](int64_t k) { return k >= 0; })) continue;
        wp[r] = weight_ptr(edge_weight_dict->at(rk), col_dict.at(rk), dev);
        biased = true;
      }
    CpuEngine eng;
    if (biased)
      PYGB_TORCH_CALL(pygb200_sampler_run_weighted(s, T, R, (int)L, rels.data(), seeds.data(), n_seeds.data(), nn.data(), flags,
                                                   &eng.mt, nph.data(), eph.data(), n_nodes.data(), n_edges.data(), stream,
                                                   wp.data(), PYGB200_F32));
    else
    PYGB_TORCH_CALL(pygb200_sampler_run_temporal(s, T, R, (int)L, rels.data(), seeds.data(), n_seeds.data(), nn.data(), flags,
                                                 &eng.mt, nph.data(), eph.data(), n_nodes.data(), n_edges.data(), stream,
                                                 any ? &tmp : nullptr));
    eng.commit();
  }
  TORCH_CHECK(directed, "Undirected heterogeneous graphs not yet supported");  // neighbor_kernel.cpp:824

  const auto opt = first_seed.options();
  c10::Dict<rel_type, at::Tensor> out_row, out_col;
  c10::Dict<node_type, at::Tensor> out_node;
  std::optional<c10::Dict<rel_type, at::Tensor>> out_eid = std::nullopt;
  if (return_edge_id) out_eid = c10::Dict<rel_type, at::Tensor>();
  c10::Dict<node_type, std::vector<int64_t>> out_nph;
  c10::Dict<rel_type, std::vector<int64_t>> out_eph;
  const bool direct_out = pygb200_sampler_outputs_direct(s) != 0;
  for (const auto& t : node_types) {
    const int i = tix[t];
    at::Tensor node;
    if (direct_out) {
      node = d_node[i].narrow(0, 0, n_nodes[i]);
      if ((double)n_nodes[i] < kDirectMinFill * (double)d_node[i].numel()) node = node.clone();
    } else {
      node = disjoint ? at::empty({n_nodes[i], 2}, opt) : at::empty({n_nodes[i]}, opt);
      PYGB_TORCH_CALL(pygb200_sampler_export_nodes(s, i, node.data_ptr(), idx32, stream));
    }
    out_node.insert(t, node);
    out_nph.insert(t, std::vector<int64_t>(nph.begin() + (size_t)i * (L + 1), nph.begin() + (size_t)(i + 1) * (L + 1)));
  }
  for (int r = 0; r < R; ++r) {
    const rel_type rk = to_rel_type(edge_types[r]);
    at::Tensor row, colv, eid;
    if (direct_out) {
      row = d_row[r].narrow(0, 0, n_edges[r]); colv = d_col[r].narrow(0, 0, n_edges[r]);
      if (return_edge_id) eid = d_eid[r].narrow(0, 0, n_edges[r]);
      if ((double)n_edges[r] < kDirectMinFill * (double)d_row[r].numel()) {
        row = row.clone(); colv = colv.clone();
        if (return_edge_id) eid = eid.clone();
      }
    } else {
      row = at::empty({n_edges[r]}, opt); colv = at::empty({n_edges[r]}, opt);
      if (return_edge_id) eid = at::empty({n_edges[r]}, opt);
      PYGB_TORCH_CALL(pygb200_sampler_export_edges(s, r, row.data_ptr(), colv.data_ptr(),
                                                   return_edge_id ? eid.data_ptr() : nullptr, idx32, stream));
    }
    if (csc) std::swap(row, colv);
    out_row.insert(rk, row);
    out_col.insert(rk, colv);
    if (return_edge_id) out_eid->insert(rk, eid);
    out_eph.insert(rk, std::vector<int64_t>(eph.begin() + (size_t)r * L, eph.begin() + (size_t)(r + 1) * L));
  }
  return std::make_tuple(out_row, out_col, out_node, out_eid, out_nph, out_eph);
}

}  // namespace

TORCH_LIBRARY_FRAGMENT(pyg, m) {
  m.def(TORCH_SELECTIVE_SCHEMA(
      "pyg::neighbor_sample(Tensor rowptr, Tensor col, Tensor seed, int[] "
      "num_neighbors, Tensor? node_time = None, Tensor? edge_time = None, "
      "Tensor? seed_time = None, Tensor? edge_weight = None, bool csc = False, "
      "bool replace = False, bool directed = True, bool disjoint = False, "
      "str temporal_strategy = 'uniform', bool return_edge_id = True) -> "
      "(Tensor, Tensor, Tensor, Tensor?, int[], int[])"));
  m.def(TORCH_SELECTIVE_SCHEMA(
      "pyg::hetero_neighbor_sample(str[] node_types, (str, str, str)[] "
      "edge_types, Dict(str, Tensor) rowptr_dict, Dict(str, Tensor) col_dict, "
      "Dict(str, Tensor) seed_dict, Dict(str, int[]) num_neighbors_dict, "
      "Dict(str, Tensor)? node_time_dict = None, Dict(str, Tensor)? "
      "edge_time_dict = None, Dict(str, Tensor)? seed_time_dict = None, "
      "Dict(str, Tensor)? edge_weight_dict = None, bool csc = False, "
      "bool replace = False, bool directed = True, bool disjoint = False, "
      "str temporal_strategy = 'uniform', bool return_edge_id = True) -> "
      "(Dict(str, Tensor), Dict(str, Tensor), Dict(str, Tensor), "
      "Dict(str, Tensor)?, Dict(str, int[]), Dict(str, int[]))"));
  m.def(TORCH_SELECTIVE_SCHEMA(   // pyg_lib/csrc/sampler/neighbor.cpp:148-153
      "pyg::dist_neighbor_sample(Tensor rowptr, Tensor col, Tensor seed, int "
      "num_neighbors, Tensor? node_time = None, Tensor? edge_time = None, "
      "Tensor? seed_time = None, Tensor? edge_weight = None, bool csc = False, "
      "bool replace = False, bool directed = True, bool disjoint = False, "
      "str temporal_strategy = 'uniform') -> (Tensor, Tensor, int[])"));
}

TORCH_LIBRARY_IMPL(pyg, CUDA, m) {
  m.impl(TORCH_SELECTIVE_NAME("pyg::neighbor_sample"), TORCH_FN(neighbor_sample_cuda));
  m.impl(TORCH_SELECTIVE_NAME("pyg::dist_neighbor_sample"), TORCH_FN(dist_neighbor_sample_cuda));
}

TORCH_LIBRARY_IMPL(pyg, BackendSelect, m) {
  m.impl(TORCH_SELECTIVE_NAME("pyg::hetero_neighbor_sample"), TORCH_FN(hetero_neighbor_sample_cuda));
}

}  // namespace sampler
}  // namespace pyg
