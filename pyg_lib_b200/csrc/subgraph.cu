// pyg_lib_b200/csrc/subgraph.cu — induced subgraph (pyg::subgraph) for sm_90a (H100).
//
// Replaces subgraph_kernel (pyg_lib/csrc/sampler/cpu/subgraph_kernel.cpp:13-89), same two sweeps with the
// prefix sum between them, each node row handled by one warp:
//   map      nodes -> dense ids in first-occurrence order (Mapper::fill, mapper.h:29-53): open-addressing
//            table, insert + min(position) per key, first-occurrence flags, exclusive scan, ids into the table
//   count    row i: how many neighbours of nodes[i] are in the set            (:41-52)
//   scan     out_rowptr = [0, cumsum(deg)]                                    (:54-57), total -> host
//   fill     row i: the kept neighbours' ids (+ edge positions) in CSR order   (:66-82): 32 neighbours per step,
//            ballot + popc give every kept edge its place, so the order inside a row is the reference's
// HBM-bound integer work: per selected node 2 rowptr words, per incident edge one coalesced `col` read and one
// random 16-byte table probe (L2-resident for realistic set sizes); per kept edge 8(+8) bytes written.
#include <algorithm>
#include <mutex>

#include "common.cuh"

namespace pygb200 {
namespace {

constexpr int NT = 256;
constexpr u64 EMPTY = ~0ull;
constexpr int SCAN_ITEMS = 4;                 // per thread
constexpr int SCAN_TILE = NT * SCAN_ITEMS;    // per block

__device__ __forceinline__ u64 slot_of(u64 key, u64 mask) {
  return (key * 0x9E3779B97F4A7C15ull) >> (64 - __popcll(mask));   // capacity = mask + 1 = 2^k >= 2
}
__device__ __forceinline__ u32 table_insert(u64* keys, u64 mask, u64 key) {
  u64 s = slot_of(key, mask);
  while (true) {
    const u64 prev = atomicCAS(&keys[s], EMPTY, key);
    if (prev == EMPTY || prev == key) return (u32)s;
    s = (s + 1) & mask;
  }
}
// id of `key`, or -1 (table is read-only while this runs)
__device__ __forceinline__ i64 table_find(const u64* __restrict__ keys, const u64* __restrict__ vals, u64 mask, u64 key) {
  u64 s = slot_of(key, mask);
  while (true) {
    const u64 k = keys[s];
    if (k == key) return (i64)vals[s];
    if (k == EMPTY) return -1;
    s = (s + 1) & mask;
  }
}

inline int grid_for(i64 items, int per_block, int sm_count) {
  const i64 b = (std::max<i64>(items, 1) + per_block - 1) / per_block;
  return (int)std::min<i64>(b, (i64)sm_count * 16);
}

// ---- map
template <typename idx_t>
__global__ void __launch_bounds__(NT) k_sg_insert(const idx_t* __restrict__ nodes, i64 n, i64 num_nodes, u64* keys, u64* vals, u64 mask,
                                                   u32* slot, i64* err) {
  for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < n; i += (i64)gridDim.x * NT) {
    const i64 v = (i64)nodes[i];
    if (v < 0 || v >= num_nodes) { *err = 1; slot[i] = 0; continue; }
    const u32 s = table_insert(keys, mask, (u64)v);
    atomicMin(&vals[s], (u64)i);
    slot[i] = s;
  }
}
__global__ void __launch_bounds__(NT) k_sg_first(const u32* __restrict__ slot, const u64* __restrict__ vals, i64 n, i64* flag) {
  for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < n; i += (i64)gridDim.x * NT) flag[i] = vals[slot[i]] == (u64)i ? 1 : 0;
}
__global__ void __launch_bounds__(NT) k_sg_assign(const u32* __restrict__ slot, const i64* __restrict__ flag, const i64* __restrict__ ids,
                                                   i64 n, u64* vals) {
  for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < n; i += (i64)gridDim.x * NT)
    if (flag[i]) vals[slot[i]] = (u64)ids[i];
}
__global__ void __launch_bounds__(NT) k_sg_clean(const u32* __restrict__ slot, i64 n, u64* keys, u64* vals) {
  for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < n; i += (i64)gridDim.x * NT) { keys[slot[i]] = EMPTY; vals[slot[i]] = EMPTY; }
}

// ---- exclusive scan of i64 (three launches: tile scans, scan of the tile sums by one block, add)
__global__ void __launch_bounds__(NT) k_scan_tiles(const i64* __restrict__ in, i64* __restrict__ out, i64 n, i64* __restrict__ tile_sum) {
  __shared__ i64 s_w[NT / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (i64 tile = blockIdx.x; tile * SCAN_TILE < n; tile += gridDim.x) {
    const i64 base = tile * SCAN_TILE + (i64)threadIdx.x * SCAN_ITEMS;
    i64 v[SCAN_ITEMS], sum = 0;
#pragma unroll
    for (int q = 0; q < SCAN_ITEMS; ++q) { v[q] = base + q < n ? in[base + q] : 0; sum += v[q]; }
    i64 inc = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const i64 o = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc += o;
    }
    if (lane == 31) s_w[wid] = inc;
    __syncthreads();
    i64 pre = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < NT / 32; ++w) { if (w < wid) pre += s_w[w]; tot += s_w[w]; }
    i64 ex = pre + inc - sum;
#pragma unroll
    for (int q = 0; q < SCAN_ITEMS; ++q) { if (base + q < n) out[base + q] = ex; ex += v[q]; }
    if (threadIdx.x == 0) tile_sum[tile] = tot;
    __syncthreads();
  }
}
__global__ void __launch_bounds__(NT) k_scan_sums(i64* tile_sum, i64 ntiles, i64* total) {
  __shared__ i64 s_w[NT / 32];
  __shared__ i64 carry;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (i64 base = 0; base < ntiles; base += NT) {
    const i64 t = base + threadIdx.x;
    const i64 v = t < ntiles ? tile_sum[t] : 0;
    i64 inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const i64 o = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc += o;
    }
    if (lane == 31) s_w[wid] = inc;
    __syncthreads();
    i64 pre = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < NT / 32; ++w) { if (w < wid) pre += s_w[w]; tot += s_w[w]; }
    const i64 c0 = carry;
    if (t < ntiles) tile_sum[t] = c0 + pre + inc - v;
    __syncthreads();
    if (threadIdx.x == 0) carry = c0 + tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry;
}
// out[i] += offset of its tile; optionally also the caller-typed copy dst[i] (+ dst[n] = total)
template <typename out_t>
__global__ void __launch_bounds__(NT) k_scan_add(i64* __restrict__ out, i64 n, const i64* __restrict__ tile_sum, const i64* __restrict__ total,
                                                  out_t* __restrict__ dst) {
  for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i <= n; i += (i64)gridDim.x * NT) {
    if (i == n) { if (dst) dst[n] = (out_t)*total; continue; }
    const i64 v = out[i] + tile_sum[i / SCAN_TILE];
    out[i] = v;
    if (dst) dst[i] = (out_t)v;
  }
}

// ---- count / fill: one warp per selected node
template <typename idx_t>
__global__ void __launch_bounds__(NT) k_sg_count(const idx_t* __restrict__ rowptr, const idx_t* __restrict__ col, const idx_t* __restrict__ nodes,
                                                  i64 n, i64 num_nodes, const u64* __restrict__ keys, const u64* __restrict__ vals, u64 mask,
                                                  i64* __restrict__ deg) {
  const int lane = threadIdx.x & 31;
  const i64 warps = (i64)gridDim.x * (NT / 32);
  for (i64 i = (i64)blockIdx.x * (NT / 32) + (threadIdx.x >> 5); i < n; i += warps) {
    const i64 v = (i64)nodes[i];
    if (v < 0 || v >= num_nodes) { if (lane == 0) deg[i] = 0; continue; }   // (reported by k_sg_insert; never read out of bounds)
    const i64 rs = (i64)rowptr[v], re = (i64)rowptr[v + 1];
    int cnt = 0;
    for (i64 j = rs + lane; j < re; j += 32) cnt += table_find(keys, vals, mask, (u64)(i64)col[j]) >= 0;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, d);
    if (lane == 0) deg[i] = cnt;
  }
}
template <typename idx_t>
__global__ void __launch_bounds__(NT) k_sg_fill(const idx_t* __restrict__ rowptr, const idx_t* __restrict__ col, const idx_t* __restrict__ nodes,
                                                 i64 n, const u64* __restrict__ keys, const u64* __restrict__ vals, u64 mask,
                                                 const i64* __restrict__ offs, idx_t* __restrict__ out_col, idx_t* __restrict__ out_eid) {
  const int lane = threadIdx.x & 31;
  const i64 warps = (i64)gridDim.x * (NT / 32);
  for (i64 i = (i64)blockIdx.x * (NT / 32) + (threadIdx.x >> 5); i < n; i += warps) {
    const i64 v = (i64)nodes[i];
    const i64 rs = (i64)rowptr[v], re = (i64)rowptr[v + 1];
    i64 off = offs[i];
    for (i64 j0 = rs; j0 < re; j0 += 32) {   // (warp-uniform trip count: the ballot below is collective)
      const i64 j = j0 + lane;
      const i64 w = j < re ? table_find(keys, vals, mask, (u64)(i64)col[j]) : -1;
      const unsigned kept = __ballot_sync(0xffffffffu, w >= 0);
      if (w >= 0) {
        const i64 p = off + __popc(kept & ((1u << lane) - 1u));
        out_col[p] = (idx_t)w;
        if (out_eid) out_eid[p] = (idx_t)j;
      }
      off += __popc(kept);
    }
  }
}

// ---- relabel_neighborhood (dist_relabel_kernel.cpp:30-95): positions 0..S-1 are the seeds, S.. the sampled nodes
// (with duplicates); a node's id is its rank among the first occurrences of that sequence.  Disjoint: the key is
// (batch, node) — a seed is its own batch (`:70-73`), a sampled node brings its batch id.
template <typename idx_t>
__global__ void __launch_bounds__(NT) k_rl_insert(const idx_t* __restrict__ seed, i64 S, i64 seed_batch0, const idx_t* __restrict__ sampled,
                                                   const idx_t* __restrict__ batch, i64 M, u64* keys, u64* vals, u64 mask, u32* slot, i64* err) {
  for (i64 p = (i64)blockIdx.x * NT + threadIdx.x; p < S + M; p += (i64)gridDim.x * NT) {
    const i64 v = p < S ? (i64)seed[p] : (i64)sampled[p - S];
    const i64 b = batch ? (p < S ? seed_batch0 + p : (i64)batch[p - S]) : 0;
    if (v < 0 || v >= ((i64)1 << 40) || b < 0 || b >= ((i64)1 << 23)) { *err = 1; slot[p] = 0; continue; }
    const u32 s = table_insert(keys, mask, ((u64)b << 40) | (u64)v);
    atomicMin(&vals[s], (u64)p);
    slot[p] = s;
  }
}
template <typename idx_t>
__global__ void __launch_bounds__(NT) k_rl_cols(const u32* __restrict__ slot, const u64* __restrict__ vals, i64 S, i64 M, idx_t* __restrict__ out_col) {
  for (i64 j = (i64)blockIdx.x * NT + threadIdx.x; j < M; j += (i64)gridDim.x * NT) out_col[j] = (idx_t)vals[slot[S + j]];
}
// row[j] = index of the source node whose run of sampled neighbours holds position j (`:76-88`): the last i with
// offs[i] <= j (offs = exclusive prefix of the per-node counts; nodes without neighbours share an offset with their successor)
template <typename idx_t>
__global__ void __launch_bounds__(NT) k_rl_rows(const i64* __restrict__ offs, i64 n_counts, i64 M, idx_t* __restrict__ out_row) {
  for (i64 j = (i64)blockIdx.x * NT + threadIdx.x; j < M; j += (i64)gridDim.x * NT) {
    i64 lo = 0, hi = n_counts;   // first i with offs[i] > j
    while (lo < hi) {
      const i64 mid = lo + ((hi - lo) >> 1);
      if (offs[mid] > j) hi = mid; else lo = mid + 1;
    }
    out_row[j] = (idx_t)(lo - 1);
  }
}

// hetero relabel: output edge j of a relation lies in source segment s (the last s with offs[s] <= j); its row is that
// segment's source index and its col the id at the segment's position in the destination type's id list
template <typename idx_t>
__global__ void __launch_bounds__(NT) k_rl_expand(const i64* __restrict__ offs, i64 n_seg, i64 M, const i64* __restrict__ seg_row,
                                                   const i64* __restrict__ seg_pos, const idx_t* __restrict__ ids, idx_t* __restrict__ out_row,
                                                   idx_t* __restrict__ out_col) {
  for (i64 j = (i64)blockIdx.x * NT + threadIdx.x; j < M; j += (i64)gridDim.x * NT) {
    i64 lo = 0, hi = n_seg;
    while (lo < hi) {
      const i64 mid = lo + ((hi - lo) >> 1);
      if (offs[mid] > j) hi = mid; else lo = mid + 1;
    }
    const i64 sgm = lo - 1;
    out_row[j] = (idx_t)seg_row[sgm];
    out_col[j] = ids[seg_pos[sgm] + (j - offs[sgm])];
  }
}

// merge_sampler_outputs: output element i lies in segment s (the last s with offs[s] <= i) and is a copy of element
// seg_begin[s] + (i - offs[s]) of source array seg_src[s] (broadcast: of element seg_begin[s] itself)
template <typename idx_t>
__global__ void __launch_bounds__(NT) k_seg_gather(const i64* __restrict__ offs, i64 n_seg, i64 M, const i64* __restrict__ seg_src,
                                                    const i64* __restrict__ seg_begin, const idx_t* const* __restrict__ src_table, int broadcast,
                                                    idx_t* __restrict__ out) {
  for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < M; i += (i64)gridDim.x * NT) {
    i64 lo = 0, hi = n_seg;
    while (lo < hi) {
      const i64 mid = lo + ((hi - lo) >> 1);
      if (offs[mid] > i) hi = mid; else lo = mid + 1;
    }
    const i64 sgm = lo - 1;
    out[i] = src_table[seg_src[sgm]][seg_begin[sgm] + (broadcast ? 0 : i - offs[sgm])];
  }
}

}  // namespace
}  // namespace pygb200

using namespace pygb200;

struct pygb200_subgraph {
  int device = 0, sm_count = 132;
  DevBuf keys, vals, slot, flag, ids, deg, offs, tiles, misc, segs;   // misc: {total, err}; segs: hetero relabel segment lists
  u64 tcap = 0;
  i64 n = 0;            // node count of the pending count() (fill() must follow with the same inputs)
  bool pending = false;
  std::mutex mu;
};

extern "C" int pygb200_subgraph_create(pygb200_subgraph** out) {
  PYGB_CHECK(out != nullptr, PYGB200_ERR_ARG, "pygb200_subgraph_create: null out");
  int dev = 0;
  PYGB_CUDA(cudaGetDevice(&dev));
  auto* h = new pygb200_subgraph();
  h->device = dev;
  cudaDeviceGetAttribute(&h->sm_count, cudaDevAttrMultiProcessorCount, dev);
  *out = h;
  return PYGB200_OK;
}

extern "C" void pygb200_subgraph_destroy(pygb200_subgraph* h) {
  if (!h) return;
  DevBuf* all[] = {&h->keys, &h->vals, &h->slot, &h->flag, &h->ids, &h->deg, &h->offs, &h->tiles, &h->misc, &h->segs};
  for (DevBuf* b : all) b->release();
  delete h;
}

namespace {
int scan_i64(pygb200_subgraph* h, const i64* in, i64* out, i64 n, i64* total_dev, void* dst, int index32, cudaStream_t st) {
  const i64 ntiles = std::max<i64>((n + SCAN_TILE - 1) / SCAN_TILE, 1);
  if (int e = h->tiles.ensure((size_t)ntiles * 8, 0, st)) return e;
  i64* tiles = h->tiles.as<i64>();
  PYGB_CUDA(cudaMemsetAsync(tiles, 0, (size_t)ntiles * 8, st));
  k_scan_tiles<<<grid_for(ntiles, 1, h->sm_count), NT, 0, st>>>(in, out, n, tiles);
  PYGB_LAUNCH_CHECK();
  k_scan_sums<<<1, NT, 0, st>>>(tiles, ntiles, total_dev);
  PYGB_LAUNCH_CHECK();
  const int g = grid_for(n + 1, NT, h->sm_count);
  if (dst && index32) k_scan_add<int32_t><<<g, NT, 0, st>>>(out, n, tiles, total_dev, (int32_t*)dst);
  else k_scan_add<int64_t><<<g, NT, 0, st>>>(out, n, tiles, total_dev, (int64_t*)dst);
  PYGB_LAUNCH_CHECK();
  return PYGB200_OK;
}
}  // namespace

extern "C" int pygb200_subgraph_count(pygb200_subgraph* h, const void* rowptr, const void* col, int64_t num_nodes,
                                      const void* nodes, int64_t n, int index32, void* out_rowptr, int64_t* n_edges_out,
                                      void* stream) {
  PYGB_CHECK(h && rowptr && out_rowptr && n_edges_out && n >= 0 && num_nodes >= 0 && (nodes || n == 0), PYGB200_ERR_ARG,
             "pygb200_subgraph_count: null / negative argument");
  std::lock_guard<std::mutex> lock(h->mu);
  cudaStream_t st = (cudaStream_t)stream;
  if (h->pending && h->n > 0) {   // a count() nobody followed up with fill(): its entries are still in the table
    k_sg_clean<<<grid_for(h->n, NT, h->sm_count), NT, 0, st>>>(h->slot.as<u32>(), h->n, h->keys.as<u64>(), h->vals.as<u64>());
    PYGB_LAUNCH_CHECK();
  }
  h->pending = false;
  // workspace: table at load <= 0.5 (all-EMPTY between calls), per-node scratch
  u64 cap = 2;
  while (cap < 2 * (u64)std::max<i64>(n, 1)) cap <<= 1;
  PYGB_CHECK(cap <= (1ull << 32), PYGB200_ERR_UNSUPPORTED, "subgraph: node set too large");
  if (cap > h->tcap) {
    if (int e = h->keys.ensure(cap * 8, 0, st)) return e;
    if (int e = h->vals.ensure(cap * 8, 0, st)) return e;
    PYGB_CUDA(cudaMemsetAsync(h->keys.p, 0xff, h->keys.cap, st));
    PYGB_CUDA(cudaMemsetAsync(h->vals.p, 0xff, h->vals.cap, st));
    h->tcap = cap;
  }
  const u64 mask = h->tcap - 1;
  const size_t nn = (size_t)std::max<i64>(n, 1);
  if (int e = h->slot.ensure(nn * 4, 0, st)) return e;
  if (int e = h->flag.ensure(nn * 8, 0, st)) return e;
  if (int e = h->ids.ensure(nn * 8, 0, st)) return e;
  if (int e = h->deg.ensure(nn * 8, 0, st)) return e;
  if (int e = h->offs.ensure(nn * 8, 0, st)) return e;
  if (int e = h->misc.ensure(64, 0, st)) return e;
  i64* misc = h->misc.as<i64>();
  PYGB_CUDA(cudaMemsetAsync(misc, 0, 64, st));
  u64 *keys = h->keys.as<u64>(), *vals = h->vals.as<u64>();
  u32* slot = h->slot.as<u32>();
  const int g = grid_for(n, NT, h->sm_count), gw = grid_for(n, NT / 32, h->sm_count);
  if (n > 0) {
    if (index32) k_sg_insert<int32_t><<<g, NT, 0, st>>>((const int32_t*)nodes, n, num_nodes, keys, vals, mask, slot, misc + 1);
    else k_sg_insert<int64_t><<<g, NT, 0, st>>>((const int64_t*)nodes, n, num_nodes, keys, vals, mask, slot, misc + 1);
    PYGB_LAUNCH_CHECK();
    k_sg_first<<<g, NT, 0, st>>>(slot, vals, n, h->flag.as<i64>());
    PYGB_LAUNCH_CHECK();
    if (int e = scan_i64(h, h->flag.as<i64>(), h->ids.as<i64>(), n, misc + 2, nullptr, 0, st)) return e;
    k_sg_assign<<<g, NT, 0, st>>>(slot, h->flag.as<i64>(), h->ids.as<i64>(), n, vals);
    PYGB_LAUNCH_CHECK();
    if (index32) k_sg_count<int32_t><<<gw, NT, 0, st>>>((const int32_t*)rowptr, (const int32_t*)col, (const int32_t*)nodes, n, num_nodes, keys, vals, mask, h->deg.as<i64>());
    else k_sg_count<int64_t><<<gw, NT, 0, st>>>((const int64_t*)rowptr, (const int64_t*)col, (const int64_t*)nodes, n, num_nodes, keys, vals, mask, h->deg.as<i64>());
    PYGB_LAUNCH_CHECK();
  }
  if (int e = scan_i64(h, h->deg.as<i64>(), h->offs.as<i64>(), n, misc, out_rowptr, index32, st)) return e;
  i64 host[2] = {0, 0};
  PYGB_CUDA(cudaMemcpyAsync(host, misc, 16, cudaMemcpyDeviceToHost, st));
  PYGB_CUDA(cudaStreamSynchronize(st));
  if (host[1] != 0) {   // leave the table clean: every listed slot goes back to EMPTY (bad entries used slot 0 of nothing)
    if (n > 0) {
      PYGB_CUDA(cudaMemsetAsync(h->keys.p, 0xff, h->keys.cap, st));
      PYGB_CUDA(cudaMemsetAsync(h->vals.p, 0xff, h->vals.cap, st));
    }
    set_error("subgraph: 'nodes' contains an index outside [0, num_nodes)");
    return PYGB200_ERR_ARG;
  }
  PYGB_CHECK(!index32 || host[0] < ((i64)1 << 31), PYGB200_ERR_UNSUPPORTED, "subgraph: edge count exceeds int32");
  *n_edges_out = host[0];
  h->n = n;
  h->pending = true;
  return PYGB200_OK;
}

extern "C" int pygb200_subgraph_fill(pygb200_subgraph* h, const void* rowptr, const void* col, const void* nodes, int64_t n,
                                     int index32, void* out_col, void* out_edge_id, void* stream) {
  PYGB_CHECK(h && rowptr && (nodes || n == 0), PYGB200_ERR_ARG, "pygb200_subgraph_fill: null argument");
  std::lock_guard<std::mutex> lock(h->mu);
  PYGB_CHECK(h->pending && h->n == n, PYGB200_ERR_ARG, "pygb200_subgraph_fill: no matching pygb200_subgraph_count before it");
  cudaStream_t st = (cudaStream_t)stream;
  h->pending = false;
  if (n == 0) return PYGB200_OK;
  const u64 mask = h->tcap - 1;
  const int g = grid_for(n, NT, h->sm_count), gw = grid_for(n, NT / 32, h->sm_count);
  if (out_col) {
    if (index32) k_sg_fill<int32_t><<<gw, NT, 0, st>>>((const int32_t*)rowptr, (const int32_t*)col, (const int32_t*)nodes, n, h->keys.as<u64>(), h->vals.as<u64>(), mask,
                                                        h->offs.as<i64>(), (int32_t*)out_col, (int32_t*)out_edge_id);
    else k_sg_fill<int64_t><<<gw, NT, 0, st>>>((const int64_t*)rowptr, (const int64_t*)col, (const int64_t*)nodes, n, h->keys.as<u64>(), h->vals.as<u64>(), mask,
                                                h->offs.as<i64>(), (int64_t*)out_col, (int64_t*)out_edge_id);
    PYGB_LAUNCH_CHECK();
  }
  k_sg_clean<<<g, NT, 0, st>>>(h->slot.as<u32>(), n, h->keys.as<u64>(), h->vals.as<u64>());
  PYGB_LAUNCH_CHECK();
  return PYGB200_OK;
}

namespace {
// ids of `sampled` [n_sampled] among the first occurrences of [seed | sampled] -> out_col (caller dtype); leaves the
// map clean.  Caller holds h->mu.  The error flag (misc[1]) is read by the caller after its own sync.
int relabel_ids_locked(pygb200_subgraph* h, const void* seed, i64 n_seed, i64 seed_batch0, const void* sampled, const void* batch,
                       i64 n_sampled, int index32, void* out_col, cudaStream_t st) {
  if (h->pending && h->n > 0) {   // an abandoned pygb200_subgraph_count still owns table entries
    k_sg_clean<<<grid_for(h->n, NT, h->sm_count), NT, 0, st>>>(h->slot.as<u32>(), h->n, h->keys.as<u64>(), h->vals.as<u64>());
    PYGB_LAUNCH_CHECK();
  }
  h->pending = false;
  if (int e = h->misc.ensure(64, 0, st)) return e;
  i64* misc = h->misc.as<i64>();
  PYGB_CUDA(cudaMemsetAsync(misc, 0, 64, st));
  if (n_sampled == 0) return PYGB200_OK;
  const i64 N = n_seed + n_sampled;
  u64 cap = 2;
  while (cap < 2 * (u64)N) cap <<= 1;
  PYGB_CHECK(cap <= (1ull << 32), PYGB200_ERR_UNSUPPORTED, "relabel_neighborhood: too many nodes");
  if (cap > h->tcap) {
    if (int e = h->keys.ensure(cap * 8, 0, st)) return e;
    if (int e = h->vals.ensure(cap * 8, 0, st)) return e;
    PYGB_CUDA(cudaMemsetAsync(h->keys.p, 0xff, h->keys.cap, st));
    PYGB_CUDA(cudaMemsetAsync(h->vals.p, 0xff, h->vals.cap, st));
    h->tcap = cap;
  }
  const u64 mask = h->tcap - 1;
  if (int e = h->slot.ensure((size_t)N * 4, 0, st)) return e;
  if (int e = h->flag.ensure((size_t)N * 8, 0, st)) return e;
  if (int e = h->ids.ensure((size_t)N * 8, 0, st)) return e;
  u64 *keys = h->keys.as<u64>(), *vals = h->vals.as<u64>();
  u32* slot = h->slot.as<u32>();
  const int g = grid_for(N, NT, h->sm_count), gm = grid_for(n_sampled, NT, h->sm_count);
  if (index32) k_rl_insert<int32_t><<<g, NT, 0, st>>>((const int32_t*)seed, n_seed, seed_batch0, (const int32_t*)sampled, (const int32_t*)batch, n_sampled, keys, vals, mask, slot, misc + 1);
  else k_rl_insert<int64_t><<<g, NT, 0, st>>>((const int64_t*)seed, n_seed, seed_batch0, (const int64_t*)sampled, (const int64_t*)batch, n_sampled, keys, vals, mask, slot, misc + 1);
  PYGB_LAUNCH_CHECK();
  k_sg_first<<<g, NT, 0, st>>>(slot, vals, N, h->flag.as<i64>());
  PYGB_LAUNCH_CHECK();
  if (int e = scan_i64(h, h->flag.as<i64>(), h->ids.as<i64>(), N, misc + 2, nullptr, 0, st)) return e;
  k_sg_assign<<<g, NT, 0, st>>>(slot, h->flag.as<i64>(), h->ids.as<i64>(), N, vals);
  PYGB_LAUNCH_CHECK();
  if (index32) k_rl_cols<int32_t><<<gm, NT, 0, st>>>(slot, vals, n_seed, n_sampled, (int32_t*)out_col);
  else k_rl_cols<int64_t><<<gm, NT, 0, st>>>(slot, vals, n_seed, n_sampled, (int64_t*)out_col);
  PYGB_LAUNCH_CHECK();
  k_sg_clean<<<g, NT, 0, st>>>(slot, N, keys, vals);
  PYGB_LAUNCH_CHECK();
  return PYGB200_OK;
}
int relabel_check_error(pygb200_subgraph* h, cudaStream_t st) {
  i64 err = 0;
  PYGB_CUDA(cudaMemcpyAsync(&err, h->misc.as<i64>() + 1, 8, cudaMemcpyDeviceToHost, st));
  PYGB_CUDA(cudaStreamSynchronize(st));   // (also keeps host lists alive until their copies are done)
  PYGB_CHECK(err == 0, PYGB200_ERR_ARG, "relabel_neighborhood: node id outside [0, 2^40) or batch id outside [0, 2^23)");
  return PYGB200_OK;
}
}  // namespace

extern "C" int pygb200_relabel_neighborhood(pygb200_subgraph* h, const void* seed, int64_t n_seed, const void* sampled,
                                            const void* batch, int64_t n_sampled, const int64_t* counts_host, int64_t n_counts,
                                            int index32, void* out_row, void* out_col, void* stream) {
  PYGB_CHECK(h && n_seed >= 0 && n_sampled >= 0 && n_counts >= 0 && (seed || n_seed == 0) && (sampled || n_sampled == 0) &&
                 (counts_host || n_counts == 0) && ((out_row && out_col) || n_sampled == 0),
             PYGB200_ERR_ARG, "pygb200_relabel_neighborhood: null / negative argument");
  i64 total = 0;
  for (i64 i = 0; i < n_counts; ++i) {
    PYGB_CHECK(counts_host[i] >= 0, PYGB200_ERR_ARG, "relabel_neighborhood: negative neighbour count");
    total += counts_host[i];
  }
  PYGB_CHECK(total == n_sampled, PYGB200_ERR_ARG, "relabel_neighborhood: the neighbour counts do not add up to the number of sampled nodes");
  std::lock_guard<std::mutex> lock(h->mu);
  cudaStream_t st = (cudaStream_t)stream;
  if (int e = relabel_ids_locked(h, seed, n_seed, 0, sampled, batch, n_sampled, index32, out_col, st)) return e;
  if (n_sampled == 0) return PYGB200_OK;
  // rows: per-node counts (a host list in the reference's API) -> offsets -> one binary search per edge
  if (int e = h->deg.ensure((size_t)n_counts * 8, 0, st)) return e;
  if (int e = h->offs.ensure((size_t)n_counts * 8, 0, st)) return e;
  PYGB_CUDA(cudaMemcpyAsync(h->deg.p, counts_host, (size_t)n_counts * 8, cudaMemcpyHostToDevice, st));
  if (int e = scan_i64(h, h->deg.as<i64>(), h->offs.as<i64>(), n_counts, h->misc.as<i64>(), nullptr, 0, st)) return e;
  const int gm = grid_for(n_sampled, NT, h->sm_count);
  if (index32) k_rl_rows<int32_t><<<gm, NT, 0, st>>>(h->offs.as<i64>(), n_counts, n_sampled, (int32_t*)out_row);
  else k_rl_rows<int64_t><<<gm, NT, 0, st>>>(h->offs.as<i64>(), n_counts, n_sampled, (int64_t*)out_row);
  PYGB_LAUNCH_CHECK();
  return relabel_check_error(h, st);
}

extern "C" int pygb200_relabel_ids(pygb200_subgraph* h, const void* seed, int64_t n_seed, int64_t seed_batch0, const void* sampled,
                                   const void* batch, int64_t n_sampled, int index32, void* out_ids, void* stream) {
  PYGB_CHECK(h && n_seed >= 0 && n_sampled >= 0 && seed_batch0 >= 0 && (seed || n_seed == 0) && (sampled || n_sampled == 0) &&
                 (out_ids || n_sampled == 0),
             PYGB200_ERR_ARG, "pygb200_relabel_ids: null / negative argument");
  std::lock_guard<std::mutex> lock(h->mu);
  cudaStream_t st = (cudaStream_t)stream;
  if (int e = relabel_ids_locked(h, seed, n_seed, seed_batch0, sampled, batch, n_sampled, index32, out_ids, st)) return e;
  return relabel_check_error(h, st);
}

extern "C" int pygb200_relabel_expand(pygb200_subgraph* h, const int64_t* seg_count_host, const int64_t* seg_row_host,
                                      const int64_t* seg_pos_host, int64_t n_seg, const void* ids, int64_t n_ids, int index32,
                                      void* out_row, void* out_col, void* stream) {
  PYGB_CHECK(h && n_seg >= 0 && n_ids >= 0 && ((seg_count_host && seg_row_host && seg_pos_host) || n_seg == 0), PYGB200_ERR_ARG,
             "pygb200_relabel_expand: null / negative argument");
  i64 total = 0;
  for (i64 i = 0; i < n_seg; ++i) {
    PYGB_CHECK(seg_count_host[i] >= 0 && seg_pos_host[i] >= 0 && seg_pos_host[i] + seg_count_host[i] <= n_ids, PYGB200_ERR_ARG,
               "relabel_expand: segment outside the id list");
    total += seg_count_host[i];
  }
  if (total == 0) return PYGB200_OK;
  PYGB_CHECK(ids && out_row && out_col, PYGB200_ERR_ARG, "pygb200_relabel_expand: null output");
  std::lock_guard<std::mutex> lock(h->mu);
  cudaStream_t st = (cudaStream_t)stream;
  if (int e = h->deg.ensure((size_t)n_seg * 8, 0, st)) return e;
  if (int e = h->offs.ensure((size_t)n_seg * 8, 0, st)) return e;
  if (int e = h->segs.ensure((size_t)n_seg * 16, 0, st)) return e;
  if (int e = h->misc.ensure(64, 0, st)) return e;
  i64* seg_row = h->segs.as<i64>();
  i64* seg_pos = seg_row + n_seg;
  PYGB_CUDA(cudaMemcpyAsync(h->deg.p, seg_count_host, (size_t)n_seg * 8, cudaMemcpyHostToDevice, st));
  PYGB_CUDA(cudaMemcpyAsync(seg_row, seg_row_host, (size_t)n_seg * 8, cudaMemcpyHostToDevice, st));
  PYGB_CUDA(cudaMemcpyAsync(seg_pos, seg_pos_host, (size_t)n_seg * 8, cudaMemcpyHostToDevice, st));
  if (int e = scan_i64(h, h->deg.as<i64>(), h->offs.as<i64>(), n_seg, h->misc.as<i64>(), nullptr, 0, st)) return e;
  const int gm = grid_for(total, NT, h->sm_count);
  if (index32) k_rl_expand<int32_t><<<gm, NT, 0, st>>>(h->offs.as<i64>(), n_seg, total, seg_row, seg_pos, (const int32_t*)ids, (int32_t*)out_row, (int32_t*)out_col);
  else k_rl_expand<int64_t><<<gm, NT, 0, st>>>(h->offs.as<i64>(), n_seg, total, seg_row, seg_pos, (const int64_t*)ids, (int64_t*)out_row, (int64_t*)out_col);
  PYGB_LAUNCH_CHECK();
  PYGB_CUDA(cudaStreamSynchronize(st));   // the host lists may go away after the call
  return PYGB200_OK;
}

// ---- merge_sampler_outputs (pyg_lib/csrc/sampler/cpu/dist_merge_outputs_kernel.cpp:15-137)
// Host arithmetic only (no CUDA call): where seed j's neighbours sit in the output of the partition that sampled it.
extern "C" int pygb200_merge_plan(const int64_t* cumsum_flat, const int64_t* cumsum_off, int64_t num_partitions,
                                  const int64_t* partition_ids, const int64_t* partition_orders, int64_t p_size,
                                  const int64_t* node_numel, const int64_t* edge_numel, int64_t* seg_node_begin,
                                  int64_t* seg_edge_begin, int64_t* seg_count) {
  PYGB_CHECK(num_partitions >= 0 && p_size >= 0 && (p_size == 0 || (cumsum_flat && cumsum_off && partition_ids && partition_orders &&
                                                                    node_numel && edge_numel && seg_node_begin && seg_edge_begin && seg_count)),
             PYGB200_ERR_ARG, "pygb200_merge_plan: null / negative argument");
  for (i64 j = 0; j < p_size; ++j) {
    const i64 p = partition_ids[j], o = partition_orders[j];
    PYGB_CHECK(p >= 0 && p < num_partitions, PYGB200_ERR_ARG, "merge_sampler_outputs: partition id out of range");
    const int64_t* cs = cumsum_flat + cumsum_off[p];
    const i64 len = cumsum_off[p + 1] - cumsum_off[p];
    PYGB_CHECK(o >= 0 && o + 1 < len, PYGB200_ERR_ARG, "merge_sampler_outputs: sampling order outside the partition's cumulative counts");
    // node ids start with the partition's seeds (cs[0] of them); edge ids have no such prefix (:85-92)
    const i64 begin_node = cs[o], end_node = cs[o + 1], begin_edge = begin_node - cs[0];
    PYGB_CHECK(end_node >= begin_node && begin_node >= 0 && end_node <= node_numel[p] && begin_edge >= 0 &&
                   begin_edge + (end_node - begin_node) <= edge_numel[p],
               PYGB200_ERR_ARG, "merge_sampler_outputs: cumulative counts do not fit the partition's outputs");
    seg_node_begin[j] = begin_node;
    seg_edge_begin[j] = begin_edge;
    seg_count[j] = end_node - begin_node;
  }
  return PYGB200_OK;
}

extern "C" int pygb200_segment_gather(pygb200_subgraph* h, const void* const* src_ptrs_host, int64_t n_src, const int64_t* seg_src_host,
                                      const int64_t* seg_begin_host, const int64_t* seg_count_host, int64_t n_seg, int broadcast,
                                      int index32, void* out, void* stream) {
  PYGB_CHECK(h && n_src >= 0 && n_seg >= 0 && (n_seg == 0 || (src_ptrs_host && seg_src_host && seg_begin_host && seg_count_host)),
             PYGB200_ERR_ARG, "pygb200_segment_gather: null / negative argument");
  i64 total = 0;
  for (i64 i = 0; i < n_seg; ++i) {
    PYGB_CHECK(seg_count_host[i] >= 0 && seg_begin_host[i] >= 0 && seg_src_host[i] >= 0 && seg_src_host[i] < n_src, PYGB200_ERR_ARG,
               "segment_gather: bad segment");
    total += seg_count_host[i];
  }
  if (total == 0) return PYGB200_OK;
  PYGB_CHECK(out != nullptr, PYGB200_ERR_ARG, "pygb200_segment_gather: null output");
  std::lock_guard<std::mutex> lock(h->mu);
  cudaStream_t st = (cudaStream_t)stream;
  if (int e = h->deg.ensure((size_t)n_seg * 8, 0, st)) return e;
  if (int e = h->offs.ensure((size_t)n_seg * 8, 0, st)) return e;
  if (int e = h->segs.ensure((size_t)(2 * n_seg + n_src) * 8, 0, st)) return e;
  if (int e = h->misc.ensure(64, 0, st)) return e;
  i64* seg_src = h->segs.as<i64>();
  i64* seg_begin = seg_src + n_seg;
  void** table = reinterpret_cast<void**>(seg_begin + n_seg);
  PYGB_CUDA(cudaMemcpyAsync(h->deg.p, seg_count_host, (size_t)n_seg * 8, cudaMemcpyHostToDevice, st));
  PYGB_CUDA(cudaMemcpyAsync(seg_src, seg_src_host, (size_t)n_seg * 8, cudaMemcpyHostToDevice, st));
  PYGB_CUDA(cudaMemcpyAsync(seg_begin, seg_begin_host, (size_t)n_seg * 8, cudaMemcpyHostToDevice, st));
  PYGB_CUDA(cudaMemcpyAsync(table, src_ptrs_host, (size_t)n_src * 8, cudaMemcpyHostToDevice, st));
  if (int e = scan_i64(h, h->deg.as<i64>(), h->offs.as<i64>(), n_seg, h->misc.as<i64>(), nullptr, 0, st)) return e;
  const int g = grid_for(total, NT, h->sm_count);
  if (index32) k_seg_gather<int32_t><<<g, NT, 0, st>>>(h->offs.as<i64>(), n_seg, total, seg_src, seg_begin, (const int32_t* const*)table, broadcast, (int32_t*)out);
  else k_seg_gather<int64_t><<<g, NT, 0, st>>>(h->offs.as<i64>(), n_seg, total, seg_src, seg_begin, (const int64_t* const*)table, broadcast, (int64_t*)out);
  PYGB_LAUNCH_CHECK();
  PYGB_CUDA(cudaStreamSynchronize(st));   // the host lists may go away after the call
  return PYGB200_OK;
}
