/*
 * include/pyg_b200.h — C ABI of libpyg_b200.so: the H100 (sm_90a) implementation of pyg-lib's two
 * data-parallel hot paths.  Plain pointers and sizes only; no torch types.  Everything that is a
 * "const void* / void*" tensor argument is DEVICE memory on the current CUDA device unless it says
 * "host".  `stream` is a cudaStream_t passed as void*.
 *
 * The reference has no FFI layer for these paths: its boundary is the PyTorch dispatcher registry
 * (`TORCH_LIBRARY_FRAGMENT(pyg, m)`).  Each entry point below names the reference operator kernel
 * it replaces (paths relative to the pyg-lib tree); libpyg.so (pyg_lib_b200/csrc/torch/) is the thin
 * registration layer that binds those dispatcher ops to this ABI — see INTEGRATION.md.
 *
 * All functions return 0 on success and a negative code on failure; pygb200_last_error() gives a
 * thread-local message.  There is no CPU fallback anywhere behind this ABI.
 */
#ifndef PYG_B200_H_
#define PYG_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PYGB200_OK 0
#define PYGB200_ERR_CUDA -1
#define PYGB200_ERR_ARG -2
#define PYGB200_ERR_UNSUPPORTED -3
#define PYGB200_ERR_INTERNAL -4

/* element types of matmul operands */
#define PYGB200_F32 0
#define PYGB200_BF16 1
#define PYGB200_F16 2

/* flags for the matmul entry points */
#define PYGB200_MM_ALLOW_TF32 1u  /* fp32 inputs may use TF32 tensor-core math
                                     (== torch.get_float32_matmul_precision() != 'highest',
                                     pyg_lib/csrc/ops/cuda/matmul_kernel.cu:159-165) */
#define PYGB200_MM_FORCE_SIMT 2u  /* debugging: never take the tensor-core paths */

/* flags for the sampler entry points */
#define PYGB200_S_REPLACE 1u
#define PYGB200_S_DISJOINT 2u
#define PYGB200_S_INDEX32 4u      /* rowptr/col/seed are int32 (else int64) */
#define PYGB200_S_DEFER_CLEANUP 8u /* single node type only: the hash-table reset is done by the following
                                     pygb200_sampler_export_all (or by the next run) instead of its own launch */
#define PYGB200_S_NO_DEDUP 16u     /* distributed one-hop sampling (dist_neighbor_sample_kernel, neighbor_kernel.cpp:957-978,
                                     296-303): one node type / relation / hop; sampled neighbours are NOT mapped — after
                                     the run `col` of pygb200_sampler_export_edges holds their GLOBAL ids in emission
                                     order, `row` the index of the seed they came from, and
                                     pygb200_sampler_export_cumsum gives cumsum_neighbors_per_node */

const char* pygb200_last_error(void);
int pygb200_cuda_version(void);          /* CUDA_VERSION the library was built with
                                            (pyg_lib/csrc/library.cpp:19-29 `pyg::cuda_version`) */
int pygb200_kernel_launches(void);       /* number of kernels this library launched so far
                                            (process-wide counter; bench.py reports deltas) */

/* Per-kernel device timing for bench.py's roofline: when enabled, selected kernels are bracketed with
 * CUDA events on their launching stream.  `pygb200_profile_read` synchronises the pending events and
 * returns accumulated milliseconds, launch count and work units (sampler kernels: edges; matmul: rows)
 * for `name` in {"sample","count","mark","assign","lookup","segment_matmul","grouped_gemm"} and, for the throughput /
 * sharded schedule, {"seed","insert","pref","reduce","xbarrier","final","cleanup","export"}, then resets that accumulator.  Returns 0, or PYGB200_ERR_ARG for an unknown name. */
void pygb200_profile_enable(int on);
int pygb200_profile_read(const char* name, double* ms, int64_t* launches, int64_t* work);

/* Debug timeline of the sampler's kernel chain: when enabled, every sampler kernel stamps %globaltimer (ns)
 * when its block 0 starts working / finishes, and when its serial "last block" section starts / ends.
 * Each word is (id << 56) | (smid << 48) | (time & 2^48-1); id = kernel (1 seed, 2 count, 3 sample, 4 mark, 5 assign, 6 final,
 * 7 export) | 8 for the last-block section | 16 for an end stamp.  `pygb200_timeline_read` synchronises the
 * device, copies up to `cap` words (in stamping order) and clears the buffer; returns the word count. */
int pygb200_timeline_enable(int on);
int64_t pygb200_timeline_read(uint64_t* out, int64_t cap);

/* ------------------------------------------------------------------------------------ matmul
 * out[ptr[b]:ptr[b+1], :] = x[ptr[b]:ptr[b+1], :] @ w[b]        (row-major, contiguous)
 *   x [N,K], w [B,K,M], out [N,M] of `dtype`; ptr_dev [B+1] int64 on the DEVICE.
 * Replaces segment_matmul_kernel / grouped_matmul_out_kernel / run_grouped_gemm
 * (pyg_lib/csrc/ops/cuda/matmul_kernel.cu:304-319,121-287,21-100; CUTLASS 2.x sm80 GemmGrouped)
 * with a persistent sm_90a kernel: TMA-staged tiles -> wgmma (register accumulators) -> epilogue.
 * bias (optional, [B,M], may be NULL) is fused into the epilogue — it replaces the Python loop of
 * pyg_lib/ops/__init__.py:169-171.
 */
int pygb200_segment_matmul(const void* x, const int64_t* ptr_dev, const void* w, const void* bias,
                           void* out, int64_t N, int64_t K, int64_t M, int64_t B, int dtype,
                           unsigned flags, void* stream);

/* dW[b] = x[ptr[b]:ptr[b+1], :]^T @ dy[ptr[b]:ptr[b+1], :]     x [N,K], dy [N,M], dw [B,K,M]
 * Replaces the per-segment torch::matmul loop + at::stack of SegmentMatmul::backward
 * (pyg_lib/csrc/ops/autograd/matmul_kernel.cpp:92-107). */
int pygb200_segment_matmul_wgrad(const void* x, const int64_t* ptr_dev, const void* dy, void* dw,
                                 int64_t N, int64_t K, int64_t M, int64_t B, int dtype,
                                 unsigned flags, void* stream);

/* Independent problems C_i[n_i,m_i] = A_i[n_i,k_i] @ B_i[k_i,m_i] with arbitrary row strides (so
 * transposed views need no copy when their inner stride is 1).  All descriptor arrays are HOST
 * arrays of length `count`; a/b/c are device pointers.  lda/ldb/ldc are ROW strides in elements;
 * a_colmajor[i] / b_colmajor[i] != 0 means that operand is stored transposed (column stride ==
 * ld, row stride == 1).  Replaces grouped_matmul_kernel (matmul_kernel.cu:289-302). */
typedef struct {
  const void* a; const void* b; void* c;
  int64_t n, k, m;
  int64_t lda, ldb, ldc;
  int32_t a_colmajor, b_colmajor;
} pygb200_gemm_problem;
int pygb200_grouped_matmul(const pygb200_gemm_problem* problems_host, int64_t count, int dtype,
                           unsigned flags, void* stream);

/* ------------------------------------------------------------------------------------ sampler
 * Bit-exact reproduction of NeighborSampler / sample<> / hetero sample<>
 * (pyg_lib/csrc/sampler/cpu/neighbor_kernel.cpp:22-328,337-514,529-841) including the RNG stream
 * of RandintEngine (pyg_lib/csrc/random/cpu/rand_engine.h:26-97) drawn from torch's CPU mt19937.
 */

/* torch mt19937 engine state (ATen/core/MT19937RNGEngine.h mt19937_data_pod: state_, left_, next_).
 * Host struct, in/out: on success it is advanced exactly as the reference advances the default CPU
 * generator (whole 128-word blocks of at::randint). */
typedef struct {
  uint32_t state[624];
  int32_t left;
  int32_t next;
} pygb200_mt19937;

typedef struct pygb200_sampler pygb200_sampler; /* opaque: persistent device workspace */

int pygb200_sampler_create(pygb200_sampler** out);
void pygb200_sampler_destroy(pygb200_sampler* s);

/* One relation's CSR (device) plus its endpoints as indices into the node-type list. For csc=True
 * callers pass src_type = the relation's dst and dst_type = its src (neighbor_kernel.cpp:718-719). */
typedef struct {
  const void* rowptr;   /* [num_src_nodes + 1] */
  const void* col;      /* [num_edges] */
  int64_t num_src_nodes;
  int64_t num_edges;
  int32_t src_type;
  int32_t dst_type;
} pygb200_relation;

/* Runs all hops on `stream`, then synchronises the stream once and fills the host count arrays.
 *   T node types, R relations (in the reference's `edge_types` order), L hops.
 *   seeds[t] device pointer (or NULL), n_seeds[t] counts; seed order == seed_dict order only matters
 *   for disjoint batch numbering, which follows type index order.
 *   num_neighbors host [R*L] (row r = relation r; -1 == all neighbours).
 * Outputs (host): nodes_per_hop [T*(L+1)], edges_per_hop [R*L], n_nodes [T], n_edges [R].
 * The sampled subgraph stays in the workspace until the next run; copy it out with the export calls.
 */
int pygb200_sampler_run(pygb200_sampler* s, int32_t T, int32_t R, int32_t L,
                        const pygb200_relation* rels_host, const void* const* seeds,
                        const int64_t* n_seeds, const int64_t* num_neighbors, unsigned flags,
                        pygb200_mt19937* mt_inout, int64_t* nodes_per_hop, int64_t* edges_per_hop,
                        int64_t* n_nodes, int64_t* n_edges, void* stream);

/* Temporal sampling (node_temporal_sample / edge_temporal_sample, neighbor_kernel.cpp:74-144,417-428,
 * 742-787): neighbourhoods must be sorted by time; only neighbours with time <= the seed time of the
 * frontier node's subgraph are candidates (`strategy_last`: the latest `fan-out` of them).  Requires
 * PYGB200_S_DISJOINT.  All arrays are int64 on the device; any pointer / entry may be NULL:
 *   node_time[t]  time of the nodes of type t (applies to relations whose DST type is t)
 *   edge_time[r]  time of relation r's edges (wins over node_time)
 *   seed_time[t]  per seed of type t; default node_time[t][seed]. */
typedef struct {
  const int64_t* const* node_time;   /* [T] */
  const int64_t* const* edge_time;   /* [R] */
  const int64_t* const* seed_time;   /* [T] */
  int32_t strategy_last;
} pygb200_temporal;
int pygb200_sampler_run_temporal(pygb200_sampler* s, int32_t T, int32_t R, int32_t L,
                                 const pygb200_relation* rels_host, const void* const* seeds,
                                 const int64_t* n_seeds, const int64_t* num_neighbors, unsigned flags,
                                 pygb200_mt19937* mt_inout, int64_t* nodes_per_hop,
                                 int64_t* edges_per_hop, int64_t* n_nodes, int64_t* n_edges, void* stream,
                                 const pygb200_temporal* temporal);

/* Biased sampling (edge_weight; _biased_sample, neighbor_kernel.cpp:245-285): per frontier node the whole neighbourhood
 * (fan-out >= degree without replacement), at::multinomial with replacement, or the `fan-out` largest keys
 * log(u) / weight without — reproducing the reference bit for bit INCLUDING the CPU generator stream it consumes
 * (uniform_/random64 outputs), torch's CPU float32 log (MKL; table of its deviations from the correctly rounded log)
 * and at::topk's libstdc++ tie behaviour.  edge_weight[r]: device pointer to relation r's weights (one per edge,
 * weight_dtype = PYGB200_F32) or NULL: that relation samples uniformly (the reference's interleaving of the two kinds of
 * draws on one generator is reproduced; such runs synchronise with the host after every pass).  All flags of pygb200_sampler_run apply (PYGB200_S_DISJOINT,
 * PYGB200_S_REPLACE, PYGB200_S_NO_DEDUP = the reference's distributed one-hop sampling, -1 fan-outs).  Limits
 * (PYGB200_ERR_UNSUPPORTED): with replacement no fan-out of 1 (at::multinomial(n_sample=1)
 * samples from an MKL VSL stream); one GPU; not temporal (the reference refuses that too).  Invalid weights under replacement
 * (negative, NaN/inf, zero row sum) return PYGB200_ERR_ARG with at::multinomial's message.  One host synchronisation per
 * (hop, relation): the number of engine outputs a pass consumes is data dependent. */
int pygb200_sampler_run_weighted(pygb200_sampler* s, int32_t T, int32_t R, int32_t L,
                                 const pygb200_relation* rels_host, const void* const* seeds,
                                 const int64_t* n_seeds, const int64_t* num_neighbors, unsigned flags,
                                 pygb200_mt19937* mt_inout, int64_t* nodes_per_hop,
                                 int64_t* edges_per_hop, int64_t* n_nodes, int64_t* n_edges, void* stream,
                                 const void* const* edge_weight, int32_t weight_dtype);

/* Frontier-sharded run for multi-GPU sampling of ONE batch (SURVEY 8e; the reference's own split of
 * the work is dist_neighbor_sample -> merge -> relabel, neighbor_kernel.cpp:296-303,957-978,
 * dist_relabel_kernel.cpp:30-94).  One process per GPU; every rank holds the full CSR and calls this with
 * identical arguments and identical engine state, and every rank ends with the identical, reference-exact
 * result.  Per pass each rank counts the whole frontier (edge offsets and bit-stream positions are global)
 * and draws only its contiguous slice of frontier nodes.  Two transports:
 *
 *  (a) peer memory (`exchange` != NULL; homogeneous, non-disjoint, fan-outs >= 0, node ids < 2^32-1, world <= 16):
 *      the sampling kernel stores the (dst, edge id) of its edges straight into every rank's exchange region
 *      over NVLink (the all-gather of sampled edges is fused into the kernel), dedup is partitioned by key hash,
 *      the per-edge refs are reduced slice-wise with coalesced peer loads/stores, and cross-GPU ordering uses
 *      flag words in peer memory — no host sync and no collective call per hop.  `exchange` is a HOST
 *      all-gather of small blobs (out[q*bytes .. (q+1)*bytes) = rank q's `mine`), called only when the exchange
 *      regions are (re)allocated, to swap cudaIpcMemHandle_t's; it doubles as a host barrier.
 *  (b) callback all-gather (`exchange` == NULL): the callback all-gathers the drawn EDGE IDS in place: on return
 *      buf[seg_begin[q] .. seg_begin[q+1]) must hold rank q's elements for every q (int64 elements, offsets
 *      relative to buf; seg_begin is a HOST array of world+1 entries; the call is made on `stream`'s timeline).
 *      Dedup / relabel then run replicated.  Also covers disjoint runs; world <= 64. */
typedef int (*pygb200_allgather_fn)(void* user, void* buf_dev, const int64_t* seg_begin, int32_t world,
                                    void* stream);
typedef int (*pygb200_exchange_fn)(void* user, const void* mine_host, void* all_host, int64_t bytes);
typedef struct {
  int32_t rank, world;
  pygb200_allgather_fn allgather;
  void* user;
  pygb200_exchange_fn exchange;
} pygb200_shard;
int pygb200_sampler_run_sharded(pygb200_sampler* s, int32_t T, int32_t R, int32_t L,
                                const pygb200_relation* rels_host, const void* const* seeds,
                                const int64_t* n_seeds, const int64_t* num_neighbors, unsigned flags,
                                pygb200_mt19937* mt_inout, int64_t* nodes_per_hop,
                                int64_t* edges_per_hop, int64_t* n_nodes, int64_t* n_edges, void* stream,
                                const pygb200_shard* shard);

/* Results without an export pass (latency path).  `pygb200_sampler_bounds` gives the static upper bounds of a
 * run — nodes per type, edges per relation — from the seed counts and fan-outs alone (the recurrence of
 * neighbor_kernel.cpp:430-475: every frontier node emits at most `k` edges, every edge at most one new node);
 * PYGB200_ERR_UNSUPPORTED if a fan-out is -1 or the worst case exceeds 8 GiB.  `pygb200_sampler_bind_outputs`
 * hands the sampler caller-owned int64 device arrays of at least those capacities (edge_id may be NULL, or hold
 * NULL entries, when edge ids are not wanted) for the NEXT run only: that run's kernels then write rows, local
 * column ids, edge ids and the per-type node lists straight into them — the first n_edges_out[r] /
 * n_nodes_out[t] entries are the result, there is nothing to export, and the hash tables are reset behind the
 * run.  The binding is honoured for bounded, int64, non-disjoint, non-sharded runs whose bounds fit the
 * capacities; `pygb200_sampler_outputs_direct` says whether the last run used it (1) or the caller has to
 * export as usual (0).  After a direct run the export functions fail with PYGB200_ERR_ARG. */
int pygb200_sampler_bounds(int32_t T, int32_t R, int32_t L, const pygb200_relation* rels, const int64_t* n_seeds,
                           const int64_t* num_neighbors, int64_t* node_cap, int64_t* edge_cap);
int pygb200_sampler_bind_outputs(pygb200_sampler* s, int32_t T, int32_t R, void* const* row, void* const* col,
                                 void* const* edge_id, void* const* node, const int64_t* edge_cap,
                                 const int64_t* node_cap);
int pygb200_sampler_outputs_direct(pygb200_sampler* s);

/* After a PYGB200_S_NO_DEDUP run: out [n_seeds + 1] (int64, device) = n_seeds + number of edges emitted by seeds
 * 0..i-1, i.e. the reference's cumsum_neighbors_per_node (neighbor_kernel.cpp:386-388,446-492). */
int pygb200_sampler_export_cumsum(pygb200_sampler* s, int64_t* out, void* stream);

/* Asynchronous copies (cast to int32 when index32 != 0) of the last run's results into caller
 * buffers of exactly n_edges[r] / n_nodes[t] elements.  row = local index of the source (frontier)
 * node, col = local index of the sampled neighbour, edge_id = position in the relation's `col`
 * (neighbor_kernel.cpp:309-315).  Pass NULL to skip an array.  node_batch is only valid for disjoint
 * runs (node_id_out then receives [n,2] pairs (batch,node) like cpu/convert.h:17-24). */
int pygb200_sampler_export_edges(pygb200_sampler* s, int32_t rel, void* row_out, void* col_out,
                                 void* edge_id_out, int index32, void* stream);
int pygb200_sampler_export_nodes(pygb200_sampler* s, int32_t type, void* node_id_out, int index32,
                                 void* stream);

/* Both of the above for one relation and one node type in a single launch (homogeneous fast path). */
int pygb200_sampler_export_all(pygb200_sampler* s, int32_t rel, void* row_out, void* col_out,
                               void* edge_id_out, int32_t type, void* node_id_out, int index32,
                               void* stream);

/* Homogeneous convenience wrapper == T=1, R=1 (neighbor_sample_kernel, neighbor_kernel.cpp:899-926). */
int pygb200_neighbor_sample_run(pygb200_sampler* s, const void* rowptr, const void* col,
                                int64_t num_nodes, int64_t num_edges, const void* seed,
                                int64_t n_seed, const int64_t* num_neighbors, int32_t L,
                                unsigned flags, pygb200_mt19937* mt_inout, int64_t* nodes_per_hop,
                                int64_t* edges_per_hop, int64_t* n_nodes, int64_t* n_edges,
                                void* stream);

/* ---------------------------------------------------------------------------------- subgraph
 * Induced subgraph of the CSR graph (rowptr, col) on `nodes` — replaces subgraph_kernel
 * (pyg_lib/csrc/sampler/cpu/subgraph_kernel.cpp:13-89; schema pyg::subgraph, sampler/subgraph.cpp:28-32).
 * `nodes` [n] (same index dtype as rowptr/col; may repeat, need not be sorted) are numbered in first-occurrence
 * order like Mapper::fill (mapper.h:29-53); output row i lists, in CSR order, the neighbours of nodes[i] that are
 * in the set, as those ids.  Two calls, because the caller allocates the result between them like the reference
 * does (`:59-64`):
 *   pygb200_subgraph_count  builds the id map, writes out_rowptr [n+1] (device, index dtype) and returns the
 *                           number of kept edges (one host sync); PYGB200_ERR_ARG for a node outside
 *                           [0, num_nodes);
 *   pygb200_subgraph_fill   with the same rowptr/col/nodes: writes out_col [n_edges] and, unless NULL,
 *                           out_edge_id [n_edges] (positions in `col`), then resets the map.
 * A handle owns the map and scratch (device of the creating thread; one per stream; serialises its calls). */
typedef struct pygb200_subgraph pygb200_subgraph;
int pygb200_subgraph_create(pygb200_subgraph** out);
void pygb200_subgraph_destroy(pygb200_subgraph* h);
int pygb200_subgraph_count(pygb200_subgraph* h, const void* rowptr, const void* col, int64_t num_nodes,
                           const void* nodes, int64_t n, int index32, void* out_rowptr, int64_t* n_edges_out,
                           void* stream);
int pygb200_subgraph_fill(pygb200_subgraph* h, const void* rowptr, const void* col, const void* nodes, int64_t n,
                          int index32, void* out_col, void* out_edge_id, void* stream);

/* relabel_neighborhood (pyg_lib/csrc/sampler/cpu/dist_relabel_kernel.cpp:30-95; schema pyg::relabel_neighborhood,
 * sampler/dist_relabel.cpp:71-76): local (row, col) of edges whose global endpoints were sampled without mapping
 * (pyg::dist_neighbor_sample).  `sampled` [n_sampled] are the neighbours with duplicates, in source-node order;
 * counts_host [n_counts] (HOST, like the reference's int[] argument) says how many belong to source node i, so
 * out_row[j] = i; out_col[j] = id of sampled[j], ids numbering the first occurrences of [seed | sampled] — seeds
 * first, exactly Mapper::fill + insert.  `batch` (NULL, or [n_sampled]) switches to disjoint keys (batch, node) with
 * seed i in batch i.  Uses the map/scratch of a pygb200_subgraph handle; one host sync (error flag). */
int pygb200_relabel_neighborhood(pygb200_subgraph* h, const void* seed, int64_t n_seed, const void* sampled,
                                 const void* batch, int64_t n_sampled, const int64_t* counts_host, int64_t n_counts,
                                 int index32, void* out_row, void* out_col, void* stream);

/* The two halves of the heterogeneous version (hetero relabel<disjoint>, dist_relabel_kernel.cpp:97-273), where the
 * schedule — which positions of a destination type's sampled list belong to which (layer, edge type, source node)
 * — is host bookkeeping over the reference's int[][] count lists:
 *   pygb200_relabel_ids     ids of one node type's `sampled` list among the first occurrences of [seed | sampled]
 *                           (out_ids [n_sampled], index dtype); disjoint (batch != NULL): seed i has batch seed_batch0 + i;
 *   pygb200_relabel_expand  one relation: HOST lists of n_seg source segments (count, source index, first position in
 *                           the destination type's id list `ids` [n_ids]) -> out_row / out_col [sum of counts]. */
int pygb200_relabel_ids(pygb200_subgraph* h, const void* seed, int64_t n_seed, int64_t seed_batch0, const void* sampled,
                        const void* batch, int64_t n_sampled, int index32, void* out_ids, void* stream);
int pygb200_relabel_expand(pygb200_subgraph* h, const int64_t* seg_count_host, const int64_t* seg_row_host,
                           const int64_t* seg_pos_host, int64_t n_seg, const void* ids, int64_t n_ids, int index32,
                           void* out_row, void* out_col, void* stream);

/* merge_sampler_outputs (pyg_lib/csrc/sampler/cpu/dist_merge_outputs_kernel.cpp:15-137): the per-partition outputs of
 * pyg::dist_neighbor_sample are put back into the order of the seeds.  Seed j was sampled as the partition_orders[j]-th
 * seed of partition partition_ids[j]; its neighbours are node_ids[p][c[o] : c[o+1]] and edge_ids[p][c[o]-c[0] : c[o+1]-c[0]]
 * (c = that partition's cumsum_neighbors_per_node).
 *   pygb200_merge_plan      HOST arithmetic only: cumsum lists flattened (list p = cumsum_flat[cumsum_off[p] : cumsum_off[p+1]])
 *                           -> per seed the begin in its partition's node / edge ids and the neighbour count
 *                           (= num_sampled_neighbors_per_node); validates against the arrays' lengths;
 *   pygb200_segment_gather  out = concatenation of n_seg segments, segment s = seg_count[s] elements of device array
 *                           src_ptrs[seg_src[s]] from seg_begin[s] (broadcast != 0: seg_count[s] copies of that one element,
 *                           used for the batch vector).  Lists are HOST arrays; uses the scratch of a subgraph handle. */
int pygb200_merge_plan(const int64_t* cumsum_flat, const int64_t* cumsum_off, int64_t num_partitions,
                       const int64_t* partition_ids, const int64_t* partition_orders, int64_t p_size,
                       const int64_t* node_numel, const int64_t* edge_numel, int64_t* seg_node_begin,
                       int64_t* seg_edge_begin, int64_t* seg_count);
int pygb200_segment_gather(pygb200_subgraph* h, const void* const* src_ptrs_host, int64_t n_src, const int64_t* seg_src_host,
                           const int64_t* seg_begin_host, const int64_t* seg_count_host, int64_t n_seg, int broadcast,
                           int index32, void* out, void* stream);

/* ------------------------------------------------------------------------------------ random walk
 * Uniform random walks (pyg::random_walk with p == q == 1; replaces random_walk_kernel,
 * pyg_lib/csrc/sampler/cuda/random_walk_kernel.cu:27-85).  rowptr [num_nodes + 1] / col [num_edges] / seed [S] of one
 * index dtype (index32 != 0: int32, else int64); rand [walk_length, S] float32 draws in [0, 1), row-major (the caller
 * fills it, e.g. with at::rand, so the generator is consumed exactly as the reference consumes it); out [S, walk_length + 1]
 * row-major in the index dtype.  out[i][0] = seed[i]; step j moves v to col[rowptr[v] + min(int(rand[j][i] * float(deg)),
 * deg - 1)] when deg = rowptr[v+1] - rowptr[v] > 0 and stays on v otherwise.  One kernel launch, no host sync.  A node
 * index outside [0, num_nodes) in seed / col, or a row outside [0, num_edges), is never dereferenced: that walk stops
 * there and the NEXT call returns PYGB200_ERR_ARG (the output of the call that met it is undefined). */
int pygb200_random_walk(const void* rowptr, const void* col, int64_t num_nodes, int64_t num_edges, const void* seed,
                        int64_t S, int64_t walk_length, const float* rand, void* out, int index32, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PYG_B200_H_ */
