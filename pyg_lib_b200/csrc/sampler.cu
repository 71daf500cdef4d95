// pyg_lib_b200/csrc/sampler.cu — neighbor_sample / hetero_neighbor_sample for sm_90a (H100).
//
// Replaces the single-threaded CPU loops of pyg_lib/csrc/sampler/cpu/neighbor_kernel.cpp
// (NeighborSampler :22-328, homogeneous sample<> :337-514, hetero sample<> :529-841) and reproduces
// them bit-for-bit, including the order in which the sequential RandintEngine stream
// (pyg_lib/csrc/random/cpu/rand_engine.h:26-97) is consumed.
//
// One "pass" = (hop, relation).  Sizes never leave the device while a pass runs.  Device bodies shared by both
// schedules: count_tile (degree -> #edges + the node's RNG "advance function", phase-in -> units consumed),
// sample_node (draws: Robert Floyd / with replacement / full row; coalesced writes of (row, global dst, edge id);
// hash insert keyed by global id with a min-reduction of the flat emission position = first-occurrence order),
// mark_tile (an edge is "first" iff its position won the reduction; tile-local ranks).
// Three schedules:
//   latency      k_seed_fused (+ the first pass's count) -> per pass k_count_s, k_sample_s, k_mark_s, k_assign_s
//                -> k_final: write-once counters, every block scans the <= 1024 tile aggregates itself, the run is
//                published to the host by its last pass (DESIGN.md 3.3).  Small bounded runs.
//   v2           (sampler_v2.cuh) k_v2_seed -> per pass k_count, k_v2_sample (+ inserts), k_v2_mark, k_v2_assign -> k_final:
//                packed 32-bit table, refs instead of lookups, peer-memory frontier sharding.  The other bounded,
//                non-disjoint runs whose node ids fit 32 bits.
//   wide table   k_seed* -> per pass k_count, k_sample, k_mark, k_assign (last block scans, running counters)
//                -> k_final: any size, full neighbourhoods (host-synced sizing), disjoint / temporal runs, collective
//                frontier sharding, no-dedup hop.
// Host work per call: bounds, launches, ONE wait on a mapped flag (the API returns host counts).  make_plan decides
// everything about a run before its first CUDA call; Run<idx_t> executes it phase by phase.
#include <dlfcn.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <mutex>
#include <vector>

#include "common.cuh"
#include "mt19937.cuh"

namespace pygb200 {

// ------------------------------------------------------------------------------- error plumbing
static thread_local std::string g_err;
static std::atomic<int> g_launches{0};
void set_error(const std::string& msg) { g_err = msg; }
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

// ---- optional per-kernel timing
namespace {
struct ProfPending { cudaEvent_t a, b; int slot; long long work; };
struct ProfAcc { const char* name; double ms; long long launches, work; };
std::mutex g_prof_mu;
std::atomic<bool> g_prof_on{false};
std::vector<ProfPending> g_prof_pending;
ProfAcc g_prof_acc[] = {{"sample", 0, 0, 0}, {"count", 0, 0, 0}, {"mark", 0, 0, 0}, {"assign", 0, 0, 0},
                        {"lookup", 0, 0, 0}, {"segment_matmul", 0, 0, 0}, {"grouped_gemm", 0, 0, 0},
                        {"insert", 0, 0, 0}, {"pref", 0, 0, 0}, {"reduce", 0, 0, 0}, {"xbarrier", 0, 0, 0},
                        {"seed", 0, 0, 0}, {"final", 0, 0, 0}, {"cleanup", 0, 0, 0}, {"export", 0, 0, 0}, {"rows", 0, 0, 0}, {"push", 0, 0, 0},
                        {"mtgen", 0, 0, 0}};
constexpr int N_PROF = sizeof(g_prof_acc) / sizeof(g_prof_acc[0]);
int prof_slot(const char* name) {
  for (int i = 0; i < N_PROF; ++i) if (strcmp(g_prof_acc[i].name, name) == 0) return i;
  return -1;
}
void prof_drain_locked() {
  for (auto& p : g_prof_pending) {
    float ms = 0.f;
    if (cudaEventSynchronize(p.b) == cudaSuccess && cudaEventElapsedTime(&ms, p.a, p.b) == cudaSuccess) {
      g_prof_acc[p.slot].ms += ms; g_prof_acc[p.slot].launches += 1; g_prof_acc[p.slot].work += p.work;
    }
    cudaEventDestroy(p.a); cudaEventDestroy(p.b);
  }
  g_prof_pending.clear();
}
}  // namespace
bool prof_enabled() { return g_prof_on.load(std::memory_order_relaxed); }
void* prof_begin(cudaStream_t st) {
  if (!prof_enabled()) return nullptr;
  auto* p = new ProfPending();
  cudaEventCreate(&p->a); cudaEventCreate(&p->b);
  cudaEventRecord(p->a, st);
  return p;
}
void prof_end(void* token, const char* name, cudaStream_t st, long long work) {
  if (!token) return;
  auto* p = static_cast<ProfPending*>(token);
  cudaEventRecord(p->b, st);
  p->slot = prof_slot(name); p->work = work;
  std::lock_guard<std::mutex> lock(g_prof_mu);
  if (p->slot >= 0) g_prof_pending.push_back(*p); else { cudaEventDestroy(p->a); cudaEventDestroy(p->b); }
  delete p;
}

namespace {

constexpr int NT = 256;              // threads per block everywhere in this file
constexpr int ETILE = 1024;          // edges per mark/assign tile (NT x 4)
constexpr u64 EMPTY = ~0ull;
constexpr u64 POS_BASE = 1ull << 62; // vals >= POS_BASE are flat positions of the running pass
constexpr u32 NO_SLOT = 0xffffffffu;

// state buffer (device, i64 words); a pinned mirror is read by the host after the final sync
enum {
  ST_CURSOR = 0,    // RNG units consumed so far (end of last scanned pass)
  ST_SPARE = 1,
  ST_PASS_F = 2,    // frontier size of the running pass
  ST_PASS_E = 3,    // edges emitted by the running pass
  ST_PASS_BASE = 4, // offset of the running pass inside its relation's edge arrays
  ST_PASS_NEW = 5,  // new nodes found by the running pass
  ST_LIST_BASE = 6, // dst list length before the running pass
  ST_IDS_BASE = 7,  // dst id counter before the running pass
  ST_ERROR = 8,
  ST_MT_NEXT = 9, ST_MT_LEFT = 10, ST_BLOCKS = 11,
  ST_TICKET_A = 12, ST_TICKET_B = 13,
  ST_W_WORDS = 14, ST_W_SCR = 15,   // biased pass: engine words it consumes, scratch entries it needs (k_w_count)
  ST_HDR = 16
};

struct NodeRec {   // per frontier node of the running pass (written by k_count, read by k_sample)
  i64 rs;          // rowptr[v]
  u32 deg;         // degree (clamped; degrees >= 2^32 are rejected on the host side)
  u32 loc_off;     // edges emitted by earlier nodes of the same 256-node tile
  u32 pf[4];       // RNG units consumed by earlier nodes of the tile, per entry phase
};

struct PassArgs {
  const void* rowptr; const void* col;
  const i64* src_nodes; const i64* src_batch;
  i64* dst_nodes; i64* dst_batch; u32* dst_slot;
  u64* keys; u64* vals; u64 mask;
  i64* row; i64* colv; i64* eid;
  u32* eslot; u32* erank;
  NodeRec* rec; i64* tile_out; u32* tile_func; i64* tile_off; i64* tile_pos;
  i64* mtile;      // per edge tile: count of firsts, then exclusive offset
  i64* st;
  int o_src_begin, o_src_end, o_dst_list, o_dst_ids, o_rel_edges, o_eph;
  u32* raw; i64* gen; i64 out0; i64 raw_cap;   // mt19937 raw stream, #words generated, raw index of this call's output 0
  i64 fanout; int replace; int disjoint; int seed_mode;
  // lookup of the PREVIOUS pass, deferred into this pass's k_count / the final kernel (null = none)
  i64* lk_colv; const u64* lk_vals;
  // end-of-hop bookkeeping folded into the last pass's k_mark (he_T == 0: not the last pass of its hop)
  int he_T, he_L, he_hop, he_list, he_begin, he_end, he_nph;
  // frontier sharding (multi-GPU): phase 0 = normal; 1 = draw only, frontier nodes [shard_lo, shard_hi),
  // writes edge ids; 2 = expand ALL nodes from the (all-gathered) edge ids: gather col, rows, hash insert
  int phase; i64 shard_lo, shard_hi;
  int group;       // k_sample: lanes per frontier node (sample_group_lanes)
  // temporal sampling (neighbor_kernel.cpp:74-144): time_mode 1 = node time of the neighbour (time[col[e]]),
  // 2 = edge time (time[e]); seed_times indexed by the frontier node's batch id; time_last = strategy 'last'
  const i64* time; const i64* seed_times; int time_mode, time_last;
  // Latency path (k_*_s kernels): the counters of a run are WRITE-ONCE words of `st` whose indices the host
  // fixes from its static pass schedule, so no kernel updates a word another block of the same launch reads and
  // no pass needs a serial "last block" section.  A value is st[w_x] when w_x >= 0, else the constant c_x.
  int ssa;
  int w_begin, w_end, w_list_in, w_pbase, w_cur_in;      // frontier slice, dst list length, relation offset, RNG cursor
  i64 c_begin, c_end, c_list_in;                          // (pbase / cursor constants are 0)
  int w_E, w_cur_out, w_relcum_out, w_list_out;          // written by this pass (block 0 of k_sample_s / k_assign_s)
  int w_new;                                              // new nodes of this pass (summed up by k_mark_s)
  int w_seed_list, w_seed_ids;                            // dst type: seeds listed / distinct seeds (ids = list - dups)
  int lk_w_E, lk_w_pbase;                                 // previous pass (deferred lookup)
  // publication of the run's counters + final engine state to the host (publish_run): by k_final, or — latency
  // path — already by the last pass's k_assign_s, as soon as the last counter is known
  i64* pub_host; i64* pub_zero; i64 pub_serial; int pub_words, pub_o_mt;
  i64 pub_wwords;                                         // engine outputs consumed by biased passes (beside the RandintEngine's blocks)
  // ---- v2 schedule (sampler_v2.cuh): packed 32-bit table of the dst type, refs, optional peer-memory sharding
  u64* pk; int pk_bits;            // slot = node id << 32 | value
  u64* pk_main; int pk_main_bits;  // sharded seeds: `pk` is the replicated seed scratch table, ids go into this one
  u32* fref;                       // ref of every edge of the running pass
  int xw, xr, x_eid64;             // world size (1 = single GPU), rank, wire type of edge ids
  int v2_writeback, o_shard;
  i64 x_off_bar, x_off_dst, x_off_eid, x_off_fref;               // byte offsets inside an exchange region
  i64 x_off_exc, x_off_exc_n, x_off_xcnt, x_exc_cap;             // ref exceptions: W lists of (position, ref), their lengths, my counter
  u64 x_sig_epoch, x_timeout_ns;                                 // cross-GPU flags raised at the end of a kernel (0 = none)
  int sd_begin, sd_end, sd_nph;                                  // seed pass: frontier-slice words its mark kernel sets (k_seed_end folded in; 0 = not)
  unsigned char* xpeer[16];        // exchange region of every rank (own one included), peer-mapped
};
__device__ __forceinline__ i64 ldw(const i64* st, int w, i64 c) { return w >= 0 ? st[w] : c; }

// ------------------------------------------------------------------------------------- helpers
// Programmatic dependent launch: the kernels of a run form a chain on one stream.  Each waits for its
// predecessor's completion + memory flush here, then lets its successor's blocks be scheduled early
// (they park in their own pdl_enter), which hides launch latency and the block-scheduling ramp.
// Debug timeline (pygb200_timeline_enable): %globaltimer stamps by thread 0 of block 0 (or of the calling
// block for tl_mark_any), word 0 of the buffer counts the stamps.  Off: one constant-bank load per mark.
__constant__ u64* g_tl = nullptr;
constexpr int TL_CAP = 8192;
__device__ __forceinline__ void tl_mark_any(int id) {
  u64* tl = g_tl;
  if (tl == nullptr || threadIdx.x != 0) return;
  u64 t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  const u64 i = atomicAdd(tl, 1ull);
  u32 smid;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
  if (i < TL_CAP) tl[1 + i] = ((u64)id << 56) | ((u64)(smid & 0xff) << 48) | (t & ((1ull << 48) - 1));
}
__device__ __forceinline__ void tl_mark(int id) { if (blockIdx.x == 0) tl_mark_any(id); }
enum { TL_SEED = 1, TL_COUNT = 2, TL_SAMPLE = 3, TL_MARK = 4, TL_ASSIGN = 5, TL_FINAL = 6, TL_EXPORT = 7, TL_LAST = 8, TL_END = 16 };

__device__ __forceinline__ void pdl_enter(int id = 0) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (id) tl_mark(id);
}

// open addressing, linear probing; returns the slot holding `key`
__device__ __forceinline__ u32 table_insert(u64* keys, u64 mask, u64 key) {
  // Fibonacci hashing: one multiply, top log2(capacity) bits (capacity = mask + 1 is a power of two >= 2)
  u64 s = (key * 0x9E3779B97F4A7C15ull) >> (64 - __popcll(mask));
  while (true) {
    const u64 prev = atomicCAS(&keys[s], EMPTY, key);
    if (prev == EMPTY || prev == key) return (u32)s;
    s = (s + 1) & mask;
  }
}

// min-reduction without a return value, as one RED instruction: the addresses of a warp's inserts are almost
// always distinct, so the match/elect/redux aggregation the compiler wraps around atomicMin only costs here
__device__ __forceinline__ void red_min_u64(u64* addr, u64 v) {
  asm volatile("red.global.min.u64 [%0], %1;" ::"l"(addr), "l"(v) : "memory");
}

__device__ __forceinline__ u64 make_key(i64 node, i64 batch, int disjoint) {
  return disjoint ? (((u64)batch << 40) | (u64)node) : (u64)node;
}

struct Func4 { u32 d[4]; };
// (entry selected with a chain of selects: a run-time index into d[] would put the struct in local memory)
template <typename F>
__device__ __forceinline__ auto sel4(const F& f, unsigned ph) -> decltype(f.d[0] + 0) {
  return ph == 0 ? f.d[0] : (ph == 1 ? f.d[1] : (ph == 2 ? f.d[2] : f.d[3]));
}
// apply a first, then b
__device__ __forceinline__ Func4 compose(const Func4& a, const Func4& b) {
  Func4 c;
#pragma unroll
  for (int p = 0; p < 4; ++p) c.d[p] = a.d[p] + sel4(b, (p + a.d[p]) & 3u);
  return c;
}
struct Func4L { u64 d[4]; };
__device__ __forceinline__ Func4L composeL(const Func4L& a, const Func4L& b) {
  Func4L c;
#pragma unroll
  for (int p = 0; p < 4; ++p) c.d[p] = a.d[p] + sel4(b, (unsigned)((p + a.d[p]) & 3u));
  return c;
}

// how a frontier node is sampled (neighbor_kernel.cpp:58-72,177-243)
enum { MODE_NONE = 0, MODE_FULL = 1, MODE_REPLACE = 2, MODE_FLOYD = 3 };
__device__ __forceinline__ int classify(i64 deg, i64 k, int replace, i64* n_out, i64* n16, i64* n32, i64* n64) {
  *n16 = *n32 = *n64 = 0;
  if (deg == 0 || k == 0) { *n_out = 0; return MODE_NONE; }
  if (k < 0 || (!replace && k >= deg)) { *n_out = deg; return MODE_FULL; }
  *n_out = k;
  if (replace) {
    const int wu = rng_width_units((u64)deg);
    if (wu == 1) *n16 = k; else if (wu == 2) *n32 = k; else *n64 = k;
    return MODE_REPLACE;
  }
  // Floyd: ranges deg-k+1 .. deg, increasing
  const i64 lo = deg - k;  // range_j = lo + 1 + j
  i64 a = 65535 - lo; a = a < 0 ? 0 : (a > k ? k : a);
  i64 b = 4294967295ll - lo; b = b < 0 ? 0 : (b > k ? k : b);
  *n16 = a; *n32 = b - a; *n64 = k - b;
  return MODE_FLOYD;
}

// ordered exclusive scan of (u32 sum, Func4) over the NT threads of a block
__device__ __forceinline__ void block_scan_pair(u32 v, Func4 f, u32* ex_v, Func4* ex_f, u32* tot_v, Func4* tot_f) {
  __shared__ u32 s_v[NT / 32];
  __shared__ Func4 s_f[NT / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  u32 iv = v; Func4 iff = f;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const u32 ov = __shfl_up_sync(0xffffffffu, iv, d);
    Func4 of;
#pragma unroll
    for (int p = 0; p < 4; ++p) of.d[p] = __shfl_up_sync(0xffffffffu, iff.d[p], d);
    if (lane >= d) { iv += ov; iff = compose(of, iff); }
  }
  if (lane == 31) { s_v[wid] = iv; s_f[wid] = iff; }
  __syncthreads();
  u32 pv = 0; Func4 pfx = {{0, 0, 0, 0}};
  for (int w = 0; w < wid; ++w) { pv += s_v[w]; pfx = compose(pfx, s_f[w]); }
  // exclusive = prefix of earlier warps, then inclusive of the previous lane
  u32 ev = __shfl_up_sync(0xffffffffu, iv, 1);
  Func4 ef;
#pragma unroll
  for (int p = 0; p < 4; ++p) ef.d[p] = __shfl_up_sync(0xffffffffu, iff.d[p], 1);
  if (lane == 0) { ev = 0; ef = {{0, 0, 0, 0}}; }
  *ex_v = pv + ev;
  *ex_f = compose(pfx, ef);
  u32 tv = 0; Func4 tf = {{0, 0, 0, 0}};
  for (int w = 0; w < NT / 32; ++w) { tv += s_v[w]; tf = compose(tf, s_f[w]); }
  *tot_v = tv; *tot_f = tf;
  __syncthreads();
}

// Ordered exclusive scan of two u32 sums over the NT threads of a block.
__device__ __forceinline__ void block_scan_sums(u32 v, u32 u, u32* ex_v, u32* ex_u, u32* tot_v, u32* tot_u) {
  __shared__ u32 s_a[NT / 32], s_b[NT / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  u32 iv = v, iu = u;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const u32 ov = __shfl_up_sync(0xffffffffu, iv, d), ou = __shfl_up_sync(0xffffffffu, iu, d);
    if (lane >= d) { iv += ov; iu += ou; }
  }
  if (lane == 31) { s_a[wid] = iv; s_b[wid] = iu; }
  __syncthreads();
  u32 pv = 0, pu = 0, tv = 0, tu = 0;
#pragma unroll
  for (int w = 0; w < NT / 32; ++w) {
    const u32 xa = s_a[w], xb = s_b[w];
    if (w < wid) { pv += xa; pu += xb; }
    tv += xa; tu += xb;
  }
  *ex_v = pv + iv - v; *ex_u = pu + iu - u;
  *tot_v = tv; *tot_u = tu;
  __syncthreads();
}

// block_scan_pair for advance functions that are almost always plain additions: a draw from a range below 2^16
// takes one 16-bit unit whatever the phase, so f is uniform (d[0..3] equal) unless a node has >= 2^16 candidate
// neighbours, and uniform functions compose by adding.  One block-wide vote picks the cheap scan.
__device__ __forceinline__ void block_scan_nodes(u32 v, Func4 f, u32* ex_v, Func4* ex_f, u32* tot_v, Func4* tot_f) {
  const int uni = f.d[0] == f.d[1] && f.d[1] == f.d[2] && f.d[2] == f.d[3];
  if (__syncthreads_and(uni)) {
    u32 eu, tu;
    block_scan_sums(v, f.d[0], ex_v, &eu, tot_v, &tu);
    ex_f->d[0] = ex_f->d[1] = ex_f->d[2] = ex_f->d[3] = eu;
    tot_f->d[0] = tot_f->d[1] = tot_f->d[2] = tot_f->d[3] = tu;
  } else {
    block_scan_pair(v, f, ex_v, ex_f, tot_v, tot_f);
  }
}

// Single-block ordered scan of the frontier tile aggregates: edge offsets and absolute RNG positions.
// Runs in the last block of k_count, a section nothing overlaps (device timeline r2k: 26 us for the 3840 tiles of a
// 983 k-node frontier when every thread walked its tiles in global memory, 12 us even for 256 tiles).  The aggregates
// are staged in shared memory with coalesced loads, SCAN_CHUNK tiles per round; a thread scans 4 consecutive staged
// tiles, one block-wide scan orders the threads.  Uniform advance functions (every pass unless a node has >= 2^16
// candidates) are plain sums; the general case composes the 4-entry functions in the same order.
constexpr int SCAN_PER = 4, SCAN_CHUNK = NT * SCAN_PER;   // (5 staged words per tile + k_count's 16 KB RNG window fit 48 KB)
constexpr int MSCAN_PER = 16, MSCAN_CHUNK = NT * MSCAN_PER;
__device__ void scan_frontier_tiles(const PassArgs& a, i64 ntiles) {
  __shared__ u32 s_out[SCAN_CHUNK];
  __shared__ u32 s_f[4][SCAN_CHUNK];
  __shared__ i64 s_sum[NT / 32];
  __shared__ Func4L s_fun[NT / 32];
  __shared__ i64 c_off, c_pos;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (threadIdx.x == 0) { c_off = 0; c_pos = a.st[ST_CURSOR]; }
  for (i64 base = 0; base < ntiles; base += SCAN_CHUNK) {
    const int n = (int)(ntiles - base < SCAN_CHUNK ? ntiles - base : SCAN_CHUNK);
    int uni = 1;
    for (int j = threadIdx.x; j < n; j += NT) {   // coalesced staging
      s_out[j] = (u32)__ldcg(&a.tile_out[base + j]);
      const uint4 w = __ldcg(reinterpret_cast<const uint4*>(a.tile_func + 4 * (base + j)));
      s_f[0][j] = w.x; s_f[1][j] = w.y; s_f[2][j] = w.z; s_f[3][j] = w.w;
      uni &= w.x == w.y && w.y == w.z && w.z == w.w;
    }
    uni = __syncthreads_and(uni);   // (also publishes the staged tiles and c_off / c_pos)
    const int j0 = threadIdx.x * SCAN_PER, j1 = j0 + SCAN_PER < n ? j0 + SCAN_PER : n;
    i64 v = 0; Func4L f = {{0, 0, 0, 0}};
    if (uni) {
      u64 u = 0;
      for (int j = j0; j < j1; ++j) { v += s_out[j]; u += s_f[0][j]; }
      f.d[0] = f.d[1] = f.d[2] = f.d[3] = u;
    } else {
      for (int j = j0; j < j1; ++j) {
        v += s_out[j];
        Func4L g; g.d[0] = s_f[0][j]; g.d[1] = s_f[1][j]; g.d[2] = s_f[2][j]; g.d[3] = s_f[3][j];
        f = composeL(f, g);
      }
    }
    i64 iv = v; Func4L iff = f;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const i64 ov = __shfl_up_sync(0xffffffffu, iv, d);
      Func4L of;
#pragma unroll
      for (int p = 0; p < 4; ++p) of.d[p] = __shfl_up_sync(0xffffffffu, iff.d[p], d);
      if (lane >= d) { iv += ov; iff = composeL(of, iff); }
    }
    if (lane == 31) { s_sum[wid] = iv; s_fun[wid] = iff; }
    __syncthreads();
    i64 pv = 0; Func4L pfx = {{0, 0, 0, 0}};
    for (int w = 0; w < wid; ++w) { pv += s_sum[w]; pfx = composeL(pfx, s_fun[w]); }
    i64 ev = __shfl_up_sync(0xffffffffu, iv, 1);
    Func4L ef;
#pragma unroll
    for (int p = 0; p < 4; ++p) ef.d[p] = __shfl_up_sync(0xffffffffu, iff.d[p], 1);
    if (lane == 0) { ev = 0; ef = {{0, 0, 0, 0}}; }
    const i64 off0 = c_off, pos0 = c_pos;
    i64 off = off0 + pv + ev;              // edges emitted before this thread's tiles
    Func4L adv = composeL(pfx, ef);        // RNG advance (per entry phase) of this round's tiles before them
    for (int j = j0; j < j1; ++j) {
      a.tile_off[base + j] = off;
      a.tile_pos[base + j] = pos0 + (i64)sel4(adv, (unsigned)(pos0 & 3));
      off += s_out[j];
      Func4L g; g.d[0] = s_f[0][j]; g.d[1] = s_f[1][j]; g.d[2] = s_f[2][j]; g.d[3] = s_f[3][j];
      adv = composeL(adv, g);
    }
    i64 tv = 0; Func4L tf = {{0, 0, 0, 0}};
    for (int w = 0; w < NT / 32; ++w) { tv += s_sum[w]; tf = composeL(tf, s_fun[w]); }
    __syncthreads();                        // everybody has read c_off / c_pos and the staged tiles
    if (threadIdx.x == 0) { c_off = off0 + tv; c_pos = pos0 + (i64)sel4(tf, (unsigned)(pos0 & 3)); }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const i64 E = c_off;
    a.st[ST_PASS_E] = E;
    a.st[ST_CURSOR] = c_pos;
    if (!a.seed_mode) {
      a.st[ST_PASS_BASE] = a.st[a.o_rel_edges];
      a.st[a.o_rel_edges] += E;
      a.st[a.o_eph] = E;
    }
  }
  __syncthreads();
}

// mt19937 raw-stream extension by the calling block (blockDim.x == NT): same recurrence as
// k_mt_extend but with NT threads per step (several words per thread).
template <int KL>
__device__ void mt_extend_block(u32* __restrict__ raw, i64* gen, i64 need, i64 cap_words, i64* st, u32* win) {
  const i64 target = ((need + MT_N - 1) / MT_N) * MT_N;
  i64 m = *gen;
  if (target <= m) return;
  if (target > cap_words) {
    if (threadIdx.x == 0) st[ST_ERROR] = 1;
    return;
  }
  constexpr int HIST = MT_N + MT_LAG * (KL - 1);
  const i64 h0 = m > HIST ? m - HIST : 0;
  for (i64 i = h0 + threadIdx.x; i < m; i += blockDim.x) win[i & (MT_WIN - 1)] = __ldcg(&raw[i]);
  __syncthreads();
  while (m < target) {
    int k = (int)((m - MT_N) / MT_LAG) + 1;
    if (k > KL) k = KL;
    i64 n = (i64)MT_LAG * k;
    if (n > MT_N - 1) n = MT_N - 1;
    if (n > target - m) n = target - m;
    for (i64 idx = threadIdx.x; idx < n; idx += blockDim.x) {
      const i64 mm = m + idx;
      u32 x = win[(mm - (i64)MT_LAG * k) & (MT_WIN - 1)];
#pragma unroll
      for (int j = 0; j < KL; ++j)
        if (j < k)
          x ^= mt_twist(win[(mm - MT_N - MT_LAG * j) & (MT_WIN - 1)], win[(mm - MT_N + 1 - MT_LAG * j) & (MT_WIN - 1)]);
      win[mm & (MT_WIN - 1)] = x;
      raw[mm] = x;
    }
    __syncthreads();
    m += n;
  }
  mt_publish(gen, m);
  __syncthreads();
}

// "last block done" ticket: returns true in exactly one block, after all other blocks' global
// writes issued before their call are visible.
__device__ __forceinline__ bool last_block(i64* ticket) {
  __shared__ int s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const u64 t = atomicAdd((u64*)ticket, 1ull);
    s_last = (t == (u64)gridDim.x - 1);
    if (s_last) *ticket = 0;
  }
  __syncthreads();
  if (s_last) __threadfence();
  return s_last != 0;
}

// same, for kernels that stored to PEER memory: the fence in front of the ticket is system-wide
__device__ __forceinline__ bool last_block_sys(i64* ticket) {
  __shared__ int s_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();   // one fence per block, behind the block barrier, orders every thread's stores (cumulativity)
    const u64 t = atomicAdd((u64*)ticket, 1ull);
    s_last = (t == (u64)gridDim.x - 1);
    if (s_last) *ticket = 0;
  }
  __syncthreads();
  if (s_last) __threadfence_system();
  return s_last != 0;
}

// ------------------------------------------------------------------------------------ kernels
// local ids of the previous pass's edges (its k_assign has completed: kernel boundary)
__device__ __forceinline__ void deferred_lookup(const PassArgs& a) {
  if (a.lk_colv == nullptr) return;
  const i64 E = a.ssa ? a.st[a.lk_w_E] : a.st[ST_PASS_E];
  const i64 pbase = a.ssa ? ldw(a.st, a.lk_w_pbase, 0) : a.st[ST_PASS_BASE];
  for (i64 p = (i64)blockIdx.x * NT + threadIdx.x; p < E; p += (i64)gridDim.x * NT)
    a.lk_colv[pbase + p] = (i64)a.lk_vals[a.eslot[p]];
}

// What frontier node v (batch id `batch`, only read for temporal sampling) contributes to a pass: its (possibly
// time-windowed) row, the number of edges it emits and its RNG advance function (neighbor_kernel.cpp:58-144).
template <typename idx_t>
__device__ __forceinline__ void node_degree(const PassArgs& a, i64 v, i64 batch, i64* rs_out, i64* deg_out, u32* n_out_out, Func4* f_out) {
  const idx_t* __restrict__ rowptr = (const idx_t*)a.rowptr;
  i64 rs = (i64)rowptr[v];
  i64 re = (i64)rowptr[v + 1];
  if (a.time_mode && re > rs && a.fanout != 0) {
    // neighbours that fulfil the temporal constraint: std::upper_bound on the (time-sorted) row
    const i64 st = a.seed_times[batch];
    const idx_t* __restrict__ colp = (const idx_t*)a.col;
    i64 lo = rs, hi = re;
    while (lo < hi) {
      const i64 mid = lo + ((hi - lo) >> 1);
      const i64 key = a.time_mode == 1 ? a.time[(i64)colp[mid]] : a.time[mid];
      if (st < key) hi = mid; else lo = mid + 1;
    }
    re = lo;
    if (a.time_last && a.fanout >= 0 && re - a.fanout > rs) rs = re - a.fanout;
  }
  const i64 deg = re - rs;
  i64 n_out, n16, n32, n64;
  classify(deg, a.fanout, a.replace, &n_out, &n16, &n32, &n64);
  Func4 f;
  if (n32 == 0 && n64 == 0) {
    f.d[0] = f.d[1] = f.d[2] = f.d[3] = (u32)n16;
  } else {
#pragma unroll
    for (int p = 0; p < 4; ++p) f.d[p] = (u32)(rng_node_end(p, n16, n32, n64) - p);
  }
  *rs_out = rs; *deg_out = deg; *n_out_out = (u32)n_out; *f_out = f;
}

// one 256-node frontier tile: per-node records + the tile's aggregate (blockDim.x == NT)
template <typename idx_t>
__device__ __forceinline__ void count_tile(const PassArgs& a, i64 begin, i64 F, i64 tile) {
  const i64 i = tile * NT + threadIdx.x;
  i64 rs = 0, deg = 0; u32 n_out = 0;
  Func4 f = {{0, 0, 0, 0}};
  if (i < F) node_degree<idx_t>(a, a.src_nodes[begin + i], a.time_mode ? a.src_batch[begin + i] : 0, &rs, &deg, &n_out, &f);
  u32 ex_v, tot_v; Func4 ex_f, tot_f;
  block_scan_nodes(n_out, f, &ex_v, &ex_f, &tot_v, &tot_f);
  if (i < F) {
    NodeRec r;
    r.rs = rs; r.deg = (u32)deg; r.loc_off = ex_v;
    r.pf[0] = ex_f.d[0]; r.pf[1] = ex_f.d[1]; r.pf[2] = ex_f.d[2]; r.pf[3] = ex_f.d[3];
    a.rec[i] = r;
  }
  if (threadIdx.x == 0) {
    a.tile_out[tile] = tot_v;
#pragma unroll
    for (int p = 0; p < 4; ++p) a.tile_func[4 * tile + p] = tot_f.d[p];
  }
}

template <typename idx_t>
__global__ void __launch_bounds__(NT) k_count(const PassArgs a) {
  __shared__ u32 s_win[MT_WIN];
  pdl_enter(TL_COUNT);
  deferred_lookup(a);  // must precede the ticket: the last block overwrites ST_PASS_E / ST_PASS_BASE
  const i64 begin = a.st[a.o_src_begin], end = a.st[a.o_src_end];
  const i64 F = end - begin;
  const i64 ntiles = ceil_div(F, NT);
  for (i64 tile = blockIdx.x; tile < ntiles; tile += gridDim.x) count_tile<idx_t>(a, begin, F, tile);
  tl_mark(TL_COUNT | TL_END);
  if (last_block(&a.st[ST_TICKET_A])) {
    tl_mark_any(TL_COUNT | TL_LAST);
    if (threadIdx.x == 0) a.st[ST_PASS_F] = F;
    scan_frontier_tiles(a, ntiles);
    if (a.xw > 1 && (int)threadIdx.x <= a.xw) {   // sharded: flat position of the first edge of every rank's frontier slice
      const i64 i = (i64)((__int128)F * threadIdx.x / a.xw);
      a.st[a.o_shard + threadIdx.x] = i < F ? a.tile_off[i / NT] + (i64)a.rec[i].loc_off : a.st[ST_PASS_E];
    }
    mt_extend_block<3>(a.raw, a.gen, a.out0 + 256 * rng_blocks_for_units(a.st[ST_CURSOR]), a.raw_cap, a.st, s_win);
    tl_mark_any(TL_COUNT | TL_LAST | TL_END);
  }
}

// Sampling of ONE frontier node by a group of `g` consecutive lanes of a warp (g = min(fan-out, 32): a warp
// takes 32 / g nodes, so a fan-out of 10 keeps 30 of its 32 lanes busy).  `r` = the node's record, `off` =
// pass-local flat position of its first edge, `pos0` = RNG position (16-bit units) of its first draw, `gl` = lane
// within the group, `gbase` = the group's first lane, `gmask` = its lanes.
// Robert Floyd's algorithm (neighbor_kernel.cpp:231-241) is sequential in the draws — draw j falls back to lo + j
// when its random value was already CHOSEN by an earlier draw — but only through the chosen values: every lane
// takes one draw and the conflicts are settled with g shuffles.  Fan-outs beyond 32 go in rounds of 32 and
// re-read what earlier rounds emitted.
// The draws of one node, with the emission left to the caller: emit(j, e) receives the index of the draw within the
// node and the chosen edge position; prev(t) must return the edge position emitted as draw t of this node in an
// earlier round (only called for fan-outs beyond the group width).
template <typename EmitF, typename PrevF>
__device__ __forceinline__ void sample_draws(const PassArgs& a, const NodeRec& r, i64 pos0, int g, int gl, int gbase, unsigned gmask,
                                             EmitF emit, PrevF prev) {
  const u32* __restrict__ raw = a.raw;
  const i64 out0 = a.out0;
  const i64 deg = r.deg, rs = r.rs, k = a.fanout;
  i64 n_out, n16, n32, n64;
  const int mode = classify(deg, k, a.replace, &n_out, &n16, &n32, &n64);
  if (mode == MODE_FULL) {
    for (i64 j = gl; j < deg; j += g) emit(j, rs + j);
  } else if (mode == MODE_REPLACE) {
    const int wu = rng_width_units((u64)deg);
    for (i64 j = gl; j < k; j += g) {
      const i64 pos = (wu == 1) ? pos0 + j : rng_align(rng_run(pos0, wu, j), wu);
      emit(j, rs + (i64)rng_draw(raw, out0, pos, wu, (u64)deg));
    }
  } else if (mode == MODE_FLOYD) {
    // (in-row offsets fit 32 bits: NodeRec::deg is u32, larger degrees are rejected by the host)
    const u32 lo = (u32)(deg - k);  // draw j: range lo+1+j, fallback value lo+j
    const u32 k32 = (u32)k;
    for (u32 c0 = 0; c0 < k32; c0 += g) {
      const u32 j = c0 + gl;
      const bool act = j < k32;
      u32 rnd = 0xffffffffu, c = 0xffffffffu;
      if (act) {
        int wu;
        const i64 pos = (n32 == 0 && n64 == 0) ? (wu = 1, pos0 + j) : rng_draw_start(pos0, n16, n32, j, &wu);
        rnd = (u32)rng_draw(raw, out0, pos, wu, (u64)lo + 1 + j);
        c = rnd;
        // already chosen in an earlier round of this node? (only when fanout > 32)
        for (u32 t = 0; t < c0; ++t)
          if ((u32)(prev(t) - rs) == rnd) { c = lo + j; break; }
      }
      const int lim = (int)((k32 - c0) < (u32)g ? (k32 - c0) : (u32)g);
      for (int jj = 0; jj < lim; ++jj) {
        const u32 cj = __shfl_sync(gmask, c, gbase + jj);
        if (act && gl > jj && rnd == cj) c = lo + j;
      }
      if (act) emit(j, rs + c);
      if (c0 + g < k32) __syncwarp(gmask);
    }
  }
}

template <typename idx_t, bool PHASED>
__device__ __forceinline__ void sample_node(const PassArgs& a, const NodeRec& r, i64 off, i64 pos0, i64 src_pos, i64 pbase,
                                            int g, int gl, int gbase, unsigned gmask) {
  const idx_t* __restrict__ col = (const idx_t*)a.col;
  const i64 sbatch = a.disjoint ? a.src_batch[src_pos] : 0;
  auto emit = [&](i64 j, i64 e) {
    const i64 p = off + j;
    if (PHASED && a.phase == 1) { a.eid[pbase + p] = e; return; }
    const i64 d = (i64)col[e];
    a.row[pbase + p] = src_pos;
    a.eid[pbase + p] = e;
    a.colv[pbase + p] = d;  // global id for now; the (deferred) lookup overwrites it with the local id
    if (PHASED && a.phase == 3) return;   // distributed one-hop sampling: no mapping at all (neighbor_kernel.cpp:296-303)
    const u32 s = table_insert(a.keys, a.mask, make_key(d, sbatch, a.disjoint));
    red_min_u64(&a.vals[s], POS_BASE + (u64)p);
    a.eslot[p] = s;
  };
  auto prev = [&](u32 t) { return __ldcg(&a.eid[pbase + off + t]); };
  if (PHASED && a.phase == 2) {
    i64 n_out, n16, n32, n64;
    classify((i64)r.deg, a.fanout, a.replace, &n_out, &n16, &n32, &n64);
    for (i64 j = gl; j < n_out; j += g) emit(j, a.eid[pbase + off + j]);
  } else {
    sample_draws(a, r, pos0, g, gl, gbase, gmask, emit, prev);
  }
}

// Lanes per frontier node: the power of two that holds the fan-out, 4..32 (full neighbourhoods: a warp per node).
// Measured on C2's second hop (15k nodes x 10): 16 lanes, 960 CTAs in two waves 24 us; exact groups of 10 (three
// nodes per warp, one wave) 33 us; 8 lanes with two draws per lane 34 us — more nodes in flight per SM lengthen
// every gather / table insert more than the saved wave is worth, so the kernel stays with one draw per lane.
inline int sample_group_lanes(i64 k) {
  if (k < 0 || k > 16) return 32;
  return k > 8 ? 16 : (k > 4 ? 8 : 4);
}
inline int sample_nodes_per_block(int g) { return (NT / 32) * (32 / g); }

#ifndef SAMPLE_MIN_BLOCKS
#define SAMPLE_MIN_BLOCKS 4   // resident CTAs per SM the register allocation aims for
#endif
template <typename idx_t>
__global__ void __launch_bounds__(NT, SAMPLE_MIN_BLOCKS) k_sample(const PassArgs a) {
  pdl_enter(TL_SAMPLE);
  const i64 F = a.st[ST_PASS_F];
  const i64 begin = a.st[a.o_src_begin];
  const i64 pbase = a.st[ST_PASS_BASE];
  const int g = a.group, lane = threadIdx.x & 31, per_warp = 32 / g;
  const int gi = lane / g, gl = lane - gi * g, gbase = gi * g;
  const unsigned gmask = (g == 32) ? 0xffffffffu : (((1u << g) - 1u) << gbase);
  const int npb = (NT / 32) * per_warp;
  const i64 i_lo = a.phase == 1 ? a.shard_lo : 0;
  const i64 i_hi = a.phase == 1 ? (a.shard_hi < F ? a.shard_hi : F) : F;
  if (gi >= per_warp) return;   // (lanes beyond the last whole group of the warp)
  for (i64 i = i_lo + (i64)blockIdx.x * npb + (threadIdx.x >> 5) * per_warp + gi; i < i_hi; i += (i64)gridDim.x * npb) {
    const NodeRec r = a.rec[i];
    const i64 tile = i / NT;
    const i64 tpos = a.tile_pos[tile];
    const i64 off = a.tile_off[tile] + r.loc_off;    // pass-local flat position of the node's first edge
    const int ph = (int)(tpos & 3);
    const u32 pfv = ph == 0 ? r.pf[0] : (ph == 1 ? r.pf[1] : (ph == 2 ? r.pf[2] : r.pf[3]));
    // RNG position of the first draw; begin + i == local id of the source node (neighbor_kernel.cpp:453)
    sample_node<idx_t, true>(a, r, off, tpos + pfv, begin + i, pbase, g, gl, gbase, gmask);
  }
  tl_mark(TL_SAMPLE | TL_END);
}

// seed time per batch id (neighbor_kernel.cpp:417-428): explicit seed_time wins, else node_time[seed]
template <typename idx_t>
__global__ void __launch_bounds__(NT) k_seed_times(i64* __restrict__ out, const idx_t* __restrict__ seeds, i64 n, i64 batch0,
                                                    const i64* __restrict__ seed_time, const i64* __restrict__ node_time) {
  for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < n; i += (i64)gridDim.x * NT)
    out[batch0 + i] = seed_time ? seed_time[i] : node_time[(i64)seeds[i]];
}

// flat edge offset of the first frontier node of every shard (frontier split evenly by node index)
__global__ void k_shard_bounds(const PassArgs a, int W, int o_shard) {
  const int q = threadIdx.x;
  if (q > W) return;
  const i64 F = a.st[ST_PASS_F], E = a.st[ST_PASS_E];
  const i64 i = (i64)((__int128)F * q / W);
  a.st[o_shard + q] = (i < F) ? a.tile_off[i / NT] + a.rec[i].loc_off : E;
}

// seeds: list them, insert them (first-occurrence order == seed order)
template <typename idx_t>
__global__ void __launch_bounds__(NT) k_seed(const PassArgs a, const idx_t* __restrict__ seeds, i64 n, i64 batch0) {
  for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < n; i += (i64)gridDim.x * NT) {
    const i64 v = (i64)seeds[i];
    a.dst_nodes[i] = v;
    if (a.disjoint) a.dst_batch[i] = batch0 + i;
    const u32 s = table_insert(a.keys, a.mask, make_key(v, batch0 + i, a.disjoint));
    red_min_u64(&a.vals[s], POS_BASE + (u64)i);
    a.eslot[i] = s;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    a.st[ST_PASS_E] = n;
    a.st[ST_PASS_BASE] = 0;
  }
}

#include "sampler_v2.cuh"
#include "sampler_weighted.cuh"
const u32 kMklLogfTable[] = {
#include "mkl_logf_table.inc"
};
constexpr int kMklLogfTableN = (int)(sizeof(kMklLogfTable) / sizeof(u32));

// first occurrences of the running pass + tile-local ranks; last block scans the tile counts and
// updates the dst type's counters.
// one 1024-edge tile: first-occurrence flags + tile-local ranks, count of firsts -> mtile[tile]
__device__ __forceinline__ void mark_tile(const PassArgs& a, i64 E, i64 tile, u32* s_w) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const i64 p0 = tile * ETILE + threadIdx.x * 4;
  u32 fl[4]; u32 cnt = 0;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const i64 p = p0 + q;
    fl[q] = 0;
    if (p < E) fl[q] = (a.vals[a.eslot[p]] == POS_BASE + (u64)p) ? 1u : 0u;
    cnt += fl[q];
  }
  u32 inc = cnt;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const u32 o = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += o;
  }
  if (lane == 31) s_w[wid] = inc;
  __syncthreads();
  u32 pre = 0, tot = 0;
  for (int w = 0; w < NT / 32; ++w) { if (w < wid) pre += s_w[w]; tot += s_w[w]; }
  u32 ex = pre + inc - cnt;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const i64 p = p0 + q;
    if (p < E) a.erank[p] = fl[q] ? (0x80000000u | ex) : 0u;
    ex += fl[q];
  }
  if (threadIdx.x == 0) a.mtile[tile] = tot;
  __syncthreads();
}

__global__ void __launch_bounds__(NT) k_mark(const PassArgs a) {
  __shared__ u32 s_w[NT / 32];
  pdl_enter(TL_MARK);
  const i64 E = a.st[ST_PASS_E];
  const i64 ntiles = ceil_div(E, ETILE);
  for (i64 tile = blockIdx.x; tile < ntiles; tile += gridDim.x) mark_tile(a, E, tile, s_w);
  tl_mark(TL_MARK | TL_END);
  if (last_block(&a.st[ST_TICKET_B])) {
    tl_mark_any(TL_MARK | TL_LAST);
    mark_finish(a, E, ntiles);   // ordered exclusive scan of the tile counts by one block + the pass's counters
    tl_mark_any(TL_MARK | TL_LAST | TL_END);
  }
}

__global__ void __launch_bounds__(NT) k_assign(const PassArgs a) {
  pdl_enter(TL_ASSIGN);
  const i64 E = a.st[ST_PASS_E];
  const i64 pbase = a.st[ST_PASS_BASE];
  const i64 list_base = a.st[ST_LIST_BASE], ids_base = a.st[ST_IDS_BASE];
  for (i64 p = (i64)blockIdx.x * NT + threadIdx.x; p < E; p += (i64)gridDim.x * NT) {
    const u32 er = a.erank[p];
    if (a.seed_mode) {
      if (er & 0x80000000u) {
        const i64 rank = a.mtile[p / ETILE] + (er & 0x7fffffffu);
        a.vals[a.eslot[p]] = (u64)rank;
        a.dst_slot[p] = a.eslot[p];
      } else {
        a.dst_slot[p] = NO_SLOT;
      }
    } else if (er & 0x80000000u) {
      const i64 rank = a.mtile[p / ETILE] + (er & 0x7fffffffu);
      const u32 s = a.eslot[p];
      a.vals[s] = (u64)(ids_base + rank);
      a.dst_nodes[list_base + rank] = a.colv[pbase + p];
      if (a.disjoint) a.dst_batch[list_base + rank] = a.src_batch[a.row[pbase + p]];
      a.dst_slot[list_base + rank] = s;
    }
  }
}

// The run's counters and the final engine state go straight into mapped host memory; the host polls the flag
// word behind them (no DMA copy, no event round trip) and everything else it does is stream-ordered behind the
// run's remaining kernels, so this may happen as soon as the last counter exists.  Called by one whole block.
// Engine state = the generation holding the last consumed output (see mt19937.cuh); at least one 128-word block
// is always consumed (rand_engine.h:28).  The stream must already cover it.
// flag word = run serial (24 bits) above a 40-bit payload
__host__ __device__ __forceinline__ i64 flag_word(i64 serial, i64 payload) {
  return (i64)((((u64)serial & 0xffffffull) << 40) | ((u64)payload & 0xffffffffffull));
}
__device__ void publish_run(const PassArgs& a, i64 cursor, bool with_flag) {
  i64* host_st = a.pub_host;
  const int n_words = a.pub_words, o_mt = a.pub_o_mt;
  // counters first: these loads overlap the stream -> engine-state chain below
  for (int i = threadIdx.x; i < n_words; i += blockDim.x)
    if ((i < o_mt || i >= o_mt + MT_N / 2) && (i < ST_ERROR || i > ST_BLOCKS)) host_st[i] = a.st[i];
  // the state buffer is double-buffered: the half the NEXT run uses is cleared here (nobody reads it any more)
  if (a.pub_zero) for (int i = threadIdx.x; i < n_words; i += blockDim.x) a.pub_zero[i] = 0;
  const i64 blocks = rng_blocks_for_units(cursor);
  const i64 q = a.out0 + 256 * blocks + a.pub_wwords;
  const i64 g = (q - 1) / MT_N;
  u32* hout = reinterpret_cast<u32*>(host_st + o_mt);
  for (int i = threadIdx.x; i < MT_N; i += blockDim.x) hout[i] = __ldcg(&a.raw[g * MT_N + i]);
  if (threadIdx.x == 0) {
    const i64 nxt = q - g * MT_N;
    host_st[ST_MT_NEXT] = nxt; host_st[ST_MT_LEFT] = 625 - nxt; host_st[ST_BLOCKS] = blocks;
    host_st[ST_ERROR] = a.st[ST_ERROR];
  }
  if (!with_flag) return;   // (a later kernel adds the last counter and raises the flag: publish_last)
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) { *reinterpret_cast<volatile i64*>(host_st + n_words) = flag_word(a.pub_serial, 0); __threadfence_system(); }
}
// One thread of a LATER kernel (everything publish_run wrote is visible by then): the flag word carries the one
// counter that was still missing, so a single 8-byte store completes the run for the host.
__device__ __forceinline__ void publish_last(const PassArgs& a, i64 value) {
  *reinterpret_cast<volatile i64*>(a.pub_host + a.pub_words) = flag_word(a.pub_serial, value);
  __threadfence_system();
}

// ============================================================================ latency path
// Small bounded runs (every pass <= LAT_TILES frontier tiles and edge tiles, seeds <= SEED_FUSED_MAX per type)
// are a chain of tiny kernels whose cost is the length of their dependent-latency chains, not their work.  The
// k_*_s kernels cut the two serial sections of a pass (the "last block" tile scans of k_count and k_mark and
// the tickets in front of them): the producer only writes per-tile aggregates, and EVERY block of the consumer
// scans them for itself (<= 1024 aggregates, 4 per thread).  The run's counters become write-once words (see
// PassArgs), written by block 0 of the consumer for later kernels only.
constexpr int LAT_TILES = 1024;

__device__ __forceinline__ u32 pick4(const Func4& f, int ph) {
  return ph == 0 ? f.d[0] : (ph == 1 ? f.d[1] : (ph == 2 ? f.d[2] : f.d[3]));
}

template <typename idx_t>
__global__ void __launch_bounds__(NT) k_count_s(const PassArgs a) {
  pdl_enter(TL_COUNT);
  deferred_lookup(a);
  const i64 begin = ldw(a.st, a.w_begin, a.c_begin), end = ldw(a.st, a.w_end, a.c_end);
  const i64 F = end - begin;
  const i64 ntiles = ceil_div(F, NT);
  for (i64 tile = blockIdx.x; tile < ntiles; tile += gridDim.x) count_tile<idx_t>(a, begin, F, tile);
  tl_mark(TL_COUNT | TL_END);
}

template <typename idx_t>
__global__ void __launch_bounds__(NT, SAMPLE_MIN_BLOCKS) k_sample_s(const PassArgs a) {
  __shared__ u32 s_off[LAT_TILES], s_pos[LAT_TILES];
  __shared__ u32 s_win[MT_WIN];   // (block 0, stream shortfall only)
  pdl_enter(TL_SAMPLE);
  const i64 gen0 = *reinterpret_cast<volatile i64*>(a.gen);
  const i64 begin = ldw(a.st, a.w_begin, a.c_begin), end = ldw(a.st, a.w_end, a.c_end);
  const i64 cur_in = ldw(a.st, a.w_cur_in, 0), pbase = ldw(a.st, a.w_pbase, 0);
  const i64 F = end - begin;
  const int ntiles = (int)ceil_div(F, NT);
  const int ph0 = (int)(cur_in & 3);
  const int g = a.group, lane = threadIdx.x & 31, per_warp = 32 / g;
  const int gi = lane / g, gl = lane - gi * g, gbase = gi * g;
  const unsigned gmask = (g == 32) ? 0xffffffffu : (((1u << g) - 1u) << gbase);
  const int npb = (NT / 32) * per_warp;
  // this group's first node: its record is fetched now, beside the tile aggregates (rec[] is sized for the bound)
  const i64 i_first = (i64)blockIdx.x * npb + (threadIdx.x >> 5) * per_warp + (gi < per_warp ? gi : 0);
  // (a record = two 16-byte loads kept as eight scalars: selecting between whole NodeRec structs put pf[] in local memory)
  uint4 ra_first = make_uint4(0, 0, 0, 0), rb_first = make_uint4(0, 0, 0, 0);
  if (i_first < F) { const uint4* rp = reinterpret_cast<const uint4*>(a.rec + i_first); ra_first = rp[0]; rb_first = rp[1]; }
  // ---- every block: exclusive scan of the tile aggregates (edge offsets, RNG positions relative to cur_in)
  u32 E, adv;
  {
    const int t0 = threadIdx.x * 4;
    auto tile_agg = [&](int t, u32* v, Func4* f) {
      *v = (u32)a.tile_out[t];
      const uint4 w = *reinterpret_cast<const uint4*>(a.tile_func + 4 * (size_t)t);
      f->d[0] = w.x; f->d[1] = w.y; f->d[2] = w.z; f->d[3] = w.w;
    };
    u32 lv = 0; Func4 lf = {{0, 0, 0, 0}};
    int uni = 1;
    for (int q = 0; q < 4 && t0 + q < ntiles; ++q) {
      u32 v; Func4 f;
      tile_agg(t0 + q, &v, &f);
      uni &= f.d[0] == f.d[1] && f.d[1] == f.d[2] && f.d[2] == f.d[3];
      lv += v; lf = compose(lf, f);
    }
    if (__syncthreads_and(uni)) {   // (the rule: no multi-word draw in this pass) advances just add up
      u32 ex_v, ex_u, tot_v, tot_u;
      block_scan_sums(lv, lf.d[0], &ex_v, &ex_u, &tot_v, &tot_u);
      for (int q = 0; q < 4 && t0 + q < ntiles; ++q) {   // (second look at the aggregates: L1 hits)
        s_off[t0 + q] = ex_v; s_pos[t0 + q] = ex_u;
        ex_v += (u32)a.tile_out[t0 + q]; ex_u += a.tile_func[4 * (size_t)(t0 + q)];
      }
      E = tot_v; adv = tot_u;
    } else {
      u32 ex_v, tot_v; Func4 ex_f, tot_f;
      block_scan_pair(lv, lf, &ex_v, &ex_f, &tot_v, &tot_f);
      for (int q = 0; q < 4 && t0 + q < ntiles; ++q) {
        u32 v; Func4 f;
        tile_agg(t0 + q, &v, &f);
        s_off[t0 + q] = ex_v; s_pos[t0 + q] = pick4(ex_f, ph0);
        ex_v += v; ex_f = compose(ex_f, f);
      }
      E = tot_v; adv = pick4(tot_f, ph0);
    }
    __syncthreads();
  }
  const i64 cur_out = cur_in + adv;
  // ---- the stream must cover this pass; it does unless a node drew multi-word values (deg >= 2^16)
  const i64 need = a.out0 + 256 * rng_blocks_for_units(cur_out);
  const i64 target = ((need + MT_N - 1) / MT_N) * MT_N;
  if (blockIdx.x == 0) {
    if (threadIdx.x == 0) {
      a.st[a.w_E] = E;
      a.st[a.w_cur_out] = cur_out;
      a.st[a.w_relcum_out] = pbase + E;
    }
    if (gen0 < target) mt_extend_block<3>(a.raw, a.gen, need, a.raw_cap, a.st, s_win);
    if (a.pub_words) {   // last pass of the run: everything but the final length of its dst list is known now
      __syncthreads();
      publish_run(a, cur_out, false);
    }
  } else if (gen0 < target) {
    if (threadIdx.x == 0) {
      while (*reinterpret_cast<volatile i64*>(a.gen) < target && *reinterpret_cast<volatile i64*>(a.st + ST_ERROR) == 0) { }
      __threadfence();
    }
    __syncthreads();
  }
  // ---- one group of g lanes per frontier node
  if (gi >= per_warp) return;   // (lanes beyond the last whole group of the warp; no block-wide sync below)
  for (i64 i = i_first; i < F; i += (i64)gridDim.x * npb) {
    uint4 ra = ra_first, rb = rb_first;
    if (i != i_first) { const uint4* rp = reinterpret_cast<const uint4*>(a.rec + i); ra = rp[0]; rb = rp[1]; }
    NodeRec r;
    r.rs = (i64)(((u64)ra.y << 32) | (u64)ra.x); r.deg = ra.z; r.loc_off = ra.w;
    r.pf[0] = r.pf[1] = r.pf[2] = r.pf[3] = 0;   // (the advance is picked from the scalars below)
    const int tile = (int)(i / NT);
    const i64 tpos = cur_in + s_pos[tile];
    const i64 off = (i64)s_off[tile] + r.loc_off;
    const int ph = (int)(tpos & 3);
    const u32 pfv = ph == 0 ? rb.x : (ph == 1 ? rb.y : (ph == 2 ? rb.z : rb.w));
    sample_node<idx_t, false>(a, r, off, tpos + pfv, begin + i, pbase, g, gl, gbase, gmask);
  }
  tl_mark(TL_SAMPLE | TL_END);
}

__global__ void __launch_bounds__(NT) k_mark_s(const PassArgs a) {
  __shared__ u32 s_w[NT / 32];
  pdl_enter(TL_MARK);
  const i64 E = a.st[a.w_E];
  const i64 ntiles = ceil_div(E, ETILE);
  u32 mine = 0;
  for (i64 tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    mark_tile(a, E, tile, s_w);
    if (threadIdx.x == 0) mine += (u32)a.mtile[tile];
  }
  // the pass's total of new nodes: the host-facing counter of the run's last pass is published from it
  if (threadIdx.x == 0 && mine) atomicAdd(reinterpret_cast<unsigned long long*>(a.st + a.w_new), (unsigned long long)mine);
  tl_mark(TL_MARK | TL_END);
}

__global__ void __launch_bounds__(NT) k_assign_s(const PassArgs a) {
  __shared__ u32 s_excl[LAT_TILES];
  __shared__ u32 s_w[NT / 32];
  pdl_enter(TL_ASSIGN);
  const i64 E = a.st[a.w_E];
  const i64 pbase = ldw(a.st, a.w_pbase, 0);
  const i64 list_base = ldw(a.st, a.w_list_in, a.c_list_in);
  const i64 ids_base = list_base - (a.st[a.w_seed_list] - a.st[a.w_seed_ids]);   // duplicate seeds are listed, not numbered
  const int ntiles = (int)ceil_div(E, ETILE);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (a.pub_words && blockIdx.x == 0 && threadIdx.x == 0) {   // last pass of the run: its dst list length was the last counter
    publish_last(a, list_base + a.st[a.w_new]);
    tl_mark(TL_FINAL);
  }
  // this thread's first edge: fetched now, beside the tile counts
  const i64 p_first = (i64)blockIdx.x * NT + threadIdx.x;
  u32 er_first = 0, sl_first = 0;
  if (p_first < E) { er_first = a.erank[p_first]; sl_first = a.eslot[p_first]; }
  // ---- every block: exclusive scan of the per-tile counts of first occurrences
  u32 nnew;
  {
    const int t0 = threadIdx.x * 4;
    u32 pv[4]; u32 lv = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int t = t0 + q;
      pv[q] = lv;
      if (t < ntiles) lv += (u32)a.mtile[t];
    }
    u32 inc = lv;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const u32 o = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc += o;
    }
    if (lane == 31) s_w[wid] = inc;
    __syncthreads();
    u32 pre = 0, tot = 0;
    for (int w = 0; w < NT / 32; ++w) { if (w < wid) pre += s_w[w]; tot += s_w[w]; }
    const u32 ex = pre + inc - lv;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int t = t0 + q;
      if (t < ntiles) s_excl[t] = ex + pv[q];
    }
    nnew = tot;
    __syncthreads();
  }
  if (blockIdx.x == 0) {
    if (threadIdx.x == 0) a.st[a.w_list_out] = list_base + nnew;
  }
  for (i64 p = p_first; p < E; p += (i64)gridDim.x * NT) {
    const u32 er = p == p_first ? er_first : a.erank[p];
    if (er & 0x80000000u) {
      const i64 rank = (i64)s_excl[p / ETILE] + (er & 0x7fffffffu);
      const u32 s = p == p_first ? sl_first : a.eslot[p];
      a.vals[s] = (u64)(ids_base + rank);
      a.dst_nodes[list_base + rank] = a.colv[pbase + p];
      if (a.disjoint) a.dst_batch[list_base + rank] = a.src_batch[a.row[pbase + p]];
      a.dst_slot[list_base + rank] = s;
    }
  }
}

__global__ void __launch_bounds__(NT) k_lookup(const PassArgs a) {
  const i64 E = a.st[ST_PASS_E];
  const i64 pbase = a.st[ST_PASS_BASE];
  for (i64 p = (i64)blockIdx.x * NT + threadIdx.x; p < E; p += (i64)gridDim.x * NT)
    a.colv[pbase + p] = (i64)a.vals[a.eslot[p]];
}

// end of hop: advance every type's frontier slice and record nodes-per-hop (neighbor_kernel.cpp:807-812)
__global__ void k_hop_end(i64* st, int T, int L, int hop, int o_list, int o_begin, int o_end, int o_nph) {
  const int t = threadIdx.x;
  if (t < T) {
    const i64 n = st[o_list + t], e = st[o_end + t];
    st[o_nph + t * (L + 1) + hop + 1] = n - e;
    st[o_begin + t] = e;
    st[o_end + t] = n;
  }
}

__global__ void k_seed_end(i64* st, int t, int L, int o_list, int o_begin, int o_end, int o_nph) {
  st[o_begin + t] = 0;
  st[o_end + t] = st[o_list + t];
  st[o_nph + t * (L + 1)] = st[o_list + t];
}

// Last kernel of a run: deferred lookup of the last pass; block 0 publishes the run unless that has happened.
__global__ void __launch_bounds__(NT) k_final(const PassArgs a) {
  __shared__ u32 s_win[MT_WIN];
  pdl_enter(TL_FINAL);
  if (blockIdx.x == 0 && a.pub_words) {
    const i64 cursor = a.ssa ? ldw(a.st, a.w_cur_in, 0) : a.st[ST_CURSOR];
    mt_extend_block<3>(a.raw, a.gen, a.out0 + 256 * rng_blocks_for_units(cursor), a.raw_cap, a.st, s_win);
    publish_run(a, cursor, true);
  }
  deferred_lookup(a);
  tl_mark(TL_FINAL | TL_END);
}

// Seeds of one node type in ONE block (n <= SEED_FUSED_MAX): list, insert, first-occurrence ranks, ids.
// Equivalent to k_seed + k_mark + k_assign + k_seed_end (neighbor_kernel.cpp:409-416, mapper.h:29-46).
constexpr int SEED_NT = 1024;
constexpr int SEED_FUSED_MAX = 16384;
template <typename idx_t>
__global__ void __launch_bounds__(SEED_NT) k_seed_fused(const PassArgs a, const idx_t* __restrict__ seeds, int n, i64 batch0,
                                                         int L, int o_begin, int o_end, int o_nph, const PassArgs c) {
  __shared__ int s_w[SEED_NT / 32];
  __shared__ int s_carry;
  pdl_enter(TL_SEED);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (blockIdx.x > 0) {
    // ---- latency path: blocks 1.. do the k_count of the run's first pass `c` beside the dedup of block 0.  Its
    // frontier is this seed list as given (duplicates included) and nothing it needs comes out of the hash
    // table, so one launch covers both.  Each block takes 1024 seeds = four 256-node tiles (same records and
    // tile aggregates as count_tile).
    __shared__ u32 s_tv[SEED_NT / 32];
    __shared__ Func4 s_tf[SEED_NT / 32];
    const int base = ((int)blockIdx.x - 1) * SEED_NT;
    const int i = base + threadIdx.x;
    i64 rs = 0, deg = 0; u32 n_out = 0;
    Func4 f = {{0, 0, 0, 0}};
    if (i < n) node_degree<idx_t>(c, (i64)seeds[i], batch0 + i, &rs, &deg, &n_out, &f);
    u32 iv = n_out; Func4 iff = f;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const u32 ov = __shfl_up_sync(0xffffffffu, iv, d);
      Func4 of;
#pragma unroll
      for (int p = 0; p < 4; ++p) of.d[p] = __shfl_up_sync(0xffffffffu, iff.d[p], d);
      if (lane >= d) { iv += ov; iff = compose(of, iff); }
    }
    if (lane == 31) { s_tv[wid] = iv; s_tf[wid] = iff; }
    __syncthreads();
    const int w0 = wid & ~7;   // first warp of this thread's 256-node tile
    u32 pv = 0; Func4 pfx = {{0, 0, 0, 0}};
    for (int w = w0; w < wid; ++w) { pv += s_tv[w]; pfx = compose(pfx, s_tf[w]); }
    u32 ev = __shfl_up_sync(0xffffffffu, iv, 1);
    Func4 ef;
#pragma unroll
    for (int p = 0; p < 4; ++p) ef.d[p] = __shfl_up_sync(0xffffffffu, iff.d[p], 1);
    if (lane == 0) { ev = 0; ef = {{0, 0, 0, 0}}; }
    const Func4 exf = compose(pfx, ef);
    if (i < n) {
      NodeRec r;
      r.rs = rs; r.deg = (u32)deg; r.loc_off = pv + ev;
      r.pf[0] = exf.d[0]; r.pf[1] = exf.d[1]; r.pf[2] = exf.d[2]; r.pf[3] = exf.d[3];
      c.rec[i] = r;
    }
    if (lane == 31 && (wid & 7) == 7) {   // last thread of a tile: the tile's totals
      const int tile = (base >> 8) + (wid >> 3);
      if (tile * NT < n) {
        const Func4 tf = compose(pfx, iff);
        c.tile_out[tile] = pv + iv;
#pragma unroll
        for (int p = 0; p < 4; ++p) c.tile_func[4 * tile + p] = tf.d[p];
      }
    }
    return;
  }
  for (int i = threadIdx.x; i < n; i += SEED_NT) {
    const i64 v = (i64)seeds[i];
    a.dst_nodes[i] = v;
    if (a.disjoint) a.dst_batch[i] = batch0 + i;
    const u32 s = table_insert(a.keys, a.mask, make_key(v, batch0 + i, a.disjoint));
    red_min_u64(&a.vals[s], POS_BASE + (u64)i);
    a.eslot[i] = s;
  }
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();   // block-scope: all atomicMin of this block are visible
  for (int base = 0; base < n; base += SEED_NT) {
    const int i = base + threadIdx.x;
    u32 s = 0; int first = 0;
    if (i < n) {
      s = a.eslot[i];
      first = (a.vals[s] == POS_BASE + (u64)i) ? 1 : 0;
    }
    int inc = first;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int o = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc += o;
    }
    if (lane == 31) s_w[wid] = inc;
    __syncthreads();
    int pre = 0, tot = 0;
    for (int w = 0; w < SEED_NT / 32; ++w) { if (w < wid) pre += s_w[w]; tot += s_w[w]; }
    const int c0 = s_carry;
    if (i < n) a.dst_slot[i] = first ? s : NO_SLOT;
    __syncthreads();   // every thread has read vals[] of this chunk before ranks overwrite them
    if (first) a.vals[s] = (u64)(c0 + pre + inc - 1);
    if (threadIdx.x == 0) s_carry = c0 + tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    a.st[a.o_dst_list] = n;        // every seed is listed, duplicates included
    a.st[a.o_dst_ids] = s_carry;   // ids count distinct seeds only
    a.st[o_begin] = 0;
    a.st[o_end] = n;
    a.st[o_nph] = n;
  }
  tl_mark(TL_SEED | TL_END);
}

__global__ void __launch_bounds__(NT) k_cleanup(u64* keys, u64* vals, const u32* __restrict__ slots, const i64* n_ptr) {
  pdl_enter();
  const i64 n = *n_ptr;
  for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < n; i += (i64)gridDim.x * NT) {
    const u32 s = slots[i];
    if (s != NO_SLOT) { keys[s] = EMPTY; vals[s] = EMPTY; }
  }
}

// pyg::dist_neighbor_sample: cumsum_neighbors_per_node = seeds, then seeds + edges emitted by seeds 0..i
// (neighbor_kernel.cpp:386-388,446-492) from the records of the run's only pass
__global__ void __launch_bounds__(NT) k_dist_cumsum(const NodeRec* __restrict__ rec, const i64* __restrict__ tile_off, i64 n_seeds, i64 n_edges,
                                                     int have_pass, i64* __restrict__ out) {
  for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i <= n_seeds; i += (i64)gridDim.x * NT)
    out[i] = n_seeds + (i == n_seeds ? n_edges : (have_pass ? tile_off[i / NT] + (i64)rec[i].loc_off : 0));
}

// table growth (only the synced path): move every listed node's entry into the new table
__global__ void __launch_bounds__(NT) k_rehash(const u64* __restrict__ old_keys, const u64* __restrict__ old_vals,
                                               u64* new_keys, u64* new_vals, u64 new_mask, u32* slots, i64 n) {
  for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < n; i += (i64)gridDim.x * NT) {
    const u32 s = slots[i];
    if (s == NO_SLOT) continue;
    const u32 ns = table_insert(new_keys, new_mask, old_keys[s]);
    new_vals[ns] = old_vals[s];
    slots[i] = ns;
  }
}

template <typename out_t>
__global__ void __launch_bounds__(NT) k_export(const i64* __restrict__ src, out_t* __restrict__ dst, i64 n) {
  for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < n; i += (i64)gridDim.x * NT) dst[i] = (out_t)src[i];
}
// row / col / edge_id of one relation in one launch (null dst = skip)
template <typename out_t>
__global__ void __launch_bounds__(NT) k_export3(const i64* __restrict__ s0, const i64* __restrict__ s1, const i64* __restrict__ s2,
                                                 out_t* __restrict__ d0, out_t* __restrict__ d1, out_t* __restrict__ d2, i64 n) {
  for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < n; i += (i64)gridDim.x * NT) {
    if (d0) d0[i] = (out_t)s0[i];
    if (d1) d1[i] = (out_t)s1[i];
    if (d2) d2[i] = (out_t)s2[i];
  }
}
// one relation's edges + one type's node list in a single launch (homogeneous fast path)
template <typename out_t>
__global__ void __launch_bounds__(NT) k_export4(const i64* __restrict__ s0, const i64* __restrict__ s1, const i64* __restrict__ s2,
                                                 out_t* __restrict__ d0, out_t* __restrict__ d1, out_t* __restrict__ d2, i64 n_edges,
                                                 const i64* __restrict__ node, const i64* __restrict__ batch, out_t* __restrict__ dn,
                                                 i64 n_nodes, u64* keys, u64* vals, const u32* __restrict__ slots) {
  pdl_enter(TL_EXPORT);
  const i64 n = n_edges > n_nodes ? n_edges : n_nodes;
  for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < n; i += (i64)gridDim.x * NT) {
    if (keys && i < n_nodes) {   // deferred table reset (PYGB200_S_DEFER_CLEANUP)
      const u32 sl = slots[i];
      if (sl != NO_SLOT) { keys[sl] = EMPTY; vals[sl] = EMPTY; }
    }
    if (i < n_edges) {
      if (d0) d0[i] = (out_t)s0[i];
      if (d1) d1[i] = (out_t)s1[i];
      if (d2) d2[i] = (out_t)s2[i];
    }
    if (i < n_nodes && dn) {
      if (batch) { dn[2 * i] = (out_t)batch[i]; dn[2 * i + 1] = (out_t)node[i]; }
      else dn[i] = (out_t)node[i];
    }
  }
  tl_mark(TL_EXPORT | TL_END);
}
template <typename out_t>
__global__ void __launch_bounds__(NT) k_export_pairs(const i64* __restrict__ batch, const i64* __restrict__ node,
                                                      out_t* __restrict__ dst, i64 n) {
  for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < n; i += (i64)gridDim.x * NT) {
    dst[2 * i] = (out_t)batch[i];
    dst[2 * i + 1] = (out_t)node[i];
  }
}

inline int grid_for(i64 work_items, int per_block, int sm_count) {
  i64 b = ceil_div(work_items > 0 ? work_items : 1, per_block);
  const i64 cap = (i64)sm_count * 8;
  return (int)(b < cap ? b : cap);
}

inline i64 sat_mul(i64 a, i64 b) {
  if (a == 0 || b == 0) return 0;
  const i64 LIM = (i64)1 << 60;
  if (a > LIM / b) return LIM;
  return a * b;
}
inline i64 sat_add(i64 a, i64 b) {
  const i64 LIM = (i64)1 << 60;
  return (a + b > LIM) ? LIM : a + b;
}
inline u64 pow2_ge(u64 x) { u64 p = 1024; while (p < x) p <<= 1; return p; }

}  // namespace
}  // namespace pygb200

using namespace pygb200;

// ------------------------------------------------------------------------------------- handle
struct pygb200_sampler {
  int device = -1;
  int sm_count = 132;
  struct TypeBuf {
    DevBuf nodes, batch, slot, keys, vals;
    // v2: packed tables (node id << 32 | value) and the slot lists that say which entries a run touched, TWO of each:
    // consecutive runs alternate, so that the reset of run i's table (random 8-byte stores: 144 us per 65,536-seed call on
    // the papers100M-shaped graph, bench r2l) runs on a side stream beside run i+1 instead of in front of it
    DevBuf pk[2], vslot[2];
    int pk_bits[2] = {0, 0};   // log2 of the capacities (0 = not allocated)
    u64 tcap = 0;       // table capacity (slots, power of two); table is all-EMPTY between runs
    i64 n_nodes = 0;    // result of the last run
  };
  struct RelBuf { DevBuf row, colv, eid; i64 n_edges = 0; };
  std::vector<TypeBuf> types;
  std::vector<RelBuf> rels;
  // caller-owned result arrays for the NEXT run (pygb200_sampler_bind_outputs): the run's kernels write rows /
  // local cols / edge ids / node lists straight into them, so no export pass follows
  struct Bound { std::vector<i64*> row, col, eid, node; std::vector<i64> ecap, ncap; bool armed = false; } bound;
  bool last_direct = false;   // the last run wrote into the bound arrays (exports are refused)
  bool last_nodedup = false;  // the last run was a PYGB200_S_NO_DEDUP run (pygb200_sampler_export_cumsum is valid)
  i64 nd_seeds = 0;
  DevBuf eslot, erank, rec, tile_out, tile_func, tile_off, tile_pos, mtile, raw, st, gen;
  DevBuf fref;              // v2, single GPU: ref of every edge of the running pass
  DevBuf wkey, widx, wl_bits, wl_tab;   // biased sampling: key / index scratch, MKL logf deviations (bitmap + sorted list)
  DevBuf eraw;              // mixed biased / uniform relations: the RandintEngine's blocks, compacted (see sampler_run_impl)
  bool wl_ready = false;
  DevBuf seedpk[2];         // v2, sharded: scratch tables for the replicated dedup of the seeds (all-EMPTY between runs; one per side)
  int seedpk_bits[2] = {0, 0};
  int v2_side = 0;          // which of the two packed tables the current / last v2 run uses
  cudaStream_t clean_stream = nullptr;
  cudaEvent_t clean_done[2] = {nullptr, nullptr}, final_ev = nullptr;
  bool clean_pending[2] = {false, false};
  // v2, frontier sharding over peer memory: this rank's exchange region and the peer mappings of the others'
  struct XRegion {
    unsigned char* base = nullptr;
    size_t bytes = 0;
    i64 cap = 0;            // edges per pass the region is laid out for
    int world = 0, rank = 0;
    unsigned char* peer[16] = {nullptr};
    u64 epoch = 0;          // barrier count (flag words only grow)
    u64 passes = 0;         // sharded passes so far: parity picks the (dst, edge id) buffer
    i64 off_bar = 0, off_dst[2] = {0, 0}, off_eid[2] = {0, 0}, off_fref = 0;
    i64 off_exc = 0, off_exc_n = 0, off_xcnt = 0;
  } x;
  i64* st_host = nullptr;   // pinned + mapped mirror of the state buffer (k_final writes it directly)
  i64* st_host_dev = nullptr;   // device-side address of st_host
  i64 run_serial = 0;       // completion flag value of the current run
  bool cleanup_pending = false;   // the last run left its table reset to pygb200_sampler_export_all
  int st_o_list = 0;        // offset of the node-list counters inside `st` (for the deferred cleanup)
  // persistent mt19937 raw stream: survives between runs while torch's CPU generator is exactly where
  // the previous run left it (the common case in a sampling loop) and is extended ahead of time on a
  // side stream, so that generation stays off the critical path of the next run.
  bool mt_valid = false;          // raw[] continues the stream of `mt_expected`
  pygb200_mt19937 mt_expected;    // engine state written back by the previous run
  i64 mt_q = 0;                   // raw index of the next output
  i64 mt_gen_known = 0;           // raw words known (to the host) to be generated and visible to the main stream
  i64 mt_requested = 0;           // lower bound of the stream length once every queued generation kernel has run
  DevBuf seed_times;              // temporal sampling: seed time per batch id
  DevBuf jump_polys, jump_scratch; // jump-ahead table (tools/mt19937_jump.py) and {jump_base, ticket}
  int jump_S = 0, jump_P = 0;     // 0 = table not available: serial generation only
  bool jump_tried = false;
  i64 raw_cap_words = 0;
  cudaStream_t mt_stream = nullptr;
  // the last two pre-generation launches (side stream, in launch order): event + raw index they cover
  cudaEvent_t mt_ev[2] = {nullptr, nullptr};
  cudaEvent_t mt_order_ev = nullptr;   // main stream -> side stream ordering after an in-run extension
  i64 mt_ev_target[2] = {0, 0};
  bool mt_ev_pending[2] = {false, false};
  int mt_ev_next = 0;
  size_t st_words = 0;
  size_t st_dev_words = 0;  // layout size the device state halves were cleared for (0 = both halves need a memset)
  int st_cur = 0;           // half of `st` the last run used (k_final clears the other one for the next run)
  i64* st_last = nullptr;   // device state of the last run
  i64 mt_defer_target = 0;  // pre-generation decided at the end of the last run, launched inside the next one
  bool disjoint = false;
  bool dirty = false;       // a run failed mid-way: tables must be wiped before reuse
  int T = 0, R = 0, L = 0;
  std::mutex mu;
};

extern "C" const char* pygb200_last_error(void) { return g_err.c_str(); }
extern "C" int pygb200_cuda_version(void) { return CUDART_VERSION; }
extern "C" int pygb200_kernel_launches(void) { return g_launches.load(); }
extern "C" void pygb200_profile_enable(int on) { g_prof_on.store(on != 0); }
static u64* g_tl_buf = nullptr;
extern "C" int pygb200_timeline_enable(int on) {
  u64* p = nullptr;
  if (on) {
    if (!g_tl_buf) PYGB_CUDA(cudaMalloc(&g_tl_buf, (size_t)(TL_CAP + 1) * 8));
    PYGB_CUDA(cudaMemset(g_tl_buf, 0, (size_t)(TL_CAP + 1) * 8));
    p = g_tl_buf;
  }
  PYGB_CUDA(cudaDeviceSynchronize());
  PYGB_CUDA(cudaMemcpyToSymbol(g_tl, &p, sizeof(p)));
  return PYGB200_OK;
}
extern "C" int64_t pygb200_timeline_read(uint64_t* out, int64_t cap) {
  if (!g_tl_buf || !out || cap <= 0) return 0;
  if (cudaDeviceSynchronize() != cudaSuccess) return 0;
  u64 n = 0;
  if (cudaMemcpy(&n, g_tl_buf, 8, cudaMemcpyDeviceToHost) != cudaSuccess) return 0;
  if (n > (u64)TL_CAP) n = TL_CAP;
  if ((i64)n > cap) n = (u64)cap;
  if (n && cudaMemcpy(out, g_tl_buf + 1, (size_t)n * 8, cudaMemcpyDeviceToHost) != cudaSuccess) return 0;
  cudaMemset(g_tl_buf, 0, 8);
  return (int64_t)n;
}
extern "C" int pygb200_profile_read(const char* name, double* ms, int64_t* launches, int64_t* work) {
  std::lock_guard<std::mutex> lock(g_prof_mu);
  prof_drain_locked();
  const int i = name ? prof_slot(name) : -1;
  if (i < 0) { set_error("pygb200_profile_read: unknown kernel name"); return PYGB200_ERR_ARG; }
  if (ms) *ms = g_prof_acc[i].ms;
  if (launches) *launches = g_prof_acc[i].launches;
  if (work) *work = g_prof_acc[i].work;
  g_prof_acc[i].ms = 0; g_prof_acc[i].launches = 0; g_prof_acc[i].work = 0;
  return PYGB200_OK;
}

extern "C" int pygb200_sampler_create(pygb200_sampler** out) {
  PYGB_CHECK(out != nullptr, PYGB200_ERR_ARG, "pygb200_sampler_create: null out");
  int dev = 0;
  PYGB_CUDA(cudaGetDevice(&dev));
  auto* s = new pygb200_sampler();
  s->device = dev;
  cudaDeviceGetAttribute(&s->sm_count, cudaDevAttrMultiProcessorCount, dev);
  *out = s;
  return PYGB200_OK;
}

extern "C" void pygb200_sampler_destroy(pygb200_sampler* s) {
  if (!s) return;
  if (s->clean_stream) { cudaStreamSynchronize(s->clean_stream); cudaStreamDestroy(s->clean_stream); }
  for (int i = 0; i < 2; ++i) if (s->clean_done[i]) cudaEventDestroy(s->clean_done[i]);
  if (s->final_ev) cudaEventDestroy(s->final_ev);
  for (auto& t : s->types) {
    t.nodes.release(); t.batch.release(); t.slot.release(); t.keys.release(); t.vals.release();
    for (int i = 0; i < 2; ++i) { t.pk[i].release(); t.vslot[i].release(); }
  }
  s->fref.release(); s->seedpk[0].release(); s->seedpk[1].release();
  s->wkey.release(); s->widx.release(); s->wl_bits.release(); s->wl_tab.release(); s->eraw.release();
  for (int q = 0; q < s->x.world; ++q) if (q != s->x.rank && s->x.peer[q]) cudaIpcCloseMemHandle(s->x.peer[q]);
  if (s->x.base) cudaFree(s->x.base);
  for (auto& r : s->rels) { r.row.release(); r.colv.release(); r.eid.release(); }
  if (s->mt_stream) { cudaStreamSynchronize(s->mt_stream); cudaStreamDestroy(s->mt_stream); }
  for (int i = 0; i < 2; ++i) if (s->mt_ev[i]) cudaEventDestroy(s->mt_ev[i]);
  if (s->mt_order_ev) cudaEventDestroy(s->mt_order_ev);
  DevBuf* all[] = {&s->eslot, &s->erank, &s->rec, &s->tile_out, &s->tile_func,
                   &s->tile_off, &s->tile_pos, &s->mtile, &s->raw, &s->st, &s->gen, &s->jump_polys, &s->jump_scratch, &s->seed_times};
  for (auto* b : all) b->release();
  if (s->st_host) cudaFreeHost(s->st_host);
  delete s;
}

namespace {

// kernel<<<grid, block, smem, st>>>(args...), as a PDL launch (with the programmatic-stream-serialization attribute, see
// pdl_enter) or a plain one, timed under the profile slot `slot` with `work` units (no slot: not timed).  Counts the
// launch and returns its error.
constexpr bool PDL = true, PLAIN = false;
template <bool pdl, typename... KP, typename... A>
int launch(const char* slot, long long work, void (*kernel)(KP...), dim3 grid, int block, size_t smem, cudaStream_t st,
           A... args) {
  void* tk = slot ? prof_begin(st) : nullptr;
  cudaError_t err = cudaSuccess;
  if constexpr (pdl) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = dim3((unsigned)block); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    err = cudaLaunchKernelEx(&cfg, kernel, KP(args)...);
  } else {
    kernel<<<grid, block, smem, st>>>(KP(args)...);
  }
  prof_end(tk, slot, st, work);
  PYGB_CUDA(err);
  PYGB_LAUNCH_CHECK();
  return PYGB200_OK;
}

constexpr int MAX_SHARDS = 64;
struct Layout { int o_list, o_ids, o_begin, o_end, o_rel, o_nph, o_eph, o_mt, o_shard, o_ssa; size_t words; };
Layout make_layout(int T, int R, int L) {
  Layout l;
  int o = ST_HDR;
  l.o_list = o; o += T; l.o_ids = o; o += T; l.o_begin = o; o += T; l.o_end = o; o += T;
  l.o_rel = o; o += R; l.o_nph = o; o += T * (L + 1); l.o_eph = o; o += R * (L > 0 ? L : 1);
  l.o_mt = o; o += MT_N / 2;
  l.o_shard = o; o += MAX_SHARDS + 2;
  l.o_ssa = o; o += 5 * R * (L > 0 ? L : 1);   // latency path: {E, cursor, relation total, dst list length, new nodes} per pass
  l.words = (size_t)o;
  return l;
}

// node list / slot list / batch list of one type: capacity for `need` entries, keeping `keep`
int ensure_type(pygb200_sampler* s, int t, i64 need, i64 keep, bool disjoint, cudaStream_t st) {
  auto& tb = s->types[t];
  if (int e = tb.nodes.ensure((size_t)need * 8, (size_t)keep * 8, st)) return e;
  if (int e = tb.slot.ensure((size_t)need * 4, (size_t)keep * 4, st)) return e;
  if (disjoint) if (int e = tb.batch.ensure((size_t)need * 8, (size_t)keep * 8, st)) return e;
  return PYGB200_OK;
}

// hash table of one type: room for `need_nodes` distinct keys at load factor <= 0.5.
// `listed` = entries currently in the table (0 between runs) -> rehash when it has to grow.
int ensure_table(pygb200_sampler* s, int t, i64 need_nodes, i64 listed, cudaStream_t st) {
  auto& tb = s->types[t];
  const u64 cap = pow2_ge(2 * (u64)(need_nodes > 0 ? need_nodes : 1));
  if (cap <= tb.tcap) return PYGB200_OK;
  PYGB_CHECK(cap <= (1ull << 32), PYGB200_ERR_UNSUPPORTED, "sampler hash table would exceed 2^32 slots");
  if (listed == 0) {
    if (int e = tb.keys.ensure(cap * 8, 0, st)) return e;
    if (int e = tb.vals.ensure(cap * 8, 0, st)) return e;
    PYGB_CUDA(cudaMemsetAsync(tb.keys.p, 0xff, cap * 8, st));
    PYGB_CUDA(cudaMemsetAsync(tb.vals.p, 0xff, cap * 8, st));
  } else {
    DevBuf nk, nv;
    if (int e = nk.ensure(cap * 8, 0, st)) return e;
    if (int e = nv.ensure(cap * 8, 0, st)) return e;
    PYGB_CUDA(cudaMemsetAsync(nk.p, 0xff, nk.cap, st));
    PYGB_CUDA(cudaMemsetAsync(nv.p, 0xff, nv.cap, st));
    if (int e = launch<PLAIN>(nullptr, 0, k_rehash, grid_for(listed, NT, s->sm_count), NT, 0, st, tb.keys.as<u64>(), tb.vals.as<u64>(),
                              nk.as<u64>(), nv.as<u64>(), cap - 1, tb.slot.as<u32>(), listed))
      return e;
    PYGB_CUDA(cudaStreamSynchronize(st));
    tb.keys.release(); tb.vals.release();
    tb.keys = nk; tb.vals = nv;
  }
  tb.tcap = cap;
  return PYGB200_OK;
}

// v2: packed table of one type with room for `need_nodes` distinct keys at load factor <= 0.5
int ensure_table_v2(pygb200_sampler* s, int t, int side, i64 need_nodes, i64 list_cap, cudaStream_t st) {
  auto& tb = s->types[t];
  if (int e = tb.vslot[side].ensure((size_t)std::max<i64>(list_cap, 1) * 4, 0, st)) return e;
  int bits = 10;
  while ((1ull << bits) < 2 * (u64)(need_nodes > 0 ? need_nodes : 1)) ++bits;
  if (bits <= tb.pk_bits[side]) return PYGB200_OK;
  PYGB_CHECK(bits <= 32, PYGB200_ERR_UNSUPPORTED, "sampler hash table would exceed 2^32 slots");
  if (int e = tb.pk[side].ensure((size_t)8 << bits, 0, st)) return e;
  PYGB_CUDA(cudaMemsetAsync(tb.pk[side].p, 0xff, (size_t)8 << bits, st));
  tb.pk_bits[side] = bits;
  return PYGB200_OK;
}

// v2 sharding: exchange region for passes of up to `cap` edges, mapped into every rank.  Collective: all ranks get
// here together (identical call sequences), `exchange` swaps the IPC handles and orders the remapping.
int ensure_xregion(pygb200_sampler* s, i64 cap, const pygb200_shard* shard, cudaStream_t st) {
  auto& x = s->x;
  const int W = shard->world;
  if (x.base && x.cap >= cap && x.world == W && x.rank == shard->rank) return PYGB200_OK;
  PYGB_CUDA(cudaStreamSynchronize(st));
  for (int q = 0; q < x.world; ++q)
    if (q != x.rank && x.peer[q]) { cudaIpcCloseMemHandle(x.peer[q]); x.peer[q] = nullptr; }
  i64 ncap = x.world == W ? std::max<i64>(x.cap, 1 << 16) : (1 << 16);
  while (ncap < cap) ncap *= 2;
  auto al = [](i64 b) { return (b + 255) / 256 * 256; };
  i64 o = 256;
  const i64 off_bar = 0;
  i64 off_dst[2], off_eid[2];
  for (int i = 0; i < 2; ++i) { off_dst[i] = o; o += al(ncap * 4); }
  for (int i = 0; i < 2; ++i) { off_eid[i] = o; o += al(ncap * 8); }
  const i64 off_fref = o; o += al(ncap * 4);
  const i64 off_exc_n = o; o += 256;                 // W list lengths (written by the source ranks)
  const i64 off_xcnt = o; o += 256;                  // this rank's running exception count
  const i64 off_exc = o; o += al((i64)W * ncap * 8); // W lists of up to ncap (position, ref) pairs

  unsigned char* nb = nullptr;
  PYGB_CUDA(cudaMalloc((void**)&nb, (size_t)o));
  PYGB_CUDA(cudaMemset(nb, 0, 256));
  PYGB_CUDA(cudaDeviceSynchronize());
  cudaIpcMemHandle_t mine;
  PYGB_CUDA(cudaIpcGetMemHandle(&mine, nb));
  std::vector<cudaIpcMemHandle_t> all((size_t)W);
  const int rc = shard->exchange(shard->user, &mine, all.data(), (int64_t)sizeof(mine));
  if (rc != 0) { cudaFree(nb); set_error("frontier-sharded sampling: handle exchange callback failed"); return PYGB200_ERR_INTERNAL; }
  // every rank closed its mappings of the old regions before it entered the exchange
  if (x.base) cudaFree(x.base);
  x.base = nb; x.bytes = (size_t)o; x.cap = ncap; x.world = W; x.rank = shard->rank;
  x.off_bar = off_bar; x.off_dst[0] = off_dst[0]; x.off_dst[1] = off_dst[1]; x.off_eid[0] = off_eid[0]; x.off_eid[1] = off_eid[1];
  x.off_fref = off_fref;
  x.off_exc = off_exc; x.off_exc_n = off_exc_n; x.off_xcnt = off_xcnt;
  x.epoch = 0; x.passes = 0;
  for (int q = 0; q < W; ++q) {
    if (q == x.rank) { x.peer[q] = nb; continue; }
    void* pp = nullptr;
    PYGB_CUDA(cudaIpcOpenMemHandle(&pp, all[(size_t)q], cudaIpcMemLazyEnablePeerAccess));
    x.peer[q] = (unsigned char*)pp;
  }
  return PYGB200_OK;
}

int ensure_rel(pygb200_sampler* s, int r, i64 need, i64 keep, cudaStream_t st) {
  auto& rb = s->rels[r];
  if (int e = rb.row.ensure((size_t)need * 8, (size_t)keep * 8, st)) return e;
  if (int e = rb.colv.ensure((size_t)need * 8, (size_t)keep * 8, st)) return e;
  if (int e = rb.eid.ensure((size_t)need * 8, (size_t)keep * 8, st)) return e;
  return PYGB200_OK;
}

int ensure_frontier_scratch(pygb200_sampler* s, i64 F, cudaStream_t st) {
  const i64 tiles = ceil_div(F > 0 ? F : 1, NT);
  if (int e = s->rec.ensure((size_t)(F > 0 ? F : 1) * sizeof(NodeRec), 0, st)) return e;
  if (int e = s->tile_out.ensure((size_t)tiles * 8, 0, st)) return e;
  if (int e = s->tile_func.ensure((size_t)tiles * 16, 0, st)) return e;
  if (int e = s->tile_off.ensure((size_t)tiles * 8, 0, st)) return e;
  if (int e = s->tile_pos.ensure((size_t)tiles * 8, 0, st)) return e;
  return PYGB200_OK;
}
int ensure_edge_scratch(pygb200_sampler* s, i64 E, cudaStream_t st) {
  const i64 e_ = E > 0 ? E : 1;
  if (int e = s->eslot.ensure((size_t)e_ * 4, 0, st)) return e;
  if (int e = s->erank.ensure((size_t)e_ * 4, 0, st)) return e;
  if (int e = s->mtile.ensure((size_t)ceil_div(e_, ETILE) * 8, 0, st)) return e;
  return PYGB200_OK;
}

// jump-ahead table: mt19937_jump.bin next to this shared library (optional; without it generation is serial)
void load_jump_table(pygb200_sampler* s, cudaStream_t st) {
  if (s->jump_tried) return;
  s->jump_tried = true;
  Dl_info info;
  if (!dladdr((void*)&pygb200_sampler_create, &info) || !info.dli_fname) return;
  std::string dir(info.dli_fname);
  const size_t slash = dir.find_last_of('/');
  dir = slash == std::string::npos ? std::string(".") : dir.substr(0, slash);
  const char* cands[] = {"/mt19937_jump.bin", "/csrc/mt19937_jump.bin"};
  for (const char* c : cands) {
    FILE* f = fopen((dir + c).c_str(), "rb");
    if (!f) continue;
    uint32_t hdr[4];
    std::vector<uint32_t> data;
    bool ok = fread(hdr, 4, 4, f) == 4 && hdr[0] == 0x4a54364du && hdr[3] == (uint32_t)MT_POLY_WORDS && hdr[2] >= 2 && hdr[2] <= 1024 &&
              hdr[1] >= 65536;
    if (ok) {
      data.resize((size_t)(hdr[2] - 1) * MT_POLY_WORDS);
      ok = fread(data.data(), 4, data.size(), f) == data.size();
    }
    fclose(f);
    if (!ok) continue;
    if (s->jump_polys.ensure(data.size() * 4, 0, st) != PYGB200_OK || s->jump_scratch.ensure(64, 0, st) != PYGB200_OK) return;
    if (cudaMemcpyAsync(s->jump_polys.p, data.data(), data.size() * 4, cudaMemcpyHostToDevice, st) != cudaSuccess) return;
    if (cudaMemsetAsync(s->jump_scratch.p, 0, 64, st) != cudaSuccess) return;
    if (cudaStreamSynchronize(st) != cudaSuccess) return;   // `data` is pageable and dies here
    s->jump_S = (int)hdr[1];
    s->jump_P = (int)hdr[2];
    return;
  }
}

// Jump-ahead has a fixed cost (~0.6 ms: serial pre-step + one polynomial pass per chunk); the one-CTA generator makes 2 G words/s
// (measured with biased sampling, which asks for 10^5..10^8 words at a time): the crossover is at ~1.2 M words.
constexpr i64 JUMP_MIN_WORDS = 1250000;

// Queue generation of the raw stream up to (at least) `target` on `st`.  Large requests are split over
// CTAs by jump-ahead (~20k-word serial pre-step + one pass over it per chunk), small ones run on one CTA.
int mt_request(pygb200_sampler* s, cudaStream_t st, i64 target) {
  target = std::min<i64>(target, s->raw_cap_words - MT_N);
  while (target > s->mt_requested) {
    const i64 amount = target - s->mt_requested;
    if (s->jump_P >= 2 && amount >= std::max<i64>(2 * (i64)s->jump_S, JUMP_MIN_WORDS)) {
      const int P_used = (int)std::min<i64>(s->jump_P, (amount + s->jump_S - 1) / s->jump_S);
      i64* jb = s->jump_scratch.as<i64>();
      if (int e = launch<PLAIN>(nullptr, 0, k_mt_jump_prestep<3>, 1, 640, 0, st, s->raw.as<u32>(), s->gen.as<i64>(), jb, s->raw_cap_words))
        return e;
      static const bool smem_ok = cudaFuncSetAttribute(k_mt_jump_generate<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, MT_JUMP_HIST * 4) == cudaSuccess;
      PYGB_CHECK(smem_ok, PYGB200_ERR_CUDA, "k_mt_jump_generate: cannot reserve shared memory for the jump history");
      if (int e = launch<PLAIN>(nullptr, 0, k_mt_jump_generate<3>, P_used, 640, MT_JUMP_HIST * 4, st, s->raw.as<u32>(), s->gen.as<i64>(), jb,
                                s->jump_polys.as<u32>(), s->jump_S, s->raw_cap_words, reinterpret_cast<unsigned long long*>(jb + 1)))
        return e;
      s->mt_requested += (i64)P_used * s->jump_S;
      if (s->mt_requested > s->raw_cap_words - MT_N) { s->mt_requested = s->raw_cap_words - MT_N; break; }
    } else {
      if (int e = launch<PLAIN>(nullptr, 0, k_mt_extend_to<3>, 1, 640, 0, st, s->raw.as<u32>(), s->gen.as<i64>(), target, s->raw_cap_words))
        return e;
      s->mt_requested = target;
    }
  }
  return PYGB200_OK;
}

int biased_error(i64 code) {
  PYGB_CHECK(code != W_ERR_NEG, PYGB200_ERR_ARG, "invalid multinomial distribution (encountering probability entry < 0)");
  PYGB_CHECK(code != W_ERR_INF, PYGB200_ERR_ARG, "invalid multinomial distribution (encountering probability entry = infinity or NaN)");
  PYGB_CHECK(code != W_ERR_SUM, PYGB200_ERR_ARG, "invalid multinomial distribution (sum of probabilities <= 0)");
  PYGB_CHECK(code != W_ERR_CATEGORIES, PYGB200_ERR_ARG, "number of categories cannot exceed 2^24");
  return PYGB200_OK;
}

u64 xbar_timeout_ns() {
  static const u64 ns = [] { const char* e = getenv("PYGB200_XBARRIER_TIMEOUT_MS"); return (u64)(e ? atoll(e) : 20000) * 1000000ull; }();
  return ns;
}

// ------------------------------------------------------------------------------------- run plan
// Static worst case of a run: frontier per (type, hop) `fb` and edges per (relation, hop) `eb` (every frontier node emits
// <= k edges, every edge adds <= one node of the relation's dst type; a fan-out < 0 adds nothing), and their sums per type
// (`nodes`) and per relation (`edges`).  Unclamped; every sum saturates at 2^60.  The relations' endpoints must be valid.
void static_bounds(int T, int R, int L, const pygb200_relation* rels, const int64_t* n_seeds, const int64_t* num_neighbors,
                   std::vector<i64>& fb, std::vector<i64>& eb, std::vector<i64>& nodes, std::vector<i64>& edges) {
  fb.assign((size_t)T * (L + 1), 0);
  eb.assign((size_t)R * (L > 0 ? L : 1), 0);
  for (int t = 0; t < T; ++t) fb[(size_t)t * (L + 1)] = n_seeds[t];
  for (int h = 0; h < L; ++h)
    for (int r = 0; r < R; ++r) {
      const i64 k = num_neighbors[(size_t)r * L + h];
      const i64 e = k >= 0 ? sat_mul(fb[(size_t)rels[r].src_type * (L + 1) + h], k) : 0;
      eb[(size_t)r * L + h] = e;
      i64& nf = fb[(size_t)rels[r].dst_type * (L + 1) + h + 1];
      nf = sat_add(nf, e);
    }
  nodes.assign(T, 0);
  edges.assign(R, 0);
  for (int t = 0; t < T; ++t)
    for (int h = 0; h <= L; ++h) nodes[t] = sat_add(nodes[t], fb[(size_t)t * (L + 1) + h]);
  for (int r = 0; r < R; ++r)
    for (int h = 0; h < L; ++h) edges[r] = sat_add(edges[r], eb[(size_t)r * L + h]);
}

// Everything a run decides before its first CUDA call: the caller's arguments, the static bounds, the mode flags and the
// schedule.
struct RunPlan {
  int T = 0, R = 0, L = 0;
  const pygb200_relation* rels = nullptr;
  const void *const *seeds = nullptr, *const *edge_weight = nullptr;
  const int64_t *n_seeds = nullptr, *num_neighbors = nullptr;
  unsigned flags = 0;
  const pygb200_shard* shard = nullptr;
  const pygb200_temporal* temporal = nullptr;
  bool replace = false, disjoint = false, idx32 = false;
  i64 total_seeds = 0;
  std::vector<i64> fb, eb, node_cap, rel_cap;   // static_bounds; the capacities clamped to >= 1
  i64 max_F = 1, max_E = 1, draw_units = 0, draw_count = 0;
  bool synced = false;   // sync after every count kernel and size buffers from actual numbers
  bool any_time = false, weighted = false, mixed = false, sharded = false, p2p = false, nodedup = false;
  std::vector<char> wrel;          // relations with edge weights
  std::vector<i64> type_nodes;     // nodes of each type, where a relation with that source type tells us (-1: unknown)
  bool lat = false, v2 = false;    // the schedule: latency, v2, else the wide table
  bool direct = false;             // results straight into the caller's bound arrays
  int XW = 1, XR = 0;              // peer-memory sharding: world size and rank
  int fuse_r = -1, fuse_t = -1;    // latency schedule: the first pass, counted inside the seed launch of its source type
  i64 k(int r, int h) const { return num_neighbors[(size_t)r * L + h]; }
  i64 F(int r, int h) const { return fb[(size_t)rels[r].src_type * (L + 1) + h]; }   // static frontier of pass (h, r)
  i64 E(int r, int h) const { return eb[(size_t)r * L + h]; }
  bool launches(int r, int h) const { return k(r, h) != 0 && F(r, h) != 0 && E(r, h) != 0; }   // bounded pass (h, r) runs
};

int make_plan(RunPlan& p, pygb200_sampler* s, bool bound_armed, int32_t T, int32_t R, int32_t L, const pygb200_relation* rels,
              const void* const* seeds, const int64_t* n_seeds, const int64_t* num_neighbors, unsigned flags,
              const pygb200_mt19937* mt, const pygb200_shard* shard, const pygb200_temporal* temporal,
              const void* const* edge_weight) {
  p.T = T; p.R = R; p.L = L; p.rels = rels; p.seeds = seeds; p.n_seeds = n_seeds; p.num_neighbors = num_neighbors;
  p.flags = flags; p.shard = shard; p.temporal = temporal; p.edge_weight = edge_weight;
  const bool replace = p.replace = (flags & PYGB200_S_REPLACE) != 0;
  const bool disjoint = p.disjoint = (flags & PYGB200_S_DISJOINT) != 0;
  const bool idx32 = p.idx32 = (flags & PYGB200_S_INDEX32) != 0;
  for (int t = 0; t < T; ++t) {
    PYGB_CHECK(n_seeds[t] >= 0, PYGB200_ERR_ARG, "negative seed count");
    PYGB_CHECK(n_seeds[t] == 0 || seeds[t] != nullptr, PYGB200_ERR_ARG, "null seed pointer");
    p.total_seeds += n_seeds[t];
  }
  for (int r = 0; r < R; ++r) {
    PYGB_CHECK(rels[r].src_type >= 0 && rels[r].src_type < T && rels[r].dst_type >= 0 && rels[r].dst_type < T,
               PYGB200_ERR_ARG, "relation endpoint out of range");
    PYGB_CHECK(rels[r].num_edges >= 0 && rels[r].num_edges < ((i64)1 << 40), PYGB200_ERR_UNSUPPORTED,
               "relations with >= 2^40 edges are not supported");
    PYGB_CHECK(rels[r].rowptr != nullptr && (rels[r].col != nullptr || rels[r].num_edges == 0), PYGB200_ERR_ARG,
               "null CSR pointer");
  }
  if (disjoint) PYGB_CHECK(p.total_seeds < ((i64)1 << 23), PYGB200_ERR_UNSUPPORTED,
                           "disjoint sampling supports < 2^23 seeds and node ids < 2^40 on this path");
  PYGB_CHECK(mt->left >= 1 && mt->left <= MT_N && mt->next >= 0 && mt->next <= MT_N, PYGB200_ERR_ARG,
             "invalid mt19937 state");

  // ---- static worst-case bounds
  static_bounds(T, R, L, rels, n_seeds, num_neighbors, p.fb, p.eb, p.node_cap, p.rel_cap);
  bool& synced = p.synced;
  for (size_t i = 0; i < (size_t)R * L; ++i) if (num_neighbors[i] < 0) synced = true;   // full neighbourhoods: no bound
  i64 total_elems = 0;
  p.max_E = std::max<i64>(p.total_seeds, 1);
  for (int t = 0; t < T; ++t) {
    for (int h = 0; h <= L; ++h) p.max_F = std::max(p.max_F, p.fb[(size_t)t * (L + 1) + h]);
    total_elems = sat_add(total_elems, p.node_cap[t]);
    p.node_cap[t] = std::max<i64>(p.node_cap[t], 1);
  }
  for (int r = 0; r < R; ++r) {
    for (int h = 0; h < L; ++h) {
      const i64 e = p.E(r, h);
      p.max_E = std::max(p.max_E, e);
      // units per draw: 1 when every range < 2^16, else at most 2 + 1 skipped (32-bit) / 4 + 3 (64-bit)
      p.draw_units = sat_add(p.draw_units, sat_mul(e, rels[r].num_edges < 65536 ? 1 : (rels[r].num_edges < ((i64)1 << 32) ? 3 : 7)));
      p.draw_count = sat_add(p.draw_count, e);
    }
    total_elems = sat_add(total_elems, sat_mul(p.rel_cap[r], 3));
    p.rel_cap[r] = std::max<i64>(p.rel_cap[r], 1);
  }
  if (total_elems > ((i64)1 << 30)) synced = true;  // > 8 GiB of worst-case int64 results: size from actuals
  bool& any_time = p.any_time;
  if (temporal) {
    for (int t = 0; t < T && temporal->node_time; ++t) any_time |= temporal->node_time[t] != nullptr;
    for (int r = 0; r < R && temporal->edge_time; ++r) any_time |= temporal->edge_time[r] != nullptr;
  }
  if (any_time) {
    PYGB_CHECK(disjoint, PYGB200_ERR_ARG, "Temporal sampling needs to create disjoint subgraphs");
    for (int t = 0; t < T; ++t)
      PYGB_CHECK(n_seeds[t] == 0 || (temporal->seed_time && temporal->seed_time[t]) || (temporal->node_time && temporal->node_time[t]),
                 PYGB200_ERR_ARG, "Seed time needs to be specified");
  }
  // biased sampling (edge_weight): per relation (neighbor_kernel.cpp:732-745).  `mixed` = some relations with weights, some without:
  // the weighted ones take engine outputs directly while the others draw from the RandintEngine, whose 256-output blocks then sit
  // wherever the generator happened to be when a block ran out — see Run::hops_synced.
  p.wrel.assign((size_t)std::max(R, 1), 0);
  if (edge_weight) {
    int nw = 0;
    for (int r = 0; r < R; ++r) { p.wrel[r] = edge_weight[r] != nullptr; nw += p.wrel[r]; }
    p.weighted = nw > 0;
    p.mixed = nw > 0 && nw < R;
    PYGB_CHECK(!p.weighted || !any_time, PYGB200_ERR_ARG, "Biased temporal sampling not yet supported");   // neighbor_kernel.cpp:377-380
    if (p.weighted && replace)
      for (int r = 0; r < R; ++r)
        for (int h = 0; h < L && p.wrel[r]; ++h)
          PYGB_CHECK(p.k(r, h) != 1, PYGB200_ERR_UNSUPPORTED,
                     "biased sampling with replacement and a fan-out of 1: at::multinomial(n_sample=1) draws from an MKL VSL stream "
                     "(exponential_), which this path does not reproduce");
  }
  if (p.mixed) synced = true;   // the host follows the engine's block count pass by pass
  const bool sharded = p.sharded = shard != nullptr && shard->world > 1;
  const bool nodedup = p.nodedup = (flags & PYGB200_S_NO_DEDUP) != 0;
  if (nodedup) PYGB_CHECK(T == 1 && R == 1 && L == 1 && !sharded, PYGB200_ERR_ARG,
                          "PYGB200_S_NO_DEDUP (distributed one-hop sampling) takes one node type, one relation, one hop");
  s->last_nodedup = false;
  if (sharded) {
    PYGB_CHECK(!synced, PYGB200_ERR_UNSUPPORTED, "frontier-sharded sampling needs bounded fan-outs (no -1, < 8 GiB worst case)");
    PYGB_CHECK(shard->world <= MAX_SHARDS && shard->rank >= 0 && shard->rank < shard->world && (shard->allgather || shard->exchange),
               PYGB200_ERR_ARG, "bad shard descriptor");
  }
  // ---- which schedule?  latency path (k_*_s: write-once counters, no serial sections) for small bounded runs,
  // v2 (sampler_v2.cuh: packed table, refs, peer-memory sharding) for the other bounded non-disjoint runs whose node
  // ids provably fit 32 bits, the wide-table throughput path for everything else.
  static const bool no_lat = getenv("PYGB200_NO_LATENCY_PATH") != nullptr;
  static const bool no_v2 = getenv("PYGB200_NO_V2") != nullptr;
  bool& lat = p.lat;
  lat = !synced && !sharded && !nodedup && L > 0 && !no_lat && !p.weighted;
  for (int t = 0; t < T && lat; ++t) lat = n_seeds[t] <= SEED_FUSED_MAX;
  for (int h = 0; h < L && lat; ++h)
    for (int r = 0; r < R && lat; ++r) {
      if (p.k(r, h) == 0) continue;
      lat = p.F(r, h) <= (i64)LAT_TILES * NT && p.E(r, h) <= (i64)LAT_TILES * ETILE;
    }
  const bool p2p = p.p2p = sharded && shard->exchange != nullptr;
  bool& v2 = p.v2;
  v2 = !lat && !synced && !nodedup && !disjoint && !any_time && L > 0 && (!sharded || p2p) && (!no_v2 || p2p || p.weighted);
  p.type_nodes.assign((size_t)T, -1);
  for (int r = 0; r < R; ++r) p.type_nodes[rels[r].src_type] = std::max(p.type_nodes[rels[r].src_type], (i64)rels[r].num_src_nodes);
  if (v2)   // every node type's id range must be known and fit the packed key (a type that is never a source has no bound)
    for (int t = 0; t < T && v2; ++t) v2 = idx32 || (p.type_nodes[t] >= 0 && p.type_nodes[t] < 0xffffffffll);
  if (p2p) PYGB_CHECK(v2 && T == 1 && R == 1 && shard->world <= V2_MAX_W, PYGB200_ERR_UNSUPPORTED,
                      "peer-memory frontier sharding: homogeneous, non-disjoint, bounded fan-outs, node ids < 2^32-1, world <= 16");
  if (p.weighted) PYGB_CHECK(!sharded, PYGB200_ERR_UNSUPPORTED, "biased sampling is not frontier-sharded: one GPU per batch");
  p.XW = p2p ? shard->world : 1;
  p.XR = p2p ? shard->rank : 0;

  // ---- results straight into the caller's arrays?  (bounded int64 non-disjoint runs only; the binding is one-shot)
  bool& direct = p.direct;
  direct = bound_armed && !synced && (!sharded || shard->exchange != nullptr) && !nodedup && !idx32 && !disjoint &&
           (int)s->bound.node.size() == T && (int)s->bound.row.size() == R;
  for (int t = 0; t < T && direct; ++t) direct = s->bound.node[t] != nullptr && s->bound.ncap[t] >= p.node_cap[t];
  for (int r = 0; r < R && direct; ++r)
    direct = s->bound.row[r] != nullptr && s->bound.col[r] != nullptr && s->bound.ecap[r] >= p.rel_cap[r];

  // the first pass that will run (hop 0) is counted inside the seed launch of its source type (extra blocks)
  if (lat)
    for (int r = 0; r < R; ++r)
      if (p.launches(r, 0)) { p.fuse_r = r; p.fuse_t = rels[r].src_type; break; }
  return PYGB200_OK;
}

// ------------------------------------------------------------------------------------- run
// latency schedule: a counter is the write-once word st[w] (w >= 0), else the constant c
struct Wd { int w; i64 c; };

// One run: its state, and one member function per phase (sampler_run_impl calls them in order).  idx_t is the index type
// of the caller's seeds and CSR (PYGB200_S_INDEX32); every kernel that reads them is launched as its idx_t instance.
template <typename idx_t>
struct Run {
  pygb200_sampler* s;
  cudaStream_t st;
  const RunPlan& p;
  Layout lay{};
  i64* dst = nullptr;         // this run's half of the device state
  i64* dst_other = nullptr;   // the other half (cleared by whoever publishes the run, for the next one)
  i64 out0 = 0;               // raw index of this run's first engine output
  i64 raw_cap = 0;            // raw stream capacity (words) the kernels are given
  i64 run_outputs = 0, run_outputs_max = 0;   // see mt_stream
  i64 wwords = 0;             // engine outputs consumed by biased passes so far
  i64 eng_blocks_max = 1;     // mixed: upper bound of the RandintEngine blocks fetched so far
  // lookup of the last pass, deferred into the next k_count / the final kernel
  i64* lk_colv = nullptr; const u64* lk_vals = nullptr; i64 lk_E = 0;
  // latency schedule: the static pass schedule decides which write-once word holds what
  std::vector<Wd> cur_list, sl_begin, sl_end, relcum, list_end;
  std::vector<int> eph_w;
  Wd cursor{-1, 0};
  int lk_w_E = -1, lk_w_pbase = -1;
  bool published = false;   // the last pass publishes the run (else k_final does)
  int pub_w_list = -1;      // the counter that arrives as the flag word's payload

  // ---- workspace
  int workspace() {
    const int T = p.T, R = p.R, L = p.L;
    if (s->cleanup_pending && !s->types.empty() && s->types[0].tcap) {   // nobody exported the previous run: reset its table now
      if (int e = cleanup_table(0, (i64)(s->types[0].slot.cap / 4), s->st_last + s->st_o_list)) return e;
      s->cleanup_pending = false;
    }
    if ((int)s->types.size() < T) s->types.resize(T);
    if ((int)s->rels.size() < R) s->rels.resize(R);
    s->T = T; s->R = R; s->L = L; s->disjoint = p.disjoint;
    lay = make_layout(T, R, L);
    if (lay.words > s->st_words) {
      if (s->st_host) cudaFreeHost(s->st_host);
      s->st_host = nullptr; s->st_words = 0;
      PYGB_CUDA(cudaHostAlloc((void**)&s->st_host, (lay.words + 8) * 8, cudaHostAllocMapped));
      PYGB_CUDA(cudaHostGetDevicePointer((void**)&s->st_host_dev, s->st_host, 0));
      memset(s->st_host, 0, (lay.words + 8) * 8);
      s->st_words = lay.words;
    }
    if (int e = s->st.ensure(2 * lay.words * 8, 0, st)) return e;
    if (int e = s->gen.ensure(64, 0, st)) return e;
    if (!s->mt_stream) {
      PYGB_CUDA(cudaStreamCreateWithFlags(&s->mt_stream, cudaStreamNonBlocking));
      for (int i = 0; i < 2; ++i) PYGB_CUDA(cudaEventCreateWithFlags(&s->mt_ev[i], cudaEventDisableTiming));
      PYGB_CUDA(cudaEventCreateWithFlags(&s->mt_order_ev, cudaEventDisableTiming));
    }
    if (s->dirty) {  // previous run aborted: wipe tables, forget the stream
      for (auto& tb : s->types) if (tb.tcap) {
        PYGB_CUDA(cudaMemsetAsync(tb.keys.p, 0xff, tb.tcap * 8, st));
        PYGB_CUDA(cudaMemsetAsync(tb.vals.p, 0xff, tb.tcap * 8, st));
      }
      for (int i = 0; i < 2; ++i) if (s->clean_pending[i]) { PYGB_CUDA(cudaStreamWaitEvent(st, s->clean_done[i], 0)); s->clean_pending[i] = false; }
      for (auto& tb : s->types)
        for (int i = 0; i < 2; ++i) if (tb.pk_bits[i]) PYGB_CUDA(cudaMemsetAsync(tb.pk[i].p, 0xff, (size_t)8 << tb.pk_bits[i], st));
      for (int i = 0; i < 2; ++i) if (s->seedpk_bits[i]) PYGB_CUDA(cudaMemsetAsync(s->seedpk[i].p, 0xff, (size_t)8 << s->seedpk_bits[i], st));
      s->mt_valid = false;
      s->st_dev_words = 0;
    }
    s->dirty = true;
    if (p.v2) {
      if (!s->clean_stream) {
        PYGB_CUDA(cudaStreamCreateWithFlags(&s->clean_stream, cudaStreamNonBlocking));
        for (int i = 0; i < 2; ++i) PYGB_CUDA(cudaEventCreateWithFlags(&s->clean_done[i], cudaEventDisableTiming));
        PYGB_CUDA(cudaEventCreateWithFlags(&s->final_ev, cudaEventDisableTiming));
      }
      s->v2_side ^= 1;   // the other table: the previous v2 run's one may still be resetting on the side stream
      if (s->clean_pending[s->v2_side]) { PYGB_CUDA(cudaStreamWaitEvent(st, s->clean_done[s->v2_side], 0)); s->clean_pending[s->v2_side] = false; }
      for (int t = 0; t < T; ++t) {
        if (int e = ensure_type(s, t, p.node_cap[t], 0, false, st)) return e;
        // distinct keys <= min(static bound, nodes of the type): a products-sized graph (2.4 M nodes) keeps its table
        // L2-resident (64 MB) whatever the batch; a rank's table holds the keys it owns: 1/W of them (+25 % for imbalance)
        const i64 keys = p.type_nodes[t] >= 0 ? std::min(p.node_cap[t], p.type_nodes[t]) : p.node_cap[t];
        const i64 own = p.XW == 1 ? keys : keys / p.XW + keys / (4 * p.XW) + 1024;
        if (int e = ensure_table_v2(s, t, s->v2_side, own, p.node_cap[t], st)) return e;
      }
      for (int r = 0; r < R; ++r) if (int e = ensure_rel(s, r, p.rel_cap[r], 0, st)) return e;
      if (int e = ensure_frontier_scratch(s, p.max_F, st)) return e;
      if (int e = ensure_edge_scratch(s, p.max_E, st)) return e;
      if (p.p2p) {
        if (int e = ensure_xregion(s, p.max_E, p.shard, st)) return e;
        int bits = 10;
        while ((1ull << bits) < 2 * (u64)std::max<i64>(p.total_seeds, 1)) ++bits;
        if (bits > s->seedpk_bits[s->v2_side]) {
          if (int e = s->seedpk[s->v2_side].ensure((size_t)8 << bits, 0, st)) return e;
          PYGB_CUDA(cudaMemsetAsync(s->seedpk[s->v2_side].p, 0xff, (size_t)8 << bits, st));
          s->seedpk_bits[s->v2_side] = bits;
        }
      } else if (int e = s->fref.ensure((size_t)p.max_E * 4, 0, st)) return e;
    } else if (!p.synced) {
      for (int t = 0; t < T; ++t) {
        if (int e = ensure_type(s, t, p.node_cap[t], 0, p.disjoint, st)) return e;
        if (int e = ensure_table(s, t, p.node_cap[t], 0, st)) return e;
      }
      for (int r = 0; r < R; ++r) if (int e = ensure_rel(s, r, p.rel_cap[r], 0, st)) return e;
      if (int e = ensure_frontier_scratch(s, p.max_F, st)) return e;
      if (int e = ensure_edge_scratch(s, p.max_E, st)) return e;
    } else {
      for (int t = 0; t < T; ++t) {
        if (int e = ensure_type(s, t, std::max<i64>(p.n_seeds[t], 1), 0, p.disjoint, st)) return e;
        if (int e = ensure_table(s, t, std::max<i64>(p.n_seeds[t], 1), 0, st)) return e;
      }
      for (int r = 0; r < R; ++r) if (int e = ensure_rel(s, r, 1, 0, st)) return e;
      if (int e = ensure_edge_scratch(s, p.total_seeds, st)) return e;
    }
    return PYGB200_OK;
  }

  // ---- mt19937 raw stream: continue the persistent one or (re)start from the caller's engine state.
  // Pre-generation runs TWO runs ahead on the side stream: the launch made at the end of run i-1 already
  // covers run i+1, so in a steady loop this run only waits for an event that completed long ago while
  // the launch made at the end of run i (for run i+2) overlaps run i+1.
  // run_outputs     : what a run is EXPECTED to consume at most (one 16-bit unit per draw — exact unless a
  //                   frontier node has >= 2^16 neighbours); pre-generation targets use it, a shortfall is
  //                   extended by the last block of k_count;
  // run_outputs_max : the worst case (32/64-bit draws incl. skipped units), used only for capacity.
  int wait_all_pregen() {
    for (int i = 0; i < 2; ++i) if (s->mt_ev_pending[i]) { PYGB_CUDA(cudaStreamWaitEvent(st, s->mt_ev[i], 0)); s->mt_ev_pending[i] = false; }
    return PYGB200_OK;
  }
  int mt_stream(const pygb200_mt19937* mt) {
    const bool synced = p.synced, weighted = p.weighted;
    run_outputs = synced ? 256 * 2 : 256 * (rng_blocks_for_units(p.draw_count) + 1);
    run_outputs_max = synced ? 256 * 2 : 256 * (rng_blocks_for_units(p.draw_units) + 1);
    bool cont = s->mt_valid && memcmp(&s->mt_expected, mt, sizeof(*mt)) == 0 &&
                s->mt_q + run_outputs_max + run_outputs + 6 * MT_N <= s->raw_cap_words;
    if (synced || weighted) {  // these runs extend the stream themselves (k_count / between passes): nothing may run beside them
      if (int e = wait_all_pregen()) return e;
      s->mt_gen_known = 0;
    }
    if (!cont || synced || weighted) s->mt_defer_target = 0;
    if (cont) {
      out0 = s->mt_q;
      const i64 need = out0 + run_outputs + MT_N;
      // oldest pending launch that covers this run (mt_ev_next is the older slot)
      const int older = s->mt_ev_next, newer = s->mt_ev_next ^ 1;
      if (s->mt_gen_known >= need) {
        // covered by a launch this stream has already waited for; newer launches keep running beside us
      } else if (s->mt_ev_pending[older] && s->mt_ev_target[older] >= need) {
        PYGB_CUDA(cudaStreamWaitEvent(st, s->mt_ev[older], 0));
        s->mt_ev_pending[older] = false;
        s->mt_gen_known = std::max(s->mt_gen_known, s->mt_ev_target[older]);
      } else if (s->mt_ev_pending[newer] && s->mt_ev_target[newer] >= need) {
        // same side stream: once the newer launch is complete so is the older one
        PYGB_CUDA(cudaStreamWaitEvent(st, s->mt_ev[newer], 0));
        s->mt_ev_pending[older] = s->mt_ev_pending[newer] = false;
        s->mt_gen_known = std::max(s->mt_gen_known, s->mt_ev_target[newer]);
      } else {
        // not covered ahead of time (first continued run, or a run larger than the previous one): extend here
        if (int e = wait_all_pregen()) return e;
        if (int e = mt_request(s, st, need)) return e;
        s->mt_gen_known = need;
        // the side stream continues from here: order its next launch behind this one
        PYGB_CUDA(cudaEventRecord(s->mt_order_ev, st));
        PYGB_CUDA(cudaStreamWaitEvent(s->mt_stream, s->mt_order_ev, 0));
      }
    } else {
      if (int e = wait_all_pregen()) return e;
      static const i64 pref_cap = [] { const char* e = getenv("PYGB200_MT_CAP_WORDS"); return e ? (i64)atoll(e) : (i64)1 << 23; }();
      load_jump_table(s, st);
      const i64 want = std::max<i64>((i64)MT_N + 4 * (run_outputs_max + run_outputs) + 8 * MT_N + 2 * (i64)s->jump_S, pref_cap);  // default 32 MB of raw words
      if (want > s->raw_cap_words) {
        if (int e = s->raw.ensure((size_t)want * 4, 0, st)) return e;
        s->raw_cap_words = want;
      }
      MTPodParam pod;
      memcpy(pod.state, mt->state, sizeof(pod.state));
      if (int e = launch<PLAIN>(nullptr, 0, k_mt_init, 1, NT, 0, st, s->raw.as<u32>(), s->gen.as<i64>(), pod)) return e;
      out0 = mt_next0(mt->left);
      s->mt_gen_known = MT_N;
      s->mt_requested = MT_N;
      if (!synced) {  // cover this run's expected need up front so that no pass has to extend the stream itself
        if (int e = mt_request(s, st, out0 + run_outputs + MT_N)) return e;
        s->mt_gen_known = out0 + run_outputs + MT_N;
      }
    }
    s->mt_valid = false;  // until this run completes
    raw_cap = s->raw_cap_words;
    if (p.mixed) {   // the engine's first block (fetched by its constructor, before anything else draws) opens the compacted copy
      if (int e = mt_request(s, st, out0 + 512 + MT_N)) return e;
      if (int e = s->eraw.ensure(512 * 4, 0, st)) return e;
      PYGB_CUDA(cudaMemcpyAsync(s->eraw.p, s->raw.as<u32>() + out0, 256 * 4, cudaMemcpyDeviceToDevice, st));
    }
    return PYGB200_OK;
  }

  // The raw stream buffer grows to `need` words, keeping what has been generated.
  int grow_raw(i64 need) {
    i64 gen_now = 0;
    PYGB_CUDA(cudaMemcpyAsync(&gen_now, s->gen.p, 8, cudaMemcpyDeviceToHost, st));
    PYGB_CUDA(cudaStreamSynchronize(st));
    if (int e = s->raw.ensure((size_t)need * 4, (size_t)gen_now * 4, st)) return e;
    raw_cap = s->raw_cap_words = (i64)(s->raw.cap / 4);
    return PYGB200_OK;
  }

  // ---- init: zero state.  Two halves: the previous run's k_final already cleared the one this run uses.
  int init_state() {
    if (s->st_dev_words != lay.words) {
      PYGB_CUDA(cudaMemsetAsync(s->st.p, 0, 2 * lay.words * 8, st));
      s->st_dev_words = lay.words;
      s->st_cur = 0;
    } else {
      s->st_cur ^= 1;
    }
    dst = s->st.as<i64>() + (size_t)s->st_cur * lay.words;
    dst_other = s->st.as<i64>() + (size_t)(s->st_cur ^ 1) * lay.words;
    s->st_last = dst;
    if (p.weighted && !s->wl_ready) {   // biased sampling: MKL logf deviations, once per sampler
      if (int e = s->wl_tab.ensure(sizeof(kMklLogfTable), 0, st)) return e;
      if (int e = s->wl_bits.ensure((size_t)1 << 21, 0, st)) return e;
      PYGB_CUDA(cudaMemcpyAsync(s->wl_tab.p, kMklLogfTable, sizeof(kMklLogfTable), cudaMemcpyHostToDevice, st));
      PYGB_CUDA(cudaMemsetAsync(s->wl_bits.p, 0, (size_t)1 << 21, st));
      if (int e = launch<PLAIN>(nullptr, 0, k_w_log_bitmap, ceil_div(kMklLogfTableN, NT), NT, 0, st, s->wl_tab.as<u32>(), kMklLogfTableN,
                                s->wl_bits.as<u32>()))
        return e;
      s->wl_ready = true;
    }
    return PYGB200_OK;
  }

  PassArgs make_args(int src_t, int dst_t, int rel) const {
    PassArgs a;
    memset(&a, 0, sizeof(a));
    auto& td = s->types[dst_t];
    a.dst_nodes = td.nodes.as<i64>(); a.dst_batch = td.batch.as<i64>(); a.dst_slot = td.slot.as<u32>();
    a.keys = td.keys.as<u64>(); a.vals = td.vals.as<u64>(); a.mask = td.tcap - 1;
    if (src_t >= 0) { a.src_nodes = s->types[src_t].nodes.as<i64>(); a.src_batch = s->types[src_t].batch.as<i64>(); }
    if (rel >= 0) {
      a.rowptr = p.rels[rel].rowptr; a.col = p.rels[rel].col;
      a.row = s->rels[rel].row.as<i64>(); a.colv = s->rels[rel].colv.as<i64>(); a.eid = s->rels[rel].eid.as<i64>();
      a.o_rel_edges = lay.o_rel + rel;
    }
    if (p.direct) {
      a.dst_nodes = s->bound.node[dst_t];
      if (src_t >= 0) a.src_nodes = s->bound.node[src_t];
      if (rel >= 0) {
        a.row = s->bound.row[rel]; a.colv = s->bound.col[rel];
        if (s->bound.eid[rel]) a.eid = s->bound.eid[rel];
      }
    }
    a.eslot = s->eslot.as<u32>(); a.erank = s->erank.as<u32>(); a.rec = s->rec.as<NodeRec>();
    a.tile_out = s->tile_out.as<i64>(); a.tile_func = s->tile_func.as<u32>();
    a.tile_off = s->tile_off.as<i64>(); a.tile_pos = s->tile_pos.as<i64>(); a.mtile = s->mtile.as<i64>();
    a.st = dst;
    a.o_src_begin = lay.o_begin + (src_t >= 0 ? src_t : 0); a.o_src_end = lay.o_end + (src_t >= 0 ? src_t : 0);
    a.o_dst_list = lay.o_list + dst_t; a.o_dst_ids = lay.o_ids + dst_t;
    a.raw = s->raw.as<u32>(); a.gen = s->gen.as<i64>(); a.out0 = out0; a.raw_cap = raw_cap;
    a.replace = p.replace; a.disjoint = p.disjoint;
    if (p.v2) {
      a.pk = td.pk[s->v2_side].as<u64>(); a.pk_bits = td.pk_bits[s->v2_side];
      a.dst_slot = td.vslot[s->v2_side].as<u32>();
      a.xw = p.XW; a.xr = p.XR; a.o_shard = lay.o_shard;
      a.fref = s->fref.as<u32>();
      if (p.p2p) {
        const auto& x = s->x;
        for (int q = 0; q < p.XW; ++q) a.xpeer[q] = x.peer[q];
        a.x_off_bar = x.off_bar; a.x_off_fref = x.off_fref;
        a.x_off_exc = x.off_exc; a.x_off_exc_n = x.off_exc_n; a.x_off_xcnt = x.off_xcnt; a.x_exc_cap = x.cap;
        a.x_off_dst = x.off_dst[x.passes & 1]; a.x_off_eid = x.off_eid[x.passes & 1];
        a.fref = reinterpret_cast<u32*>(x.base + x.off_fref);
        a.x_eid64 = (rel >= 0 && p.rels[rel].num_edges > 0xffffffffll) ? 1 : 0;
      }
    }
    if (p.any_time && rel >= 0) {  // edge time of the relation wins over node time of its dst type (:742-787)
      const pygb200_temporal* temporal = p.temporal;
      if (temporal->edge_time && temporal->edge_time[rel]) { a.time_mode = 2; a.time = reinterpret_cast<const i64*>(temporal->edge_time[rel]); }
      else if (temporal->node_time && temporal->node_time[dst_t]) { a.time_mode = 1; a.time = reinterpret_cast<const i64*>(temporal->node_time[dst_t]); }
      a.seed_times = s->seed_times.as<i64>();
      a.time_last = temporal->strategy_last;
    }
    return a;
  }
  // the arguments of pass (hop h, relation r); mixed runs point the uniform relations at the compacted engine blocks
  PassArgs pass_args(int r, int h) const {
    PassArgs a = make_args(p.rels[r].src_type, p.rels[r].dst_type, r);
    a.fanout = p.k(r, h);
    a.o_eph = lay.o_eph + r * p.L + h;
    if (p.mixed && !p.wrel[r]) { a.raw = s->eraw.as<u32>(); a.out0 = 0; a.raw_cap = (i64)(s->eraw.cap / 4); }
    return a;
  }
  // the last pass of hop h folds the end-of-hop bookkeeping into its k_mark
  void with_hop_end(PassArgs& a, int h) const {
    a.he_T = p.T; a.he_L = p.L; a.he_hop = h; a.he_list = lay.o_list; a.he_begin = lay.o_begin; a.he_end = lay.o_end;
    a.he_nph = lay.o_nph;
  }
  // the same, standalone, for a hop whose last pass did not run it
  int hop_end(int h) { return launch<PLAIN>(nullptr, 0, k_hop_end, 1, 1024, 0, st, dst, p.T, p.L, h, lay.o_list, lay.o_begin, lay.o_end, lay.o_nph); }
  int read_state() {
    PYGB_CUDA(cudaMemcpyAsync(s->st_host, dst, lay.words * 8, cudaMemcpyDeviceToHost, st));
    PYGB_CUDA(cudaStreamSynchronize(st));
    return PYGB200_OK;
  }

  // a count kernel's grid: F frontier nodes, and the deferred lookup of the previous pass (E_prev edges)
  int count_grid(const PassArgs& a, i64 F, i64 E_prev) const {
    return std::max(grid_for(F, NT, s->sm_count), a.lk_colv ? grid_for(E_prev, NT, s->sm_count) : 1);
  }
  // the publication of the run's counters and engine state to the host (by k_final, or the latency schedule's last pass)
  void publish(PassArgs& a) const {
    a.pub_host = s->st_host_dev; a.pub_zero = dst_other; a.pub_serial = s->run_serial; a.pub_words = (int)lay.words;
    a.pub_o_mt = lay.o_mt;
  }

  // ---- the wide-table pass kernels
  int count(const PassArgs& a, i64 F, i64 E_prev) { return launch<PDL>("count", F, k_count<idx_t>, count_grid(a, F, E_prev), NT, 0, st, a); }
  int sample(const PassArgs& a_in, i64 F, i64 E) {
    PassArgs a = a_in;
    a.group = sample_group_lanes(a.fanout);
    return launch<PDL>("sample", E, k_sample<idx_t>, grid_for(F, sample_nodes_per_block(a.group), s->sm_count), NT, 0, st, a);
  }
  int rest(const PassArgs& a, i64 F, i64 E, bool lookup_now, bool with_sample = true) {
    if (with_sample) if (int e = sample(a, F, E)) return e;
    if (int e = launch<PDL>("mark", E, k_mark, grid_for(E, ETILE, s->sm_count), NT, 0, st, a)) return e;
    if (int e = launch<PDL>("assign", E, k_assign, grid_for(E, NT, s->sm_count), NT, 0, st, a)) return e;
    if (lookup_now) return launch<PLAIN>("lookup", E, k_lookup, grid_for(E, NT, s->sm_count), NT, 0, st, a);
    return PYGB200_OK;
  }
  // a pass whose edge ids are already drawn (biased draws, all-gathered shards): expand from them (gather col, rows, hash
  // insert), then mark / assign
  int expand(const PassArgs& a, i64 F, i64 E, bool lookup_now) {
    PassArgs d = a;
    d.phase = 2;
    if (int e = sample(d, F, E)) return e;
    return rest(a, F, E, lookup_now, false);
  }

  // ---- v2: from the inserts of a pass (or of the seeds) to ids.  Single GPU: mark reads the refs from the table.
  // Sharded: refs of owned positions -> barrier -> slice-wise reduction over the peers, result stored to all ->
  // barrier -> the same mark on the full ref array.  Then ids (replicated, streaming).
  int xbarrier(const PassArgs& a) {   // wait until every rank has raised the flags of the current epoch
    return launch<PDL>("xbarrier", 1, k_xbarrier, 1, 32, 0, st, a, (u64)s->x.epoch, xbar_timeout_ns());
  }
  int v2_ids(const PassArgs& a, i64 Eb) {
    if (p.p2p) {
      PassArgs b = a;
      b.x_timeout_ns = xbar_timeout_ns();
      b.x_sig_epoch = ++s->x.epoch;   // the last block of k_v2_exc raises the flags ...
      if (int e = launch<PDL>("pref", Eb, k_v2_exc, grid_for(Eb, 4 * NT, s->sm_count), NT, 0, st, b)) return e;
      b.x_sig_epoch = 0;
      if (int e = xbarrier(a)) return e;   // ... and k_v2_scatter starts behind everybody's
      if (int e = launch<PDL>("reduce", Eb, k_v2_scatter, dim3((unsigned)grid_for(ceil_div(Eb, p.XW), NT, s->sm_count), (unsigned)p.XW), NT, 0,
                              st, b))
        return e;
      if (int e = launch<PDL>("mark", Eb, k_v2_mark<false>, grid_for(Eb, ETILE, s->sm_count), NT, 0, st, a)) return e;
      return launch<PDL>("assign", Eb, k_v2_assign<true>, grid_for(Eb, 4 * NT, s->sm_count), NT, 0, st, a);
    }
    if (int e = launch<PDL>("mark", Eb, k_v2_mark<true>, grid_for(Eb, ETILE, s->sm_count), NT, 0, st, a)) return e;
    return launch<PDL>("assign", Eb, k_v2_assign<false>, grid_for(Eb, 4 * NT, s->sm_count), NT, 0, st, a);
  }

  // ---- biased (edge_weight) pass: count -> the host reads the totals (one synchronisation) -> the raw stream and the key
  // scratch are sized -> draws -> inserts -> ids.  The engine outputs of biased passes follow the RandintEngine's first
  // (and, on this path, only) block of 256.
  // step 1: degrees -> per-node edge / engine-word / scratch offsets; the host reads the pass's totals (st_host)
  int biased_count(const PassArgs& a, i64 F_grid, i64 E_prev) {
    if (int e = launch<PDL>("count", F_grid, k_w_count<idx_t>, count_grid(a, F_grid, E_prev), NT, 0, st, a)) return e;
    if (int e = read_state()) return e;
    return biased_error(s->st_host[ST_ERROR]);
  }
  // step 2: size the key scratch and the raw stream from those totals, then draw: row / edge id / global dst id of every
  // sampled edge at its final position (what the schedules' insert stages start from)
  int biased_draws(PassArgs& a, int r) {
    const i64 F = s->st_host[ST_PASS_F], E = s->st_host[ST_PASS_E], W = s->st_host[ST_W_WORDS], S = s->st_host[ST_W_SCR];
    if (int e = s->wkey.ensure((size_t)std::max<i64>(S, 1) * 4, 0, st)) return e;
    if (int e = s->widx.ensure((size_t)std::max<i64>(S, 1) * 4, 0, st)) return e;
    // the engine outputs of this pass follow whatever the generator has handed out so far: the RandintEngine's blocks (one,
    // fetched by its constructor, unless uniform relations have drawn from it: `mixed`) and the earlier biased passes
    const i64 eng_words = 256 * rng_blocks_for_units(s->st_host[ST_CURSOR]);
    const i64 need = out0 + eng_words + wwords + W + 2 * MT_N;
    const i64 cap_need = need + 2 * (i64)s->jump_S + 8 * MT_N;
    if (cap_need > raw_cap) {
      PYGB_CHECK(cap_need < ((i64)1 << 33), PYGB200_ERR_UNSUPPORTED, "biased sampling: a run may consume at most 2^33 engine outputs");
      if (int e = grow_raw(cap_need)) return e;
    }
    void* tkm = prof_begin(st);
    if (int e = mt_request(s, st, need)) return e;
    prof_end(tkm, "mtgen", st, W);   // (raw mt19937 words of this pass: jump-ahead generation when there are many)
    a.raw = s->raw.as<u32>(); a.raw_cap = raw_cap;
    WArgs wa;
    wa.weight = reinterpret_cast<const float*>(p.edge_weight[r]);
    wa.skey = s->wkey.as<float>(); wa.sidx = s->widx.as<u32>();
    wa.lbits = s->wl_bits.as<u32>(); wa.ltab = s->wl_tab.as<u32>(); wa.ltab_n = kMklLogfTableN;
    wa.wbase = out0 + eng_words + wwords;
    wwords += W;
    const int gw = (int)std::min<i64>(std::max<i64>(ceil_div(F, NT / 32), 1), (i64)s->sm_count * 16);
    static const bool smem_ok = cudaFuncSetAttribute(k_w_sample<idx_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, W_LIST_MAX * 2048) == cudaSuccess;
    PYGB_CHECK(smem_ok, PYGB200_ERR_CUDA, "k_w_sample: cannot reserve shared memory for the candidate lists");
    const i64 kf = a.fanout;
    const size_t smem = (!a.replace && kf >= 0 && kf + 1 <= W_LIST_MAX) ? (size_t)(kf + 1) * (NT / 32) * 32 * 8 : 0;
    return launch<PDL>("sample", E, k_w_sample<idx_t>, gw, NT, smem, st, a, wa);
  }
  // v2 schedule: count -> draws -> inserts -> ids
  int biased_pass(PassArgs& a, int r, i64 Fb) {
    if (int e = biased_count(a, Fb, 0)) return e;
    if (int e = biased_draws(a, r)) return e;
    const i64 Eg = std::max<i64>(s->st_host[ST_PASS_E], 1);
    if (int e = launch<PDL>("insert", Eg, k_v2_insert<false>, grid_for(Eg, 4 * NT, s->sm_count), NT, 0, st, a)) return e;
    return v2_ids(a, Eg);
  }

  // ---- seeds (neighbor_kernel.cpp:409-416, :669-704)
  int seeds() {
    const int T = p.T, L = p.L;
    const int64_t* n_seeds = p.n_seeds;
    if (p.any_time) if (int e = s->seed_times.ensure((size_t)std::max<i64>(p.total_seeds, 1) * 8, 0, st)) return e;
    i64 batch0 = 0;
    for (int t = 0; t < T; batch0 += p.disjoint ? n_seeds[t] : 0, ++t) {
      const idx_t* seed = (const idx_t*)p.seeds[t];
      const i64 n = n_seeds[t];
      PassArgs a = make_args(-1, t, -1);
      a.seed_mode = 1;
      PassArgs c = a;
      int count_blocks = 0;
      if (t == p.fuse_t) {
        const int r = p.fuse_r;
        c = make_args(p.rels[r].src_type, p.rels[r].dst_type, r);
        c.fanout = p.k(r, 0);
        count_blocks = (int)ceil_div(n, SEED_NT);
      }
      if (p.any_time && n > 0) {
        const pygb200_temporal* temporal = p.temporal;
        const i64* stt = temporal->seed_time ? reinterpret_cast<const i64*>(temporal->seed_time[t]) : nullptr;
        const i64* ntt = temporal->node_time ? reinterpret_cast<const i64*>(temporal->node_time[t]) : nullptr;
        if (int e = launch<PLAIN>(nullptr, 0, k_seed_times<idx_t>, grid_for(n, NT, s->sm_count), NT, 0, st, s->seed_times.as<i64>(), seed, n,
                                  batch0, stt, ntt))
          return e;
      }
      if (p.v2) {
        if (n == 0) continue;   // the zeroed state already says "empty list, empty slice"
        if (p.p2p) { a.pk_main = a.pk; a.pk_main_bits = a.pk_bits; a.pk = s->seedpk[s->v2_side].as<u64>(); a.pk_bits = s->seedpk_bits[s->v2_side]; }
        a.sd_begin = lay.o_begin + t; a.sd_end = lay.o_end + t; a.sd_nph = lay.o_nph + t * (L + 1);   // (k_seed_end folded into the mark kernel)
        if (int e = launch<PDL>("seed", n, k_v2_seed<idx_t>, grid_for(n, NT, s->sm_count), NT, 0, st, a, seed, n)) return e;
        if (p.p2p) {
          // seeds: every rank dedups ALL of them in a scratch table of its own (65 k CAS, L2-resident) — no exchange, no
          // barrier; only the ids of the seeds a rank owns go into its partition of the real table (k_v2_assign)
          if (int e = launch<PDL>("mark", n, k_v2_mark<true>, grid_for(n, ETILE, s->sm_count), NT, 0, st, a)) return e;
          if (int e = launch<PDL>("assign", n, k_v2_assign<true>, grid_for(n, 4 * NT, s->sm_count), NT, 0, st, a)) return e;
          // (the scratch table is wiped on the side stream with this side's table reset, behind the run)
        } else if (int e = v2_ids(a, n)) return e;
        continue;
      }
      if (n > 0 && n <= SEED_FUSED_MAX) {
        if (int e = launch<PDL>(nullptr, 0, k_seed_fused<idx_t>, 1 + count_blocks, SEED_NT, 0, st, a, seed, (int)n, batch0, (int)L,
                                lay.o_begin + t, lay.o_end + t, lay.o_nph + t * (L + 1), c))
          return e;
      } else if (n > 0) {
        const int g = grid_for(n, NT, s->sm_count);
        if (int e = launch<PLAIN>(nullptr, 0, k_seed<idx_t>, g, NT, 0, st, a, seed, n, batch0)) return e;
        if (int e = launch<PDL>(nullptr, 0, k_mark, grid_for(n, ETILE, s->sm_count), NT, 0, st, a)) return e;
        if (int e = launch<PDL>(nullptr, 0, k_assign, g, NT, 0, st, a)) return e;
        if (int e = launch<PLAIN>(nullptr, 0, k_seed_end, 1, 1, 0, st, dst, t, L, lay.o_list, lay.o_begin, lay.o_end, lay.o_nph)) return e;
      }  // n == 0: the zeroed state already says "empty list, empty slice"
    }
    return PYGB200_OK;
  }

  // ---- hops, latency schedule: every pass's counters are write-once words fixed here, no host synchronisation
  int hops_latency() {
    const int T = p.T, R = p.R, L = p.L;
    cur_list.resize(T); sl_begin.resize(T); sl_end.resize(T); relcum.assign(R, Wd{-1, 0});
    list_end.resize((size_t)T * (L + 1)); eph_w.assign((size_t)R * L, -1);
    for (int t = 0; t < T; ++t) {
      cur_list[t] = Wd{-1, p.n_seeds[t]}; sl_begin[t] = Wd{-1, 0}; sl_end[t] = Wd{-1, p.n_seeds[t]};
      list_end[(size_t)t * (L + 1)] = cur_list[t];
    }
    int P = 0, P_total = 0;
    for (int h = 0; h < L; ++h)
      for (int r = 0; r < R; ++r) P_total += p.launches(r, h);
    for (int h = 0; h < L; ++h) {
      for (int r = 0; r < R; ++r) {
        // k == 0: nothing emitted, no RNG consumed (neighbor_kernel.cpp:67-68)
        if (!p.launches(r, h)) continue;
        const i64 k = p.k(r, h), Fb = p.F(r, h), Eb = p.E(r, h);
        const int src_t = p.rels[r].src_type, dst_t = p.rels[r].dst_type;
        PassArgs a = make_args(src_t, dst_t, r);
        if (P == P_total - 1) {   // the last pass publishes the run from its k_assign_s
          publish(a);
          published = true;
        }
        const int base = lay.o_ssa + 5 * P++;
        a.fanout = k;
        a.ssa = 1;
        a.w_begin = sl_begin[src_t].w; a.c_begin = sl_begin[src_t].c;
        a.w_end = sl_end[src_t].w; a.c_end = sl_end[src_t].c;
        a.w_list_in = cur_list[dst_t].w; a.c_list_in = cur_list[dst_t].c;
        a.w_pbase = relcum[r].w;
        a.w_cur_in = cursor.w;
        a.w_E = base; a.w_cur_out = base + 1; a.w_relcum_out = base + 2; a.w_list_out = base + 3; a.w_new = base + 4;
        if (a.pub_words) pub_w_list = base + 3;
        a.w_seed_list = lay.o_list + dst_t; a.w_seed_ids = lay.o_ids + dst_t;
        a.lk_colv = lk_colv; a.lk_vals = lk_vals; a.lk_w_E = lk_w_E; a.lk_w_pbase = lk_w_pbase;
        if (!(h == 0 && r == p.fuse_r))   // (else: counted inside the seed launch)
          if (int e = launch<PDL>("count", Fb, k_count_s<idx_t>, count_grid(a, Fb, lk_E), NT, 0, st, a)) return e;
        a.group = sample_group_lanes(k);
        const int gs = grid_for(Fb, sample_nodes_per_block(a.group), s->sm_count);
        if (int e = launch<PDL>("sample", Eb, k_sample_s<idx_t>, gs, NT, 0, st, a)) return e;
        if (int e = launch<PDL>("mark", Eb, k_mark_s, grid_for(Eb, ETILE, s->sm_count), NT, 0, st, a)) return e;
        if (int e = launch<PDL>("assign", Eb, k_assign_s, grid_for(Eb, NT, s->sm_count), NT, 0, st, a)) return e;
        lk_colv = a.colv; lk_vals = a.vals; lk_E = Eb; lk_w_E = base; lk_w_pbase = relcum[r].w;
        cursor = Wd{base + 1, 0}; relcum[r] = Wd{base + 2, 0}; cur_list[dst_t] = Wd{base + 3, 0};
        eph_w[(size_t)r * L + h] = base;
      }
      for (int t = 0; t < T; ++t) {   // end of hop: next frontier = what the hop added (neighbor_kernel.cpp:807-812)
        sl_begin[t] = sl_end[t]; sl_end[t] = cur_list[t];
        list_end[(size_t)t * (L + 1) + h + 1] = cur_list[t];
      }
    }
    return PYGB200_OK;
  }

  // ---- hops, bounded (v2 and wide-table) runs: buffers are sized from the static bounds, every pass's lookup is deferred
  // into the next k_count / the final kernel
  int hops_bounded() {
    const int R = p.R, L = p.L;
    for (int h = 0; h < L; ++h) {
      int last_r = -1;   // last pass of this hop that will actually be launched (it also does the end-of-hop bookkeeping)
      for (int r = 0; r < R; ++r) if (p.launches(r, h)) last_r = r;
      bool hop_closed = false;
      for (int r = 0; r < R; ++r) {
        // k == 0: nothing emitted, no RNG consumed (neighbor_kernel.cpp:67-68)
        if (!p.launches(r, h)) continue;
        const i64 Fb = p.F(r, h), Eb = p.E(r, h);
        PassArgs a = pass_args(r, h);
        a.lk_colv = lk_colv; a.lk_vals = lk_vals;
        if (r == last_r) with_hop_end(a, h);
        if (!p.wrel[r]) if (int e = count(a, Fb, lk_E)) return e;
        if (p.v2) {
          if (int e = pass_v2(a, r, h)) return e;
        } else if (p.wrel[r]) {   // wide table (disjoint / 64-bit ids): biased draws, then the expand-from-edge-ids stage the sharded path uses
          if (int e = biased_count(a, Fb, lk_E)) return e;
          if (int e = biased_draws(a, r)) return e;
          if (p.nodedup) continue;   // (row / edge id / global id are already what a distributed hop returns)
          if (int e = expand(a, Fb, Eb, false)) return e;
          lk_colv = a.colv; lk_vals = a.vals; lk_E = Eb;
        } else if (p.nodedup) {   // draw + gather only: global ids stay in `colv`, nothing is mapped, no lookup follows
          PassArgs d = a;
          d.phase = 3;
          if (int e = sample(d, Fb, Eb)) return e;
          continue;
        } else {
          if (int e = p.sharded ? pass_collective(a, Fb, Eb) : rest(a, Fb, Eb, false)) return e;
          lk_colv = a.colv; lk_vals = a.vals; lk_E = Eb;
        }
        if (r == last_r) hop_closed = true;
      }
      if (!hop_closed) if (int e = hop_end(h)) return e;
    }
    return PYGB200_OK;
  }
  // v2 pass after its count (a biased one counts itself): draws, inserts, ids
  int pass_v2(PassArgs& a, int r, int h) {
    const int R = p.R, L = p.L, dst_t = p.rels[r].dst_type;
    const i64 Fb = p.F(r, h), Eb = p.E(r, h);
    // does any later pass insert into this dst type's table?  (else the ids need not be written back)
    a.v2_writeback = 0;
    for (int h2 = h; h2 < L && !a.v2_writeback; ++h2)
      for (int r2 = (h2 == h ? r + 1 : 0); r2 < R && !a.v2_writeback; ++r2)
        a.v2_writeback = p.rels[r2].dst_type == dst_t && p.launches(r2, h2);
    if (p.wrel[r]) return biased_pass(a, r, Fb);
    a.group = sample_group_lanes(a.fanout);
    const int gs = grid_for(p.p2p ? ceil_div(Fb, p.XW) + 1 : Fb, sample_nodes_per_block(a.group), s->sm_count);
    if (!p.p2p) {   // draws and table inserts in one kernel
      if (int e = launch<PDL>("sample", Eb, k_v2_sample<idx_t, false>, gs, NT, 0, st, a)) return e;
      return v2_ids(a, Eb);
    }
    // (the positions of the ranks' frontier slices were written by the last block of k_count)
    if (int e = launch<PDL>("sample", Eb, k_v2_sample<idx_t, true>, gs, NT, 0, st, a)) return e;
    // own slice -> every peer with 16-byte stores; its last block raises this rank's flag at the peers ("my slice
    // has been delivered"), so the peers' flags arrive while the rows are written and k_v2_insert only has to look
    a.x_timeout_ns = xbar_timeout_ns();
    a.x_sig_epoch = ++s->x.epoch;
    if (int e = launch<PDL>("push", Eb, k_v2_push, grid_for(ceil_div(Eb, p.XW) + 1, 4 * NT, s->sm_count), NT, 0, st, a)) return e;
    a.x_sig_epoch = 0;
    if (int e = launch<PDL>("rows", Eb, k_v2_rows, grid_for(Fb, NT, s->sm_count), NT, 0, st, a)) return e;
    if (int e = xbarrier(a)) return e;   // until everybody's (dst, edge id) have arrived
    if (int e = launch<PDL>("insert", Eb, k_v2_insert<true>, grid_for(Eb, 4 * NT, s->sm_count), NT, 0, st, a)) return e;
    if (int e = v2_ids(a, Eb)) return e;
    s->x.passes += 1;
    return PYGB200_OK;
  }
  // collective frontier sharding, after the count: every rank counted the whole frontier (offsets and bit-stream positions
  // are global); draw only this rank's slice, all-gather the edge ids, then expand/dedup everything (replicated)
  int pass_collective(const PassArgs& a, i64 Fb, i64 Eb) {
    const pygb200_shard* shard = p.shard;
    const int W = shard->world;
    if (int e = launch<PLAIN>(nullptr, 0, k_shard_bounds, 1, 128, 0, st, a, W, lay.o_shard)) return e;
    if (int e = read_state()) return e;
    const i64 F = s->st_host[ST_PASS_F], E = s->st_host[ST_PASS_E], pbase = s->st_host[ST_PASS_BASE];
    PassArgs d = a;
    d.phase = 1;
    d.shard_lo = (i64)((__int128)F * shard->rank / W);
    d.shard_hi = (i64)((__int128)F * (shard->rank + 1) / W);
    if (d.shard_hi > d.shard_lo) if (int e = sample(d, d.shard_hi - d.shard_lo, E)) return e;
    if (E > 0) {
      const int rc = shard->allgather(shard->user, a.eid + pbase, reinterpret_cast<const int64_t*>(s->st_host + lay.o_shard), W, (void*)st);
      PYGB_CHECK(rc == 0, PYGB200_ERR_INTERNAL, "frontier-sharded sampling: all-gather callback failed");
    }
    return expand(a, Fb, Eb, false);
  }

  // ---- hops, host-synced runs (-1 fan-outs, > 8 GiB worst case, mixed biased / uniform relations): the host reads every
  // hop's frontier and every pass's count, and sizes the buffers from the actual numbers
  int hops_synced() {
    const int R = p.R, L = p.L;
    const i64* hs = s->st_host;
    for (int h = 0; h < L; ++h) {
      if (int e = read_state()) return e;  // actual frontier slices of this hop
      auto frontier = [&](int r) { return hs[lay.o_end + p.rels[r].src_type] - hs[lay.o_begin + p.rels[r].src_type]; };
      int last_r = -1;   // last pass of this hop that will actually be launched (it also does the end-of-hop bookkeeping)
      for (int r = 0; r < R; ++r) if (p.k(r, h) != 0 && frontier(r) != 0) last_r = r;
      bool hop_closed = false;
      for (int r = 0; r < R; ++r) {
        const i64 k = p.k(r, h);
        const int dst_t = p.rels[r].dst_type;
        const bool wrel = p.wrel[r];
        if (k == 0) continue;  // nothing emitted, no RNG consumed (neighbor_kernel.cpp:67-68)
        const i64 F = frontier(r);
        if (F == 0) continue;
        if (int e = ensure_frontier_scratch(s, F, st)) return e;
        if (k > 0 && !wrel) {  // draws possible: make sure the raw stream buffer can hold this pass
          const i64 upu = p.rels[r].num_edges < 65536 ? 1 : (p.rels[r].num_edges < ((i64)1 << 32) ? 3 : 7);
          if (int e = read_state()) return e;
          const i64 eng_blocks = rng_blocks_for_units(hs[ST_CURSOR] + sat_mul(sat_mul(F, k), upu)) + 1;   // engine blocks this pass may touch
          const i64 need = out0 + 256 * eng_blocks + wwords + 3 * MT_N + (p.mixed ? 2 * (i64)s->jump_S + 8 * MT_N : 0);
          if (need > raw_cap) if (int e = grow_raw(need)) return e;
          if (p.mixed) {
            // ---- mixed biased / uniform relations.  The reference's RandintEngine fetches a block of 256 engine outputs whenever it
            // runs out (rand_engine.h:53-61,80-85); biased relations take outputs in between, so block b of the engine sits at
            // out0 + 256 b + (outputs the biased passes had consumed when b was fetched).  The uniform kernels index a stream in
            // which the blocks are contiguous: that stream is kept as a compacted copy (`eraw`).  Blocks the engine has already
            // fetched (b < used) stay; every block it may fetch during this pass is (re)copied from where it would sit NOW.
            const i64 used = rng_blocks_for_units(hs[ST_CURSOR]);
            if (int e = mt_request(s, st, out0 + 256 * eng_blocks + wwords + 2 * MT_N)) return e;
            if (int e = s->eraw.ensure((size_t)eng_blocks * 256 * 4, (size_t)used * 256 * 4, st)) return e;
            PYGB_CUDA(cudaMemcpyAsync(s->eraw.as<u32>() + 256 * used, s->raw.as<u32>() + out0 + 256 * used + wwords,
                                      (size_t)(eng_blocks - used) * 256 * 4, cudaMemcpyDeviceToDevice, st));
            eng_blocks_max = std::max(eng_blocks_max, eng_blocks);
          }
        }
        PassArgs a = pass_args(r, h);
        if (wrel) {
          if (int e = biased_count(a, F, 0)) return e;
        } else {
          if (int e = count(a, F, 0)) return e;
          if (int e = read_state()) return e;
        }
        const i64 E = hs[ST_PASS_E];
        if (E == 0) continue;  // (a hop whose last pass emits nothing is closed by the standalone kernel below)
        const i64 rel_before = hs[ST_PASS_BASE], list_now = hs[lay.o_list + dst_t];
        if (int e = ensure_rel(s, r, rel_before + E, rel_before, st)) return e;
        if (int e = ensure_edge_scratch(s, E, st)) return e;
        if (int e = ensure_type(s, dst_t, list_now + E, list_now, p.disjoint, st)) return e;
        if (int e = ensure_table(s, dst_t, list_now + E, list_now, st)) return e;
        a = pass_args(r, h);  // pointers may have moved
        if (wrel) if (int e = biased_draws(a, r)) return e;   // (row / edge id / global dst id of every sampled edge)
        if (p.nodedup) {
          if (wrel) continue;
          a.phase = 3;
          if (int e = sample(a, F, E)) return e;
          continue;
        }
        if (r == last_r) with_hop_end(a, h);
        if (int e = wrel ? expand(a, F, E, true) : rest(a, F, E, true)) return e;
        if (r == last_r) hop_closed = true;
      }
      if (!hop_closed) if (int e = hop_end(h)) return e;
    }
    return PYGB200_OK;
  }

  // ---- final kernel (deferred lookup of the last pass + engine state), table cleanup, the wait for the run, results
  int finish(pygb200_mt19937* mt, int64_t* nodes_per_hop, int64_t* edges_per_hop, int64_t* n_nodes_out, int64_t* n_edges_out) {
    const int T = p.T;
    if (p.mixed) if (int e = mt_request(s, st, out0 + 256 * eng_blocks_max + wwords + 2 * MT_N)) return e;   // (the state k_final publishes)
    {
      PassArgs a = make_args(-1, 0, -1);
      a.lk_colv = lk_colv; a.lk_vals = lk_vals;
      if (p.lat) { a.ssa = 1; a.lk_w_E = lk_w_E; a.lk_w_pbase = lk_w_pbase; a.w_cur_in = cursor.w; }
      if (!published) publish(a);
      a.pub_wwords = wwords;
      if (int e = launch<PDL>("final", 1, k_final, lk_colv ? grid_for(lk_E, NT, s->sm_count) : 1, NT, 0, st, a)) return e;
    }
    // table cleanup is stream-ordered after k_final; the host does not wait for it.  With
    // PYGB200_S_DEFER_CLEANUP (homogeneous fast path) it rides along with pygb200_sampler_export_all instead.
    s->cleanup_pending = (p.flags & PYGB200_S_DEFER_CLEANUP) && T == 1 && !p.direct && !p.v2;
    s->last_direct = p.direct;
    s->last_nodedup = p.nodedup;
    s->nd_seeds = p.nodedup ? p.n_seeds[0] : 0;
    if (p.v2) PYGB_CUDA(cudaEventRecord(s->final_ev, st));   // the table reset of this run waits for it on the side stream (below)
    for (int t = 0; t < T && !s->cleanup_pending && !p.v2; ++t)
      if (int e = cleanup_table(t, p.synced ? (i64)(s->types[t].slot.cap / 4) : p.node_cap[t], dst + list_word(t))) return e;
    // pre-generation for the run after this one (decided when the previous run ended): launched now, on the side
    // stream, while the GPU is busy with this run and the host has nothing to do but wait
    if (s->mt_defer_target > 0) {
      const int slot = s->mt_ev_next;
      if (!s->mt_ev_pending[slot] && mt_request(s, s->mt_stream, s->mt_defer_target) == PYGB200_OK &&
          cudaEventRecord(s->mt_ev[slot], s->mt_stream) == cudaSuccess) {
        s->mt_ev_pending[slot] = true;
        s->mt_ev_target[slot] = s->mt_defer_target;
        s->mt_ev_next = slot ^ 1;
      }
      s->mt_defer_target = 0;
    }
    if (int e = wait_published()) return e;
    if (pub_w_list >= 0) s->st_host[pub_w_list] = (i64)((u64)s->st_host[lay.words] & 0xffffffffffull);
    const i64* hs = s->st_host;
    PYGB_CHECK(hs[ST_ERROR] != 2, PYGB200_ERR_INTERNAL, "sampler: a peer rank did not reach a cross-GPU barrier in time (frontier-sharded run; PYGB200_XBARRIER_TIMEOUT_MS)");
    if (int e = biased_error(hs[ST_ERROR])) return e;
    PYGB_CHECK(hs[ST_ERROR] == 0, PYGB200_ERR_INTERNAL, "sampler: mt19937 stream buffer too small (internal bound violated)");
    s->dirty = false;
    read_counters(nodes_per_hop, edges_per_hop, n_nodes_out, n_edges_out);
    if (p.v2) {
      // reset the entries this run touched, on the side stream, behind k_final: the next run uses the other table and does
      // not wait for it (the one after that does: clean_pending).  List lengths are host values by now.
      PYGB_CUDA(cudaStreamWaitEvent(s->clean_stream, s->final_ev, 0));
      for (int t = 0; t < T; ++t) {
        auto& tb = s->types[t];
        const i64 n = s->types[t].n_nodes;
        if (n == 0) continue;
        if (int e = launch<PLAIN>("cleanup", n, k_v2_cleanup, grid_for(n, NT, s->sm_count), NT, 0, s->clean_stream, tb.pk[s->v2_side].as<u64>(),
                                  (const u32*)tb.vslot[s->v2_side].as<u32>(), n))
          return e;
      }
      if (p.p2p && s->seedpk_bits[s->v2_side])
        PYGB_CUDA(cudaMemsetAsync(s->seedpk[s->v2_side].p, 0xff, (size_t)8 << s->seedpk_bits[s->v2_side], s->clean_stream));
      PYGB_CUDA(cudaEventRecord(s->clean_done[s->v2_side], s->clean_stream));
      s->clean_pending[s->v2_side] = true;
    }
    memcpy(mt->state, hs + lay.o_mt, sizeof(mt->state));
    mt->next = (int32_t)hs[ST_MT_NEXT];
    mt->left = (int32_t)hs[ST_MT_LEFT];
    // the stream persists: remember where it is and pre-generate what a run like this one will need,
    // on the side stream (one CTA, overlaps the caller's work and the next run's first kernels)
    s->st_o_list = list_word(0);
    s->mt_expected = *mt;
    s->mt_q = out0 + 256 * hs[ST_BLOCKS] + wwords;
    s->mt_valid = true;
    if (!p.synced && !p.weighted) {
      const i64 target = std::min<i64>(s->raw_cap_words - 2 * MT_N, s->mt_q + 2 * run_outputs + 2 * MT_N);
      // this run's kernels (which may extend the stream themselves) are done; the launch itself is left to the
      // next run (see above) so that it costs no host time between two runs
      s->mt_defer_target = target > s->mt_q ? target : 0;
    }
    return PYGB200_OK;
  }
  // the wide table of type t back to all-EMPTY: the *n_ptr listed nodes (<= n_grid) lose their entries
  int cleanup_table(int t, i64 n_grid, const i64* n_ptr) {
    auto& tb = s->types[t];
    return launch<PDL>(nullptr, 0, k_cleanup, grid_for(n_grid, NT, s->sm_count), NT, 0, st, tb.keys.as<u64>(), tb.vals.as<u64>(),
                       (const u32*)tb.slot.as<u32>(), n_ptr);
  }
  // the state word that holds the node list length of type t at the end of the run
  int list_word(int t) const { return p.lat && cur_list[t].w >= 0 ? cur_list[t].w : lay.o_list + t; }
  // wait for k_final's flag (spin on mapped memory; keep an eye on the stream in case the run died)
  int wait_published() {
    volatile i64* flag = s->st_host + lay.words;
    unsigned long long spins = 0;
    auto done = [&]() { return (((u64)*flag) >> 40) == ((u64)s->run_serial & 0xffffffull); };
    while (!done()) {
      if ((++spins & 0xfffff) == 0) {
        const cudaError_t q = cudaStreamQuery(st);
        if (q != cudaErrorNotReady) {
          if (q == cudaSuccess && done()) break;
          set_error(std::string("sampler: run did not complete: ") + cudaGetErrorString(q == cudaSuccess ? cudaErrorUnknown : q));
          return PYGB200_ERR_CUDA;
        }
      }
#if defined(__x86_64__)
      __builtin_ia32_pause();
#endif
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    return PYGB200_OK;
  }
  // node / edge counts of the run: from the write-once words of the latency schedule, else from the running counters
  void read_counters(int64_t* nodes_per_hop, int64_t* edges_per_hop, int64_t* n_nodes_out, int64_t* n_edges_out) {
    const int T = p.T, R = p.R, L = p.L;
    const i64* hs = s->st_host;
    if (p.lat) {
      auto val = [&](const Wd& x) { return x.w >= 0 ? hs[x.w] : x.c; };
      for (int t = 0; t < T; ++t) {
        const i64 n = val(cur_list[t]);
        s->types[t].n_nodes = n;
        if (n_nodes_out) n_nodes_out[t] = n;
        if (nodes_per_hop) {
          nodes_per_hop[(size_t)t * (L + 1)] = p.n_seeds[t];
          for (int j = 1; j <= L; ++j)
            nodes_per_hop[(size_t)t * (L + 1) + j] = val(list_end[(size_t)t * (L + 1) + j]) - val(list_end[(size_t)t * (L + 1) + j - 1]);
        }
      }
      for (int r = 0; r < R; ++r) {
        const i64 n = val(relcum[r]);
        s->rels[r].n_edges = n;
        if (n_edges_out) n_edges_out[r] = n;
        if (edges_per_hop) for (int j = 0; j < L; ++j) edges_per_hop[(size_t)r * L + j] = eph_w[(size_t)r * L + j] >= 0 ? hs[eph_w[(size_t)r * L + j]] : 0;
      }
      return;
    }
    for (int t = 0; t < T; ++t) {
      s->types[t].n_nodes = hs[lay.o_list + t];
      if (n_nodes_out) n_nodes_out[t] = hs[lay.o_list + t];
      if (nodes_per_hop) for (int j = 0; j <= L; ++j) nodes_per_hop[(size_t)t * (L + 1) + j] = hs[lay.o_nph + t * (L + 1) + j];
    }
    for (int r = 0; r < R; ++r) {
      s->rels[r].n_edges = hs[lay.o_rel + r];
      if (n_edges_out) n_edges_out[r] = hs[lay.o_rel + r];
      if (edges_per_hop) for (int j = 0; j < L; ++j) edges_per_hop[(size_t)r * L + j] = hs[lay.o_eph + r * L + j];
    }
  }

  int run(pygb200_mt19937* mt, int64_t* nodes_per_hop, int64_t* edges_per_hop, int64_t* n_nodes_out, int64_t* n_edges_out) {
    if (int e = workspace()) return e;
    if (int e = mt_stream(mt)) return e;
    if (int e = init_state()) return e;
    if (int e = seeds()) return e;
    s->run_serial += 1;
    if (int e = p.lat ? hops_latency() : p.synced ? hops_synced() : hops_bounded()) return e;
    return finish(mt, nodes_per_hop, edges_per_hop, n_nodes_out, n_edges_out);
  }
};

// The checks every run entry point makes (`fn` names it in their messages), then the run, under the sampler's mutex.
int sampler_run_impl(const char* fn, pygb200_sampler* s, int32_t T, int32_t R, int32_t L, const pygb200_relation* rels,
                     const void* const* seeds, const int64_t* n_seeds, const int64_t* num_neighbors, unsigned flags,
                     pygb200_mt19937* mt, int64_t* nodes_per_hop, int64_t* edges_per_hop, int64_t* n_nodes_out,
                     int64_t* n_edges_out, void* stream, const pygb200_shard* shard, const pygb200_temporal* temporal,
                     const void* const* edge_weight, int32_t weight_dtype) {
  PYGB_CHECK(s && seeds && n_seeds && mt && (rels || R == 0) && (num_neighbors || L == 0 || R == 0), PYGB200_ERR_ARG,
             std::string(fn) + ": null argument");
  PYGB_CHECK(T >= 1 && T <= 1024 && R >= 0 && L >= 0, PYGB200_ERR_ARG, std::string(fn) + ": bad T/R/L");
  PYGB_CHECK(weight_dtype == PYGB200_F32, PYGB200_ERR_UNSUPPORTED,
             "biased sampling: float32 edge weights only (the reference's random stream and key arithmetic depend on the weight dtype)");
  std::lock_guard<std::mutex> lock(s->mu);
  // the output binding is one-shot: it is consumed here, before any check can return early, so that a failed run
  // never leaves pointers to arrays its caller is about to free (ADVICE r1)
  const bool bound_armed = s->bound.armed;
  s->bound.armed = false;
  s->last_direct = false;
  RunPlan p;
  if (int e = make_plan(p, s, bound_armed, T, R, L, rels, seeds, n_seeds, num_neighbors, flags, mt, shard, temporal, edge_weight)) return e;
  cudaStream_t st = (cudaStream_t)stream;
  if (p.idx32) return Run<int32_t>{s, st, p}.run(mt, nodes_per_hop, edges_per_hop, n_nodes_out, n_edges_out);
  return Run<int64_t>{s, st, p}.run(mt, nodes_per_hop, edges_per_hop, n_nodes_out, n_edges_out);
}

}  // namespace

extern "C" int pygb200_sampler_run(pygb200_sampler* s, int32_t T, int32_t R, int32_t L,
                                   const pygb200_relation* rels, const void* const* seeds,
                                   const int64_t* n_seeds, const int64_t* num_neighbors, unsigned flags,
                                   pygb200_mt19937* mt, int64_t* nodes_per_hop, int64_t* edges_per_hop,
                                   int64_t* n_nodes_out, int64_t* n_edges_out, void* stream) {
  return sampler_run_impl("pygb200_sampler_run", s, T, R, L, rels, seeds, n_seeds, num_neighbors, flags, mt, nodes_per_hop,
                          edges_per_hop, n_nodes_out, n_edges_out, stream, nullptr, nullptr, nullptr, PYGB200_F32);
}

extern "C" int pygb200_sampler_run_temporal(pygb200_sampler* s, int32_t T, int32_t R, int32_t L,
                                            const pygb200_relation* rels, const void* const* seeds,
                                            const int64_t* n_seeds, const int64_t* num_neighbors, unsigned flags,
                                            pygb200_mt19937* mt, int64_t* nodes_per_hop, int64_t* edges_per_hop,
                                            int64_t* n_nodes_out, int64_t* n_edges_out, void* stream,
                                            const pygb200_temporal* temporal) {
  return sampler_run_impl("pygb200_sampler_run_temporal", s, T, R, L, rels, seeds, n_seeds, num_neighbors, flags, mt, nodes_per_hop,
                          edges_per_hop, n_nodes_out, n_edges_out, stream, nullptr, temporal, nullptr, PYGB200_F32);
}

extern "C" int pygb200_sampler_run_weighted(pygb200_sampler* s, int32_t T, int32_t R, int32_t L,
                                            const pygb200_relation* rels, const void* const* seeds,
                                            const int64_t* n_seeds, const int64_t* num_neighbors, unsigned flags,
                                            pygb200_mt19937* mt, int64_t* nodes_per_hop, int64_t* edges_per_hop,
                                            int64_t* n_nodes_out, int64_t* n_edges_out, void* stream,
                                            const void* const* edge_weight, int32_t weight_dtype) {
  return sampler_run_impl("pygb200_sampler_run_weighted", s, T, R, L, rels, seeds, n_seeds, num_neighbors, flags, mt, nodes_per_hop,
                          edges_per_hop, n_nodes_out, n_edges_out, stream, nullptr, nullptr, edge_weight, weight_dtype);
}

extern "C" int pygb200_sampler_run_sharded(pygb200_sampler* s, int32_t T, int32_t R, int32_t L,
                                           const pygb200_relation* rels, const void* const* seeds,
                                           const int64_t* n_seeds, const int64_t* num_neighbors, unsigned flags,
                                           pygb200_mt19937* mt, int64_t* nodes_per_hop, int64_t* edges_per_hop,
                                           int64_t* n_nodes_out, int64_t* n_edges_out, void* stream,
                                           const pygb200_shard* shard) {
  return sampler_run_impl("pygb200_sampler_run_sharded", s, T, R, L, rels, seeds, n_seeds, num_neighbors, flags, mt, nodes_per_hop,
                          edges_per_hop, n_nodes_out, n_edges_out, stream, shard, nullptr, nullptr, PYGB200_F32);
}

extern "C" int pygb200_sampler_bounds(int32_t T, int32_t R, int32_t L, const pygb200_relation* rels,
                                      const int64_t* n_seeds, const int64_t* num_neighbors, int64_t* node_cap,
                                      int64_t* edge_cap) {
  PYGB_CHECK(n_seeds && node_cap && (rels || R == 0) && (edge_cap || R == 0) && (num_neighbors || L == 0 || R == 0),
             PYGB200_ERR_ARG, "pygb200_sampler_bounds: null argument");
  PYGB_CHECK(T >= 1 && T <= 1024 && R >= 0 && L >= 0, PYGB200_ERR_ARG, "pygb200_sampler_bounds: bad T/R/L");
  for (int r = 0; r < R; ++r)
    PYGB_CHECK(rels[r].src_type >= 0 && rels[r].src_type < T && rels[r].dst_type >= 0 && rels[r].dst_type < T,
               PYGB200_ERR_ARG, "pygb200_sampler_bounds: relation node type out of range");
  for (int h = 0; h < L; ++h)
    for (int r = 0; r < R; ++r)
      PYGB_CHECK(num_neighbors[(size_t)r * L + h] >= 0, PYGB200_ERR_UNSUPPORTED, "pygb200_sampler_bounds: a fan-out of -1 has no static bound");
  // the run's static bounds, unclamped, with this function's own size limit (4 int64 words per edge)
  std::vector<i64> fb, eb, nodes, edges;
  static_bounds(T, R, L, rels, n_seeds, num_neighbors, fb, eb, nodes, edges);
  i64 total = 0;
  for (const i64 e : eb) total = sat_add(total, sat_mul(e, 4));
  std::copy(nodes.begin(), nodes.end(), node_cap);
  std::copy(edges.begin(), edges.end(), edge_cap);
  PYGB_CHECK(total <= ((i64)1 << 30), PYGB200_ERR_UNSUPPORTED, "pygb200_sampler_bounds: worst case too large for static sizing");
  return PYGB200_OK;
}

extern "C" int pygb200_sampler_bind_outputs(pygb200_sampler* s, int32_t T, int32_t R, void* const* row, void* const* col,
                                            void* const* edge_id, void* const* node, const int64_t* edge_cap,
                                            const int64_t* node_cap) {
  PYGB_CHECK(s && node && node_cap && (R == 0 || (row && col && edge_cap)) && T >= 1 && R >= 0, PYGB200_ERR_ARG,
             "pygb200_sampler_bind_outputs: null argument");
  std::lock_guard<std::mutex> lock(s->mu);
  auto& b = s->bound;
  b.row.assign(R, nullptr); b.col.assign(R, nullptr); b.eid.assign(R, nullptr); b.ecap.assign(R, 0);
  b.node.assign(T, nullptr); b.ncap.assign(T, 0);
  for (int r = 0; r < R; ++r) {
    b.row[r] = (i64*)row[r]; b.col[r] = (i64*)col[r]; b.eid[r] = edge_id ? (i64*)edge_id[r] : nullptr;
    b.ecap[r] = edge_cap[r];
  }
  for (int t = 0; t < T; ++t) { b.node[t] = (i64*)node[t]; b.ncap[t] = node_cap[t]; }
  b.armed = true;
  return PYGB200_OK;
}

extern "C" int pygb200_sampler_outputs_direct(pygb200_sampler* s) {
  if (!s) return 0;
  std::lock_guard<std::mutex> lock(s->mu);
  return s->last_direct ? 1 : 0;
}

extern "C" int pygb200_sampler_export_cumsum(pygb200_sampler* s, int64_t* out, void* stream) {
  PYGB_CHECK(s && out, PYGB200_ERR_ARG, "export_cumsum: null argument");
  PYGB_CHECK(s->last_nodedup, PYGB200_ERR_ARG, "export_cumsum: the last run was not a PYGB200_S_NO_DEDUP run");
  cudaStream_t st = (cudaStream_t)stream;
  const i64 ne = s->rels[0].n_edges;
  return launch<PLAIN>(nullptr, 0, k_dist_cumsum, grid_for(s->nd_seeds + 1, NT, s->sm_count), NT, 0, st, s->rec.as<NodeRec>(),
                       s->tile_off.as<i64>(), s->nd_seeds, ne, ne > 0 ? 1 : 0, reinterpret_cast<i64*>(out));
}

extern "C" int pygb200_sampler_export_edges(pygb200_sampler* s, int32_t rel, void* row_out, void* col_out,
                                            void* edge_id_out, int index32, void* stream) {
  PYGB_CHECK(s && rel >= 0 && rel < s->R, PYGB200_ERR_ARG, "export_edges: bad relation");
  PYGB_CHECK(!s->last_direct, PYGB200_ERR_ARG, "export: the last run wrote its results into the bound output arrays");
  cudaStream_t st = (cudaStream_t)stream;
  const i64 n = s->rels[rel].n_edges;
  if (n == 0) return PYGB200_OK;
  const int g = grid_for(n, NT, s->sm_count);
  const i64 *s0 = s->rels[rel].row.as<i64>(), *s1 = s->rels[rel].colv.as<i64>(), *s2 = s->rels[rel].eid.as<i64>();
  if (index32)
    return launch<PLAIN>("export", n, k_export3<int32_t>, g, NT, 0, st, s0, s1, s2, (int32_t*)row_out, (int32_t*)col_out, (int32_t*)edge_id_out, n);
  return launch<PLAIN>("export", n, k_export3<int64_t>, g, NT, 0, st, s0, s1, s2, (int64_t*)row_out, (int64_t*)col_out, (int64_t*)edge_id_out, n);
}

extern "C" int pygb200_sampler_export_all(pygb200_sampler* s, int32_t rel, void* row_out, void* col_out, void* edge_id_out,
                                          int32_t type, void* node_id_out, int index32, void* stream) {
  PYGB_CHECK(s && rel >= 0 && rel < s->R && type >= 0 && type < s->T, PYGB200_ERR_ARG, "export_all: bad relation / node type");
  PYGB_CHECK(!s->last_direct, PYGB200_ERR_ARG, "export: the last run wrote its results into the bound output arrays");
  cudaStream_t st = (cudaStream_t)stream;
  const i64 ne = s->rels[rel].n_edges, nn = s->types[type].n_nodes;
  const bool clean = s->cleanup_pending && type == 0;
  if (ne == 0 && nn == 0) { if (clean) s->cleanup_pending = false; return PYGB200_OK; }
  u64* ck = clean ? s->types[0].keys.as<u64>() : nullptr;
  u64* cv = clean ? s->types[0].vals.as<u64>() : nullptr;
  const u32* cs = clean ? s->types[0].slot.as<u32>() : nullptr;
  if (clean) s->cleanup_pending = false;
  const int g = grid_for(std::max(ne, nn), NT, s->sm_count);
  const i64 *s0 = s->rels[rel].row.as<i64>(), *s1 = s->rels[rel].colv.as<i64>(), *s2 = s->rels[rel].eid.as<i64>();
  const i64* node = s->types[type].nodes.as<i64>();
  const i64* batch = s->disjoint ? s->types[type].batch.as<i64>() : nullptr;
  if (index32)
    return launch<PDL>(nullptr, 0, k_export4<int32_t>, g, NT, 0, st, s0, s1, s2, (int32_t*)row_out, (int32_t*)col_out, (int32_t*)edge_id_out,
                       ne, node, batch, (int32_t*)node_id_out, nn, ck, cv, cs);
  return launch<PDL>(nullptr, 0, k_export4<int64_t>, g, NT, 0, st, s0, s1, s2, (int64_t*)row_out, (int64_t*)col_out, (int64_t*)edge_id_out,
                     ne, node, batch, (int64_t*)node_id_out, nn, ck, cv, cs);
}

extern "C" int pygb200_sampler_export_nodes(pygb200_sampler* s, int32_t type, void* node_id_out, int index32,
                                            void* stream) {
  PYGB_CHECK(s && type >= 0 && type < s->T, PYGB200_ERR_ARG, "export_nodes: bad node type");
  PYGB_CHECK(!s->last_direct, PYGB200_ERR_ARG, "export: the last run wrote its results into the bound output arrays");
  cudaStream_t st = (cudaStream_t)stream;
  const i64 n = s->types[type].n_nodes;
  if (n == 0 || !node_id_out) return PYGB200_OK;
  const int g = grid_for(n, NT, s->sm_count);
  const i64* node = s->types[type].nodes.as<i64>();
  if (s->disjoint) {
    const i64* batch = s->types[type].batch.as<i64>();
    if (index32) return launch<PLAIN>(nullptr, 0, k_export_pairs<int32_t>, g, NT, 0, st, batch, node, (int32_t*)node_id_out, n);
    return launch<PLAIN>(nullptr, 0, k_export_pairs<int64_t>, g, NT, 0, st, batch, node, (int64_t*)node_id_out, n);
  }
  if (index32) return launch<PLAIN>(nullptr, 0, k_export<int32_t>, g, NT, 0, st, node, (int32_t*)node_id_out, n);
  PYGB_CUDA(cudaMemcpyAsync(node_id_out, node, (size_t)n * 8, cudaMemcpyDeviceToDevice, st));
  return PYGB200_OK;
}

extern "C" int pygb200_neighbor_sample_run(pygb200_sampler* s, const void* rowptr, const void* col,
                                           int64_t num_nodes, int64_t num_edges, const void* seed,
                                           int64_t n_seed, const int64_t* num_neighbors, int32_t L,
                                           unsigned flags, pygb200_mt19937* mt, int64_t* nodes_per_hop,
                                           int64_t* edges_per_hop, int64_t* n_nodes, int64_t* n_edges,
                                           void* stream) {
  pygb200_relation rel;
  rel.rowptr = rowptr; rel.col = col; rel.num_src_nodes = num_nodes; rel.num_edges = num_edges;
  rel.src_type = 0; rel.dst_type = 0;
  const void* seeds[1] = {seed};
  return pygb200_sampler_run(s, 1, 1, L, &rel, seeds, &n_seed, num_neighbors, flags, mt, nodes_per_hop,
                             edges_per_hop, n_nodes, n_edges, stream);
}
