// pyg_lib_b200/csrc/random_walk.cu — uniform random walks (pyg::random_walk with p == q == 1) for sm_90a (H100).
//
// Same walk as the reference's CUDA walker (pyg_lib/csrc/sampler/cuda/random_walk_kernel.cu:27-51) on the same
// draws: the caller fills rand [walk_length, S] with at::rand (so values and generator advance are ATen's own), and
// walk i takes step j to col[rowptr[v] + int(rand[j][i] * float(deg))], or stays put on an isolated node.
// Differences, none of which changes a result for draws at::rand can produce:
//   * the result is written in its final [S, walk_length + 1] layout.  One thread walks one seed; a block stages
//     CHUNK steps of its BLOCK walks in shared memory and stores them row by row, so the stores stay coalesced
//     without the reference's [walk_length + 1, S] buffer and its transposing copy;
//   * the neighbour index is clamped to deg - 1.  For rand <= 1 - 2^-24 (the largest float at::rand returns) the
//     correctly rounded float product never reaches deg, whatever the degree, so the clamp only matters to ABI
//     callers that pass their own draws (rand == 1.0 would make the reference read col[row_end]);
//   * every node index is checked before it is dereferenced: a seed or `col` entry outside [0, num_nodes), or a
//     row outside [0, num_edges), stops that walk where it is and raises the process-wide asynchronous error flag,
//     which the next call reports (no host synchronisation on the way).  The reference reads out of bounds.
// Per step: one 4-byte draw (streamed), two rowptr words and one col word (dependent gathers), one output word.
#include "common.cuh"

namespace pygb200 {
namespace {

constexpr int RW_BLOCK = 128;   // walks per block
constexpr int RW_CHUNK = 16;    // steps staged in shared memory between two stores

}  // namespace

template <typename idx_t>
__global__ void __launch_bounds__(RW_BLOCK) k_random_walk(const idx_t* __restrict__ rowptr, const idx_t* __restrict__ col,
                                                          i64 num_nodes, i64 num_edges, const idx_t* __restrict__ seed,
                                                          i64 S, i64 walk_length, const float* __restrict__ rand,
                                                          idx_t* __restrict__ out, int* err) {
  __shared__ idx_t tile[RW_BLOCK][RW_CHUNK + 1];   // (+1: a column of the tile spreads over the banks)
  const i64 base = (i64)blockIdx.x * RW_BLOCK;
  const i64 i = base + threadIdx.x;
  const int rows = (int)min((i64)RW_BLOCK, S - base);
  const i64 width = walk_length + 1;
  i64 v = 0;
  bool ok = i < S;
  if (ok) {
    v = (i64)seed[i];
    if (v < 0 || v >= num_nodes) { ok = false; if (err) *err = 1; }
  }
  for (i64 j0 = 0; j0 < width; j0 += RW_CHUNK) {
    const int cols = (int)min((i64)RW_CHUNK, width - j0);
    float r[RW_CHUNK];
#pragma unroll
    for (int c = 0; c < RW_CHUNK; ++c) {   // the draws do not depend on the walk: issue them ahead of the chain
      const i64 j = j0 + c;
      r[c] = (i < S && j >= 1 && c < cols) ? __ldcs(rand + (j - 1) * S + i) : 0.f;
    }
#pragma unroll
    for (int c = 0; c < RW_CHUNK; ++c) {
      if (c < cols && j0 + c >= 1 && ok) {
        const i64 rs = (i64)rowptr[v], re = (i64)rowptr[v + 1];
        const i64 deg = re - rs;
        if (deg > 0) {
          if (rs < 0 || re > num_edges) {
            ok = false;
            if (err) *err = 1;
          } else {
            const i64 k = min((i64)(r[c] * (float)deg), deg - 1);
            const i64 w = (i64)col[rs + k];
            if (w < 0 || w >= num_nodes) { ok = false; if (err) *err = 1; }
            else v = w;
          }
        }
      }
      tile[threadIdx.x][c] = (idx_t)v;
    }
    __syncthreads();
    // rows base .. base + rows - 1, columns j0 .. j0 + cols - 1 of out: `rows` runs of `cols` consecutive words
    for (int e = threadIdx.x; e < rows * cols; e += RW_BLOCK) {
      const int rr = e / cols, cc = e - rr * cols;
      __stcs(out + (base + rr) * width + j0 + cc, tile[rr][cc]);
    }
    __syncthreads();
  }
}

}  // namespace pygb200

using namespace pygb200;

extern "C" int pygb200_random_walk(const void* rowptr, const void* col, int64_t num_nodes, int64_t num_edges, const void* seed,
                                   int64_t S, int64_t walk_length, const float* rand, void* out, int index32, void* stream) {
  PYGB_CHECK(S >= 0 && walk_length >= 0 && num_nodes >= 0 && num_edges >= 0, PYGB200_ERR_ARG,
             "random_walk: negative size ('walk_length' must be >= 0)");
  PYGB_CHECK(!take_async_error(ASYNC_ERR_RANDOM_WALK), PYGB200_ERR_ARG,
             "random_walk: an EARLIER random_walk call met a node index outside [0, num_nodes) in 'seed' or 'col' (or a row "
             "outside 'col' in 'rowptr'); that call's output is undefined");
  if (S == 0) return PYGB200_OK;
  PYGB_CHECK(rowptr && seed && out && (col || num_edges == 0) && (rand || walk_length == 0), PYGB200_ERR_ARG,
             "pygb200_random_walk: null pointer");
  PYGB_CHECK(ceil_div(S, RW_BLOCK) < (1ll << 31), PYGB200_ERR_UNSUPPORTED, "random_walk: too many seeds");
  cudaStream_t st = (cudaStream_t)stream;
  int* err = async_error_flag_dev(ASYNC_ERR_RANDOM_WALK);
  const unsigned grid = (unsigned)ceil_div(S, RW_BLOCK);
  if (index32)
    k_random_walk<int32_t><<<grid, RW_BLOCK, 0, st>>>((const int32_t*)rowptr, (const int32_t*)col, num_nodes, num_edges,
                                                      (const int32_t*)seed, S, walk_length, rand, (int32_t*)out, err);
  else
    k_random_walk<int64_t><<<grid, RW_BLOCK, 0, st>>>((const int64_t*)rowptr, (const int64_t*)col, num_nodes, num_edges,
                                                      (const int64_t*)seed, S, walk_length, rand, (int64_t*)out, err);
  PYGB_LAUNCH_CHECK();
  return PYGB200_OK;
}
