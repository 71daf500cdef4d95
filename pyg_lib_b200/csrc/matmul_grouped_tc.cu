// pyg_lib_b200/csrc/matmul_grouped_tc.cu — grouped GEMM on Hopper tensor cores (wgmma + TMA + mbarrier, sm_90a).
//
// Replaces the reference's TensorOp grouped GEMM (pyg_lib/csrc/ops/cuda/matmul_kernel.cu:121-287: CUTLASS 2.x
// GemmGrouped, mma.sync) with one hand-written persistent kernel that serves every tensor-core matmul of the library:
//   * pyg::segment_matmul in bf16 / fp16 (any K, M that are multiples of 8 elements — the TMA row-pitch rule) and in
//     fp32 storage with TF32 math when the caller allows it; the problem list is built ON THE DEVICE from `ptr`, so a
//     device-resident `ptr` costs no host sync;
//   * pyg::grouped_matmul (matmul_kernel.cu:289-302) — independent problems C_i = A_i @ B_i, including the transposed
//     VIEWS its backward passes in (dX = dY @ W^T, dW = X^T @ dY): an operand stored transposed is consumed MN-major
//     through wgmma's transpose bit — no copies;
//   * the weight gradient dW[b] = X_b^T dY_b of segment_matmul (contraction over the rows of a segment).
// One CTA per SM, 384 threads:
//   warpgroup 0, one thread   TMA producer: per K step one stage = A tile [128 rows x 128 bytes of K] + B tile
//                             [128 bytes of K x 128 columns], 4-stage mbarrier ring, SWIZZLE_128B; out-of-range K / M /
//                             rows are zero-filled by TMA, so tails need no special cases;
//   warpgroups 1, 2           wgmma m64n128 (k16 for 16-bit, k8 for TF32) on rows [0, 64) / [64, 128) of the tile,
//                             fp32 accumulators in registers; epilogue: registers -> fp32 staging tile in shared memory
//                             -> (+bias) -> storage type -> coalesced 16-byte row stores, predicated on the tails.
// Tiles of all problems form one flat list dealt round-robin to the CTAs (column tiles of one row tile are adjacent, so
// their A loads meet in L2).  Long contractions with few output tiles are split over K chunks whose fp32 partials are
// added in chunk order by k_gt_finish (bit-reproducible, no atomics).
// H100: 132 SMs, up to 227 KB of shared memory per block — the 4 x 32 KB ring plus 2 x 33 KB staging tiles fit one CTA.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "matmul_common.cuh"

namespace pygb200 {
namespace {

#include "hopper_ptx.cuh"

constexpr int GT_TM = 128;       // rows per tile: two consumer warpgroups x wgmma M = 64
constexpr int GT_BN = 128;       // columns per tile == wgmma N
constexpr int GT_STAGES = 4;
constexpr int GT_NT = 384;
constexpr u32 GT_A_BYTES = GT_TM * 128;                    // 16 KB: 128 rows x one 128-byte swizzle row of K
constexpr u32 GT_STAGE_BYTES = GT_A_BYTES + GT_BN * 128;   // 32 KB
constexpr int GT_SP = GT_BN + 4;                           // fp32 staging pitch (floats)
constexpr u32 GT_OUT_BYTES = 64 * GT_SP * 4;               // one consumer warpgroup's staging tile
constexpr int MAX_SEG = 1024;                              // segments of the TF32 / weight-gradient paths

// element kinds of the kernel
constexpr int ET_F16 = 0, ET_BF16 = 1, ET_TF32 = 2;
inline int et_of(int dtype) { return dtype == PYGB200_BF16 ? ET_BF16 : ET_F16; }   // bf16 / fp16 storage

struct GProb {
  const CUtensorMap* map_a;    // K-major A: dims [k, rows]; MN-major A (transposed view): dims [n, k]
  const CUtensorMap* map_b;    // MN-major B: dims [m, k, z]; K-major B (transposed view): dims [k, m, z]
  unsigned char* c;            // row-major output of this problem (storage type; fp32 in the TF32 kernel)
  const unsigned char* bias;   // [m] or null (storage type of c)
  i64 ldc;                     // elements
  int n, k, m;
  int a_off;                   // K-major A: row of this problem's first row in map_a; MN-major A: its first k
  int b_k0;                    // first k of this problem in map_b
  int b_z;                     // third coordinate into map_b (segment index)
  int a_mn, b_k;               // operand stored transposed
  int c_vec;                   // rows of C are 16-byte aligned
  int zero_ktail;              // k past `k` in the last stage are rows of the next segment: zero them in shared memory
  int tile0, tiles_n;          // first flat tile of the problem; number of column tiles
  int ksplit, ksteps_chunk;    // K chunks (work items per output tile) and K steps per chunk
  float* part;                 // non-null: [ksplit][n, m] fp32 partial products, added in chunk order by k_gt_finish
};

struct TileRef { int p, i, j, kc; };
__device__ __forceinline__ TileRef find_tile(const GProb* __restrict__ probs, int P, int t) {
  int lo = 0, hi = P - 1;
  while (lo < hi) {   // largest p with tile0 <= t (empty problems share their successor's tile0 and are skipped)
    const int mid = (lo + hi + 1) >> 1;
    if (probs[mid].tile0 <= t) lo = mid; else hi = mid - 1;
  }
  const int local = t - probs[lo].tile0, tn = probs[lo].tiles_n, tm = (probs[lo].n + GT_TM - 1) / GT_TM;
  const int mn = local % (tm * tn);   // K chunks outermost: the chunks of one output tile run on different CTAs
  return {lo, mn / tn, mn % tn, local / (tm * tn)};
}

// the four wgmma of one stage (K = 64 16-bit or 32 TF32 elements) for consumer warpgroup `c`
template <int ET, int TA, int TB>
__device__ __forceinline__ void mma_stage(float (&d)[64], u32 a_base, u32 b_base, int c) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    // K-major: 32 bytes per K step inside the 128-byte swizzle row; MN-major: 16 K rows = 2 KB per step, 64-wide groups
    const u64 da = TA ? make_desc(a_base + c * 8192 + kk * 2048, 8192, 1024) : make_desc(a_base + c * 8192 + kk * 32, 16, 1024);
    const u64 db = TB ? make_desc(b_base + kk * 2048, 8192, 1024) : make_desc(b_base + kk * 32, 16, 1024);
    if constexpr (ET == ET_TF32) wgmma_tf32(d, da, db);
    else wgmma_16<ET == ET_BF16, TA, TB>(d, da, db);
  }
}

// LAYOUT: operand major-ness, per problem at run time (LAY_ANY: grouped_matmul) or fixed for the whole launch (segment
// paths) — a fixed one keeps the wgmma of a stage free of branches, so ptxas does not serialise them
constexpr int LAY_ANY = 0, LAY_FWD = 1, LAY_WGRAD = 2;

template <int ET, int LAYOUT>
__global__ void __launch_bounds__(GT_NT, 1) k_grouped_wgmma(const GProb* __restrict__ probs, int P, const int* __restrict__ total_ptr) {
  constexpr int BK = ET == ET_TF32 ? 32 : 64;   // K elements per stage: one 128-byte swizzle row
  extern __shared__ unsigned char smem_raw[];
  const u32 raw = smem_u32(smem_raw);
  const u32 base = (raw + 1023u) & ~1023u;
  unsigned char* sm = smem_raw + (base - raw);
  const u32 off_out = GT_STAGES * GT_STAGE_BYTES, off_bar = off_out + 2 * GT_OUT_BYTES;
  const u32 bar0 = base + off_bar;
  auto FULL = [&](int s) { return bar0 + 8u * (u32)s; };
  auto EMPTY = [&](int s) { return bar0 + 8u * (u32)(GT_STAGES + s); };
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;

  if (threadIdx.x == 0) {
    for (int s = 0; s < GT_STAGES; ++s) { mbar_init(FULL(s), 1); mbar_init(EMPTY(s), 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int total = *total_ptr;

  if (wg == 0) {
    // ================================ TMA producer ================================
    if (t != 0) return;
    int stage = 0, last_p = -1;
    u32 phase = 0;
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
      const TileRef tr = find_tile(probs, P, tile);
      const GProb& pb = probs[tr.p];
      if (tr.p != last_p) { fence_tensormap(pb.map_a); fence_tensormap(pb.map_b); last_p = tr.p; }
      const int ks0 = tr.kc * pb.ksteps_chunk, ks1 = min((pb.k + BK - 1) / BK, ks0 + pb.ksteps_chunk);
      for (int ks = ks0; ks < ks1; ++ks) {
        mbar_wait(EMPTY(stage), phase ^ 1);
        const u32 a_dst = base + stage * GT_STAGE_BYTES, b_dst = a_dst + GT_A_BYTES, full = FULL(stage);
        const int k0 = ks * BK;
        mbar_expect_tx(full, GT_STAGE_BYTES);   // (boxes partly or wholly out of range still deliver their full size)
        if (!pb.a_mn) {   // box [BK x 128 rows] -> [128][128 B]
          tma_load_2d(a_dst, pb.map_a, k0, pb.a_off + tr.i * GT_TM, full);
        } else {          // two boxes [64 n x 64 k]: MN-major atoms, 8 KB per 64 rows of the tile
          tma_load_2d(a_dst, pb.map_a, tr.i * GT_TM, pb.a_off + k0, full);
          tma_load_2d(a_dst + 8192, pb.map_a, tr.i * GT_TM + 64, pb.a_off + k0, full);
        }
        if (pb.b_k) {     // box [BK x 128 columns] -> [128][128 B]
          tma_load_3d(b_dst, pb.map_b, pb.b_k0 + k0, tr.j * GT_BN, pb.b_z, full);
        } else {          // two boxes [64 columns x 64 k]
          tma_load_3d(b_dst, pb.map_b, tr.j * GT_BN, pb.b_k0 + k0, pb.b_z, full);
          tma_load_3d(b_dst + 8192, pb.map_b, tr.j * GT_BN + 64, pb.b_k0 + k0, pb.b_z, full);
        }
        if (++stage == GT_STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ================================ consumers: wgmma + epilogue ================================
  const int c = wg - 1, warp = t >> 5, lane = t & 31;
  float* stg = reinterpret_cast<float*>(sm + off_out + c * GT_OUT_BYTES);
  int stage = 0;
  u32 phase = 0;
  for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
    const TileRef tr = find_tile(probs, P, tile);
    const GProb& pb = probs[tr.p];
    const int ks0 = tr.kc * pb.ksteps_chunk, ks1 = min((pb.k + BK - 1) / BK, ks0 + pb.ksteps_chunk);
    float d[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = 0.f;
    for (int ks = ks0; ks < ks1; ++ks) {
      mbar_wait(FULL(stage), phase);
      const u32 a_base = base + stage * GT_STAGE_BYTES, b_base = a_base + GT_A_BYTES;
      if (ET != ET_TF32 && pb.zero_ktail && (ks + 1) * BK > pb.k) {
        // rows [valid, 64) of the four [64 k][128 B] boxes (A and B are both MN-major here) belong to the next segment;
        // a row is one 128-byte line whatever the swizzle
        const int valid = pb.k - ks * BK, per_box = (BK - valid) * 8;
        unsigned char* st = sm + stage * GT_STAGE_BYTES;
        for (int q = threadIdx.x - 128; q < 4 * per_box; q += 256) {
          const int box = q / per_box, rem = q - box * per_box;
          *reinterpret_cast<uint4*>(st + box * 8192 + (valid + (rem >> 3)) * 128 + (rem & 7) * 16) = make_uint4(0, 0, 0, 0);
        }
        fence_proxy_async();
        named_bar(1, 256);
      }
      wg_fence();
      if constexpr (ET == ET_TF32) {
        mma_stage<ET, 0, 0>(d, a_base, b_base, c);
      } else if constexpr (LAYOUT == LAY_FWD) {
        mma_stage<ET, 0, 1>(d, a_base, b_base, c);
      } else if constexpr (LAYOUT == LAY_WGRAD) {
        mma_stage<ET, 1, 1>(d, a_base, b_base, c);
      } else {
        if (pb.a_mn) {
          if (pb.b_k) mma_stage<ET, 1, 0>(d, a_base, b_base, c); else mma_stage<ET, 1, 1>(d, a_base, b_base, c);
        } else {
          if (pb.b_k) mma_stage<ET, 0, 0>(d, a_base, b_base, c); else mma_stage<ET, 0, 1>(d, a_base, b_base, c);
        }
      }
      wg_commit();
      wg_wait_all();
      if (t == 0) mbar_arrive(EMPTY(stage));   // this warpgroup's reads of the stage are done
      if (++stage == GT_STAGES) { stage = 0; phase ^= 1; }
    }

    // fragment -> staging: thread holds rows warp*16 + lane/4 (+8), columns 8j + 2(lane%4) (+1)
    named_bar(2 + c, 128);   // the previous tile's stores have finished reading the staging tile
    {
      const int r = warp * 16 + (lane >> 2), col = 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        *reinterpret_cast<float2*>(stg + r * GT_SP + 8 * j + col) = make_float2(d[4 * j], d[4 * j + 1]);
        *reinterpret_cast<float2*>(stg + (r + 8) * GT_SP + 8 * j + col) = make_float2(d[4 * j + 2], d[4 * j + 3]);
      }
    }
    named_bar(2 + c, 128);
    // staging -> global: 16-byte chunks, consecutive threads along a row
    const int col0 = tr.j * GT_BN, cols = min(GT_BN, pb.m - col0);
    const i64 row0 = (i64)tr.i * GT_TM + c * 64;
    const int rows = (int)min((i64)64, (i64)pb.n - row0);
    if (rows <= 0) continue;
    if (pb.part != nullptr || ET == ET_TF32) {
      // fp32 out: a split-K partial (no bias) or the TF32 kernel's result
      const bool partial = pb.part != nullptr;
      float* cb = partial ? pb.part + (i64)tr.kc * pb.n * pb.m : reinterpret_cast<float*>(pb.c);
      const i64 ldc = partial ? (i64)pb.m : pb.ldc;
      const bool vec = partial ? (pb.m & 3) == 0 : pb.c_vec != 0;
      const float* bias = partial ? nullptr : reinterpret_cast<const float*>(pb.bias);
      for (int q = t; q < rows * 32; q += 128) {
        const int r = q >> 5, cc = (q & 31) * 4;
        if (cc >= cols) continue;
        const float4 v4 = *reinterpret_cast<const float4*>(stg + r * GT_SP + cc);
        float e[4] = {v4.x, v4.y, v4.z, v4.w};
        if (bias) {
#pragma unroll
          for (int u = 0; u < 4; ++u) if (cc + u < cols) e[u] += bias[col0 + cc + u];
        }
        float* dst = cb + (row0 + r) * ldc + col0 + cc;
        if (vec && cc + 4 <= cols) {
          *reinterpret_cast<float4*>(dst) = make_float4(e[0], e[1], e[2], e[3]);
        } else {
#pragma unroll
          for (int u = 0; u < 4; ++u) if (cc + u < cols) dst[u] = e[u];
        }
      }
    } else if constexpr (ET != ET_TF32) {
      constexpr bool BF = ET == ET_BF16;
      for (int q = t; q < rows * 16; q += 128) {
        const int r = q >> 4, cc = (q & 15) * 8;
        if (cc >= cols) continue;
        const float4 v0 = *reinterpret_cast<const float4*>(stg + r * GT_SP + cc);
        const float4 v1 = *reinterpret_cast<const float4*>(stg + r * GT_SP + cc + 4);
        float e[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
        if (pb.bias) {
#pragma unroll
          for (int u = 0; u < 8; ++u) if (cc + u < cols) e[u] += ld_bias<BF>(pb.bias, col0 + cc + u);
        }
        unsigned short* dst = reinterpret_cast<unsigned short*>(pb.c) + (row0 + r) * pb.ldc + col0 + cc;
        if (pb.c_vec && cc + 8 <= cols) {
          *reinterpret_cast<uint4*>(dst) = make_uint4(pack2<BF>(e[0], e[1]), pack2<BF>(e[2], e[3]), pack2<BF>(e[4], e[5]), pack2<BF>(e[6], e[7]));
        } else {
#pragma unroll
          for (int u = 0; u < 8; ++u) if (cc + u < cols) dst[u] = (unsigned short)(pack2<BF>(e[u], 0.f) & 0xffffu);
        }
      }
    }
  }
}

// segment mode: problems[b] for segment b (all share map_a / map_b), flat tile prefix (build_segment_list).
//   mode 0 (forward)  C_b = X[ptr_b:ptr_b+1] @ W[b]  (n = len, k = K, m = M); W enters MN-major ([K, M] per segment) or,
//                      for TF32, K-major ([M, K] per segment, b_k = 1)
//   mode 1 (wgrad)    dW[b] = X_b^T @ dY_b          (n = K, k = len, m = M): both operands MN-major, every segment split
//                      into K chunks of `kchunk_steps` stages whose fp32 partials k_gt_finish adds (empty segment: zeros)
__global__ void __launch_bounds__(1024) k_gt_build_segments(GProb* probs, int* total, const i64* __restrict__ ptr, const CUtensorMap* map_a,
                                    const CUtensorMap* map_b, unsigned char* out, const unsigned char* bias, int K, int M, int B,
                                    int c_vec, i64 N, int* err, int mode, int esize, int b_k, float* part, int kchunk_steps) {
  const int tiles_n = (M + GT_BN - 1) / GT_BN, bk = 128 / esize;
  const int tiles_mn = ((K + GT_TM - 1) / GT_TM) * tiles_n;   // wgrad: output tiles of one dW[b]
  build_segment_list<int>(probs, total, ptr, B, N, err, [&](int b, i64 r0, i64 len, GProb& p) {
    memset(&p, 0, sizeof(p));
    p.map_a = map_a; p.map_b = map_b; p.ldc = M; p.m = M; p.a_off = (int)r0; p.tiles_n = tiles_n; p.c_vec = c_vec;
    if (mode == 0) {
      p.c = out + r0 * M * esize; p.bias = bias ? bias + (i64)b * M * esize : nullptr;
      p.n = (int)len; p.k = K; p.b_z = b; p.b_k = b_k;
      p.ksplit = 1; p.ksteps_chunk = (K + bk - 1) / bk;
      return (int)((len + GT_TM - 1) / GT_TM) * tiles_n;
    }
    p.c = out + (i64)b * K * M * esize;
    p.n = K; p.k = (int)len; p.a_mn = 1; p.b_k0 = (int)r0; p.zero_ktail = 1;
    p.ksteps_chunk = kchunk_steps;
    p.ksplit = (int)((len + (i64)kchunk_steps * bk - 1) / ((i64)kchunk_steps * bk));
    return tiles_mn * p.ksplit;
  }, [&](GProb& p) {
    // wgrad: every segment has the same output tile grid, so tile0 / tiles_mn numbers the K chunks of all segments
    // consecutively — chunk c of this segment owns partial buffer tile0 / tiles_mn + c
    if (mode == 1) p.part = part + (i64)(p.tile0 / tiles_mn) * K * M;
  });
}

// split-K epilogue: C = sum over the K chunks' partials, in chunk order (bit-reproducible), rounded to the storage type
template <bool BF16>
__global__ void k_gt_finish(const GProb* __restrict__ probs, int P) {
  for (int b = blockIdx.y; b < P; b += gridDim.y) {
    const GProb pb = probs[b];
    if (pb.part)
      finish_split_problem(reinterpret_cast<unsigned short*>(pb.c), pb.ldc, pb.part, pb.n, pb.m, pb.ksplit,
                           [](float v) { return (unsigned short)(pack2<BF16>(v, 0.f) & 0xffffu); });
  }
}

// W[b] [K, M] -> Wt[b] [M, K] (TF32 wgmma reads both operands K-major)
__global__ void k_transpose_w_f32(const float* __restrict__ w, float* __restrict__ wt, int K, int M) {
  __shared__ float tile[32][33];
  const float* src = w + (size_t)blockIdx.z * K * M;
  float* dst = wt + (size_t)blockIdx.z * K * M;
  const int k0 = blockIdx.y * 32, m0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int k = k0 + i, m = m0 + threadIdx.x;
    tile[i][threadIdx.x] = (k < K && m < M) ? src[(size_t)k * M + m] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int m = m0 + i, k = k0 + threadIdx.x;
    if (m < M && k < K) dst[(size_t)m * K + k] = tile[threadIdx.x][i];
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn gt_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

// innermost dimension contiguous: dims / strides (bytes, for dims 1..) / box, 128-byte swizzle, zero fill
int gt_map(CUtensorMap* m, const void* ptr, int et, int rank, const cuuint64_t* dims, const cuuint64_t* strides, const cuuint32_t* box) {
  EncodeTiledFn enc = gt_encode();
  PYGB_CHECK(enc != nullptr, PYGB200_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint32_t estr[3] = {1, 1, 1};
  const CUtensorMapDataType dt = et == ET_TF32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                 : et == ET_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const CUresult r = enc(m, dt, (cuuint32_t)rank, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with code " + std::to_string((int)r));
    return PYGB200_ERR_CUDA;
  }
  return PYGB200_OK;
}

constexpr size_t GT_SMEM = 1024 + (size_t)GT_STAGES * GT_STAGE_BYTES + 2 * (size_t)GT_OUT_BYTES + 2 * GT_STAGES * 8;

template <int ET, int LAYOUT>
int gt_launch_et(const GProb* probs, int P, const int* total, int grid, cudaStream_t st) {
  PYGB_CUDA(cudaFuncSetAttribute(k_grouped_wgmma<ET, LAYOUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GT_SMEM));
  k_grouped_wgmma<ET, LAYOUT><<<grid, GT_NT, GT_SMEM, st>>>(probs, P, total);
  return PYGB200_OK;
}

template <int LAYOUT>
int gt_launch_16(const GProb* probs, int P, const int* total, int grid, bool bf16, cudaStream_t st) {
  return bf16 ? gt_launch_et<ET_BF16, LAYOUT>(probs, P, total, grid, st) : gt_launch_et<ET_F16, LAYOUT>(probs, P, total, grid, st);
}

int gt_launch(const GProb* probs, int P, const int* total, i64 tiles_bound, int et, int layout, const char* name, cudaStream_t st) {
  const int grid = (int)std::max<i64>(1, std::min<i64>(tiles_bound, num_sms()));
  void* tk = prof_begin(st);
  const bool bf16 = et == ET_BF16;
  const int rc = et == ET_TF32 ? gt_launch_et<ET_TF32, LAY_FWD>(probs, P, total, grid, st)
                 : layout == LAY_FWD ? gt_launch_16<LAY_FWD>(probs, P, total, grid, bf16, st)
                 : layout == LAY_WGRAD ? gt_launch_16<LAY_WGRAD>(probs, P, total, grid, bf16, st)
                                       : gt_launch_16<LAY_ANY>(probs, P, total, grid, bf16, st);
  if (rc != PYGB200_OK) return rc;
  prof_end(tk, name, st, tiles_bound);
  PYGB_LAUNCH_CHECK();
  return PYGB200_OK;
}

int finish_launch(const GProb* probs, int P, bool bf16, cudaStream_t st) {
  const dim3 grid(64, (unsigned)std::min(P, 4096));
  if (bf16) k_gt_finish<true><<<grid, 256, 0, st>>>(probs, P);
  else k_gt_finish<false><<<grid, 256, 0, st>>>(probs, P);
  PYGB_LAUNCH_CHECK();
  return PYGB200_OK;
}

inline bool al16(const void* p) { return ((uintptr_t)p & 15) == 0; }

// Segment-mode launch shared by the three segment paths: upload the two tensor maps, build the problem list from `ptr`
// on the device, run the GEMM (and, for the weight gradient, the ordered sum of the K chunks).
int segment_run(const CUtensorMap (&hm)[2], const i64* ptr_dev, void* out, const void* bias, i64 N, i64 K, i64 M, i64 B, int et,
                int mode, int c_vec, int b_k, int kchunk_steps, size_t part_bytes, i64 tiles_bound, cudaStream_t st) {
  const size_t prob_off = 256, total_off = prob_off + (((size_t)B * sizeof(GProb) + 15) & ~(size_t)15);
  const size_t part_off = (total_off + 16 + 255) & ~(size_t)255;
  AsyncScratch sc;   // (freed on every return path)
  if (int e = sc.alloc(part_off + part_bytes, st)) return e;
  unsigned char* dbuf = (unsigned char*)sc.p;
  PYGB_CUDA(cudaMemcpyAsync(dbuf, hm, sizeof(hm), cudaMemcpyHostToDevice, st));
  const CUtensorMap* dm = reinterpret_cast<const CUtensorMap*>(dbuf);
  GProb* probs = reinterpret_cast<GProb*>(dbuf + prob_off);
  int* total = reinterpret_cast<int*>(dbuf + total_off);
  k_gt_build_segments<<<1, 1024, 0, st>>>(probs, total, ptr_dev, dm, dm + 1, reinterpret_cast<unsigned char*>(out),
                                          reinterpret_cast<const unsigned char*>(bias), (int)K, (int)M, (int)B, c_vec, N,
                                          async_error_flag_dev(ASYNC_ERR_MATMUL), mode, et == ET_TF32 ? 4 : 2, b_k,
                                          reinterpret_cast<float*>(dbuf + part_off), kchunk_steps);
  PYGB_LAUNCH_CHECK();
  if (int e = gt_launch(probs, (int)B, total, tiles_bound, et, mode == 0 ? LAY_FWD : LAY_WGRAD, "segment_matmul", st)) return e;
  if (mode == 1) return finish_launch(probs, (int)B, et == ET_BF16, st);
  return PYGB200_OK;
}

}  // namespace

// ---- pyg::grouped_matmul: can every problem go through the tensor cores?  (TMA: 16-byte aligned bases and row pitches)
bool grouped_tc_supported(const pygb200_gemm_problem* ps, i64 count, int dtype) {
  if (dtype != PYGB200_BF16 && dtype != PYGB200_F16) return false;
  if (count < 1 || count > 65536) return false;
  i64 tiles = 0;
  for (i64 i = 0; i < count; ++i) {
    const auto& q = ps[i];
    if (q.n == 0 || q.m == 0) continue;
    if (q.n >= ((i64)1 << 31) || q.k >= ((i64)1 << 31) || q.m >= ((i64)1 << 31)) return false;
    if (q.k == 0) continue;   // empty contraction: the output is zeroed by a memset, no tile is scheduled
    if (!al16(q.a) || !al16(q.b) || q.lda % 8 != 0 || q.ldb % 8 != 0) return false;
    // the extent along the contiguous dimension must fit the pitch
    if (q.lda < (q.a_colmajor ? q.n : q.k) || q.ldb < (q.b_colmajor ? q.k : q.m) || q.ldc < q.m) return false;
    tiles += ((q.n + GT_TM - 1) / GT_TM) * ((q.m + GT_BN - 1) / GT_BN);
  }
  return tiles > 0 && tiles < ((i64)1 << 31);
}

int grouped_matmul_tc(const pygb200_gemm_problem* ps, i64 count, int dtype, cudaStream_t st) {
  const int et = et_of(dtype);
  const int sms = num_sms();
  // Split-K plan: a weight-gradient-shaped list (few output tiles, very long K: dW = X^T dY of a HeteroDictLinear) would
  // keep a handful of CTAs busy for thousands of K steps.  When the output tiles do not fill the machine twice, every
  // problem's K steps are cut into chunks (>= 8 steps = 512 of K each) that become work items of their own; chunk c
  // stores an fp32 partial and k_gt_finish adds the partials in order.  256 MB of partials at most.
  i64 base_tiles = 0;
  for (i64 i = 0; i < count; ++i)
    if (ps[i].n > 0 && ps[i].m > 0 && ps[i].k > 0) base_tiles += ((ps[i].n + GT_TM - 1) / GT_TM) * ((ps[i].m + GT_BN - 1) / GT_BN);
  const i64 want = base_tiles > 0 && base_tiles < 2 * (i64)sms ? (2 * (i64)sms + base_tiles - 1) / base_tiles : 1;
  std::vector<int> ksplit((size_t)count, 1);
  size_t part_bytes = 0;
  for (i64 i = 0; i < count && want > 1; ++i) {
    const auto& q = ps[i];
    if (q.n <= 0 || q.m <= 0 || q.k <= 0) continue;
    const i64 ksteps = (q.k + 63) / 64;
    const i64 sp = std::max<i64>(1, std::min<i64>(want, ksteps / 8));
    const size_t bytes = (size_t)sp * q.n * q.m * 4;
    if (sp > 1 && part_bytes + bytes <= ((size_t)256 << 20)) { ksplit[(size_t)i] = (int)sp; part_bytes += (bytes + 255) & ~(size_t)255; }
  }
  // one upload: [tensor maps: 2 per problem | problem list | tile total]; partials behind it
  const size_t map_bytes = (size_t)count * 2 * sizeof(CUtensorMap);
  const size_t prob_off = (map_bytes + 255) & ~(size_t)255, total_off = prob_off + (((size_t)count * sizeof(GProb) + 15) & ~(size_t)15);
  const size_t part_off = (total_off + 16 + 255) & ~(size_t)255;
  std::vector<unsigned char> h(total_off + 16, 0);
  AsyncScratch sc;   // (freed on every return path)
  if (int e = sc.alloc(part_off + part_bytes, st)) return e;
  unsigned char* dbuf = (unsigned char*)sc.p;
  CUtensorMap* hmaps = reinterpret_cast<CUtensorMap*>(h.data());
  GProb* hp = reinterpret_cast<GProb*>(h.data() + prob_off);
  const CUtensorMap* dmaps = reinterpret_cast<const CUtensorMap*>(dbuf);
  i64 tiles = 0;
  size_t part_used = 0;
  bool any_split = false;
  int rc = PYGB200_OK;
  for (i64 i = 0; i < count && rc == PYGB200_OK; ++i) {
    const auto& q = ps[i];
    GProb p;
    memset(&p, 0, sizeof(p));
    p.tile0 = (int)tiles; p.tiles_n = 1; p.ksplit = 1; p.ksteps_chunk = 1;
    p.n = (int)q.n; p.k = (int)q.k; p.m = (int)q.m;
    if (q.n > 0 && q.m > 0 && q.k == 0) {   // empty contraction: zeros
      if (cudaMemset2DAsync(q.c, (size_t)q.ldc * 2, 0, (size_t)q.m * 2, (size_t)q.n, st) != cudaSuccess) rc = PYGB200_ERR_CUDA;
    } else if (q.n > 0 && q.m > 0) {
      CUtensorMap ma, mb;
      cuuint64_t d[3], s[2]; cuuint32_t box[3];
      if (!q.a_colmajor) { d[0] = (cuuint64_t)q.k; d[1] = (cuuint64_t)q.n; box[0] = 64; box[1] = GT_TM; }
      else { d[0] = (cuuint64_t)q.n; d[1] = (cuuint64_t)q.k; box[0] = 64; box[1] = 64; }
      s[0] = (cuuint64_t)q.lda * 2;
      rc = gt_map(&ma, q.a, et, 2, d, s, box);
      if (rc != PYGB200_OK) break;
      if (!q.b_colmajor) { d[0] = (cuuint64_t)q.m; d[1] = (cuuint64_t)q.k; box[1] = 64; }
      else { d[0] = (cuuint64_t)q.k; d[1] = (cuuint64_t)q.m; box[1] = GT_BN; }
      d[2] = 1; s[0] = (cuuint64_t)q.ldb * 2; s[1] = s[0] * d[1]; box[0] = 64; box[2] = 1;
      rc = gt_map(&mb, q.b, et, 3, d, s, box);
      if (rc != PYGB200_OK) break;
      hmaps[2 * i] = ma; hmaps[2 * i + 1] = mb;
      p.map_a = dmaps + 2 * i; p.map_b = dmaps + 2 * i + 1;
      p.c = reinterpret_cast<unsigned char*>(q.c); p.bias = nullptr; p.ldc = q.ldc;
      p.a_mn = q.a_colmajor ? 1 : 0; p.b_k = q.b_colmajor ? 1 : 0;
      p.c_vec = (al16(q.c) && q.ldc % 8 == 0) ? 1 : 0;
      p.tiles_n = (int)((q.m + GT_BN - 1) / GT_BN);
      const int ksteps = (int)((q.k + 63) / 64);
      p.ksplit = ksplit[(size_t)i];
      p.ksteps_chunk = (ksteps + p.ksplit - 1) / p.ksplit;
      p.ksplit = (ksteps + p.ksteps_chunk - 1) / p.ksteps_chunk;   // (no empty chunk)
      if (p.ksplit > 1) {
        p.part = reinterpret_cast<float*>(dbuf + part_off + part_used);
        part_used += ((size_t)p.ksplit * q.n * q.m * 4 + 255) & ~(size_t)255;
        any_split = true;
      }
      tiles += ((q.n + GT_TM - 1) / GT_TM) * p.tiles_n * p.ksplit;
    }
    hp[i] = p;
  }
  if (rc == PYGB200_OK && tiles > 0) {
    *reinterpret_cast<int*>(h.data() + total_off) = (int)tiles;
    // pageable source: the copy is staged by the driver before the call returns, so `h` may die at the end of the scope
    if (cudaMemcpyAsync(dbuf, h.data(), h.size(), cudaMemcpyHostToDevice, st) != cudaSuccess) rc = PYGB200_ERR_CUDA;
    const GProb* dprobs = reinterpret_cast<const GProb*>(dbuf + prob_off);
    if (rc == PYGB200_OK) rc = gt_launch(dprobs, (int)count, reinterpret_cast<const int*>(dbuf + total_off), tiles, et, LAY_ANY, "grouped_gemm", st);
    if (rc == PYGB200_OK && any_split) rc = finish_launch(dprobs, (int)count, et == ET_BF16, st);
  }
  return rc;
}

// ---- pyg::segment_matmul, bf16 / fp16
bool segment_tc_supported(i64 N, i64 K, i64 M, i64 B, int dtype, const void* x, const void* w, const void* out) {
  if (dtype != PYGB200_BF16 && dtype != PYGB200_F16) return false;
  if (K < 1 || M < 1 || K % 8 != 0 || M % 8 != 0) return false;
  if (B < 1 || N < 1 || N >= ((i64)1 << 31) || B >= ((i64)1 << 24) || K >= ((i64)1 << 31) || M >= ((i64)1 << 31)) return false;
  if ((N / GT_TM + B) * ((M + GT_BN - 1) / GT_BN) >= ((i64)1 << 31)) return false;
  return al16(x) && al16(w) && al16(out);
}

int segment_matmul_tc(const void* x, const i64* ptr_dev, const void* w, const void* bias, void* out, i64 N, i64 K, i64 M, i64 B,
                      int dtype, cudaStream_t st) {
  const int et = et_of(dtype);
  CUtensorMap hm[2];
  cuuint64_t d[3] = {(cuuint64_t)K, (cuuint64_t)N, 1}, s[2] = {(cuuint64_t)K * 2, 0};
  cuuint32_t box[3] = {64, GT_TM, 1};
  if (int e = gt_map(&hm[0], x, et, 2, d, s, box)) return e;
  cuuint64_t dw[3] = {(cuuint64_t)M, (cuuint64_t)K, (cuuint64_t)B}, sw[2] = {(cuuint64_t)M * 2, (cuuint64_t)K * M * 2};
  cuuint32_t bw[3] = {64, 64, 1};
  if (int e = gt_map(&hm[1], w, et, 3, dw, sw, bw)) return e;
  // rows of out are M * 2 bytes apart and M % 8 == 0: 16-byte aligned
  return segment_run(hm, ptr_dev, out, bias, N, K, M, B, et, 0, 1, 0, 0, 0, (N / GT_TM + B) * ((M + GT_BN - 1) / GT_BN), st);
}

// ---- pyg::segment_matmul, fp32 storage with TF32 math (taken when the caller allows TF32:
// torch.get_float32_matmul_precision() != 'highest', like the reference's TensorOp kernel, matmul_kernel.cu:159-190).
// TF32 wgmma reads both operands K-major, so W is transposed once per call into a [B, M, K] scratch.
bool tf32_supported(i64 N, i64 K, i64 M, i64 B, const void* x, const void* w, const void* out) {
  if (K < 64 || K > 256 || K % 64 != 0) return false;
  if (M < 32 || M > 256 || M % 32 != 0) return false;
  if (B < 1 || B > MAX_SEG || N < 1 || N >= ((i64)1 << 31) || B * K >= ((i64)1 << 31)) return false;
  return al16(x) && al16(w) && al16(out);
}

int segment_matmul_tf32(const void* x, const i64* ptr_dev, const void* w, const void* bias, void* out, i64 N, i64 K, i64 M, i64 B,
                        cudaStream_t st) {
  AsyncScratch sc;   // (freed on every return path)
  if (int e = sc.alloc((size_t)B * K * M * 4, st)) return e;
  float* wt = (float*)sc.p;
  k_transpose_w_f32<<<dim3((unsigned)((M + 31) / 32), (unsigned)((K + 31) / 32), (unsigned)B), dim3(32, 8), 0, st>>>(
      (const float*)w, wt, (int)K, (int)M);
  PYGB_LAUNCH_CHECK();
  CUtensorMap hm[2];
  cuuint64_t d[3] = {(cuuint64_t)K, (cuuint64_t)N, 1}, s[2] = {(cuuint64_t)K * 4, 0};
  cuuint32_t box[3] = {32, GT_TM, 1};
  if (int e = gt_map(&hm[0], x, ET_TF32, 2, d, s, box)) return e;
  cuuint64_t dw[3] = {(cuuint64_t)K, (cuuint64_t)M, (cuuint64_t)B}, sw[2] = {(cuuint64_t)K * 4, (cuuint64_t)K * M * 4};
  cuuint32_t bw[3] = {32, GT_BN, 1};
  if (int e = gt_map(&hm[1], wt, ET_TF32, 3, dw, sw, bw)) return e;
  return segment_run(hm, ptr_dev, out, bias, N, K, M, B, ET_TF32, 0, 1, 1, 0, 0, (N / GT_TM + B) * ((M + GT_BN - 1) / GT_BN), st);
}

// ---- weight gradient dW[b] = X_b^T @ dY_b, bf16 / fp16 (replaces the B torch::matmul calls + at::stack of
// SegmentMatmul::backward, pyg_lib/csrc/ops/autograd/matmul_kernel.cpp:92-107; deterministic like them)
bool wgrad_tc_supported(i64 N, i64 K, i64 M, i64 B, int dtype, const void* x, const void* dy, const void* dw) {
  if (dtype != PYGB200_BF16 && dtype != PYGB200_F16) return false;
  if (K != 128) return false;
  if (M < 64 || M > 256 || M % 64 != 0) return false;
  if (B < 1 || B > MAX_SEG || N < 1 || N >= ((i64)1 << 31)) return false;
  return al16(x) && al16(dy) && al16(dw);
}

int segment_wgrad_tc(const void* x, const i64* ptr_dev, const void* dy, void* dw, i64 N, i64 K, i64 M, i64 B, int dtype,
                     cudaStream_t st) {
  const int et = et_of(dtype);
  CUtensorMap hm[2];
  cuuint64_t d[3] = {(cuuint64_t)K, (cuuint64_t)N, 1}, s[2] = {(cuuint64_t)K * 2, 0};
  cuuint32_t box[3] = {64, 64, 1};   // MN-major A = X^T: box [64 columns of X x 64 rows]
  if (int e = gt_map(&hm[0], x, et, 2, d, s, box)) return e;
  cuuint64_t dd[3] = {(cuuint64_t)M, (cuuint64_t)N, 1}, sd[2] = {(cuuint64_t)M * 2, (cuuint64_t)N * M * 2};
  if (int e = gt_map(&hm[1], dy, et, 3, dd, sd, box)) return e;
  // K chunks of 2048 rows (32 stages) at least; longer when the partials of (N / chunk + B) chunks would pass 256 MB
  const i64 km_bytes = K * M * 4, slots = ((i64)256 << 20) / km_bytes;
  i64 chunk = 2048;
  if (slots > B + 1) chunk = std::max<i64>(chunk, ceil_div(N, slots - B - 1));
  else chunk = std::max<i64>(N, 64);
  chunk = ceil_div(chunk, (i64)64) * 64;
  const i64 chunks = ceil_div(N, chunk) + B;
  const i64 tiles_mn = ceil_div(K, (i64)GT_TM) * ceil_div(M, (i64)GT_BN);
  return segment_run(hm, ptr_dev, dw, nullptr, N, K, M, B, et, 1, 1, 0, (int)(chunk / 64), (size_t)chunks * km_bytes,
                     chunks * tiles_mn, st);
}

}  // namespace pygb200
