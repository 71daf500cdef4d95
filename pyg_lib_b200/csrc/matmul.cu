// pyg_lib_b200/csrc/matmul.cu — segment_matmul / grouped_matmul entry points of the C ABI and the
// general (any shape, any stride, fp32-exact) grouped GEMM they fall back to.
//
// Replaces pyg_lib/csrc/ops/cuda/matmul_kernel.cu (CUTLASS 2.x sm80 GemmGrouped, fp32 only):
//   * problems are described ON THE DEVICE (built from `ptr` by a tiny kernel), so a device-resident
//     `ptr` needs no D2H sync (the reference does size_from_ptr(ptr).cpu(), matmul_kernel.cu:307);
//   * one launch walks a flat work list over all problems: (128x128 output tile) x (K chunk); ragged
//     segments load-balance by tiles, and long reductions (the weight gradient dW[b] = X_b^T dY_b, whose
//     K is the segment length) are split over K chunks whose fp32 partials k_finish_split adds in chunk order;
//   * bf16 / fp16 / fp32 storage with fp32 FMA accumulation; optional fused bias.
// The tensor-core paths (bf16 / fp16, TF32, and the weight gradient for TMA-aligned shapes) live in
// matmul_grouped_tc.cu; this file is the path for fp32 ('highest' precision == the reference's SIMT kernels,
// matmul_kernel.cu:227-282) and for shapes or strides TMA cannot read.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <vector>

#include "matmul_common.cuh"

namespace pygb200 {

// matmul_grouped_tc.cu: the Hopper tensor-core (wgmma) grouped GEMM behind every bf16 / fp16 / TF32 path
bool segment_tc_supported(i64 N, i64 K, i64 M, i64 B, int dtype, const void* x, const void* w, const void* out);
int segment_matmul_tc(const void* x, const i64* ptr_dev, const void* w, const void* bias, void* out, i64 N, i64 K, i64 M, i64 B,
                      int dtype, cudaStream_t st);
bool tf32_supported(i64 N, i64 K, i64 M, i64 B, const void* x, const void* w, const void* out);
int segment_matmul_tf32(const void* x, const i64* ptr_dev, const void* w, const void* bias, void* out, i64 N, i64 K, i64 M,
                        i64 B, cudaStream_t st);
bool wgrad_tc_supported(i64 N, i64 K, i64 M, i64 B, int dtype, const void* x, const void* dy, const void* dw);
int segment_wgrad_tc(const void* x, const i64* ptr_dev, const void* dy, void* dw, i64 N, i64 K, i64 M, i64 B, int dtype,
                     cudaStream_t st);
bool grouped_tc_supported(const pygb200_gemm_problem* ps, i64 count, int dtype);
int grouped_matmul_tc(const pygb200_gemm_problem* ps, i64 count, int dtype, cudaStream_t st);

// "invalid ptr" flag of the segment kernels: one int in pinned, mapped, portable host memory.  The kernels validate
// `ptr` while they read it (ptr[0] == 0, non-decreasing, ptr[B] == N — what the reference's split_with_sizes checks on
// the host after its D2H copy, matmul_kernel.cu:307) and raise the flag instead of touching memory; the NEXT matmul
// call on this process reports it (like CUDA's own asynchronous errors), so a device-resident ptr still costs no sync.
// random_walk.cu raises its own slot of the same allocation for node indices outside the graph.
static int* g_mm_err_host = nullptr;
static int* g_mm_err_dev = nullptr;
int* async_error_flag_dev(int slot) {
  static bool tried = false;
  if (!tried) {
    tried = true;
    if (cudaHostAlloc((void**)&g_mm_err_host, ASYNC_ERR_SLOTS * sizeof(int), cudaHostAllocMapped | cudaHostAllocPortable) == cudaSuccess) {
      for (int s = 0; s < ASYNC_ERR_SLOTS; ++s) g_mm_err_host[s] = 0;
      if (cudaHostGetDevicePointer((void**)&g_mm_err_dev, g_mm_err_host, 0) != cudaSuccess) g_mm_err_dev = nullptr;
    }
  }
  return g_mm_err_dev ? g_mm_err_dev + slot : nullptr;
}
bool take_async_error(int slot) {
  if (g_mm_err_host && reinterpret_cast<volatile int*>(g_mm_err_host)[slot]) { g_mm_err_host[slot] = 0; return true; }
  return false;
}

namespace {

struct Problem {       // C[n,m] = A[n,k] @ B[k,m] (+ bias[m]);  element strides
  const void* a; const void* b; void* c; const void* bias;
  float* acc;          // non-null: this problem is split over K; K chunk c stores its partial product to acc + c*n*m
                       // ([n,m] fp32 each, ld = m) and k_finish_split adds the chunks in order (deterministic, no atomics)
  i64 n, k, m;
  i64 sa0, sa1, sb0, sb1, ldc;
  i64 kchunk;          // K extent of one work item (== k when not split)
  i64 tile0;           // index of this problem's first work item in the flat list
};

constexpr int BM = 128, BN = 128, BK = 16, MM_NT = 256;
constexpr i64 WGRAD_KCHUNK = 2048;   // rows of a segment reduced by one work item of the weight gradient

template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_f<__half>(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }

__host__ __device__ inline i64 work_items(i64 n, i64 m, i64 k, i64 kchunk) {
  if (n <= 0 || m <= 0) return 0;
  const i64 kc = (k <= 0) ? 1 : ceil_div(k, kchunk);   // k == 0 still needs one item to store zeros / bias
  return ceil_div(n, (i64)BM) * ceil_div(m, (i64)BN) * kc;
}

// problems[b] for segment b of a segment_matmul, and the flat work-item prefix (build_segment_list).
//   mode 0: forward   C_b = X[ptr_b:ptr_b+1] @ W[b]            (n=len, k=K, m=M)
//   mode 1: wgrad     dW[b] = X_b^T @ dY_b                      (n=K, k=len, m=M), split over K chunks
__global__ void __launch_bounds__(1024) k_build_segments(Problem* probs, i64* total_tiles, const i64* __restrict__ ptr, const char* x,
                                 const char* w, const char* bias, char* out, float* acc, i64 K, i64 M, i64 B, int esize,
                                 int mode, i64 N, int* err, i64 wgrad_kchunk) {
  const i64 tiles_mn = ceil_div(K, (i64)BM) * ceil_div(M, (i64)BN);   // wgrad: output tiles of one dW[b]
  build_segment_list<i64>(probs, total_tiles, ptr, B, N, err, [&](i64 b, i64 r0, i64 len, Problem& p) {
    if (mode == 0) {
      p.a = x + r0 * K * esize; p.b = w + b * K * M * esize; p.c = out + r0 * M * esize;
      p.bias = bias ? bias + b * M * esize : nullptr; p.acc = nullptr;
      p.n = len; p.k = K; p.m = M; p.sa0 = K; p.sa1 = 1; p.sb0 = M; p.sb1 = 1; p.ldc = M; p.kchunk = K > 0 ? K : 1;
    } else {
      p.a = x + r0 * K * esize; p.b = w + r0 * M * esize; p.c = out + b * K * M * esize; p.bias = nullptr;
      p.n = K; p.k = len; p.m = M; p.sa0 = 1; p.sa1 = K; p.sb0 = M; p.sb1 = 1; p.ldc = M;
      p.kchunk = wgrad_kchunk;
      p.acc = (acc != nullptr && len > wgrad_kchunk) ? acc : nullptr;   // (offset past earlier segments' chunks below)
      if (p.acc == nullptr) p.kchunk = len > 0 ? len : 1;   // short segment: one item, direct store
    }
    return work_items(p.n, p.m, p.k, p.kchunk);
  }, [&](Problem& p) {
    // weight gradient: every segment has the same K x M tile grid, so tile0 / tiles_mn numbers the K chunks of all
    // segments consecutively — chunk c of this segment owns the partial buffer tile0 / tiles_mn + c
    if (p.acc) p.acc += (p.tile0 / tiles_mn) * K * M;
  });
}

// Generic grouped GEMM.  Work item = (problem, 128x128 output tile, K chunk), taken grid-stride from the
// flat list; 256 threads, 8x8 register micro-tile (two 4-wide strips per dimension, 64 apart, so shared
// memory reads are 128-bit and conflict-free), BK = 16, next K step prefetched into registers while the
// current one is multiplied.  Loads are scalar with arbitrary element strides; the thread->element
// mapping follows the operand's contiguous dimension so that they coalesce.
template <typename T>
__global__ void __launch_bounds__(MM_NT) k_grouped_gemm(const Problem* __restrict__ probs, i64 P,
                                                         const i64* __restrict__ total_tiles_ptr) {
  __shared__ __align__(16) float sA[BK][BM + 4];   // +4: the transposed stores of a K-fastest A tile spread over banks
  __shared__ __align__(16) float sB[BK][BN];
  const i64 total = *total_tiles_ptr;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;  // 16 x 16 threads
  for (i64 tile = blockIdx.x; tile < total; tile += gridDim.x) {
    i64 lo = 0, hi = P - 1;
    while (lo < hi) {  // last problem with tile0 <= tile (skipping empty problems, which share tile0)
      const i64 mid = (lo + hi + 1) >> 1;
      if (probs[mid].tile0 <= tile) lo = mid; else hi = mid - 1;
    }
    const Problem& p = probs[lo];
    const i64 pn = p.n, pm = p.m, pk = p.k;
    const i64 tn = ceil_div(pm, (i64)BN), tmn = ceil_div(pn, (i64)BM) * tn;
    const i64 lt = tile - p.tile0;
    const i64 kc = lt / tmn, mn = lt % tmn;
    const i64 row0 = (mn / tn) * BM, col0 = (mn % tn) * BN;
    const i64 kbeg = kc * p.kchunk, kend = (kbeg + p.kchunk < pk) ? kbeg + p.kchunk : pk;
    // Per-thread load pattern: 8 elements of each operand tile per K step, element q at (r + q*dr, k + q*dk).
    // The mapping walks the operand's contiguous dimension with consecutive threads (coalesced).
    int a_r, a_k, a_dr, a_dk, b_c, b_k, b_dc, b_dk;
    if (p.sa1 == 1) { a_k = threadIdx.x & 15; a_r = threadIdx.x >> 4; a_dr = 16; a_dk = 0; }
    else            { a_r = threadIdx.x & 127; a_k = threadIdx.x >> 7; a_dr = 0; a_dk = 2; }
    if (p.sb1 == 1) { b_c = threadIdx.x & 127; b_k = threadIdx.x >> 7; b_dc = 0; b_dk = 2; }
    else            { b_k = threadIdx.x & 15; b_c = threadIdx.x >> 4; b_dc = 16; b_dk = 0; }
    const T* pa = (const T*)p.a + (row0 + a_r) * p.sa0 + (kbeg + a_k) * p.sa1;
    const T* pb = (const T*)p.b + (kbeg + b_k) * p.sb0 + (col0 + b_c) * p.sb1;
    const i64 a_q = a_dr * p.sa0 + a_dk * p.sa1, b_q = b_dk * p.sb0 + b_dc * p.sb1;
    const i64 a_adv = (i64)BK * p.sa1, b_adv = (i64)BK * p.sb0;
    unsigned a_ok = 0, b_ok = 0;   // bit q: row / column of element q is inside the matrix
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      a_ok |= (row0 + a_r + q * a_dr < pn ? 1u : 0u) << q;
      b_ok |= (col0 + b_c + q * b_dc < pm ? 1u : 0u) << q;
    }
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    float ra[8], rb[8];
    auto gload = [&](i64 k0) {
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        ra[q] = ((a_ok >> q) & 1u) && (k0 + a_k + q * a_dk < kend) ? to_f<T>(pa[q * a_q]) : 0.f;
        rb[q] = ((b_ok >> q) & 1u) && (k0 + b_k + q * b_dk < kend) ? to_f<T>(pb[q * b_q]) : 0.f;
      }
      pa += a_adv; pb += b_adv;
    };
    if (kbeg < kend) gload(kbeg);
    for (i64 k0 = kbeg; k0 < kend; k0 += BK) {
      __syncthreads();   // previous step's reads of sA/sB are done
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        sA[a_k + q * a_dk][a_r + q * a_dr] = ra[q];
        sB[b_k + q * b_dk][b_c + q * b_dc] = rb[q];
      }
      __syncthreads();
      if (k0 + BK < kend) gload(k0 + BK);   // in flight while we multiply
#pragma unroll
      for (int kk = 0; kk < BK; ++kk) {
        const float4 a0 = *reinterpret_cast<const float4*>(&sA[kk][ty * 4]);
        const float4 a1 = *reinterpret_cast<const float4*>(&sA[kk][64 + ty * 4]);
        const float4 b0 = *reinterpret_cast<const float4*>(&sB[kk][tx * 4]);
        const float4 b1 = *reinterpret_cast<const float4*>(&sB[kk][64 + tx * 4]);
        const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
    }
    __syncthreads();
    T* __restrict__ C = (T*)p.c;
    const T* __restrict__ bias = (const T*)p.bias;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const i64 gr = row0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
      if (gr >= pn) continue;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const i64 gc = col0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
        if (gc >= pm) continue;
        if (p.acc) {
          p.acc[(kc * pn + gr) * p.m + gc] = acc[i][j];
        } else {
          float v = acc[i][j];
          if (bias) v += to_f<T>(bias[gc]);
          C[gr * p.ldc + gc] = from_f<T>(v);
        }
      }
    }
  }
}

// split-K epilogue: fp32 accumulators -> storage dtype
template <typename T>
__global__ void k_finish_split(const Problem* __restrict__ probs, i64 P) {
  for (i64 b = blockIdx.y; b < P; b += gridDim.y) {
    const Problem p = probs[b];
    if (p.acc) finish_split_problem((T*)p.c, p.ldc, p.acc, p.n, p.m, ceil_div(p.k, p.kchunk), [](float v) { return from_f<T>(v); });
  }
}

int launch_grouped(const Problem* probs_dev, i64 P, const i64* total_dev, i64 tiles_bound, int dtype, cudaStream_t st) {
  const int sms = num_sms();
  i64 g = tiles_bound < 1 ? 1 : tiles_bound;
  if (g > (i64)sms * 2) g = (i64)sms * 2;   // 2 CTAs of 256 threads x ~128 registers per SM
  void* tk = prof_begin(st);
  switch (dtype) {
    case PYGB200_F32: k_grouped_gemm<float><<<(int)g, MM_NT, 0, st>>>(probs_dev, P, total_dev); break;
    case PYGB200_BF16: k_grouped_gemm<__nv_bfloat16><<<(int)g, MM_NT, 0, st>>>(probs_dev, P, total_dev); break;
    case PYGB200_F16: k_grouped_gemm<__half><<<(int)g, MM_NT, 0, st>>>(probs_dev, P, total_dev); break;
    default: set_error("matmul: unknown dtype"); return PYGB200_ERR_ARG;
  }
  prof_end(tk, "grouped_gemm", st, tiles_bound);
  PYGB_LAUNCH_CHECK();
  return PYGB200_OK;
}

inline int esize_of(int dtype) { return dtype == PYGB200_F32 ? 4 : 2; }

int segment_generic(const void* x, const i64* ptr_dev, const void* w, const void* bias, void* out, i64 N, i64 K, i64 M,
                    i64 B, int dtype, int mode, cudaStream_t st) {
  if (B == 0) return PYGB200_OK;
  const size_t prob_bytes = (((size_t)B * sizeof(Problem) + 16) + 255) & ~(size_t)255;
  // weight gradient: one fp32 partial [K, M] per K chunk of every split segment (<= N / kchunk + B of them), added up in
  // order afterwards.  The chunk grows until the partials fit 256 MB; if even B of them do not, segments are not split.
  i64 kchunk = WGRAD_KCHUNK;
  bool split = mode == 1 && N > WGRAD_KCHUNK;
  if (split) {
    const i64 slots = ((i64)256 << 20) / std::max<i64>(K * M * 4, 1);
    if (slots < 2 * B + 2) split = false;
    else kchunk = std::max<i64>(WGRAD_KCHUNK, ceil_div(N, slots - B - 1));
  }
  if (!split) kchunk = std::max<i64>(N, 1);
  const size_t acc_bytes = split ? (size_t)(ceil_div(N, kchunk) + B + 1) * K * M * sizeof(float) : 0;
  AsyncScratch sc;   // (freed on every return path)
  if (int e = sc.alloc(prob_bytes + acc_bytes, st)) return e;
  char* scratch = (char*)sc.p;
  Problem* probs = (Problem*)(scratch + 16);
  i64* total = (i64*)scratch;
  float* acc = split ? (float*)(scratch + prob_bytes) : nullptr;
  k_build_segments<<<1, 1024, 0, st>>>(probs, total, ptr_dev, (const char*)x, (const char*)w, (const char*)bias,
                                       (char*)out, acc, K, M, B, esize_of(dtype), mode, N, async_error_flag_dev(ASYNC_ERR_MATMUL), kchunk);
  PYGB_LAUNCH_CHECK();
  const i64 bound = mode == 0 ? (ceil_div(N, (i64)BM) + B) * ceil_div(M, (i64)BN)
                              : (ceil_div(N, kchunk) + B) * ceil_div(K, (i64)BM) * ceil_div(M, (i64)BN);
  int rc = launch_grouped(probs, B, total, bound, dtype, st);
  if (rc == PYGB200_OK && split) {
    const dim3 grid((unsigned)std::min<i64>(64, ceil_div(K * M, (i64)256)), (unsigned)std::min<i64>(B, 4096));
    switch (dtype) {
      case PYGB200_F32: k_finish_split<float><<<grid, 256, 0, st>>>(probs, B); break;
      case PYGB200_BF16: k_finish_split<__nv_bfloat16><<<grid, 256, 0, st>>>(probs, B); break;
      default: k_finish_split<__half><<<grid, 256, 0, st>>>(probs, B); break;
    }
    count_launch();
    if (cudaGetLastError() != cudaSuccess) rc = PYGB200_ERR_CUDA;
  }
  return rc;
}

}  // namespace
}  // namespace pygb200

using namespace pygb200;

extern "C" int pygb200_segment_matmul(const void* x, const int64_t* ptr_dev, const void* w, const void* bias, void* out,
                                      int64_t N, int64_t K, int64_t M, int64_t B, int dtype, unsigned flags,
                                      void* stream) {
  PYGB_CHECK(N >= 0 && K >= 0 && M >= 0 && B >= 0, PYGB200_ERR_ARG, "segment_matmul: negative size");
  PYGB_CHECK(dtype == PYGB200_F32 || dtype == PYGB200_BF16 || dtype == PYGB200_F16, PYGB200_ERR_ARG,
             "segment_matmul: dtype must be f32, bf16 or f16");
  if (N == 0 || M == 0 || B == 0) return PYGB200_OK;
  PYGB_CHECK(ptr_dev && out && (K == 0 || (x && w)), PYGB200_ERR_ARG, "segment_matmul: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  async_error_flag_dev(ASYNC_ERR_MATMUL);
  PYGB_CHECK(!take_async_error(ASYNC_ERR_MATMUL), PYGB200_ERR_ARG,
             "segment_matmul: an EARLIER segment_matmul / wgrad call received an invalid ptr (it must start at 0, be non-decreasing "
             "and end at the number of rows); that call's output is undefined");
  if (K == 0 && bias == nullptr) {
    PYGB_CUDA(cudaMemsetAsync(out, 0, (size_t)N * M * (dtype == PYGB200_F32 ? 4 : 2), st));
    return PYGB200_OK;
  }
  if (K == 0)   // empty contraction: every row of segment b is bias[b] (the generic kernel runs zero K steps and adds the bias)
    return segment_generic(x, (const i64*)ptr_dev, w, bias, out, N, K, M, B, dtype, 0, st);
  if (!(flags & PYGB200_MM_FORCE_SIMT) && (flags & PYGB200_MM_ALLOW_TF32) && dtype == PYGB200_F32 &&
      tf32_supported(N, K, M, B, x, w, out))
    return segment_matmul_tf32(x, (const i64*)ptr_dev, w, bias, out, N, K, M, B, st);
  if (!(flags & PYGB200_MM_FORCE_SIMT) && segment_tc_supported(N, K, M, B, dtype, x, w, out))
    return segment_matmul_tc(x, (const i64*)ptr_dev, w, bias, out, N, K, M, B, dtype, st);
  return segment_generic(x, (const i64*)ptr_dev, w, bias, out, N, K, M, B, dtype, 0, st);
}

extern "C" int pygb200_segment_matmul_wgrad(const void* x, const int64_t* ptr_dev, const void* dy, void* dw, int64_t N,
                                            int64_t K, int64_t M, int64_t B, int dtype, unsigned flags, void* stream) {
  PYGB_CHECK(N >= 0 && K >= 0 && M >= 0 && B >= 0, PYGB200_ERR_ARG, "segment_matmul_wgrad: negative size");
  PYGB_CHECK(dtype == PYGB200_F32 || dtype == PYGB200_BF16 || dtype == PYGB200_F16, PYGB200_ERR_ARG,
             "segment_matmul_wgrad: dtype must be f32, bf16 or f16");
  if (K == 0 || M == 0 || B == 0) return PYGB200_OK;
  PYGB_CHECK(ptr_dev && dw && (N == 0 || (x && dy)), PYGB200_ERR_ARG, "segment_matmul_wgrad: null pointer");
  async_error_flag_dev(ASYNC_ERR_MATMUL);
  PYGB_CHECK(!take_async_error(ASYNC_ERR_MATMUL), PYGB200_ERR_ARG,
             "segment_matmul_wgrad: an EARLIER segment_matmul / wgrad call received an invalid ptr; that call's output is undefined");
  if (!(flags & PYGB200_MM_FORCE_SIMT) && N > 0 && wgrad_tc_supported(N, K, M, B, dtype, x, dy, dw))
    return segment_wgrad_tc(x, (const i64*)ptr_dev, dy, dw, N, K, M, B, dtype, (cudaStream_t)stream);
  // empty segments produce zero gradients: their single work item runs the k-loop zero times and stores 0
  return segment_generic(x, (const i64*)ptr_dev, dy, nullptr, dw, N, K, M, B, dtype, 1, (cudaStream_t)stream);
}

extern "C" int pygb200_grouped_matmul(const pygb200_gemm_problem* ps, int64_t count, int dtype, unsigned flags,
                                      void* stream) {
  PYGB_CHECK(count >= 0 && (ps || count == 0), PYGB200_ERR_ARG, "grouped_matmul: bad arguments");
  PYGB_CHECK(dtype == PYGB200_F32 || dtype == PYGB200_BF16 || dtype == PYGB200_F16, PYGB200_ERR_ARG,
             "grouped_matmul: dtype must be f32, bf16 or f16");
  if (count == 0) return PYGB200_OK;
  for (i64 i = 0; i < count; ++i) PYGB_CHECK(ps[i].n >= 0 && ps[i].k >= 0 && ps[i].m >= 0, PYGB200_ERR_ARG, "grouped_matmul: negative size");
  cudaStream_t st = (cudaStream_t)stream;
  // bf16 / fp16 problems whose operands satisfy the TMA alignment rules run on the tensor cores (the reference runs
  // grouped_matmul through the same TensorOp grouped GEMM as segment_matmul, matmul_kernel.cu:289-302)
  if (!(flags & PYGB200_MM_FORCE_SIMT) && grouped_tc_supported(ps, count, dtype)) return grouped_matmul_tc(ps, count, dtype, st);
  std::vector<Problem> h((size_t)count);
  i64 tiles = 0;
  for (i64 i = 0; i < count; ++i) {
    const auto& q = ps[i];
    Problem p;
    p.a = q.a; p.b = q.b; p.c = q.c; p.bias = nullptr; p.acc = nullptr;
    p.n = q.n; p.k = q.k; p.m = q.m;
    if (q.a_colmajor) { p.sa0 = 1; p.sa1 = q.lda; } else { p.sa0 = q.lda; p.sa1 = 1; }
    if (q.b_colmajor) { p.sb0 = 1; p.sb1 = q.ldb; } else { p.sb0 = q.ldb; p.sb1 = 1; }
    p.ldc = q.ldc;
    p.kchunk = q.k > 0 ? q.k : 1;
    p.tile0 = tiles;
    tiles += work_items(q.n, q.m, q.k, p.kchunk);
    h[(size_t)i] = p;
  }
  if (tiles == 0) return PYGB200_OK;
  const size_t bytes = (size_t)count * sizeof(Problem) + 16;
  AsyncScratch sc;
  if (int e = sc.alloc(bytes, st)) return e;
  char* scratch = (char*)sc.p;
  // pageable source: the copy is staged by the driver before the call returns, so `h` may die here
  PYGB_CUDA(cudaMemcpyAsync(scratch, &tiles, 8, cudaMemcpyHostToDevice, st));
  PYGB_CUDA(cudaMemcpyAsync(scratch + 16, h.data(), (size_t)count * sizeof(Problem), cudaMemcpyHostToDevice, st));
  return launch_grouped((const Problem*)(scratch + 16), count, (const i64*)scratch, tiles, dtype, st);
}
