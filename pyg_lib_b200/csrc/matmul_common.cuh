// pyg_lib_b200/csrc/matmul_common.cuh — plumbing shared by the two grouped GEMMs of segment_matmul / grouped_matmul:
// the SIMT kernel (matmul.cu) and the tensor-core kernel (matmul_grouped_tc.cu).
#pragma once
#include "common.cuh"

namespace pygb200 {

inline int num_sms() {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

// Problem list of a segment GEMM, built on the device from `ptr` [B + 1] by one block, so that a device-resident ptr
// costs no host sync.  The block first validates ptr (ptr[0] == 0, non-decreasing, ptr[B] == N — what the reference's
// split_with_sizes checks on the host): a bad one leaves the launch without work (*total = 0) and raises *err.
// Otherwise, for each segment b with rows [r0, r0 + len), fill(b, r0, len, p) describes its problem p and returns its
// number of flat work items; an exclusive scan over the segments (one block-wide pass per blockDim.x segments, carried in
// shared memory) gives p.tile0, the index of its first item; place(p) may then use tile0 before p is stored.
// *total = the number of items.  CountT: the type of item counts and segment indices.
template <typename CountT, typename Prob, typename Fill, typename Place>
__device__ __forceinline__ void build_segment_list(Prob* probs, CountT* total, const i64* __restrict__ ptr, CountT B, i64 N,
                                                   int* err, Fill fill, Place place) {
  __shared__ CountT s_carry;
  __shared__ CountT s_w[32];
  if (threadIdx.x == 0) s_carry = 0;
  {
    int bad = 0;
    for (CountT b = threadIdx.x; b < B; b += blockDim.x) bad |= (ptr[b + 1] < ptr[b]) | (b == 0 && ptr[0] != 0) | (b == B - 1 && ptr[B] != N);
    if (__syncthreads_or(bad)) {
      if (threadIdx.x == 0) { *total = 0; if (err) *err = 1; }
      return;
    }
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (CountT base = 0; base < B; base += blockDim.x) {
    const CountT b = base + threadIdx.x;
    CountT tiles = 0;
    Prob p;
    if (b < B) tiles = fill(b, ptr[b], ptr[b + 1] - ptr[b], p);
    CountT inc = tiles;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const CountT o = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc += o;
    }
    if (lane == 31) s_w[wid] = inc;
    __syncthreads();
    CountT pre = 0, tot = 0;
    for (int q = 0; q < (int)(blockDim.x >> 5); ++q) { if (q < wid) pre += s_w[q]; tot += s_w[q]; }
    const CountT c0 = s_carry;
    if (b < B) {
      p.tile0 = c0 + pre + inc - tiles;
      place(p);
      probs[b] = p;
    }
    __syncthreads();
    if (threadIdx.x == 0) s_carry = c0 + tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = s_carry;
}

// Split-K epilogue of one problem: c[r * ldc + j] = cvt(sum of the `chunks` fp32 partials [n, m] (ld = m) at part), the
// chunks added in chunk order, so the result is bit-reproducible.  Grid-stride over the n x m elements.
template <typename T, typename Cvt>
__device__ __forceinline__ void finish_split_problem(T* c, i64 ldc, const float* part, i64 n, i64 m, i64 chunks, Cvt cvt) {
  const i64 nm = n * m;
  for (i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x; i < nm; i += (i64)gridDim.x * blockDim.x) {
    float v = 0.f;
    for (i64 k = 0; k < chunks; ++k) v += part[k * nm + i];
    c[(i / m) * ldc + i % m] = cvt(v);
  }
}

}  // namespace pygb200
