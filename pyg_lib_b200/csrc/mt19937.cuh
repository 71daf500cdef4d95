// Device-side reproduction of the random stream pyg-lib's sampler consumes.
//
// Reference semantics (restated, not copied):
//   * torch CPU generator = mt19937 (torch/include/ATen/core/MT19937RNGEngine.h:134-184); a 64-bit
//     draw is two consecutive 32-bit outputs, first one in the high half (CPUGeneratorImpl::random64).
//   * RandintEngine (pyg_lib/csrc/random/cpu/rand_engine.h:26-97) fetches blocks of 128 words
//     w = (random64() % (2^64-1)) + INT64_MIN, reads block elements from index 127 down to 0 and
//     slices each word into 16/32/64-bit fields from the low end.
//
// Design: the mt19937 *raw* (untempered) state stream is materialised in HBM by one CTA using
// the linear recurrence  raw[m] = raw[m-227] ^ T(raw[m-624], raw[m-623])  unrolled KL times, so that
// up to min(227*KL, 623) words are produced per barrier instead of one 624-word twist per three
// barriers.  Tempering, 64-bit assembly and the randint transform happen at the point of use.
#pragma once
#include "common.cuh"

namespace pygb200 {

constexpr int MT_N = 624;
constexpr int MT_M = 397;
constexpr int MT_LAG = MT_N - MT_M;  // 227

__host__ __device__ __forceinline__ u32 mt_twist(u32 u, u32 v) {
  return (((u & 0x80000000u) | (v & 0x7fffffffu)) >> 1) ^ ((v & 1u) ? 0x9908b0dfu : 0u);
}
__host__ __device__ __forceinline__ u32 mt_temper(u32 y) {
  y ^= (y >> 11);
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= (y >> 18);
  return y;
}

// Raw index of the first not-yet-consumed output for an engine pod (left_, next_):
// invariant left+next == 625 except right after seeding (left=1,next=0) where the whole state
// array is "used up" and the next output is element 0 of the next generation.
__host__ __device__ __forceinline__ i64 mt_next0(int left) { return 625 - (i64)left; }

// Number of engine outputs the reference draws for `units` consumed 16-bit units: whole blocks of
// 128 words, at least one (the constructor prefetches, rand_engine.h:28,80-85).
__host__ __device__ __forceinline__ i64 rng_blocks_for_units(i64 units) {
  i64 words = (units + 3) >> 2;
  i64 blocks = (words + 127) >> 7;
  return blocks < 1 ? 1 : blocks;
}

// Word W (0-based, in consumption order) of the RandintEngine stream.
__device__ __forceinline__ u64 rng_word(const u32* __restrict__ raw, i64 out0, i64 W) {
  const i64 b = W >> 7;
  const int e = 127 - (int)(W & 127);
  const i64 o = out0 + (b << 8) + 2 * e;
  const u64 hi = mt_temper(raw[o]), lo = mt_temper(raw[o + 1]);
  u64 v = (hi << 32) | lo;
  if (v == ~0ull) v = 0;            // v % (2^64 - 1)
  return v + 0x8000000000000000ull;  // + INT64_MIN, viewed as uint64
}

// width in 16-bit units of a draw with this range (rand_engine.h:43-50)
__host__ __device__ __forceinline__ int rng_width_units(u64 range) {
  return range < (1ull << 16) ? 1 : (range < (1ull << 32) ? 2 : 4);
}
// leftover bits too few -> skip to the next word (rand_engine.h:53-61)
__host__ __device__ __forceinline__ i64 rng_align(i64 pos, int wu) {
  const int ph = (int)(pos & 3);
  return (ph + wu > 4) ? pos + (4 - ph) : pos;
}
// position after `n` consecutive draws of the same width starting at `pos`
__host__ __device__ __forceinline__ i64 rng_run(i64 pos, int wu, i64 n) {
  if (n <= 0) return pos;
  if (wu == 1) return pos + n;
  if (wu == 4) return rng_align(pos, 4) + 4 * n;
  pos = rng_align(pos, 2) + 2;  // after one 32-bit draw the phase is 0, 2 or 3
  if (--n == 0) return pos;
  pos = rng_align(pos, 2) + 2;  // after two it is even
  return pos + 2 * (n - 1);
}
// A node's draws come as n16 16-bit draws, then n32 32-bit, then n64 64-bit (ranges only grow).
// Start position (aligned) of draw j (0-based) when the node's first draw may start at `pos`.
__host__ __device__ __forceinline__ i64 rng_draw_start(i64 pos, i64 n16, i64 n32, i64 j, int* wu_out) {
  if (j < n16) { *wu_out = 1; return pos + j; }
  pos += n16;
  if (j < n16 + n32) { *wu_out = 2; return rng_align(rng_run(pos, 2, j - n16), 2); }
  pos = rng_run(pos, 2, n32);
  *wu_out = 4;
  return rng_align(rng_run(pos, 4, j - n16 - n32), 4);
}
__host__ __device__ __forceinline__ i64 rng_node_end(i64 pos, i64 n16, i64 n32, i64 n64) {
  return rng_run(rng_run(pos + n16, 2, n32), 4, n64);
}

__device__ __forceinline__ u64 rng_draw(const u32* __restrict__ raw, i64 out0, i64 pos, int wu, u64 range) {
  if (wu == 1) {
    // 16-bit field `ph` of word W: it lies in one 32-bit half of the word, so only that engine output is loaded
    // and tempered.  rng_word's two corrections still apply: v == 2^64-1 -> 0 (both halves all-ones after
    // tempering; the other half is only looked at when this one is) and + 2^63 (flips the top bit of field 3).
    const i64 W = pos >> 2;
    const int ph = (int)(pos & 3);
    const i64 o = out0 + ((W >> 7) << 8) + 2 * (127 - (int)(W & 127));
    u32 t = mt_temper(raw[o + (ph < 2 ? 1 : 0)]);
    if (t == 0xffffffffu && mt_temper(raw[o + (ph < 2 ? 0 : 1)]) == 0xffffffffu) t = 0;
    if (ph >= 2) t ^= 0x80000000u;
    const u32 field = (ph & 1) ? (t >> 16) : (t & 0xffffu);
    return (u64)(field % (u32)range);
  }
  const u64 w = rng_word(raw, out0, pos >> 2);
  const int sh = (int)(pos & 3) * 16;
  if (wu == 2) return (u64)((u32)(w >> sh) % (u32)range);
  return w % range;
}

// ---------------------------------------------------------------------------------- generation
struct MTPodParam {
  u32 state[MT_N];
};

__global__ void k_mt_init(u32* __restrict__ raw, i64* generated, const __grid_constant__ MTPodParam pod) {
  for (int i = threadIdx.x; i < MT_N; i += blockDim.x) raw[i] = pod.state[i];
  if (threadIdx.x == 0) *generated = MT_N;
}

constexpr int MT_WIN = 4096;  // circular shared-memory window (words)

// Generates raw[m .. target) with one 640-thread CTA.  `hist_lo` = lowest raw index that holds valid
// history (0 for the stream's start; the window base after a jump).  `KL` = recurrence unroll: with
// history >= 624 + 227*(KL-1) words a step yields min(227*KL, 623) words per barrier.
template <int KL>
__device__ void mt_gen_range(u32* __restrict__ raw, i64 hist_lo, i64 m, i64 target, u32* win) {
  if (target <= m) return;
  constexpr int HIST = MT_N + MT_LAG * (KL - 1);
  const i64 h0 = (m - hist_lo) > HIST ? m - HIST : hist_lo;
  for (i64 i = h0 + threadIdx.x; i < m; i += blockDim.x) win[i & (MT_WIN - 1)] = __ldcg(&raw[i]);
  __syncthreads();
  while (m < target) {
    int k = (int)((m - hist_lo - MT_N) / MT_LAG) + 1;  // unroll factor the available history allows
    if (k > KL) k = KL;
    i64 n = (i64)MT_LAG * k;
    if (n > MT_N - 1) n = MT_N - 1;  // the T(raw[m-624], raw[m-623]) term caps the step at 623 words
    if (n > target - m) n = target - m;
    if ((i64)threadIdx.x < n) {
      const i64 mm = m + threadIdx.x;
      u32 x = win[(mm - (i64)MT_LAG * k) & (MT_WIN - 1)];
#pragma unroll
      for (int j = 0; j < KL; ++j)
        if (j < k)
          x ^= mt_twist(win[(mm - MT_N - MT_LAG * j) & (MT_WIN - 1)], win[(mm - MT_N + 1 - MT_LAG * j) & (MT_WIN - 1)]);
      win[mm & (MT_WIN - 1)] = x;  // never aliases a word read in this step (window >> history + step)
      raw[mm] = x;
    }
    __syncthreads();
    m += n;
  }
}

// Publication of a new stream length by the block that generated it: the length only ever grows (a main-stream
// kernel and the side stream may extend the same stream concurrently — they write identical words) and a
// reader that polls it (k_sample_s) must find the words behind it.
__device__ __forceinline__ void mt_publish(i64* generated, i64 m) {
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) atomicMax(reinterpret_cast<unsigned long long*>(generated), (unsigned long long)m);
}

// Extends raw[] up to (at least) raw index `target`, rounded up to a whole 624-word generation.
template <int KL>
__global__ void __launch_bounds__(640) k_mt_extend_to(u32* __restrict__ raw, i64* generated, i64 target_in, i64 cap_words) {
  __shared__ u32 win[MT_WIN];
  i64 target = ((target_in + MT_N - 1) / MT_N) * MT_N;
  if (target > cap_words) target = (cap_words / MT_N) * MT_N;
  const i64 m = *generated;
  if (target <= m) return;
  mt_gen_range<KL>(raw, 0, m, target, win);
  mt_publish(generated, target);
}

// ---- parallel generation by jump-ahead (tools/mt19937_jump.py builds the polynomial table) -------------
// raw[] is linear over GF(2): raw[t + p*S + j] = XOR_{i in g_p} raw[t + i + j] (j = 0..623) with
// g_p = x^(p*S) mod x*phi(x), deg < 19938.  So after a serial pre-step of ~20.6k words every CTA p can
// compute the 624-word window that starts its chunk and generate S words independently.
constexpr int MT_POLY_WORDS = 624;                       // 19968 bits >= degree bound 19938
constexpr i64 MT_JUMP_PRESTEP = 19938 + MT_N + MT_N;     // history the jumps read, rounded up below

// pre-step: remember where the jump base is and extend by the history the polynomials read
template <int KL>
__global__ void __launch_bounds__(640) k_mt_jump_prestep(u32* __restrict__ raw, i64* generated, i64* jump_base, i64 cap_words) {
  __shared__ u32 win[MT_WIN];
  const i64 m = *generated;
  i64 target = ((m + MT_JUMP_PRESTEP + MT_N - 1) / MT_N) * MT_N;
  if (target > cap_words) target = (cap_words / MT_N) * MT_N;
  if (threadIdx.x == 0) *jump_base = m;
  if (target <= m) return;
  mt_gen_range<KL>(raw, 0, m, target, win);
  mt_publish(generated, target);
}

// CTA p generates raw[b0 + p*S + 624 .. b0 + (p+1)*S + 624), b0 = jump_base - 624 (CTA 0 continues after the
// pre-step).  The last CTA to finish publishes the new length.
// The jump itself is ~10 k XORs of history words per thread: the history the polynomial reads (MT_JUMP_HIST words,
// 85 KB) is staged in shared memory first — read from L2 inside the bit loop, every XOR waited for one L2 round trip
// (a while(bits) loop is not unrolled, so the loads did not overlap) and the jump, not the generation, dominated a chunk.
constexpr int MT_JUMP_HIST = 19938 + MT_N + 62;   // highest history index read: deg(g) <= 19937, + 623; rounded to 20 624
template <int KL>
__global__ void __launch_bounds__(640) k_mt_jump_generate(u32* __restrict__ raw, i64* generated, const i64* jump_base,
                                                           const u32* __restrict__ polys, int S, i64 cap_words,
                                                           unsigned long long* ticket) {
  __shared__ u32 win[MT_WIN];
  __shared__ int s_last;
  extern __shared__ u32 s_hist[];   // MT_JUMP_HIST words
  const i64 b0 = *jump_base - MT_N;
  const int p = blockIdx.x, P = gridDim.x;
  i64 end_all = b0 + (i64)P * S + MT_N;
  if (end_all > cap_words) end_all = (cap_words / MT_N) * MT_N;
  i64 m, hist_lo, target = b0 + (i64)(p + 1) * S + MT_N;
  if (target > end_all) target = end_all;
  if (p == 0) {
    m = *generated;   // end of the pre-step
    hist_lo = 0;
  } else {
    const i64 w0 = b0 + (i64)p * S;   // window base of this chunk
    if (w0 + MT_N <= end_all) {
      const u32* __restrict__ g = polys + (size_t)(p - 1) * MT_POLY_WORDS;
      const u32* src = raw + b0;
      for (int i = threadIdx.x; i < MT_JUMP_HIST; i += blockDim.x) s_hist[i] = __ldcg(&src[i]);
      __syncthreads();
      if (threadIdx.x < MT_N) {
        u32 acc = 0;
        const u32* h = s_hist + threadIdx.x;
        for (int w = 0; w < MT_POLY_WORDS; ++w) {
          u32 bits = __ldg(&g[w]);
          const u32* hw = h + w * 32;
          while (bits) {
            const int i = __ffs(bits) - 1;
            bits &= bits - 1;
            acc ^= hw[i];
          }
        }
        raw[w0 + threadIdx.x] = acc;
      }
    }
    __syncthreads();
    m = w0 + MT_N;
    hist_lo = w0;
  }
  if (m < target) mt_gen_range<KL>(raw, hist_lo, m, target, win);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned long long t = atomicAdd(ticket, 1ull);
    s_last = (t == (unsigned long long)P - 1);
    if (s_last) *ticket = 0;
  }
  __syncthreads();
  if (s_last && threadIdx.x == 0) {
    __threadfence();
    atomicMax(reinterpret_cast<unsigned long long*>(generated), (unsigned long long)end_all);
  }
}

}  // namespace pygb200
