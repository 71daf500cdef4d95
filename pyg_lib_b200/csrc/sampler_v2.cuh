// pyg_lib_b200/csrc/sampler_v2.cuh — throughput schedule of the sampler ("v2"), included by sampler.cu inside its
// anonymous namespace (it uses PassArgs, NodeRec, sample_draws, pdl_enter, last_block, ... from there).
//
// Same results as the other schedules (bit-exact vs neighbor_kernel.cpp:337-514 / 529-841), different data path, built
// from what tools/p2p_microbench.cu measures: random 8-byte atomics on a table larger than L2 run more than twice as fast
// when an insert is ONE atomic than when it is CAS(keys) + min(vals) on two arrays; random 8-byte loads are faster still;
// a peer GPU takes CAS and coalesced stores over NVLink at a fraction of local rates.  So:
//   * packed table: one u64 slot = (node id : 32 | value : 32); value = V2_POS | flat position of the running pass
//     until ids are assigned, else the node's local id.  Insert = one CAS (+ one min only when the key was already
//     there with a larger position).  Needs node ids < 2^32 - 1, pass positions and local ids < 2^31 (checked by
//     the host; disjoint / temporal / unbounded runs keep the wide-table schedules).
//   * "ref" instead of a lookup pass: after all inserts of a pass, mark reads each edge's slot once: ref = value.
//     first occurrence <=> ref == V2_POS | p.  Ranks of the firsts come from per-tile counts + in-tile ranks
//     (erank[], 4 B per edge, L2-resident), so an edge's local id is ids_base + tile_prefix[q >> 10] + erank[q] with
//     q = ref's position — no second and third random pass over the table (assign's id write-back is skipped for
//     passes whose dst table is not inserted into again; the old lookup pass is gone).
//   * frontier sharding over peer memory (W ranks, one process per GPU, CSR replicated; SURVEY 8e): every rank counts
//     the whole frontier (offsets / RNG positions are global), draws only its slice of frontier nodes and STORES the
//     (dst, edge id) of its edges straight into every rank's exchange region over NVLink — the all-gather of sampled
//     edges is fused into the sampling kernel.  Dedup is partitioned by key: a rank inserts only the dst ids it owns
//     (hash of the id), so the random atomics are divided by W; it publishes the refs of owned positions, each rank
//     sums its position slice over the peers (coalesced peer loads) and stores the result to everybody.  From the
//     full ref array all ranks derive identical ids with streaming work only.  Cross-GPU ordering = flag words in
//     the exchange regions (k_xbarrier), no host involvement, no NCCL call on the data path.
#pragma once

constexpr u32 V2_POS = 0x80000000u;
constexpr int V2_MAX_W = 16;

__device__ __forceinline__ int v2_owner(u32 key, int W) {
  u32 h = key * 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;   // independent of the slot hash
  return (int)(((u64)h * (u32)W) >> 32);
}

// insert (key, position p of the running pass); returns the slot.  The slot's value ends up as the minimum position
// of the key in this pass, or stays the local id the key got in an earlier pass (ids < V2_POS <= positions).
__device__ __forceinline__ u32 v2_insert(u64* __restrict__ pk, int bits, u32 key, u32 p) {
  const u32 mask = (u32)((1ull << bits) - 1);   // (bits <= 32)
  u32 s = (u32)(((u64)key * 0x9E3779B97F4A7C15ull) >> (64 - bits));
  const u64 mine = ((u64)key << 32) | (u64)(V2_POS | p);
  while (true) {
    const u64 prev = atomicCAS(&pk[s], EMPTY, mine);
    if (prev == EMPTY) return s;
    if ((u32)(prev >> 32) == key) {
      if ((u32)prev > (V2_POS | p)) red_min_u64(&pk[s], mine);
      return s;
    }
    s = (s + 1) & mask;
  }
}

template <typename T>
__device__ __forceinline__ T* x_ptr(const PassArgs& a, int q, i64 off) { return reinterpret_cast<T*>(a.xpeer[q] + off); }

// ---- cross-GPU barrier on flag words in the exchange regions.  The last block of a kernel that stored to the peers
// tells every rank q "rank xr has reached epoch" (x_signal after last_block_sys); k_xbarrier, launched behind a kernel
// that needs nothing remote where there is one (k_v2_rows), waits for every rank's word in its own region, so the
// peers' skew hides behind local work.  Thread q waits for rank q.  A peer that never arrives is reported, not waited
// for forever.
__device__ __forceinline__ void x_signal(const PassArgs& a) {
  if ((int)threadIdx.x < a.xw && (int)threadIdx.x != a.xr)
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(x_ptr<u64>(a, threadIdx.x, a.x_off_bar) + a.xr), "l"(a.x_sig_epoch) : "memory");
}
__global__ void k_xbarrier(const PassArgs a, u64 epoch, u64 timeout_ns) {
  pdl_enter();
  const int q = threadIdx.x;
  if (q >= a.xw) return;
  __threadfence_system();
  u64* mine = x_ptr<u64>(a, a.xr, a.x_off_bar);
  if (q != a.xr) {
    u64 t0, t1, v;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    while (true) {
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(mine + q) : "memory");
      if (v >= epoch) break;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
      if (t1 - t0 > timeout_ns) { a.st[ST_ERROR] = 2; break; }
      __nanosleep(200);
    }
  }
  __threadfence_system();
}

// ---- seeds: list them and insert them at position i (first-occurrence order == seed order)
template <typename idx_t>
__global__ void __launch_bounds__(NT) k_v2_seed(const PassArgs a, const idx_t* __restrict__ seeds, i64 n) {
  pdl_enter(TL_SEED);
  for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < n; i += (i64)gridDim.x * NT) {
    const i64 v = (i64)seeds[i];
    a.dst_nodes[i] = v;
    // (sharded: `pk` is this rank's scratch table and takes ALL seeds — see k_v2_assign)
    a.eslot[i] = v2_insert(a.pk, a.pk_bits, (u32)v, (u32)i);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) { a.st[ST_PASS_E] = n; a.st[ST_PASS_BASE] = 0; }
}

// ---- sharded: the row (source-node index) of EVERY edge of the pass, one thread per frontier node — replicated on
// all ranks and cheap (F records in, E 8-byte stores out).
__global__ void __launch_bounds__(NT) k_v2_rows(const PassArgs a) {
  pdl_enter();
  const i64 F = a.st[ST_PASS_F];
  const i64 begin = a.st[a.o_src_begin];
  const i64 pbase = a.st[ST_PASS_BASE];
  for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < F; i += (i64)gridDim.x * NT) {
    const uint4 ra = __ldg(reinterpret_cast<const uint4*>(a.rec + i));   // {rs lo, rs hi, deg, loc_off}
    i64 n_out, n16, n32, n64;
    classify((i64)ra.z, a.fanout, a.replace, &n_out, &n16, &n32, &n64);
    i64* dst = a.row + pbase + __ldg(&a.tile_off[i / NT]) + ra.w;
    const i64 src_pos = begin + i;
    for (i64 j = 0; j < n_out; ++j) dst[j] = src_pos;
  }
}

// ---- sharded: this rank's slice of (dst, edge id) — contiguous flat positions [st[o_shard + r], st[o_shard + r + 1]) —
// from its own exchange region to every peer's: the all-gather of the sampled edges as 16-byte coalesced peer stores
// (the access pattern tools/p2p_microbench.cu measured at 690 GB/s).
__global__ void __launch_bounds__(NT) k_v2_push(const PassArgs a) {
  pdl_enter();
  const i64 lo = a.st[a.o_shard + a.xr], hi = a.st[a.o_shard + a.xr + 1];
  auto push_bytes = [&](i64 off, int esz) {
    // byte range of the slice inside the array: the 16-byte-aligned middle goes as uint4, the unaligned head and tail
    // (< 16 bytes each; they share their 16-byte lines with the neighbouring ranks' slices) as 4-byte stores
    const i64 b0 = lo * esz, b1 = hi * esz;
    const i64 v0 = (b0 + 15) & ~(i64)15, v1 = b1 & ~(i64)15;
    const unsigned char* src = a.xpeer[a.xr] + off;
    if (v1 > v0) {
      const i64 nv = (v1 - v0) >> 4;
      for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < nv; i += (i64)gridDim.x * NT) {
        const uint4 w = *reinterpret_cast<const uint4*>(src + v0 + (i << 4));
        for (int q = 0; q < a.xw; ++q)
          if (q != a.xr) *reinterpret_cast<uint4*>(a.xpeer[q] + off + v0 + (i << 4)) = w;
      }
    }
    // unaligned head and tail (< 16 bytes each), 4 bytes at a time, by block 0
    if (blockIdx.x == 0) {
      const i64 h1 = v1 > v0 ? v0 : b1, t0 = v1 > v0 ? v1 : b1;
      for (i64 b = b0 + 4 * threadIdx.x; b < h1; b += 4 * NT) {
        const u32 w = *reinterpret_cast<const u32*>(src + b);
        for (int q = 0; q < a.xw; ++q) if (q != a.xr) *reinterpret_cast<u32*>(a.xpeer[q] + off + b) = w;
      }
      for (i64 b = t0 + 4 * threadIdx.x; b < b1; b += 4 * NT) {
        const u32 w = *reinterpret_cast<const u32*>(src + b);
        for (int q = 0; q < a.xw; ++q) if (q != a.xr) *reinterpret_cast<u32*>(a.xpeer[q] + off + b) = w;
      }
    }
  };
  push_bytes(a.x_off_dst, 4);
  push_bytes(a.x_off_eid, a.x_eid64 ? 8 : 4);
  if (a.x_sig_epoch && last_block_sys(&a.st[ST_TICKET_B])) x_signal(a);
}

// ---- one pass's sampling.  SH = false: draw, gather, rows / edge ids / global dst into the result arrays, insert.
// SH = true: the nodes of this rank's frontier slice draw, gather and store (dst : u32, edge id : u32 | u64) at the
// edge's flat position into this rank's exchange region; k_v2_push sends the slice to every peer, k_v2_rows writes the rows.
template <typename idx_t, bool SH>
__global__ void __launch_bounds__(NT, SAMPLE_MIN_BLOCKS) k_v2_sample(const PassArgs a) {
  pdl_enter(TL_SAMPLE);
  const i64 F = a.st[ST_PASS_F];
  const i64 begin = a.st[a.o_src_begin];
  const i64 pbase = a.st[ST_PASS_BASE];
  const int g = a.group, lane = threadIdx.x & 31, per_warp = 32 / g;
  const int gi = lane / g, gl = lane - gi * g, gbase = gi * g;
  const unsigned gmask = (g == 32) ? 0xffffffffu : (((1u << g) - 1u) << gbase);
  const int npb = (NT / 32) * per_warp;
  const idx_t* __restrict__ col = (const idx_t*)a.col;
  const i64 own_lo = SH ? (i64)((__int128)F * a.xr / a.xw) : 0;
  const i64 own_hi = SH ? (i64)((__int128)F * (a.xr + 1) / a.xw) : F;
  if (gi >= per_warp) return;   // (lanes beyond the last whole group of the warp)
  for (i64 i = own_lo + (i64)blockIdx.x * npb + (threadIdx.x >> 5) * per_warp + gi; i < own_hi; i += (i64)gridDim.x * npb) {
    const NodeRec r = a.rec[i];
    const i64 tile = i / NT;
    const i64 off = a.tile_off[tile] + r.loc_off;    // pass-local flat position of the node's first edge
    const i64 src_pos = begin + i;                   // local id of the source node (neighbor_kernel.cpp:453)
    const i64 tpos = a.tile_pos[tile];
    const int ph = (int)(tpos & 3);
    const u32 pfv = ph == 0 ? r.pf[0] : (ph == 1 ? r.pf[1] : (ph == 2 ? r.pf[2] : r.pf[3]));
    auto emit = [&](i64 j, i64 e) {
      const i64 p = off + j;
      const i64 d = (i64)col[e];
      if (!SH) {
        a.eslot[p] = v2_insert(a.pk, a.pk_bits, (u32)d, (u32)p);
        a.colv[pbase + p] = d;   // global id until k_v2_assign replaces it with the local id
        a.row[pbase + p] = src_pos;
        a.eid[pbase + p] = e;
      } else {
        // into this rank's OWN exchange region; k_v2_push forwards the slice to the peers with wide, fully coalesced
        // stores — 4-byte lane stores straight to 7 peers made this kernel 227 us at 8 ranks for 1/8 of the draws
        x_ptr<u32>(a, a.xr, a.x_off_dst)[p] = (u32)d;
        if (a.x_eid64) x_ptr<u64>(a, a.xr, a.x_off_eid)[p] = (u64)e; else x_ptr<u32>(a, a.xr, a.x_off_eid)[p] = (u32)e;
      }
    };
    auto prev = [&](u32 t) -> i64 {
      if (!SH) return __ldcg(&a.eid[pbase + off + t]);
      return a.x_eid64 ? (i64)__ldcg(x_ptr<u64>(a, a.xr, a.x_off_eid) + off + t) : (i64)__ldcg(x_ptr<u32>(a, a.xr, a.x_off_eid) + off + t);
    };
    sample_draws(a, r, tpos + pfv, g, gl, gbase, gmask, emit, prev);
  }
  tl_mark(TL_SAMPLE | TL_END);
}

// ---- sharded: the owner of a dst id inserts it (all positions of the pass are streamed, 1/W of them hit the table).
// Four positions per thread (coalesced, strided by the block) with their first CAS issued back to back: the kernel is
// bound by the round trips of independent atomics, not by their number.
template <bool SH>   // SH = false: single GPU, the inserts of a biased pass (keys = the global ids in colv)
__global__ void __launch_bounds__(NT) k_v2_insert(const PassArgs a) {
  pdl_enter();
  const i64 E = a.st[ST_PASS_E];
  const i64 pbase = a.st[ST_PASS_BASE];
  const u32* __restrict__ xdst = SH ? x_ptr<u32>(a, a.xr, a.x_off_dst) : nullptr;
  const u64 mask = (1ull << a.pk_bits) - 1;
  for (i64 base = (i64)blockIdx.x * (4 * NT); base < E; base += (i64)gridDim.x * (4 * NT)) {
    u32 key[4]; u64 slot[4], prev[4]; bool own[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const i64 p = base + j * NT + threadIdx.x;
      key[j] = p < E ? (SH ? xdst[p] : (u32)a.colv[pbase + p]) : 0u;
      own[j] = p < E && (!SH || v2_owner(key[j], a.xw) == a.xr);
      slot[j] = ((u64)key[j] * 0x9E3779B97F4A7C15ull) >> (64 - a.pk_bits);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const i64 p = base + j * NT + threadIdx.x;
      prev[j] = own[j] ? atomicCAS(&a.pk[slot[j]], EMPTY, ((u64)key[j] << 32) | (u64)(V2_POS | (u32)p)) : EMPTY;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const i64 p = base + j * NT + threadIdx.x;
      if (p >= E) break;
      u32 res = NO_SLOT;
      if (own[j]) {
        const u64 mine = ((u64)key[j] << 32) | (u64)(V2_POS | (u32)p);
        u64 sl = slot[j], pv = prev[j];
        while (true) {   // (same decisions as v2_insert, continuing from the CAS already made)
          if (pv == EMPTY) break;
          if ((u32)(pv >> 32) == key[j]) { if ((u32)pv > (V2_POS | (u32)p)) red_min_u64(&a.pk[sl], mine); break; }
          sl = (sl + 1) & mask;
          pv = atomicCAS(&a.pk[sl], EMPTY, mine);
        }
        res = (u32)sl;
      }
      a.eslot[p] = res;
      if (SH) a.fref[p] = V2_POS | (u32)p;   // default ref "first occurrence"; the owners send the exceptions (k_v2_exc)
    }
  }
  if (SH && blockIdx.x == 0 && threadIdx.x == 0) *x_ptr<u64>(a, a.xr, a.x_off_xcnt) = 0;   // this pass's exception count (k_v2_exc)
}

// ---- sharded: the refs every rank needs.  A position's ref is "first occurrence" (V2_POS | p, what k_v2_insert wrote
// as the default) unless its key was seen earlier — in this pass at a smaller position, or in an earlier pass.  Only
// the owner of the key knows, and only those EXCEPTIONS travel: (position, ref) pairs appended to a list in every
// rank's exchange region (on the papers100M-shaped graph ~5 % of the positions, on a duplicate-heavy graph at most
// all of them).  One barrier later k_v2_scatter applies the W lists to the local ref array.  This replaced a
// zero-padded partial-ref array + slice-wise pull / reduce / push (two kernels, two barriers, 8 B/edge on the link).
__global__ void __launch_bounds__(NT) k_v2_exc(const PassArgs a) {
  pdl_enter();
  const i64 E = a.st[ST_PASS_E];
  u64* cnt = x_ptr<u64>(a, a.xr, a.x_off_xcnt);
  const int lane = threadIdx.x & 31;
  for (i64 base = (i64)blockIdx.x * (4 * NT); base < E; base += (i64)gridDim.x * (4 * NT)) {
    u32 s[4], v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) { const i64 p = base + j * NT + threadIdx.x; s[j] = p < E ? __ldg(&a.eslot[p]) : NO_SLOT; }
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = s[j] == NO_SLOT ? 0u : (u32)a.pk[s[j]];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const i64 p = base + j * NT + threadIdx.x;
      const bool exc = s[j] != NO_SLOT && v[j] != (V2_POS | (u32)p);
      const unsigned m = __ballot_sync(0xffffffffu, exc);   // (the loop bounds are block-uniform: all lanes are here)
      if (m == 0) continue;
      u64 pos0 = 0;
      if (lane == __ffs(m) - 1) pos0 = atomicAdd(cnt, (u64)__popc(m));   // one counter bump per warp
      pos0 = __shfl_sync(0xffffffffu, pos0, __ffs(m) - 1);
      if (exc) {
        const u64 idx = pos0 + __popc(m & ((1u << lane) - 1u)), pair = ((u64)(u32)p << 32) | (u64)v[j];
        for (int q = 0; q < a.xw; ++q) x_ptr<u64>(a, q, a.x_off_exc)[(i64)a.xr * a.x_exc_cap + idx] = pair;
      }
    }
  }
  // the list length goes to every rank once all blocks are done
  if (last_block_sys(&a.st[ST_TICKET_A])) {
    if (threadIdx.x < a.xw) x_ptr<u64>(a, threadIdx.x, a.x_off_exc_n)[a.xr] = *reinterpret_cast<volatile u64*>(cnt);
    __threadfence_system();
    __syncthreads();
    if (a.x_sig_epoch) x_signal(a);
  }
}

// blockIdx.y = source rank
__global__ void __launch_bounds__(NT) k_v2_scatter(const PassArgs a) {
  pdl_enter();
  const int sr = blockIdx.y;
  const i64 n = (i64)x_ptr<u64>(a, a.xr, a.x_off_exc_n)[sr];
  const u64* __restrict__ list = x_ptr<u64>(a, a.xr, a.x_off_exc) + (i64)sr * a.x_exc_cap;
  for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < n; i += (i64)gridDim.x * NT) {
    const u64 pair = list[i];
    a.fref[pair >> 32] = (u32)pair;
  }
}

// counters of a pass once the per-tile counts of first occurrences are known: ordered exclusive scan of the counts by
// the calling (last) block, dst list / id counters, end-of-hop bookkeeping (shared with k_mark)
__device__ void mark_finish(const PassArgs& a, i64 E, i64 ntiles) {
  // (staged in shared memory like scan_frontier_tiles: coalesced loads, 16 consecutive tiles per thread, one block-wide
  //  scan per round of 4096 tiles; a tile holds at most 1024 firsts, so the counts fit 32 bits)
  __shared__ u32 s_cnt[MSCAN_CHUNK];
  __shared__ i64 s_s[NT / 32];
  __shared__ i64 carry;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry = 0;
  for (i64 base = 0; base < ntiles; base += MSCAN_CHUNK) {
    const int n = (int)(ntiles - base < MSCAN_CHUNK ? ntiles - base : MSCAN_CHUNK);
    for (int j = threadIdx.x; j < n; j += NT) s_cnt[j] = (u32)__ldcg(&a.mtile[base + j]);
    __syncthreads();
    const int j0 = threadIdx.x * MSCAN_PER, j1 = j0 + MSCAN_PER < n ? j0 + MSCAN_PER : n;
    i64 v = 0;
    for (int j = j0; j < j1; ++j) v += s_cnt[j];
    i64 inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const i64 o = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc += o;
    }
    if (lane == 31) s_s[wid] = inc;
    __syncthreads();
    i64 pre = 0, tot = 0;
    for (int w = 0; w < NT / 32; ++w) { if (w < wid) pre += s_s[w]; tot += s_s[w]; }
    const i64 c0 = carry;
    i64 run = c0 + pre + inc - v;
    for (int j = j0; j < j1; ++j) { a.mtile[base + j] = run; run += s_cnt[j]; }
    __syncthreads();
    if (threadIdx.x == 0) carry = c0 + tot;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const i64 nnew = carry;
    a.st[ST_PASS_NEW] = nnew;
    if (a.seed_mode) {
      a.st[ST_LIST_BASE] = 0;
      a.st[ST_IDS_BASE] = 0;
      a.st[a.o_dst_list] = E;      // every seed is listed, duplicates included (neighbor_kernel.cpp:410)
      a.st[a.o_dst_ids] = nnew;    // ... but ids only count distinct ones (mapper.h:29-46)
      if (a.sd_end) { a.st[a.sd_begin] = 0; a.st[a.sd_end] = E; a.st[a.sd_nph] = E; }   // first frontier = the seed list (k_seed_end)
    } else {
      a.st[ST_LIST_BASE] = a.st[a.o_dst_list];
      a.st[ST_IDS_BASE] = a.st[a.o_dst_ids];
      a.st[a.o_dst_list] += nnew;
      a.st[a.o_dst_ids] += nnew;
    }
  }
  __syncthreads();
  // last pass of the hop: advance every type's frontier slice (neighbor_kernel.cpp:807-812)
  for (int t = threadIdx.x; t < a.he_T; t += NT) {
    const i64 n = a.st[a.he_list + t], e = a.st[a.he_end + t];
    a.st[a.he_nph + t * (a.he_L + 1) + a.he_hop + 1] = n - e;
    a.st[a.he_begin + t] = e;
    a.st[a.he_end + t] = n;
  }
}

// ---- refs -> first-occurrence flags, in-tile ranks, per-tile counts; last block: scan + counters.
// TABLE = true (single GPU): the ref of an edge is read from its slot here and kept in fref[].
template <bool TABLE>
__global__ void __launch_bounds__(NT) k_v2_mark(const PassArgs a) {
  __shared__ u32 s_w[NT / 32];
  pdl_enter(TL_MARK);
  const i64 E = a.st[ST_PASS_E];
  const i64 ntiles = ceil_div(E, ETILE);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (i64 tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const i64 p0 = tile * ETILE + threadIdx.x * 4;
    u32 fl[4]; u32 cnt = 0;
    if (p0 + 3 < E) {
      uint4 rv;
      if (TABLE) {
        const uint4 sl = *reinterpret_cast<const uint4*>(a.eslot + p0);
        rv.x = (u32)a.pk[sl.x]; rv.y = (u32)a.pk[sl.y]; rv.z = (u32)a.pk[sl.z]; rv.w = (u32)a.pk[sl.w];
        *reinterpret_cast<uint4*>(a.fref + p0) = rv;
      } else {
        rv = *reinterpret_cast<const uint4*>(a.fref + p0);
      }
      fl[0] = rv.x == (V2_POS | (u32)p0); fl[1] = rv.y == (V2_POS | (u32)(p0 + 1));
      fl[2] = rv.z == (V2_POS | (u32)(p0 + 2)); fl[3] = rv.w == (V2_POS | (u32)(p0 + 3));
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const i64 p = p0 + q;
        fl[q] = 0;
        if (p < E) {
          u32 rv;
          if (TABLE) { rv = (u32)a.pk[a.eslot[p]]; a.fref[p] = rv; } else rv = a.fref[p];
          fl[q] = rv == (V2_POS | (u32)p);
        }
      }
    }
    cnt = fl[0] + fl[1] + fl[2] + fl[3];
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
      if (p < E) a.erank[p] = ex;     // rank of p among the tile's firsts (only read for firsts)
      ex += fl[q];
    }
    if (threadIdx.x == 0) a.mtile[tile] = tot;
    __syncthreads();
  }
  tl_mark(TL_MARK | TL_END);
  if (last_block(&a.st[ST_TICKET_B])) mark_finish(a, E, ntiles);
}

// ---- ids.  An edge's dst id = its ref if the node is older than this pass, else ids_base + rank of the node's first
// position.  Firsts append their node to the dst list; the owner of the slot writes the id back unless no later pass
// inserts into this table (then nobody will read it).
// Four edges per thread: the kernel is a chain of dependent loads per edge (ref -> rank of the ref's position ->
// store), and with one edge per thread in flight — the loads of an unrolled iteration could not move above the stores
// of the previous one — it ran at a few percent issue utilisation in a profile of the first version.  Now the four refs and their four rank lookups are issued together through the read-only path (nothing
// this kernel writes is read by it, except colv by the same thread).
__device__ __forceinline__ i64 v2_rank_of(const PassArgs& a, u32 q) {
  return __ldg(&a.mtile[q / ETILE]) + (i64)__ldg(&a.erank[q]);
}
template <bool SH>
__global__ void __launch_bounds__(NT) k_v2_assign(const PassArgs a) {
  pdl_enter(TL_ASSIGN);
  const i64 E = a.st[ST_PASS_E];
  const i64 pbase = a.st[ST_PASS_BASE];
  const i64 list_base = a.st[ST_LIST_BASE], ids_base = a.st[ST_IDS_BASE];
  const u32* __restrict__ xdst = SH ? x_ptr<u32>(a, a.xr, a.x_off_dst) : nullptr;
  // a block takes 1024 consecutive edges per step, thread t the edges base + t + 256 j: every access is coalesced and
  // the four chains of a thread are independent
  for (i64 base = (i64)blockIdx.x * (4 * NT); base < E; base += (i64)gridDim.x * (4 * NT)) {
    u32 r[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const i64 p = base + j * NT + threadIdx.x;
      r[j] = p < E ? __ldg(&a.fref[p]) : 0u;
    }
    if (a.seed_mode) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const i64 p = base + j * NT + threadIdx.x;
        if (p >= E) break;
        const bool first = r[j] == (V2_POS | (u32)p);
        u32 s = a.eslot[p];
        if (first && a.pk_main == nullptr) {
          a.pk[s] = ((u64)(u32)a.dst_nodes[p] << 32) | (u64)v2_rank_of(a, (u32)p);
        } else if (first) {
          // sharded: the dedup ran in the scratch table; the id of a seed this rank owns goes into its partition of the
          // real table (empty of this key: first occurrences are distinct), the others leave no slot to clean up
          const u32 key = (u32)a.dst_nodes[p];
          s = NO_SLOT;
          if (v2_owner(key, a.xw) == a.xr) {
            const u64 mask = (1ull << a.pk_main_bits) - 1, mine = ((u64)key << 32) | (u64)v2_rank_of(a, (u32)p);
            u64 sl = ((u64)key * 0x9E3779B97F4A7C15ull) >> (64 - a.pk_main_bits);
            while (atomicCAS(&a.pk_main[sl], EMPTY, mine) != EMPTY) sl = (sl + 1) & mask;
            s = (u32)sl;
          }
        }
        a.dst_slot[p] = first ? s : NO_SLOT;
      }
      continue;
    }
    i64 id[4], rank[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {   // four independent lookups in flight
      rank[j] = (r[j] & V2_POS) ? v2_rank_of(a, r[j] & ~V2_POS) : 0;
      id[j] = (r[j] & V2_POS) ? ids_base + rank[j] : (i64)r[j];
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const i64 p = base + j * NT + threadIdx.x;
      if (p >= E) break;
      if (SH) a.eid[pbase + p] = a.x_eid64 ? (i64)x_ptr<u64>(a, a.xr, a.x_off_eid)[p] : (i64)x_ptr<u32>(a, a.xr, a.x_off_eid)[p];
      const bool first = r[j] == (V2_POS | (u32)p);
      if (first) {
        const i64 d = SH ? (i64)xdst[p] : a.colv[pbase + p];   // (global id, about to be replaced)
        const u32 s = a.eslot[p];
        a.dst_nodes[list_base + rank[j]] = d;
        a.dst_slot[list_base + rank[j]] = s;
        if (a.v2_writeback && s != NO_SLOT) a.pk[s] = ((u64)(u32)d << 32) | (u64)id[j];
      }
      a.colv[pbase + p] = id[j];
    }
  }
}

__global__ void __launch_bounds__(NT) k_v2_cleanup(u64* pk, const u32* __restrict__ slots, i64 n) {
  for (i64 i = (i64)blockIdx.x * NT + threadIdx.x; i < n; i += (i64)gridDim.x * NT) {
    const u32 s = slots[i];
    if (s != NO_SLOT) pk[s] = EMPTY;
  }
}
