// br_kernels.cu -- CUDA kernels (sm_90a) and the per-stream pipeline that drives them.
//
// Stages of job_compress: host functions that queue kernels on the job's stream and return false on a CUDA error (the
// index and snapshot stages take any stream; the test hooks below call them too).
//   stage_setup     arena, uploads, chunk table (k_build_chunks)
//   stage_index     bucket rings (hash_longest_match64_inc.h Store*): br_build_index, k_slot_pred, k_tags
//   stage_snapshot  the stored bits in S order and their prefix counts (k_build_storedS)
//   stage_fixpoint  EncodeData glue (encode.c:985) k_chain_*, and CreateBackwardReferences / FindLongestMatch: k_walk
//                   launches (a warp per scheduled chunk; k_cover, k_commit, k_verify, k_snapshot_update) to the fixpoint
//   stage_entropy   BrotliBuildMetaBlockGreedy + BrotliStoreMetaBlock: k_compact, E0..E7 (br_entropy2.h)
//   stage_assemble  metablock concatenation and the late uncompressed fallback: k_assemble_scan, k_assemble_copy
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <mutex>
#include <vector>
#include "br_params.h"
#include "br_lz77.h"
#include "br_chain.h"
#include "br_entropy.h"
#include "br_entropy2.h"
#include "br_assemble.h"
#include "br_entropy_flat.h"
#include "br_pipeline.h"
#include "br_probe.h"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { \
  fprintf(stderr, "brotli_b200: CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
  return 0; } } while (0)

// ---------------------------------------------------------------------------- hashing + sort
// Where a radix pass reads its keys: a materialised array, or (qualities 5..9, first pass) the bucket key computed from
// the input on the fly, with the overflow key P.nbuckets for the unhashable tail.  A batch job (P.multi) hashes over the
// whole concatenation, like a single stream.
template <class KT> struct BrKeyArray {
  const KT* k;
  __device__ __forceinline__ u32 operator()(u32 j) const { return k[j]; }
};
struct BrKeyHash {
  BrParams P; const u8* data; u32 hashable;
  __device__ __forceinline__ u32 operator()(u32 j) const { return j < hashable ? br_hash_key(P, data, j) : P.nbuckets; }
};

// qualities 2..4: the key is the table slot of the one-position-per-slot hashers (br_lz77.h br_quick_slot), up to 20 bits
// (+ the overflow key of the unhashable tail): 32-bit keys, three radix passes
// One CTA per input block: the slot depends on the position counted from the first byte of the block's stream (BrBlk::base).
__global__ void k_slot_keys(BrParams P, const u8* __restrict__ data, const BrBlk* __restrict__ blk, u32* __restrict__ keys) {
  const BrBlk B = blk[blockIdx.x];
  const u32 hashable = P.n >= P.htl ? P.n - P.htl + 1 : 0;
  for (u32 p = B.start + threadIdx.x; p < B.end; p += blockDim.x)
    keys[p] = p < hashable ? br_quick_slot(P, br_ld64u(data, p), p - B.base) : P.nbuckets;
}

// qualities 2..4: where the search at position p enters each of its slots' segments (br_lz77.h br_quick_pred_fill); one CTA
// per input block, a thread per position
__global__ void k_slot_pred(BrStream s, u32* __restrict__ qpred) {
  const BrBlk B = s.blk[blockIdx.x];
  for (u32 p = B.start + threadIdx.x; p < B.end; p += blockDim.x)
    br_quick_pred_fill(s, p, B.base, qpred + ((size_t)p << s.P.qk_sweep_bits));
}

// Stable LSD radix sort, 8-bit digits.  A tile of RADIX_TILE elements is one CTA of RADIX_THREADS threads; warp w owns
// the tile's elements [w * RADIX_ROWS * 32, (w + 1) * RADIX_ROWS * 32), row by row, which keeps equal digits in input order.
#define RADIX_TILE 8192
#define RADIX_THREADS 256
#define RADIX_WARPS (RADIX_THREADS / 32)
#define RADIX_ROWS (RADIX_TILE / RADIX_THREADS)
// digit histogram of one tile -> hist[d * ntiles + tile]
template <int SHIFT, class Keys>
__global__ void __launch_bounds__(RADIX_THREADS) k_radix_count(Keys keys, u32 n, u32* __restrict__ hist, u32 ntiles) {
  __shared__ u32 cnt[256];
  cnt[threadIdx.x] = 0;
  __syncthreads();
  const u32 base = blockIdx.x * RADIX_TILE, lane = threadIdx.x & 31;
  for (u32 i = threadIdx.x; i < RADIX_TILE; i += RADIX_THREADS) {
    const u32 j = base + i;
    const u32 d = j < n ? (keys(j) >> SHIFT) & 0xFFu : 0xFFFFFFFFu;
    const u32 m = __match_any_sync(0xffffffffu, d);   // one shared atomic per distinct digit of the row
    if (d != 0xFFFFFFFFu && (m & ((1u << lane) - 1)) == 0) atomicAdd(&cnt[d], (u32)__popc(m));
  }
  __syncthreads();
  hist[threadIdx.x * ntiles + blockIdx.x] = cnt[threadIdx.x];
}
static size_t radix_smem_bytes(size_t key_bytes) { return (RADIX_WARPS + 1) * 256 * 4 + RADIX_TILE * (4 + key_bytes); }
// Stable scatter of one tile.  The tile is first reordered in shared memory into digit order; then consecutive threads
// write each digit's run to consecutive addresses from hist_scanned[d * ntiles + tile] on, so the stores coalesce.
// Values: vals[j], or the position j itself in a first pass (HAS_VALS false).
// `rk` (nullable) gets rk[j] = the element's index in this pass's output, written by input index j (coalesced).  A first
// pass's rk is the inverse permutation of its scatter by position; a later pass's rk may alias `vals`, because each index
// j is read and then written by the same thread.  k_rank_compose chains them into BrStream::rank.
// (Two CTAs per SM: the tile's keys stay in registers between the count and the placement.)
template <int SHIFT, bool HAS_VALS, class KT, class Keys>
__global__ void __launch_bounds__(RADIX_THREADS, 2) k_radix_scatter(Keys keys, const u32* vals, u32 n,
    const u32* __restrict__ hist_scanned, u32 ntiles, KT* __restrict__ out_keys, u32* __restrict__ out_vals, u32* rk) {
  extern __shared__ u32 smem[];
  u32 (*wcnt)[256] = (u32 (*)[256])smem;         // per warp and digit: count, then the warp's first tile-local index
  u32* gbase = smem + RADIX_WARPS * 256;           // per digit: output index of tile-local index 0
  u32* sv = gbase + 256;                           // the tile in digit order: values ...
  KT* sk = (KT*)(sv + RADIX_TILE);                 // ... and keys
  const u32 warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (u32 i = threadIdx.x; i < RADIX_WARPS * 256; i += RADIX_THREADS) smem[i] = 0;
  __syncthreads();
  const u32 tbase = blockIdx.x * RADIX_TILE, wbase = warp * (RADIX_ROWS * 32);
  u32 k[RADIX_ROWS];
#pragma unroll
  for (u32 r = 0; r < RADIX_ROWS; ++r) {
    const u32 j = tbase + wbase + r * 32 + lane;
    k[r] = j < n ? keys(j) : 0;
  }
#pragma unroll
  for (u32 r = 0; r < RADIX_ROWS; ++r) {
    const u32 j = tbase + wbase + r * 32 + lane;
    const u32 d = j < n ? (k[r] >> SHIFT) & 0xFFu : 0xFFFFFFFFu;
    const u32 m = __match_any_sync(0xffffffffu, d);
    if (d != 0xFFFFFFFFu && (m & ((1u << lane) - 1)) == 0) wcnt[warp][d] += __popc(m);
    __syncwarp();
  }
  __syncthreads();
  {  // thread d: the digit's tile-local start (exclusive scan over the digits), its output base and the warps' starts
    __shared__ u32 wsum[RADIX_WARPS];
    const u32 d = threadIdx.x;
    u32 c = 0;
    for (u32 w = 0; w < RADIX_WARPS; ++w) c += wcnt[w][d];
    u32 x = c;
    for (int o = 1; o < 32; o <<= 1) { const u32 t = __shfl_up_sync(0xffffffffu, x, o); if (lane >= (u32)o) x += t; }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    u32 start = x - c;
    for (u32 w = 0; w < warp; ++w) start += wsum[w];
    gbase[d] = hist_scanned[d * ntiles + blockIdx.x] - start;
    for (u32 w = 0; w < RADIX_WARPS; ++w) { const u32 t = wcnt[w][d]; wcnt[w][d] = start; start += t; }
  }
  __syncthreads();
#pragma unroll
  for (u32 r = 0; r < RADIX_ROWS; ++r) {
    const u32 j = tbase + wbase + r * 32 + lane;
    const u32 d = j < n ? (k[r] >> SHIFT) & 0xFFu : 0xFFFFFFFFu;
    const u32 m = __match_any_sync(0xffffffffu, d);
    const u32 before = __popc(m & ((1u << lane) - 1));
    if (j < n) {
      const u32 loc = wcnt[warp][d] + before;
      sk[loc] = (KT)k[r];
      sv[loc] = HAS_VALS ? vals[j] : j;
      if (rk) rk[j] = gbase[d] + loc;   // (after this thread's read of vals[j]: the only access to index j)
    }
    __syncwarp();
    if (d != 0xFFFFFFFFu && before == 0) wcnt[warp][d] += __popc(m);
    __syncwarp();
  }
  __syncthreads();
  const u32 len = n - tbase < RADIX_TILE ? n - tbase : RADIX_TILE;
  for (u32 i = threadIdx.x; i < len; i += RADIX_THREADS) {
    const u32 kk = sk[i];
    const u32 dst = gbase[(kk >> SHIFT) & 0xFFu] + i;
    out_keys[dst] = (KT)kk;
    out_vals[dst] = sv[i];
  }
}
// rank[p] = r_last[r_mid[rank[p]]] (r_mid nullable), in place: on entry rank holds the first pass's rk
__global__ void k_rank_compose(u32* __restrict__ rank, const u32* __restrict__ r_mid, const u32* __restrict__ r_last, u32 n) {
  const u32 p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  u32 i = rank[p];
  if (r_mid) i = r_mid[i];
  rank[p] = r_last[i];
}
static void scan_exclusive(u32* a, u32 n, u32* tmp, cudaStream_t st);
// one radix pass: histogram, its scan, scatter
template <int SHIFT, bool HAS_VALS, class KT, class Keys>
static void radix_pass(Keys keys, const u32* vals, u32 n, u32* hist, u32* scan_tmp, KT* out_keys, u32* out_vals, u32* rk,
                       cudaStream_t st) {
  const u32 ntiles = (n + RADIX_TILE - 1) / RADIX_TILE;
  const int smem = (int)radix_smem_bytes(sizeof(KT));
  cudaFuncSetAttribute(k_radix_scatter<SHIFT, HAS_VALS, KT, Keys>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  k_radix_count<SHIFT><<<ntiles, RADIX_THREADS, 0, st>>>(keys, n, hist, ntiles);
  scan_exclusive(hist, 256 * ntiles, scan_tmp, st);
  k_radix_scatter<SHIFT, HAS_VALS, KT><<<ntiles, RADIX_THREADS, smem, st>>>(keys, vals, n, hist, ntiles, out_keys, out_vals, rk);
}
// chunk table of one input block (br_params.h br_chunk_in): one CTA per block
__global__ void k_build_chunks(const BrBlk* __restrict__ blk, BrBlockIn* __restrict__ bin, u32 ch) {
  const BrBlk B = blk[blockIdx.x];
  for (u32 c = threadIdx.x; c < B.nchunks; c += blockDim.x) bin[B.first_chunk + c] = br_chunk_in(B, blockIdx.x, c, ch);
}
// tagS[j] = tag of the position S[j] (br_lz77.h br_tag4)
__global__ void k_tags(const u8* __restrict__ data, const u32* __restrict__ S, u32 n, u16* __restrict__ tagS) {
  u32 j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) tagS[j] = (u16)br_tag4(br_ld32u(data, S[j]));
}
// seg[k] = first index in S whose key is >= k, for k in [0, nbuckets + 1]
template <class KT>
__global__ void k_seg(const KT* __restrict__ sorted_keys, u32 n, u32 nbuckets, u32* __restrict__ seg) {
  u32 j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j > n) return;
  int k0 = j == 0 ? -1 : (int)sorted_keys[j - 1];
  int k1 = j == n ? (int)nbuckets + 1 : (int)sorted_keys[j];
  for (int k = k0 + 1; k <= k1; ++k) seg[k] = j;
}

// Buffers of the position index (n elements each unless noted).  Qualities 5..9 use K1, V1, K2; qualities 2..4 the four
// 32-bit arrays qk_*.  tagS is filled by k_tags.
struct BrIndexBufs {
  u16 *K1, *K2, *tagS;                       // K2: the sorted bucket keys (BrStream::skeys)
  u32 *V1, *S, *rank, *seg;                  // seg: nbuckets + 2 words
  u32 *hist, *scan_tmp;                      // 256 * ntiles words and scan_tmp_words of that
  u32 *qk_keys, *qk_K1, *qk_V1, *qk_V2;
};
// S, rank and seg of the input (and K2 at qualities 5..9), queued on st.  blk / nblk: the input blocks (the slot keys of
// qualities 2..4 count positions from BrBlk::base).
static void br_build_index(const BrParams& P, const u8* data, const BrBlk* blk, u32 nblk, const BrIndexBufs& b, cudaStream_t st) {
  const u32 n = P.n;
  if (P.quick) {
    // sorted by (slot, position): three stable 8-bit passes over 32-bit keys (slots have up to 20 bits + the overflow key);
    // rank = r3[r2[inv1]]: the two later passes' rk alias the values they have read
    k_slot_keys<<<nblk, 256, 0, st>>>(P, data, blk, b.qk_keys);
    radix_pass<0, false>(BrKeyArray<u32>{b.qk_keys}, nullptr, n, b.hist, b.scan_tmp, b.qk_K1, b.qk_V1, b.rank, st);
    radix_pass<8, true>(BrKeyArray<u32>{b.qk_K1}, b.qk_V1, n, b.hist, b.scan_tmp, b.qk_keys, b.qk_V2, b.qk_V1, st);
    radix_pass<16, true>(BrKeyArray<u32>{b.qk_keys}, b.qk_V2, n, b.hist, b.scan_tmp, b.qk_K1, b.S, b.qk_V2, st);
    k_rank_compose<<<(n + 255) / 256, 256, 0, st>>>(b.rank, b.qk_V1, b.qk_V2, n);
    k_seg<u32><<<(n + 1 + 255) / 256, 256, 0, st>>>(b.qk_K1, n, P.nbuckets, b.seg);
  } else {
    // two passes over the 16-bit bucket keys, hashed from the input in the first; rank = r1[inv1], r1 aliasing V1
    const BrKeyHash hk{P, data, n >= P.htl ? n - P.htl + 1 : 0};
    radix_pass<0, false>(hk, nullptr, n, b.hist, b.scan_tmp, b.K1, b.V1, b.rank, st);
    radix_pass<8, true>(BrKeyArray<u16>{b.K1}, b.V1, n, b.hist, b.scan_tmp, b.K2, b.S, b.V1, st);
    k_rank_compose<<<(n + 255) / 256, 256, 0, st>>>(b.rank, nullptr, b.V1, n);
    k_seg<u16><<<(n + 1 + 255) / 256, 256, 0, st>>>(b.K2, n, P.nbuckets, b.seg);
  }
}

// ---------------------------------------------------------------------------- exclusive scan
#define SCAN_CHUNK 2048
__global__ void __launch_bounds__(256) k_scan_chunks(u32* __restrict__ a, u32 n, u32* __restrict__ sums) {
  __shared__ u32 part[256];
  u32 base = blockIdx.x * SCAN_CHUNK + threadIdx.x * 8;
  u32 v[8], acc = 0;
  for (int i = 0; i < 8; ++i) { v[i] = base + i < n ? a[base + i] : 0; acc += v[i]; }
  part[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 1; o < 256; o <<= 1) {
    u32 t = threadIdx.x >= (u32)o ? part[threadIdx.x - o] : 0;
    __syncthreads();
    part[threadIdx.x] += t;
    __syncthreads();
  }
  u32 run = part[threadIdx.x] - acc;
  for (int i = 0; i < 8; ++i) { if (base + i < n) a[base + i] = run; run += v[i]; }
  if (threadIdx.x == 255) sums[blockIdx.x] = part[255];
}
__global__ void k_scan_add(u32* __restrict__ a, u32 n, const u32* __restrict__ sums) {
  u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] += sums[i / SCAN_CHUNK];
}
// in-place exclusive scan of a[0..n); tmp must hold >= n/SCAN_CHUNK + n/SCAN_CHUNK^2 + 8 words
static void scan_exclusive(u32* a, u32 n, u32* tmp, cudaStream_t st) {
  if (n == 0) return;
  u32 chunks = (n + SCAN_CHUNK - 1) / SCAN_CHUNK;
  k_scan_chunks<<<chunks, 256, 0, st>>>(a, n, tmp);
  if (chunks > 1) {
    scan_exclusive(tmp, chunks, tmp + chunks, st);
    k_scan_add<<<(n + 255) / 256, 256, 0, st>>>(a, n, tmp);
  }
}

// ---------------------------------------------------------------------------- stored bits
// Initial speculation (br_chain.h br_init_bits): one CTA per input block (blocks cut by a FLUSH are irregular).
__global__ void k_init_bits(BrStream s) { br_init_bits(s, blockIdx.x, threadIdx.x, blockDim.x); }
// bits_latest permuted into S order + per-1024 popcounts: the first snapshot of a job (br_snapshot_update keeps it)
__global__ void __launch_bounds__(1024) k_build_storedS(BrStream s, u32* __restrict__ storedS, u32* __restrict__ blockcnt) {
  __shared__ u32 wsum[32];
  u32 j = blockIdx.x * 1024 + threadIdx.x;
  int bit = 0;
  if (j < s.P.n) { u32 q = s.S[j]; bit = (s.bits_latest[q >> 5] >> (q & 31)) & 1; }
  u32 m = __ballot_sync(0xffffffffu, bit);
  if ((threadIdx.x & 31) == 0) { storedS[j >> 5] = m; wsum[threadIdx.x >> 5] = __popc(m); }
  __syncthreads();
  if (threadIdx.x < 32) {
    u32 v = wsum[threadIdx.x];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) blockcnt[blockIdx.x] = v;
  }
}

__global__ void k_snapshot_update(BrStream s, u32* __restrict__ storedS, u32* __restrict__ cntS) {
  const u32 x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x < s.bits_words) br_snapshot_update(s, x, storedS, cntS);
}

// ---------------------------------------------------------------------------- warp-task kernels
// k_walk<F, M>: the walker form F and M as br_walk_dispatch (br_params.h) picks them; BR_WALK_WARPS warps per block
#ifndef BR_WALK1_MINB
#define BR_WALK1_MINB 8
#endif
template <int F, bool M>
__global__ void __launch_bounds__(32 * BR_WALK_WARPS, BR_FORM_G(F) <= 2 ? BR_WALK1_MINB : BR_FORM_G(F) == 4 ? 5 : 4)
k_walk(BrStream s) {
  u32 t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (t >= s.counters[5]) return;
  const u32 b = br_sched_entry(s, t);
  br_walk_block<F, M>(s, b, s.forced && b == s.counters[6]);
}
// positions covered by the runs of this launch (br_chain.h br_cover_run); before k_commit
__global__ void k_cover(BrStream s) {
  u32 t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (t >= s.counters[4]) return;
  br_cover_run(s, s.ran_list[t]);
}
__global__ void k_commit(BrStream s) {
  u32 t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (t >= s.counters[4]) return;
  br_commit_bits(s, s.ran_list[t]);
}
// qualities 2..4: every run against the committed stored-bits (br_chain.h br_verify_run); warp per chunk
__global__ void k_verify(BrStream s) {
  u32 t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (t >= s.P.nblocks) return;
  br_verify_run(s, t);
}
__global__ void k_chain_a(BrStream s) {
  u32 bi = blockIdx.x * blockDim.x + threadIdx.x;
  if (bi < s.nblk) br_chain_a(s, bi);
}
__global__ void __launch_bounds__(32) k_chain_b(BrStream s) { br_chain_b(s); }
__global__ void __launch_bounds__(128) k_chain_b1(BrStream s) {   // batch of streams: a warp per stream
  const u32 st = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (st < s.P.multi) br_chain_b1(s, st);
}
__global__ void __launch_bounds__(32) k_chain_b2(BrStream s) { br_chain_b2(s); }
__global__ void k_chain_b3(BrStream s) {
  const u32 bi = blockIdx.x * blockDim.x + threadIdx.x;
  if (bi < s.nblk) br_chain_b3(s, bi);
}
__global__ void k_chain_c(BrStream s) {
  u32 bi = blockIdx.x * blockDim.x + threadIdx.x;
  if (bi < s.nblk) br_chain_c(s, bi);
}
__global__ void k_chain_d(BrStream s) {
  u32 k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < s.P.nblocks) br_chain_d(s, k);
}
__global__ void k_compact(BrStream s, BrCmd* cmds_all, const u32* __restrict__ block_mb) {
  u32 t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (t >= s.P.nblocks) return;
  br_compact_block(s, t, cmds_all, block_mb);
}
// ---- data-parallel entropy stage (br_entropy2.h)
__global__ void k_cmd_scan_inputs(const BrCmd* __restrict__ cmds, u32 C, u32* ins, u32* span, u32* hasd) {
  u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > C) return;
  u32 a = 0, b = 0, d = 0;
  if (i < C) br_cmd_scan_inputs(cmds[i], &a, &b, &d);
  ins[i] = a; span[i] = b; hasd[i] = d;
}
__global__ void k_cmd_mb(BrStream s, u32* cmd_mb, u32 n_mbs) {
  // (grid.y is capped at 65535: 16 KiB input blocks of noise at quality 2, 3 make up to 65536 metablocks per GiB)
  for (u32 m = blockIdx.y; m < n_mbs; m += gridDim.y) {
    const BrMetaBlock mb = s.mbs[m];
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < mb.ncmd; i += gridDim.x * blockDim.x) cmd_mb[mb.cmd_off + i] = m;
  }
}
__global__ void k_expand(BrEnt e) {
  u32 w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (w * 32 >= e.total_cmds) return;
  br_expand_cmds(e, w * 32);
}
// one CTA per metablock: literal context model (its histograms in shared memory) + bookkeeping
__global__ void __launch_bounds__(256) k_mb_setup(BrStream s, BrEnt e) {
  __shared__ u32 hist[14 * 32];
  const u32 i = blockIdx.x;
  const BrMetaBlock mb = s.mbs[i];
  if (!mb.compress) return;
  u32 which = s.P.disable_ctx ? 1u : br_decide_context_modeling(s, mb.start, mb.end - mb.start, hist);
  if (threadIdx.x == 0) {
    BrMbAux a;
    br_mb_aux_init(a, mb, e, which);
    e.aux[i] = a;
  }
}
// E3's symbol arrays (br_split_syms) of every compressed metablock; grid.y = metablock (capped, see k_cmd_mb), grid.x
// strides over its literals and commands
__global__ void k_split_syms(BrStream s, BrEnt e, u32 n_mbs) {
  for (u32 m = blockIdx.y; m < n_mbs; m += gridDim.y) {
    const BrMetaBlock mb = s.mbs[m];
    if (!mb.compress) continue;
    const BrMbAux a = e.aux[m];
    const u32 n = mb.nlit > mb.ncmd ? mb.nlit : mb.ncmd;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) br_split_syms(s, e, mb, a, i);
  }
}
__global__ void __launch_bounds__(256) k_split(BrStream s, BrEnt e) {
  extern __shared__ u32 sm[];
  const u32 i = blockIdx.x; const int cat = (int)blockIdx.y;
  const BrMetaBlock mb = s.mbs[i];
  if (!mb.compress) return;
  BrMbAux& a = e.aux[i];
  u8* sc = e.scratch + e.scratch_off[i];
  BrMbMem* M = (BrMbMem*)sc;
  const u32 A = BR_SPLIT_ALPHABET(cat), nc = BR_SPLIT_CONTEXTS(cat, a.which);
  const u32 minb = BR_SPLIT_MIN_BLOCK(cat);
  const double thr = BR_SPLIT_THR(cat);
  u32* H = BR_SPLIT_HIST(M, cat);
  u32 nblk = br_mb2_nblk(cat, mb.nlit, mb.ncmd);
  br_split_cta(s, e, mb, a, cat, A, nc, minb, thr, a.nsym[cat], br_mb2_types(sc, a, cat, nblk),
               br_mb2_lengths(sc, a, cat, nblk), H, sm);
}
// E4 (br_entropy2.h): code_base[i] = number of prefix codes of metablock i (0 when it is stored raw), then scanned
__global__ void k_code_count(BrStream s, BrEnt e, u32* code_base, u32 n_mbs) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_mbs) code_base[i] = s.mbs[i].compress ? br_mb_code_count(e.aux[i]) : 0u;
  else if (i == n_mbs) code_base[i] = 0;
}
// At most BR_CODE_WARP_MAX codes in the job: one warp per code, (metablock, code) of global code t from the scanned counts.
template <bool STORE>
__global__ void __launch_bounds__(32) k_codes_warp(BrStream s, BrEnt e, const u32* __restrict__ code_base, u32 n_mbs) {
  __shared__ BrCodeSmem S;
  const u32 total = code_base[n_mbs], t = blockIdx.x;
  if (total > BR_CODE_WARP_MAX || t >= total) return;
  const u32 m = br_upper_index(code_base, n_mbs, t);
  const BrMetaBlock& mb = s.mbs[m];
  u8* sc = e.scratch + e.scratch_off[m];
  if (STORE) br_code_store_warp(mb, e.aux[m], sc, t - code_base[m], &S, e.outbits + e.out_off[m]);
  else br_code_build_warp(mb, e.aux[m], sc, t - code_base[m], &S);
}
// More codes: one thread per code, every worker taking the codes gridDim.x * blockDim.x apart.
template <bool STORE>
__global__ void __launch_bounds__(64) k_codes(BrStream s, BrEnt e, const u32* __restrict__ code_base, u32 n_mbs, BrHTree* pool) {
  const u32 wk = blockIdx.x * blockDim.x + threadIdx.x, nwk = gridDim.x * blockDim.x;
  BrHTree* tree = pool + (size_t)wk * BR_CODE_TREE_NODES;
  const u32 total = code_base[n_mbs];
  if (total <= BR_CODE_WARP_MAX) return;
  for (u32 t = wk; t < total; t += nwk) {
    const u32 m = br_upper_index(code_base, n_mbs, t);
    const BrMetaBlock& mb = s.mbs[m];
    u8* sc = e.scratch + e.scratch_off[m];
    if (STORE) br_code_store(mb, e.aux[m], sc, t - code_base[m], tree, e.outbits + e.out_off[m]);
    else br_code_build(mb, e.aux[m], sc, t - code_base[m], tree);
  }
}
__global__ void __launch_bounds__(32) k_mb_header(BrStream s, BrEnt e) {
  const u32 i = blockIdx.x;
  const BrMetaBlock mb = s.mbs[i];
  if (!mb.compress) return;
  br_mb_header(s, mb, e.aux[i], e.scratch + e.scratch_off[i], e.outbits + e.out_off[i]);
}
// qualities 2, 3: histograms + the three codes of a metablock without block splits (br_entropy_flat.h)
__global__ void __launch_bounds__(64) k_prep_flat(BrStream s, BrEnt e) {
  const u32 i = blockIdx.x;
  const BrMetaBlock mb = s.mbs[i];
  if (!mb.compress) return;
  br_prep_flat(s, e, mb, e.aux[i], e.scratch + e.scratch_off[i], e.outbits + e.out_off[i]);
}
__global__ void k_lit_bits(BrStream s, BrEnt e) {
  u32 o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o < e.total_lits) br_lit_bits(s, e, o);
  else if (o == e.total_lits) e.lit_len[o] = 0;
}
__global__ void k_cmd_bits(BrStream s, BrEnt e) {
  u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < e.total_cmds) br_cmd_bits(s, e, i);
  else if (i == e.total_cmds) e.cmd_len[i] = 0;
}
__global__ void k_emit_cmd(BrStream s, BrEnt e) {
  u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < e.total_cmds) br_emit_cmd(s, e, i);
}
__global__ void k_emit_lit(BrStream s, BrEnt e) {
  u32 o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o < e.total_lits) br_emit_lit(s, e, o);
}

// ---------------------------------------------------------------------------- stream assembly
__global__ void k_assemble_scan(BrStream s, const u64* __restrict__ out_off, u32* out, BrCopyDesc* desc, u32* res,
                                int with_header, const u32* __restrict__ cut_kind, u64* cut_end_bit, u64* stream_end) {
  if (threadIdx.x == 0) br_assemble_scan(s, out_off, out, desc, res, with_header, cut_kind, cut_end_bit, stream_end);
}
// grid.y = metablock, grid.x strides over its words (br_assemble.h br_copy_word)
__global__ void k_assemble_copy(BrStream s, const BrCopyDesc* __restrict__ desc, const u32* __restrict__ outbits, u32* out, u32 n_mbs) {
  for (u32 m = blockIdx.y; m < n_mbs; m += gridDim.y) {   // (grid.y is capped at 65535, see k_cmd_mb)
    const BrCopyDesc d = desc[m];
    const u32 nw = br_copy_words(d);
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < nw; i += gridDim.x * blockDim.x) br_copy_word(d, i, outbits, s.data, out);
  }
}

// ============================================================================ host pipeline
struct BrDeviceTables {
  int device = -1;
  u8* blob = nullptr;       // brotli_tables.bin on the device
  double* log2tab = nullptr;
  u32 log2tab_n = 0;
};
static BrDeviceTables g_tables[16];
static std::mutex g_tables_mu;

extern "C" const unsigned char br_tables_blob[];
extern "C" const unsigned int br_tables_blob_len;
extern "C" const double* br_host_log2_table(u32* n);   // br_host.cc

// Per-device constant tables, uploaded once.  Jobs of several host threads (BrotliB200CompressBatch) come here
// concurrently: the init is serialised, the uploads are synchronous copies that have completed before `device` is
// published, so kernels on any (non-blocking) stream launched afterwards see the finished tables.
static BrDeviceTables* get_tables() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 16) return nullptr;
  std::lock_guard<std::mutex> lock(g_tables_mu);
  BrDeviceTables& t = g_tables[dev];
  if (t.device == dev) return &t;
  u8* blob = nullptr; double* l2 = nullptr;
  u32 n = 0; const double* h = br_host_log2_table(&n);
  if (cudaMalloc(&blob, br_tables_blob_len) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  if (cudaMalloc(&l2, (size_t)n * 8) != cudaSuccess) { cudaGetLastError(); cudaFree(blob); return nullptr; }
  if (cudaMemcpy(blob, br_tables_blob, br_tables_blob_len, cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(l2, h, (size_t)n * 8, cudaMemcpyHostToDevice) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) {
    cudaGetLastError(); cudaFree(blob); cudaFree(l2); return nullptr;
  }
  t.blob = blob; t.log2tab = l2; t.log2tab_n = n;
  t.device = dev;
  return &t;
}

// Grow-only device arena owned by a job; all per-stream arrays are carved out of it.
struct BrArena {
  u8* base = nullptr; size_t cap = 0;
  bool reserve(size_t bytes) {
    if (bytes <= cap) return true;
    if (base) cudaFree(base);
    base = nullptr; cap = 0;
    if (cudaMalloc(&base, bytes) != cudaSuccess) { cudaGetLastError(); return false; }
    cap = bytes; return true;
  }
  void release() { if (base) cudaFree(base); base = nullptr; cap = 0; }
};
// Lays arrays out one behind the other, 256-byte aligned, from base; with base == nullptr it only counts the bytes.
struct BrCarve {
  u8* base; size_t used;
  template <class T> T* take(size_t count) {
    const size_t off = (used + 255) & ~(size_t)255;
    used = off + count * sizeof(T);
    return base ? (T*)(base + off) : nullptr;
  }
};
// Every arena is laid out by one function, carve(BrCarve&), run twice: to measure, then to assign from the arena.
template <class F> static bool br_carve(BrArena& A, F&& carve) {
  BrCarve m{nullptr, 0};
  carve(m);
  if (!A.reserve(m.used)) return false;
  BrCarve c{A.base, 0};
  carve(c);
  return true;
}

struct BrJob {
  cudaStream_t st = nullptr;
  BrArena arena, arena2;     // arena2: metablock scratch / bit buffers / output (sized after LZ77)
  u32* h_pinned = nullptr;    // small pinned readback area
  cudaEvent_t ev[10] = {};    // stage timers, created once per job
  BrJobStats stats;
};

extern "C" void br_job_destroy(BrJob* j);
extern "C" BrJob* br_job_create(void) {
  BrJob* j = new BrJob();
  if (cudaStreamCreateWithFlags(&j->st, cudaStreamNonBlocking) != cudaSuccess) { delete j; return nullptr; }
  if (cudaMallocHost(&j->h_pinned, 4096) != cudaSuccess) { cudaStreamDestroy(j->st); delete j; return nullptr; }
  for (auto& e : j->ev) if (cudaEventCreate(&e) != cudaSuccess) { br_job_destroy(j); return nullptr; }
  return j;
}
extern "C" void br_job_destroy(BrJob* j) {
  if (!j) return;
  j->arena.release(); j->arena2.release();
  for (auto& e : j->ev) if (e) cudaEventDestroy(e);
  if (j->h_pinned) cudaFreeHost(j->h_pinned);
  if (j->st) cudaStreamDestroy(j->st);
  delete j;
}
extern "C" const BrJobStats* br_job_stats(const BrJob* j) { return &j->stats; }
extern "C" void* br_job_stream(BrJob* j) { return (void*)j->st; }

static size_t scan_tmp_words(size_t n) { return n / SCAN_CHUNK + n / SCAN_CHUNK / SCAN_CHUNK + 64; }

// E4 (br_entropy2.h): every prefix code of the job built by its own worker, the headers, then every code stored.
// code_base: n_mbs + 1 words; stmp: scan_tmp_words(n_mbs + 1).  code_ctas: CTAs of thread workers (64 each) when the job
// has more than BR_CODE_WARP_MAX codes, 0 for L.code_workers of them; tree_pool holds BR_CODE_TREE_NODES for each.
static u32 codes_ctas(const BrMbLayout& L, u32 code_ctas) { return code_ctas ? code_ctas : (L.code_workers + 63) / 64; }
static void launch_codes(const BrStream& s, const BrEnt& e, const BrMbLayout& L, u32 n_mbs, u32* code_base, u32* stmp,
                         BrHTree* tree_pool, u32 code_ctas, cudaStream_t st) {
  k_code_count<<<(n_mbs + 1 + 255) / 256, 256, 0, st>>>(s, e, code_base, n_mbs);
  scan_exclusive(code_base, n_mbs + 1, stmp, st);
  const u32 ctas = L.code_workers ? codes_ctas(L, code_ctas) : 0u;
  if (L.code_warps) k_codes_warp<false><<<L.code_warps, 32, 0, st>>>(s, e, code_base, n_mbs);
  if (ctas) k_codes<false><<<ctas, 64, 0, st>>>(s, e, code_base, n_mbs, tree_pool);
  k_mb_header<<<n_mbs, 32, 0, st>>>(s, e);
  if (L.code_warps) k_codes_warp<true><<<L.code_warps, 32, 0, st>>>(s, e, code_base, n_mbs);
  if (ctas) k_codes<true><<<ctas, 64, 0, st>>>(s, e, code_base, n_mbs, tree_pool);
}
// E2 (the literal context decision and the metablock's BrMbAux) and, at qualities 4..9, E3 (the block splits and their
// histograms): what launch_codes starts from.  Returns false on a CUDA error.
static bool launch_split(const BrStream& s, const BrEnt& e, u32 n_mbs, cudaStream_t st) {
  k_mb_setup<<<n_mbs, 256, 0, st>>>(s, e);
  if (s.P.mb_kind) return true;
  k_split_syms<<<dim3(64, n_mbs < 65535u ? n_mbs : 65535u), 256, 0, st>>>(s, e, n_mbs);
  const size_t smem_split = br_split_smem_bytes(256, 13) > br_split_smem_bytes(704, 1) ? br_split_smem_bytes(256, 13) : br_split_smem_bytes(704, 1);
  CK(cudaFuncSetAttribute(k_split, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_split));
  k_split<<<dim3(n_mbs, 3), 256, smem_split, st>>>(s, e);
  return true;
}

// The position index's arrays and tagS, in arena order; at qualities 2..4 carve_index_quick adds the 32-bit sort arrays.
static void carve_index(BrCarve& A, const BrParams& P, BrIndexBufs& b) {
  const size_t n = P.n, ntiles = (n + RADIX_TILE - 1) / RADIX_TILE;
  b.K1 = A.take<u16>(n + 2); b.V1 = A.take<u32>(n);
  b.K2 = A.take<u16>(n + 2); b.S = A.take<u32>(n); b.rank = A.take<u32>(n); b.tagS = A.take<u16>(n + 2);
  b.hist = A.take<u32>(256 * ntiles); b.scan_tmp = A.take<u32>(scan_tmp_words(256 * ntiles));
  b.seg = A.take<u32>(P.nbuckets + 4);
}
static void carve_index_quick(BrCarve& A, const BrParams& P, BrIndexBufs& b) {
  if (!P.quick) return;
  const size_t n = P.n;
  b.qk_keys = A.take<u32>(n + 4); b.qk_K1 = A.take<u32>(n + 4); b.qk_V1 = A.take<u32>(n + 4); b.qk_V2 = A.take<u32>(n + 4);
}

// The job's device arrays that BrStream does not hold.  Main arena (stage_setup): the index's sort buffers, the stored
// bits of every 1024 positions of S (cntS, scanned into prefS with scan_tmp2) and the cut and stream-end records.
// arena2 (carve_entropy): the entropy stage's arrays and the assembled output.
struct BrJobBufs {
  BrIndexBufs ix; u32 *cntS, *scan_tmp2, *cut_kind; u64 *cut_end, *stream_end;
  BrEnt e; u32 *out, *res, *code_base, *stmp; BrCopyDesc* desc; BrHTree* tree_pool;
};
// arena2 in arena order: the metablocks' scratch and bit buffers (L), the output, and the entropy stage's arrays for C
// commands over n input bytes.  e gets every array and zero totals.  pool_workers: the E4 thread workers that the tree
// pool holds a tree area for.
static void carve_entropy(BrCarve& B, const BrMbLayout& L, size_t n, size_t C, size_t pool_workers, BrJobBufs& b) {
  const size_t n_mbs = L.scratch_off.size();
  BrEnt& e = b.e;
  memset(&e, 0, sizeof(e));
  e.scratch = B.take<u8>(L.scratch_bytes + 256); e.outbits = B.take<u32>(L.out_words + 64);
  b.out = B.take<u32>(L.out_cap / 4 + 16); e.cmds = B.take<BrCmd>(C + 1);
  e.scratch_off = B.take<u64>(n_mbs); e.out_off = B.take<u64>(n_mbs);
  b.desc = B.take<BrCopyDesc>(n_mbs); b.res = B.take<u32>(16);
  e.lit_ord = B.take<u32>(C + 2); e.cmd_pos = B.take<u32>(C + 2); e.dist_ord = B.take<u32>(C + 2);
  e.cmd_len = B.take<u32>(C + 2); e.lit_bit_base = B.take<u32>(C + 2); e.cmd_mb = B.take<u32>(C + 2);
  e.dist_sym = B.take<u16>(C + 16); e.cmd_sym = B.take<u16>(C + 16); e.lit_sym = B.take<u16>(n + 16);
  e.lit_pos = B.take<u32>(n + 2); e.lit_cmd = B.take<u32>(n + 2); e.lit_len = B.take<u32>(n + 2);
  e.aux = B.take<BrMbAux>(n_mbs);
  b.code_base = B.take<u32>(n_mbs + 1);
  b.tree_pool = B.take<BrHTree>(pool_workers * BR_CODE_TREE_NODES);
  b.stmp = B.take<u32>(scan_tmp_words(n + C + 8) * 2);
}
// E0 and E1 (br_entropy2.h) over the C commands of e: their ordinals with the totals read back into e (through `totals`,
// two host words), each command's metablock, each literal's position and command.  False on a CUDA error or on more
// literals than input bytes.
static bool launch_e01(const BrStream& s, BrEnt& e, u32 C, u32 n_mbs, u32* stmp, u32* totals, cudaStream_t st) {
  e.total_cmds = C;
  u32 *lit_ord = (u32*)e.lit_ord, *cmd_pos = (u32*)e.cmd_pos, *dist_ord = (u32*)e.dist_ord;
  k_cmd_scan_inputs<<<(C + 1 + 255) / 256, 256, 0, st>>>(e.cmds, C, lit_ord, cmd_pos, dist_ord);
  scan_exclusive(lit_ord, C + 1, stmp, st);
  scan_exclusive(cmd_pos, C + 1, stmp, st);
  scan_exclusive(dist_ord, C + 1, stmp, st);
  CK(cudaMemcpyAsync(totals, lit_ord + C, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(totals + 1, dist_ord + C, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  e.total_lits = totals[0]; e.total_dist = totals[1];
  if (e.total_lits > s.P.n) return false;
  k_cmd_mb<<<dim3(64, n_mbs < 65535u ? n_mbs : 65535u), 256, 0, st>>>(s, e.cmd_mb, n_mbs);
  k_expand<<<(C + 127) / 128 + 1, 128, 0, st>>>(e);
  return true;
}

// Setup: the main arena carved (s's arrays, b's), the input and the plan's tables uploaded, the chunk table built and the
// fixpoint's state cleared.  s.P: the plan's parameters.
static bool stage_setup(BrJob* job, BrStream& s, const BrDeviceTables* T, const BrStreamPlan& plan, const BrCuts* cuts,
                        const u8* d_in, BrJobBufs& b) {
  const BrParams& P = s.P;
  const u32 n = P.n, nb = P.nblocks, nblk = (u32)plan.blk.size(), ncuts = cuts ? cuts->n : 0, nstreams = plan.nstreams;
  const size_t nwords = (size_t)(n + 31) / 32 + 2;
  cudaStream_t st = job->st;
  s.bits_words = (u32)nwords; s.cmd_stride = plan.cmd_stride; s.nblk = nblk;
  auto carve = [&](BrCarve& A) {
    s.data = A.take<u8>((size_t)n + 64);
    carve_index(A, P, b.ix);
    s.bits_latest = A.take<u32>(nwords); s.bits_cur = A.take<u32>(2 * nwords);
    s.srch_latest = A.take<u32>(nwords); s.srch_cur = A.take<u32>(nwords); s.bits_prev = A.take<u32>(nwords);
    s.cover_cur = A.take<u32>(nwords);
    s.storedS = A.take<u32>(nwords + 64); s.prefS = A.take<u32>((size_t)n / 1024 + 8); b.cntS = A.take<u32>((size_t)n / 1024 + 8);
    b.scan_tmp2 = A.take<u32>(scan_tmp_words((size_t)n / 1024 + 8));
    s.bin = A.take<BrBlockIn>(nb); s.bin_used = A.take<BrBlockIn>(nb);
    s.bout = A.take<BrBlockOut>(nb);
    s.cmd_blocks = A.take<BrCmd>((size_t)nb * plan.cmd_stride);
    s.dirty = A.take<u32>(nb + 16); s.changed_bits = A.take<u32>(nb + 16);
    s.changed_epoch = A.take<int>(nb + 16); s.ext_total = A.take<u32>(nb + 16);
    s.cmd_off = A.take<u32>(nb + 16); s.force_unc = A.take<u32>(nb + 16);
    s.dirty_list = A.take<u32>(nb + 16); s.block_mb = A.take<u32>(nb + 16);
    s.ran_list = A.take<u32>(plan.ran_cap); s.lil_in = A.take<u32>(nb + 16);
    s.bitdep_epoch = A.take<int>(nb + 16);
    s.blk = A.take<BrBlk>(nblk); s.blkin = A.take<BrBlkIn>(nblk);
    s.key_flips = A.take<u32>(P.nbuckets + 8);
    s.slot_blk = A.take<u32>(plan.slot_blk.size()); b.cut_kind = A.take<u32>(ncuts + 2); b.cut_end = A.take<u64>(ncuts + 2);
    b.stream_end = A.take<u64>(nstreams + 2);
    s.epoch_cum = A.take<u32>((size_t)P.max_epochs + 2);
    s.mbs = A.take<BrMetaBlock>(nb + 1);
    s.stream_blk = A.take<u32>(nstreams + 2); s.stream_nmb = A.take<u32>(nstreams + 2); s.stream_ncmd = A.take<u32>(nstreams + 2);
    s.mbs_stage = A.take<BrMetaBlock>(nblk);
    s.counters = A.take<u32>(64); s.hist_scratch = A.take<u32>(256ull * nstreams);
    if (P.quick) {   // 32-bit sort keys, slot reads, slot entry points
      carve_index_quick(A, P, b.ix);
      s.saw = A.take<u32>(((size_t)n << P.qk_sweep_bits) + 16);
      s.qpred = A.take<u32>(((size_t)n << P.qk_sweep_bits) + 16);
    }
  };
  if (!br_carve(job->arena, carve)) return false;
  s.S = b.ix.S; s.rank = b.ix.rank; s.seg = b.ix.seg; s.skeys = b.ix.K2; s.tagS = b.ix.tagS;
  br_bind_tables(s, T->blob, T->log2tab, T->log2tab_n);

  CK(cudaMemcpyAsync((u8*)s.data, d_in, n, cudaMemcpyDeviceToDevice, st));
  CK(cudaMemsetAsync((u8*)s.data + n, 0, 64, st));
  CK(cudaMemcpyAsync(s.blk, plan.blk.data(), nblk * sizeof(BrBlk), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync((u32*)s.slot_blk, plan.slot_blk.data(), plan.slot_blk.size() * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync((u32*)s.stream_blk, plan.stream_blk.data(), (nstreams + 1) * 4ull, cudaMemcpyHostToDevice, st));
  if (ncuts) CK(cudaMemcpyAsync(b.cut_kind, cuts->kind, ncuts * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(s.bin, 0, nb * sizeof(BrBlockIn), st));
  k_build_chunks<<<nblk, 64, 0, st>>>(s.blk, s.bin, 1u << P.chunk_bits);
  CK(cudaStreamSynchronize(st));   // (the copies from the plan's host tables must be done before the arrays below are reused)
  CK(cudaMemsetAsync(s.bout, 0, nb * sizeof(BrBlockOut), st));
  CK(cudaMemsetAsync(s.bin_used, 0, nb * sizeof(BrBlockIn), st));
  CK(cudaMemsetAsync(s.changed_bits, 0, (nb + 16) * 4, st));
  CK(cudaMemsetAsync(s.changed_epoch, 0xFF, (nb + 16) * 4, st));
  CK(cudaMemsetAsync(s.bitdep_epoch, 0xFF, (nb + 16) * 4, st));
  CK(cudaMemsetAsync(s.srch_latest, 0, nwords * 4, st));
  CK(cudaMemsetAsync(s.key_flips, 0, (P.nbuckets + 8) * 4, st));
  CK(cudaMemsetAsync(s.force_unc, 0, (nb + 16) * 4, st));
  CK(cudaMemsetAsync(s.epoch_cum, 0, 64, st));
  CK(cudaMemsetAsync(s.counters, 0, 256, st));
  CK(cudaMemsetAsync(s.bits_cur, 0, 2 * (size_t)nwords * 4, st));
  return true;
}
// Index: S, rank and seg (br_build_index), at qualities 2..4 the slot entry points, and tagS when `tags`.
static void stage_index(const BrStream& s, const BrIndexBufs& ix, bool tags, cudaStream_t st) {
  br_build_index(s.P, s.data, s.blk, s.nblk, ix, st);
  if (s.P.quick) k_slot_pred<<<s.nblk, 256, 0, st>>>(s, (u32*)s.qpred);   // (the kernel reads s.S / s.rank / s.seg / s.blk / s.data only)
  if (tags) k_tags<<<(s.P.n + 255) / 256, 256, 0, st>>>(s.data, ix.S, s.P.n, ix.tagS);
}
// prefS = the exclusive scan of cntS, the stored bits of every 1024 positions of S
static void refresh_prefS(const BrStream& s, const u32* cntS, u32* scan_tmp2, cudaStream_t st) {
  const u32 nsnap = (s.P.n + 1023) / 1024;
  cudaMemcpyAsync((u32*)s.prefS, cntS, nsnap * 4ull, cudaMemcpyDeviceToDevice, st);
  scan_exclusive((u32*)s.prefS, nsnap, scan_tmp2, st);
}
// Snapshot: bits_latest in S order (storedS) and its prefix counts (prefS), for the bucket rings of qualities 5..9.  Built
// once; the fixpoint carries it along after every launch's commits (k_snapshot_update).
static void stage_snapshot(const BrStream& s, u32* cntS, u32* scan_tmp2, cudaStream_t st) {
  k_build_storedS<<<(s.P.n + 1023) / 1024, 1024, 0, st>>>(s, (u32*)s.storedS, cntS);
  refresh_prefS(s, cntS, scan_tmp2, st);
}
// Fixpoint: the chain, then walk launches until no chunk is dirty.  *n_mbs, *total_cmds: the metablocks and commands of
// the parse it settles on.  trace (BR_DEBUG_KNOBS builds): every launch, then the slowest chunk walks, on stderr.
static bool stage_fixpoint(BrJob* job, BrStream& s, const BrJobBufs& b, bool trace, u32* n_mbs, u32* total_cmds) {
  const BrParams& P = s.P;
  const u32 nb = P.nblocks, nblk = s.nblk, ch = 1u << P.chunk_bits, nwords = s.bits_words;
  cudaStream_t st = job->st; cudaEvent_t* ev = job->ev; u32* hp = job->h_pinned;
  const u32 round_epoch0 = s.epoch;
  bool walk_pending = false;
  for (;;) {
    k_chain_a<<<(nblk + 31) / 32, 32, 0, st>>>(s);
    if (P.multi) {
      k_chain_b1<<<(P.multi + 3) / 4, 128, 0, st>>>(s);
      k_chain_b2<<<1, 32, 0, st>>>(s);
      k_chain_b3<<<(nblk + 255) / 256, 256, 0, st>>>(s);
    } else k_chain_b<<<1, 32, 0, st>>>(s);
    k_chain_c<<<(nblk + 31) / 32, 32, 0, st>>>(s);
    k_chain_d<<<(nb + 255) / 256, 256, 0, st>>>(s);
    CK(cudaMemcpyAsync(hp, s.counters, 128, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    u32 n_dirty = hp[0], n_sched = hp[5]; *n_mbs = hp[1]; *total_cmds = hp[2];
    job->stats.block_runs += hp[4];
    if (hp[4] > job->stats.max_walks) job->stats.max_walks = hp[4];
    if (trace) fprintf(stderr, "epoch %u: dirty %u sched %u ran %u longest sweep %u | never %u state %u dict %u bits %u wrap %u\n", s.epoch, hp[0], hp[5], hp[4], hp[16], hp[9], hp[10], hp[11], hp[12], hp[13]);
    if (walk_pending) {
      float wms; cudaEventElapsedTime(&wms, ev[6], ev[7]); job->stats.ms_walk += wms; walk_pending = false;
      if (trace) fprintf(stderr, "   walk launch %u: %.2f ms\n", s.epoch, wms);
    }
    if (n_dirty == 0) break;
    if (s.epoch + 2 >= P.max_epochs) { fprintf(stderr, "brotli_b200: internal error: launch bound exceeded\n"); return false; }
    ++s.epoch; ++job->stats.lz77_iterations;
    s.forced = s.epoch - round_epoch0 >= P.force_epoch ? 1u : 0u;
    job->stats.forced_launches += s.forced;
    CK(cudaMemsetAsync(s.bits_cur, 0, 2 * (size_t)nwords * 4, st));
    CK(cudaMemsetAsync(s.srch_cur, 0, nwords * 4, st));
    CK(cudaMemsetAsync(s.counters + 4, 0, 4, st));
    CK(cudaMemsetAsync(s.counters + 16, 0, 4, st));
    cudaEventRecord(ev[6], st);
    const u32 wg = (n_sched + BR_WALK_WARPS - 1) / BR_WALK_WARPS;
    br_walk_dispatch(P, [&](auto g, auto m) { k_walk<decltype(g)::value, decltype(m)::value><<<wg, 32 * BR_WALK_WARPS, 0, st>>>(s); });
    cudaEventRecord(ev[7], st);
    walk_pending = true; ++job->stats.walk_launches; job->stats.launches += 6;
    job->stats.walk_bytes += (u64)n_sched * ch;
    CK(cudaMemcpyAsync((u32*)s.bits_prev, s.bits_latest, nwords * 4, cudaMemcpyDeviceToDevice, st));
    if (!P.quick) {   // (quality 2..4 check every run instead of marking: br_verify_run)
      CK(cudaMemsetAsync(s.cover_cur, 0, nwords * 4, st));
      k_cover<<<(nb * 32 + 127) / 128, 128, 0, st>>>(s);
    }
    k_commit<<<(nb * 32 + 127) / 128, 128, 0, st>>>(s);
    if (P.quick) k_verify<<<(nb * 32 + 127) / 128, 128, 0, st>>>(s);
    else {
      k_snapshot_update<<<(u32)((nwords + 255) / 256), 256, 0, st>>>(s, (u32*)s.storedS, b.cntS);
      refresh_prefS(s, b.cntS, b.scan_tmp2, st);
    }
  }
  cudaEventRecord(ev[2], st);
#ifdef BR_DEBUG_KNOBS
  if (trace) {   // the slowest chunk walks of the final state, and a per-megabyte profile
    std::vector<BrBlockOut> hb2(nb);
    cudaMemcpyAsync(hb2.data(), s.bout, nb * sizeof(BrBlockOut), cudaMemcpyDeviceToHost, st); cudaStreamSynchronize(st);
    const u32 per = (1u << 20) >> P.chunk_bits;
    for (u32 a = 0; a < nb; a += per) {
      unsigned long long cyc = 0, se = 0, ro = 0; u32 mx = 0;
      for (u32 k = a; k < a + per && k < nb; ++k) { cyc += hb2[k].dbg_kcycles; se += hb2[k].dbg_searches; ro += hb2[k].dbg_rows; if (hb2[k].dbg_kcycles > mx) mx = hb2[k].dbg_kcycles; }
      fprintf(stderr, "MiB %4u: %7.2f Mcycles per chunk (max %7.2f)  searches/chunk %5llu rows/search %5.1f\n", a / per, cyc / 1024.0 / per, mx / 1024.0, se / per, se ? (double)ro / se : 0.0);
    }
  }
#endif
  return true;
}
// Entropy: the metablocks' layout, arena2 (carve_entropy), the compacted commands and E0..E7 (br_entropy2.h): every
// compressed metablock's bits in its buffer.
static bool stage_entropy(BrJob* job, const BrStream& s, BrJobBufs& b, u32 n_mbs, u32 C) {
  const BrParams& P = s.P;
  cudaStream_t st = job->st;
  std::vector<BrMetaBlock> hm(n_mbs);
  CK(cudaMemcpyAsync(hm.data(), s.mbs, n_mbs * sizeof(BrMetaBlock), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  BrMbLayout L;
  br_mb_layout(P, hm.data(), n_mbs, L);
  if (!br_carve(job->arena2, [&](BrCarve& B) { carve_entropy(B, L, P.n, C, (L.code_workers + 63) & ~63u, b); })) return false;
  BrEnt& e = b.e;
  CK(cudaMemcpyAsync((u64*)e.scratch_off, L.scratch_off.data(), n_mbs * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync((u64*)e.out_off, L.out_off.data(), n_mbs * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(e.outbits, 0, (L.out_words + 64) * 4, st));
  CK(cudaMemsetAsync(b.out, 0, L.out_cap + 64, st));
  k_compact<<<(P.nblocks * 32 + 127) / 128, 128, 0, st>>>(s, (BrCmd*)e.cmds, s.block_mb);
  cudaEventRecord(job->ev[8], st);
  if (!launch_e01(s, e, C, n_mbs, b.stmp, job->h_pinned + 24, st) || !launch_split(s, e, n_mbs, st)) return false;
  if (P.mb_kind) k_prep_flat<<<n_mbs, 64, 0, st>>>(s, e);   // qualities 2, 3: no block split, one code per category
  else launch_codes(s, e, L, n_mbs, b.code_base, b.stmp, b.tree_pool, 0, st);
  k_lit_bits<<<(e.total_lits + 1 + 255) / 256, 256, 0, st>>>(s, e);
  k_cmd_bits<<<(C + 1 + 255) / 256, 256, 0, st>>>(s, e);
  scan_exclusive(e.lit_len, e.total_lits + 1, b.stmp, st);
  scan_exclusive(e.cmd_len, C + 1, b.stmp, st);
  k_emit_cmd<<<(C + 255) / 256, 256, 0, st>>>(s, e);
  if (e.total_lits) k_emit_lit<<<(e.total_lits + 255) / 256, 256, 0, st>>>(s, e);
  cudaEventRecord(job->ev[9], st);
  return true;
}

// Assembly: where every metablock's bits go (k_assemble_scan).  *redo: a coded metablock is larger than its input, so
// it is stored raw (encode.c:604; br_assemble_scan marked it in force_unc) and the parse behind it must be redone with
// the restored distance cache; nothing is copied then.  Otherwise the copies, and *out / *size: the stream.
static bool stage_assemble(BrJob* job, const BrStream& s, const BrJobBufs& b, int with_header, u32 n_mbs, bool* redo,
                           const u8** out, size_t* size) {
  cudaStream_t st = job->st; u32* hp = job->h_pinned;
  k_assemble_scan<<<1, 32, 0, st>>>(s, b.e.out_off, b.out, b.desc, b.res, with_header, b.cut_kind, b.cut_end, b.stream_end);
  CK(cudaMemcpyAsync(hp + 16, b.res, 16, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  *redo = hp[18] != 0;
  if (*redo) return true;
  k_assemble_copy<<<dim3(64, n_mbs < 65535u ? n_mbs : 65535u), 256, 0, st>>>(s, b.desc, b.e.outbits, b.out, n_mbs);
  *out = (const u8*)b.out; *size = ((u64)hp[17] << 32) | hp[16];
  return true;
}

// Compress one stream whose input already sits in device memory (d_in, n bytes).  The
// compressed bytes are left in device memory (*d_out, *out_size; valid until the next call on
// this job).  Returns 1 on success, 0 on failure (unsupported parameters, CUDA error).
// `cuts` (nullable): the stream is cut by FLUSH / EMIT_METADATA operations (br_pipeline.h BrCuts).
// knobs (nullable): the schedule of the test hook br_debug_compress_sched.
static int job_compress(BrJob* job, int quality, int lgwin, u32 size_hint, const u8* d_in, u32 n, const u8** d_out, size_t* out_size,
                        const BrCuts* cuts, const BrSchedKnobs* knobs) {
  BrDeviceTables* T = get_tables();
  if (!T) return 0;
  BrStreamPlan plan;
  if (!br_plan_stream(quality, lgwin, size_hint, n, cuts, knobs, &plan)) return 0;
  BrStream s; memset(&s, 0, sizeof(s));
  s.P = plan.P;
  BrParams& P = s.P;
#ifdef BR_DEBUG_KNOBS   // experiment switches: never in the release build (an environment variable must not change the bytes)
  if (getenv("BR_HEAVY_MIN")) P.heavy_min = (u32)strtoul(getenv("BR_HEAVY_MIN"), 0, 10);
  if (getenv("BR_STEP_CAP")) P.step_cap = (u32)strtoul(getenv("BR_STEP_CAP"), 0, 10);
  if (getenv("BR_SWEEP_EPOCH")) P.sweep_epoch = (u32)strtoul(getenv("BR_SWEEP_EPOCH"), 0, 10);
  if (getenv("BR_FORCE_EPOCH")) P.force_epoch = (u32)strtoul(getenv("BR_FORCE_EPOCH"), 0, 10);
  const bool trace = getenv("BR_TRACE") != nullptr;
#else
  const bool trace = false;
#endif
  const u32 ncuts = cuts ? cuts->n : 0, nstreams = plan.nstreams;
  cudaStream_t st = job->st;
  memset(&job->stats, 0, sizeof(job->stats));
  job->stats.ran_cap = plan.ran_cap;
  cudaEvent_t* ev = job->ev;
  cudaEventRecord(ev[0], st);
  BrJobBufs b;
  if (!stage_setup(job, s, T, plan, cuts, d_in, b)) return 0;
  // (the 16/32-entry rings of quality 5-6 gained nothing from tags when timed on C2, so only the deep rings of quality 7-9,
  // where most of the 256 ring entries are hash collisions whose bytes need not be fetched, use them)
  stage_index(s, b.ix, P.block_bits >= 6, st);
  CK(cudaMemsetAsync(s.bits_latest, 0, s.bits_words * 4ull, st));
  k_init_bits<<<s.nblk, 256, 0, st>>>(s);
  cudaEventRecord(ev[1], st);
  if (!P.quick) stage_snapshot(s, b.cntS, b.scan_tmp2, st);

  u32 n_mbs = 0, total_cmds = 0;
  int rounds = 0;
  const u8* final_out = nullptr; size_t final_size = 0;
  for (;;) {   // rounds: repeated only when a metablock needs the late uncompressed fallback
    ++rounds;
    if (!stage_fixpoint(job, s, b, trace, &n_mbs, &total_cmds) || !stage_entropy(job, s, b, n_mbs, total_cmds)) return 0;
    cudaEventRecord(ev[3], st);
    ++job->stats.encode_launches; job->stats.launches += 28;
    bool redo;
    if (!stage_assemble(job, s, b, plan.with_header, n_mbs, &redo, &final_out, &final_size)) return 0;
    if (!redo) break;
    if (rounds > (int)plan.max_rounds) return 0;
  }
  cudaEventRecord(ev[4], st);
  CK(cudaStreamSynchronize(st));
  CK(cudaGetLastError());
  float ms;
  cudaEventElapsedTime(&ms, ev[0], ev[1]); job->stats.ms_index = ms;
  cudaEventElapsedTime(&ms, ev[1], ev[2]); job->stats.ms_lz77 = ms;
  cudaEventElapsedTime(&ms, ev[2], ev[3]); job->stats.ms_entropy = ms;
  cudaEventElapsedTime(&ms, ev[3], ev[4]); job->stats.ms_assemble = ms;
  cudaEventElapsedTime(&ms, ev[0], ev[4]); job->stats.ms_total = ms;
  cudaEventElapsedTime(&ms, ev[8], ev[9]); job->stats.ms_encode = ms;
  job->stats.total_cmds = total_cmds; job->stats.launches += 12;
  job->stats.nblocks = P.nblocks; job->stats.n_metablocks = n_mbs; job->stats.rounds = (u32)rounds;
  job->stats.out_bytes = final_size; job->stats.in_bytes = n;
  if (cuts && cuts->end_bit && ncuts && nstreams == 1) {
    CK(cudaMemcpyAsync(cuts->end_bit, b.cut_end, ncuts * 8ull, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  if (cuts && cuts->stream_end && nstreams > 1) {
    CK(cudaMemcpyAsync(cuts->stream_end, b.stream_end, nstreams * 8ull, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  *d_out = final_out; *out_size = final_size;
  return 1;
}

extern "C" int br_job_compress_device(BrJob* job, int quality, int lgwin, u32 size_hint,
                                      const u8* d_in, u32 n, const u8** d_out, size_t* out_size, const BrCuts* cuts) {
  return job_compress(job, quality, lgwin, size_hint, d_in, n, d_out, out_size, cuts, nullptr);
}

// Test hook (tests/test_zz_gpu_schedule.py): one stream through br_job_compress_device with the fixpoint's schedule knobs
// set on the host (BrSchedKnobs).  stats (8 words): launches, chunk walks, chunks, forced launches, the most walks of one
// launch, ran_list capacity, rounds.  Returns the compressed size, 0 on failure, -1 when it does not fit out_cap.
extern "C" __attribute__((visibility("default"))) long br_debug_compress_sched(int quality, int lgwin, const u8* h_in, u32 n,
                                                                              const BrSchedKnobs* knobs, u8* h_out, size_t out_cap,
                                                                              u32* stats) {
  if (n == 0 || !knobs) return 0;
  BrJob* job = br_job_create();
  if (!job) return 0;
  long ret = 0;
  u8* d_in = nullptr;
  const u8* d_out = nullptr; size_t sz = 0;
  if (cudaMalloc(&d_in, n) == cudaSuccess && cudaMemcpy(d_in, h_in, n, cudaMemcpyHostToDevice) == cudaSuccess &&
      job_compress(job, quality, lgwin, n, d_in, n, &d_out, &sz, nullptr, knobs)) {
    if (sz > out_cap) ret = -1;
    else if (cudaMemcpy(h_out, d_out, sz, cudaMemcpyDeviceToHost) == cudaSuccess) ret = (long)sz;
    const BrJobStats& t = job->stats;
    const u32 v[8] = {t.lz77_iterations, (u32)t.block_runs, t.nblocks, t.forced_launches, t.max_walks, t.ran_cap, t.rounds, 0};
    memcpy(stats, v, sizeof(v));
  }
  cudaGetLastError();
  if (d_in) cudaFree(d_in);
  br_job_destroy(job);
  return ret;
}

// Debug / test hooks: the position index of a one-stream job, built by br_build_index and copied to the host.
// h_rank, h_keys (nullable): rank (n words) and the sorted keys (n words; the bucket keys of skeys at qualities 5..9, the
// slot keys at qualities 2..4, whose one input block starts at 0).
extern "C" __attribute__((visibility("default"))) int br_debug_index(int quality, int lgwin, const u8* h_in, u32 n, u32* h_S,
                                                                    u32* h_seg, u32* h_rank, u32* h_keys) {
  BrParams P;
  if (n == 0 || !br_derive_params(quality, lgwin, n, n, &P)) return 0;
  BrBlk B; memset(&B, 0, sizeof(B)); B.start = 0; B.end = n; B.base = 0; B.send = n;
  u8* data; BrBlk* blk; BrIndexBufs b;
  auto carve = [&](BrCarve& A) {
    data = A.take<u8>((size_t)n + 64); blk = A.take<BrBlk>(1);
    carve_index(A, P, b); carve_index_quick(A, P, b);
  };
  BrArena A;
  if (!br_carve(A, carve)) return 0;
  int ok = 0;
  std::vector<u16> k16;
  if (cudaMemset(data, 0, (size_t)n + 64) != cudaSuccess || cudaMemcpy(data, h_in, n, cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(blk, &B, sizeof(BrBlk), cudaMemcpyHostToDevice) != cudaSuccess) goto done;
  br_build_index(P, data, blk, 1, b, 0);
  if (cudaDeviceSynchronize() != cudaSuccess) goto done;
  if (cudaMemcpy(h_S, b.S, 4ull * n, cudaMemcpyDeviceToHost) != cudaSuccess ||
      cudaMemcpy(h_seg, b.seg, (P.nbuckets + 2) * 4ull, cudaMemcpyDeviceToHost) != cudaSuccess) goto done;
  if (h_rank && cudaMemcpy(h_rank, b.rank, 4ull * n, cudaMemcpyDeviceToHost) != cudaSuccess) goto done;
  if (h_keys) {
    if (P.quick) { if (cudaMemcpy(h_keys, b.qk_K1, 4ull * n, cudaMemcpyDeviceToHost) != cudaSuccess) goto done; }
    else {
      k16.resize(n);
      if (cudaMemcpy(k16.data(), b.K2, 2ull * n, cudaMemcpyDeviceToHost) != cudaSuccess) goto done;
      for (u32 j = 0; j < n; ++j) h_keys[j] = k16[j];
    }
  }
  ok = 1;
done:
  cudaGetLastError();
  A.release();
  return ok;
}
extern "C" __attribute__((visibility("default"))) int br_debug_sort(int quality, int lgwin, const u8* h_in, u32 n, u32* h_S, u32* h_seg) {
  return br_debug_index(quality, lgwin, h_in, n, h_S, h_seg, nullptr, nullptr);
}

// Test hook (tests/test_search_probe.py): one match search per probe (br_probe.h), one warp each, from a state the caller
// specifies.  The index, tagS and, at qualities 2..4, the slot entry points are built by the pipeline's index stage
// (stage_index, with tagS at every quality), the S-ordered snapshot by its snapshot stage (stage_snapshot).
template <int F>
__global__ void k_search_probe(BrStream s, u32* own, const u32* probes, u32 np, u32* res) {
  const u32 t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (t < np) br_probe_search<F>(s, own, probes + (size_t)t * BR_PROBE_WORDS, res + (size_t)t * BR_PROBE_WORDS);
}
// bounds[0 .. nstreams): the end of every stream of a batch laid end to end (bounds[nstreams - 1] == n; nstreams == 1: one
// stream).  snap / own: the two stored-bit bitmaps, (n + 31) / 32 words each.  heavy_min: 0 keeps the pipeline's value.
// probes are distinct positions (a quality 2..4 search records its slot reads per position).  res: BR_PROBE_WORDS words per
// probe for every variant of the search, variant after variant: the pipeline's row grouping G, and at qualities 7..9 also
// G = 1 and G = 8 (the fold does not depend on G).  tagS, storedS, prefS (nullable): n u16, (n + 31) / 32 words and
// (n + 1023) / 1024 words.  Returns the number of variants (0: failure).
extern "C" __attribute__((visibility("default"))) int br_debug_search(
    int quality, int lgwin, int lgblock, u32 size_hint, const u8* h_in, u32 n, const u32* h_bounds, u32 nstreams,
    const u32* h_snap, const u32* h_own, u32 heavy_min, const u32* h_probes, u32 np, u32* h_res, u16* h_tagS,
    u32* h_storedS, u32* h_prefS) {
  if (nstreams == 0 || h_bounds[nstreams - 1] != n) return 0;
  std::vector<u32> kinds(nstreams, 3);
  const BrCuts cuts = {h_bounds, kinds.data(), nstreams - 1, 1, 1, 0, nullptr, lgblock, 0, 0, nullptr};
  const BrSchedKnobs knobs = {BR_KNOB_KEEP, BR_KNOB_KEEP, BR_KNOB_KEEP, heavy_min ? heavy_min : BR_KNOB_KEEP, BR_KNOB_KEEP,
                              BR_KNOB_KEEP};
  BrStreamPlan plan;
  if (!br_plan_stream(quality, lgwin, size_hint, n, &cuts, &knobs, &plan)) return 0;
  BrDeviceTables* T = get_tables();
  if (!T) return 0;
  const BrParams& P = plan.P;
  const int nvar = !P.quick && P.quality >= 7 ? 3 : 1;
  const u32 nblk = (u32)plan.blk.size(), nwords = (n + 31) / 32 + 2, nsnap = (n + 1023) / 1024;
  const size_t nsaw = P.quick ? ((size_t)n << P.qk_sweep_bits) + 16 : 16;
  BrStream s; memset(&s, 0, sizeof(s));
  s.P = P; s.nblk = nblk; s.bits_words = nwords;
  BrJobBufs b;
  u8* data; u32 *snap, *own, *probes, *res;
  auto carve = [&](BrCarve& A) {
    s.data = data = A.take<u8>((size_t)n + 64); s.blk = A.take<BrBlk>(nblk); s.slot_blk = A.take<u32>(plan.slot_blk.size());
    carve_index(A, P, b.ix); carve_index_quick(A, P, b.ix);
    s.bits_latest = snap = A.take<u32>(nwords); own = A.take<u32>(nwords); s.storedS = A.take<u32>(nwords + 64);
    s.prefS = A.take<u32>((size_t)n / 1024 + 8); b.cntS = A.take<u32>((size_t)n / 1024 + 8);
    b.scan_tmp2 = A.take<u32>(scan_tmp_words((size_t)n / 1024 + 8));
    s.qpred = A.take<u32>(nsaw); s.saw = A.take<u32>(nsaw);
    probes = A.take<u32>((size_t)np * BR_PROBE_WORDS); res = A.take<u32>((size_t)np * BR_PROBE_WORDS * nvar);
  };
  auto probe = [&](auto g, int v) {
    k_search_probe<decltype(g)::value><<<(np + 3) / 4, 128>>>(s, own, probes, np, res + (size_t)v * np * BR_PROBE_WORDS);
  };
  BrArena A;
  if (!br_carve(A, carve)) return 0;
  s.S = b.ix.S; s.rank = b.ix.rank; s.seg = b.ix.seg; s.skeys = b.ix.K2; s.tagS = b.ix.tagS;
  br_bind_tables(s, T->blob, T->log2tab, T->log2tab_n);
  int ok = 0;
  if (cudaMemset(data, 0, (size_t)n + 64) != cudaSuccess || cudaMemcpy(data, h_in, n, cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(s.blk, plan.blk.data(), nblk * sizeof(BrBlk), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy((u32*)s.slot_blk, plan.slot_blk.data(), plan.slot_blk.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemset(snap, 0, nwords * 4ull) != cudaSuccess || cudaMemset(own, 0, nwords * 4ull) != cudaSuccess ||
      cudaMemcpy(snap, h_snap, (n + 31) / 32 * 4ull, cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(own, h_own, (n + 31) / 32 * 4ull, cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemset(s.saw, 0xEE, nsaw * 4) != cudaSuccess ||
      cudaMemcpy(probes, h_probes, (size_t)np * BR_PROBE_WORDS * 4, cudaMemcpyHostToDevice) != cudaSuccess) goto done;
  stage_index(s, b.ix, true, 0);
  stage_snapshot(s, b.cntS, b.scan_tmp2, 0);
  br_walk_dispatch(P, [&](auto g, auto) { probe(g, 0); });
  if (nvar == 3) { probe(std::integral_constant<int, 1>(), 1); probe(std::integral_constant<int, 8>(), 2); }
  if (cudaDeviceSynchronize() != cudaSuccess ||
      cudaMemcpy(h_res, res, (size_t)np * BR_PROBE_WORDS * 4 * nvar, cudaMemcpyDeviceToHost) != cudaSuccess) goto done;
  if (h_tagS && cudaMemcpy(h_tagS, b.ix.tagS, 2ull * n, cudaMemcpyDeviceToHost) != cudaSuccess) goto done;
  if (h_storedS && cudaMemcpy(h_storedS, s.storedS, (n + 31) / 32 * 4ull, cudaMemcpyDeviceToHost) != cudaSuccess) goto done;
  if (h_prefS && cudaMemcpy(h_prefS, s.prefS, nsnap * 4ull, cudaMemcpyDeviceToHost) != cudaSuccess) goto done;
  ok = nvar;
done:
  cudaGetLastError();
  A.release();
  return ok;
}

// Test hook (tests/test_entropy_codes.py): E4 alone by the pipeline's launch_codes and carve_entropy, on n_mbs synthetic
// metablocks (br_codes_synth: counts, histos).  The scratch and the thread workers' tree pool start filled with a nonzero
// pattern, as a reused arena leaves them.  code_ctas: CTAs of thread workers (0: the pipeline's count).  Per code, in code
// order: H (the smoothed counts), depth, bits (256, 704 or 64 entries each).  offsets: per compressed metablock the bit
// offset of each of its codes, then the end of its last code; per raw metablock one 0.  out: out_words words of each
// metablock's bit buffer.  info: the job's codes, the worker kind (1: a warp per code, 2: threads) and the worker count.
extern "C" __attribute__((visibility("default"))) int br_debug_codes(u32 n_mbs, const u32* h_counts, const u32* h_histos,
                                                                    u32 code_ctas, u32* h_H, u8* h_depth, u16* h_bits,
                                                                    u32* h_offsets, u32* h_out, u32 out_words, u32* info) {
  std::vector<BrMetaBlock> hm; std::vector<BrMbAux> ha; BrMbLayout L; std::vector<u8> img;
  if (n_mbs == 0 || !br_codes_synth(h_counts, n_mbs, h_histos, 0xA5, hm, ha, L, img)) return 0;
  BrDeviceTables* T = get_tables();
  if (!T) return 0;
  BrStream s; memset(&s, 0, sizeof(s));
  s.P.n = n_mbs * BR_SYNTH_MB_BYTES;
  br_bind_tables(s, T->blob, T->log2tab, T->log2tab_n);
  const u32 ctas = L.code_workers ? codes_ctas(L, code_ctas) : 0u;
  BrJobBufs b;
  const BrEnt& e = b.e;
  auto carve = [&](BrCarve& A) {   // (no commands and no input: n_mbs bytes size the scan of the code counts)
    carve_entropy(A, L, n_mbs, 0, (size_t)ctas * 64, b);
    s.mbs = A.take<BrMetaBlock>(n_mbs);
  };
  BrArena A;
  if (!br_carve(A, carve)) return 0;
  int ok = 0;
  u32 total = 0;
  std::vector<u8> sc;
  if (cudaMemcpy(e.scratch, img.data(), img.size(), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemset(e.outbits, 0, (L.out_words + 64) * 4) != cudaSuccess ||
      cudaMemcpy((u64*)e.scratch_off, L.scratch_off.data(), n_mbs * 8ull, cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy((u64*)e.out_off, L.out_off.data(), n_mbs * 8ull, cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(e.aux, ha.data(), n_mbs * sizeof(BrMbAux), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy((BrMetaBlock*)s.mbs, hm.data(), n_mbs * sizeof(BrMetaBlock), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemset(b.tree_pool, 0xA5, (size_t)ctas * 64 * BR_CODE_TREE_NODES * sizeof(BrHTree)) != cudaSuccess) goto done;
  launch_codes(s, e, L, n_mbs, b.code_base, b.stmp, b.tree_pool, code_ctas, 0);
  if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpy(&total, b.code_base + n_mbs, 4, cudaMemcpyDeviceToHost) != cudaSuccess) goto done;
  sc.resize(img.size());
  if (cudaMemcpy(sc.data(), e.scratch, img.size(), cudaMemcpyDeviceToHost) != cudaSuccess) goto done;
  for (u32 i = 0; i < n_mbs; ++i) {
    if (hm[i].compress &&
        cudaMemcpy(h_out + (size_t)i * out_words, e.outbits + L.out_off[i],
                   4ull * (i + 1 < n_mbs ? L.out_off[i + 1] - L.out_off[i] < out_words ? L.out_off[i + 1] - L.out_off[i] : out_words
                                         : L.out_words - L.out_off[i] < out_words ? L.out_words - L.out_off[i] : out_words),
                   cudaMemcpyDeviceToHost) != cudaSuccess) goto done;
  }
  br_codes_collect(hm, ha, L, sc.data(), h_H, h_depth, h_bits, h_offsets);
  info[0] = total; info[1] = total > BR_CODE_WARP_MAX ? 2u : 1u; info[2] = total > BR_CODE_WARP_MAX ? ctas * 64 : total;
  ok = 1;
done:
  cudaGetLastError();
  A.release();
  return ok;
}

// Test hook (tests/test_entropy_split.py): E0..E4 on metablocks the caller describes (br_split_synth: n input bytes, ncmd
// commands of 16 bytes, BR_SPLIT_MB_WORDS words per metablock), by the pipeline's launch_e01, launch_split and launch_codes
// over its arena layout (carve_entropy).  The scratch starts with a nonzero pattern, as a reused arena leaves it.  Writes
// the records of the compressed metablocks (br_split_record, br_split_record_bits) to out, at most out_cap words, and
// returns the words they take (0: failure); no symbol is coded and nothing is assembled.
extern "C" __attribute__((visibility("default"))) long br_debug_split(const u8* h_in, u32 n, const BrCmd* h_cmds, u32 ncmd,
                                                                     const u32* h_mbs, u32 n_mbs, int quality, u32 size_hint,
                                                                     int disable_ctx, u32* h_out, size_t out_cap) {
  if (n == 0 || n_mbs == 0 || quality < 4 || quality > 9) return 0;
  BrStream s; memset(&s, 0, sizeof(s));
  s.P.quality = quality; s.P.n = n; s.P.size_hint = size_hint; s.P.disable_ctx = disable_ctx ? 1u : 0u;
  std::vector<BrMetaBlock> hm; BrMbLayout L;
  if (!br_split_synth(s.P, h_mbs, n_mbs, h_cmds, ncmd, hm, L)) return 0;
  BrDeviceTables* T = get_tables();
  if (!T) return 0;
  br_bind_tables(s, T->blob, T->log2tab, T->log2tab_n);
  const size_t workers = (L.code_workers + 63) & ~63u;
  BrJobBufs b;
  BrEnt& e = b.e;
  auto carve = [&](BrCarve& A) {
    carve_entropy(A, L, n, ncmd, workers, b);
    s.data = A.take<u8>((size_t)n + 64); s.mbs = A.take<BrMetaBlock>(n_mbs);
  };
  BrArena A;
  if (!br_carve(A, carve)) return 0;
  long ret = 0;
  std::vector<BrMbAux> ha(n_mbs);
  std::vector<std::vector<u32>> recs;
  std::vector<u8> img;
  u32 totals[2];
  if (cudaMemset((u8*)s.data, 0, (size_t)n + 64) != cudaSuccess || cudaMemcpy((u8*)s.data, h_in, n, cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy((BrCmd*)e.cmds, h_cmds, ncmd * sizeof(BrCmd), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemset(e.scratch, 0xA5, L.scratch_bytes + 256) != cudaSuccess ||
      cudaMemset(e.outbits, 0, (L.out_words + 64) * 4) != cudaSuccess ||
      cudaMemcpy((u64*)e.scratch_off, L.scratch_off.data(), n_mbs * 8ull, cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy((u64*)e.out_off, L.out_off.data(), n_mbs * 8ull, cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy((BrMetaBlock*)s.mbs, hm.data(), n_mbs * sizeof(BrMetaBlock), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemset(b.tree_pool, 0xA5, workers * BR_CODE_TREE_NODES * sizeof(BrHTree)) != cudaSuccess) goto done;
  if (!launch_e01(s, e, ncmd, n_mbs, b.stmp, totals, 0) || !launch_split(s, e, n_mbs, 0) || cudaDeviceSynchronize() != cudaSuccess ||
      cudaMemcpy(ha.data(), e.aux, n_mbs * sizeof(BrMbAux), cudaMemcpyDeviceToHost) != cudaSuccess) goto done;
  for (u32 i = 0; i < n_mbs; ++i) {   // the splits and histograms before E4 smooths them
    if (!hm[i].compress) continue;
    img.resize(br_mb2_scratch_bytes(hm[i].nlit, hm[i].ncmd));
    if (cudaMemcpy(img.data(), e.scratch + L.scratch_off[i], img.size(), cudaMemcpyDeviceToHost) != cudaSuccess) goto done;
    recs.emplace_back();
    br_split_record(hm[i], ha[i], img.data(), recs.back());
  }
  launch_codes(s, e, L, n_mbs, b.code_base, b.stmp, b.tree_pool, 0, 0);
  if (cudaDeviceSynchronize() != cudaSuccess) goto done;
  for (u32 i = 0, r = 0; i < n_mbs; ++i) {
    if (!hm[i].compress) continue;
    u32 nbits = 0;
    if (cudaMemcpy(&nbits, e.scratch + L.scratch_off[i] + br_split_code_end_off(hm[i], ha[i]), 4, cudaMemcpyDeviceToHost) != cudaSuccess)
      goto done;
    std::vector<u32> bits((nbits + 31) / 32 + 1);
    if (cudaMemcpy(bits.data(), e.outbits + L.out_off[i], bits.size() * 4, cudaMemcpyDeviceToHost) != cudaSuccess) goto done;
    br_split_record_bits(recs[r++], bits.data(), nbits);
  }
  ret = (long)br_split_put(recs, h_out, out_cap);
done:
  cudaGetLastError();
  A.release();
  return ret;
}
