// br_q1.h -- quality 1: the two-pass fragment coder (SURVEY.md section 8, row F1), device side.
//
// Reference: c/enc/compress_fragment_two_pass.c (BrotliCompressFragmentTwoPass :612, CreateCommands
// :228, StoreCommands :458, BuildAndStoreCommandPrefixCode :58, ShouldCompress :526) driven by
// c/enc/encode.c:1425 BrotliEncoderCompressStreamFast.  Every fragment (one call of :612: at most
// 1 << lgwin bytes, fresh zeroed hash table) is independent of every other one; inside a fragment
// the 128 KiB blocks share the table.  The GPU shape:
//
//   parse   one WARP per fragment (k_q1_parse).  The reference's trawl loop visits a predictable
//           sequence of positions until a match turns up (skip heuristic :262), so the 32 lanes
//           probe the next 32 positions of that sequence at once: hash, table read, candidate
//           compare.  A lane must see the table as the earlier lanes of the same batch leave it:
//           __match_any_sync on the hash finds the latest earlier lane with the same slot.  The
//           first lane that matches wins; it and the lanes before it commit their table stores.
//           Match extension compares 256 bytes per step (8 per lane).
//   prep    one CTA per block (k_q1_prep): ShouldCompress, histograms, the three prefix codes and
//           their serialised headers into a 1 KiB per-block buffer, exact bit counts.
//   chain   one thread per stream: bit offsets of all blocks, the "larger than raw" fragment rule
//           (:635) and the stream epilogue.
//   emit    one CTA per block (k_q1_emit): code words scattered to their final bit offsets with
//           atomic OR; offsets from CTA scans over commands and warp scans over literal runs.
//
// Word layout of the intermediate command stream (u32 = code | extra << 8), :112-226:
//   [0,24) insert code c; [24,40) copy of len-2 with the last distance, copy code c-24;
//   [40,64) copy code c-40; [64,128) distance code c-64 (64 = last distance, 80.. = codes 16..).
#pragma once
#include "br_entropy2.h"

#define BR_Q1_BLOCK (1u << 17)           // compress_fragment_two_pass.h:25
#define BR_Q1_MAX_DISTANCE ((1u << 18) - 16u)   // :29 BROTLI_MAX_BACKWARD_LIMIT(18)
#define BR_Q1_HDR_WORDS 256u

struct BrQ1Stream {
  u64 in_off, out_off;     // byte offsets of the stream in the batch input / output buffers (16-aligned)
  u32 size, first_frag, nfrags;
  u32 hdr_lgwin;           // encode.c:673: max(lgwin, 18); 0 = no stream header (segment behind a FLUSH)
  u32 out_bytes;           // chain: size of the compressed stream
  u32 flush_end;           // the segment ends with a FLUSH: pad to a byte boundary (encode.c:1356)
  u32 start_bits;          // 0..7 bits of the stream's previous segment sit in byte 0 (encode.c:1445 last_bytes_); the caller ORs them in
  u32 end_bit;             // chain: bit length of the segment including start_bits (a segment that neither flushes nor finishes may end mid-byte)
};
struct BrQ1Frag {
  u32 stream, start, size; // start: offset in the stream
  u32 first_block, nblocks;
  u32 is_last, table_bits;
  u32 raw;                 // chain: stored as one raw meta-block (:635)
  u32 out_bit;             // chain: bit offset of the fragment in the stream's output
  u32 end_bit;             // chain: bit offset behind it (where the epilogue goes)
};
struct BrQ1Block {
  u32 frag, start, size;   // start: offset in the stream
  u32 ncmd, nlit;          // parse
  u32 compress;            // prep: 0 = raw meta-block (:584)
  u32 hdr_bits, body_bits; // prep
  u32 out_bit;             // chain
  u32 emit;                // chain: 0 when the whole fragment went raw
};
struct BrQ1Codes {         // prep -> emit
  u16 lit_bits[256], cmd_bits[128];
  u8 lit_depth[256], cmd_depth[128];
};
struct BrQ1 {
  const u8* in; u32* out;
  u32* cmds; u8* lits;     // one slot per input byte, at the block's input offset
  BrQ1Stream* streams; BrQ1Frag* frags; BrQ1Block* blocks;
  BrQ1Codes* codes; u32* hdr;
  int* tables; u32 table_slot;   // ints per warp slot
  u32 nstreams, nfrags, nblocks;
  u32* counters;           // [0] fragment queue head
  const double* log2tab; u32 log2tab_n;
  u32 first_width;         // lanes probing in the first step of a trawl (matches tend to follow matches)
};
struct BrQ1Smem {          // shared memory of one prep CTA
  u32 lit_histo[256], cmd_histo[128];
  u32 hdr[BR_Q1_HDR_WORDS];
  BrHTree tree[2 * 256 + 2];
  u8 ht[704], hx[704], full[704];
  u8 lit_depth[256], cmd_depth[128], perm_depth[64];
  u16 lit_bits[256], cmd_bits[128], perm_bits[64];
  u32 flag[4];
};

// ------------------------------------------------------------------ parse
// Where the fragment's input bytes and its hash table live:
//   BrQ1Glob  both in global memory (any fragment size; the table is a per-warp slot of 2^17 ints)
//   BrQ1Shm   both in SHARED memory: fragments of at most 64 KiB (positions fit 16 bits, so the 2^16-entry table the
//             reference uses for them is 128 KiB) with the input staged next to it by one TMA bulk copy (br_q1.cu)
struct BrQ1Glob {
  typedef int TT;
  static BR_DEV_M u64 ld64(const u8* d, u32 pos) { return br_ld64u(d, pos); }
  static BR_DEV_M u8 ld8(const u8* p) { return br_ldg(p); }
  static BR_DEV_M void prefetch(const void* p) { br_prefetch_l2(p); }
};
struct BrQ1Shm {
  typedef u16 TT;
  static BR_DEV_M u64 ld64(const u8* d, u32 pos) {   // d is 4-byte aligned (see br_q1_parse_fragment_shm)
    const u32* w = (const u32*)d;
    const u32 i = pos >> 2, sh = (pos & 3u) * 8u;
    const u32 a = w[i], b = w[i + 1], c = w[i + 2];
#if BR_GPU
    const u32 lo = __funnelshift_r(a, b, sh), hi = __funnelshift_r(b, c, sh);
#else
    const u64 t = ((u64)b << 32) | a, t2 = ((u64)c << 32) | b;
    const u32 lo = (u32)(t >> sh), hi = (u32)(t2 >> sh);
#endif
    return ((u64)hi << 32) | lo;
  }
  static BR_DEV_M u8 ld8(const u8* p) { return *p; }
  static BR_DEV_M void prefetch(const void*) {}
};

// :32 Hash / :39 HashBytesAtOffset; v = the 8 bytes at the position
BR_DEV u32 br_q1_hash(u64 v, u32 shift, u32 mm) {
  return (u32)(((v << ((8u - mm) * 8u)) * 0x1E35A7BDull) >> shift);
}
// :47 IsMatch with the bytes at the first position already loaded
template <class M>
BR_DEV bool br_q1_is_match(const u8* d, u64 va, u32 b, u32 mm) {
  u64 x = va ^ M::ld64(d, b);
  return mm == 4 ? (u32)x == 0 : (x & 0xFFFFFFFFFFFFull) == 0;
}
// find_match_length.h:20 over the whole warp: lane l compares bytes [8l, 8l+8) of each 8*BR_WARP step
template <class M>
BR_DEV u32 br_q1_match_len(const u8* d, u32 a, u32 b, u32 limit) {
  const u32 lane = (u32)br_lane();
  u32 done = 0;
  for (;;) {
    const u32 off = done + 8u * lane;
    const u32 n = off < limit ? br_min(8u, limit - off) : 0u;
    u32 eq = 0;
    if (n) {
      u64 x = M::ld64(d, a + off) ^ M::ld64(d, b + off);
      if (n < 8) x |= 1ull << (8u * n);
      eq = x ? (u32)br_ctz64(x) >> 3 : 8u;
    }
    const u32 stop = br_ballot(eq < 8u);
    if (stop) { const int f = br_ffs(stop) - 1; return done + 8u * (u32)f + br_shfl(eq, f); }
    done += 8u * BR_WARP;
  }
}
// sum_{t<m} (t >> 5): where the trawl stands after m - 32 probes (:276 skip++ >> 5)
BR_DEV u32 br_q1_skip_sum(u32 m) { const u32 g = m >> 5; return 16u * g * (g - 1u) + (m & 31u) * g; }

// :112 EmitInsertLen, :145 EmitCopyLen, :170 EmitCopyLenLastDistance, :213 EmitDistance as words
BR_DEV u32 br_q1_insert_word(u32 n) { const u32 c = br_ins_code(n); return c | ((n - br_ins_base(c)) << 8); }
BR_DEV u32 br_q1_copy_word(u32 n) { const u32 c = br_copy_code(n); return (c + 40u) | ((n - br_copy_base(c)) << 8); }
BR_DEV u32 br_q1_distance_word(u32 distance) {
  const u32 dd = distance + 3u, nb = br_log2floor(dd) - 1u, prefix = (dd >> nb) & 1u;
  return (2u * (nb - 1u) + prefix + 80u) | ((dd - ((2u + prefix) << nb)) << 8);
}
BR_DEV u32 br_q1_word_extra_bits(u32 code) {   // :460 kNumExtraBits
  if (code < 24) return br_ins_extra(code);
  if (code < 40) return br_copy_extra(code - 24);
  if (code < 64) return br_copy_extra(code - 40);
  if (code < 80) return 0;
  return ((code - 80u) >> 1) + 1u;
}

// :334 / :401 table refresh behind a copy that ends at ip (lane 0); returns the candidate for ip.
// `first`: the variant behind the first copy of a run, whose min_match == 4 form files ip-1 under
// the hash of ip-3 (:339 uses offset 0 twice).
template <class M>
BR_DEV u32 br_q1_refresh(const u8* d, u32 ip, u32 base, typename M::TT* table, u32 shift, u32 mm, bool first) {
  typedef typename M::TT TT;
  u32 cur;
  if (mm == 4) {
    const u64 v = M::ld64(d, ip - 3);
    cur = br_q1_hash(v >> 24, shift, 4);
    table[br_q1_hash(v, shift, 4)] = (TT)(ip - 3 - base);
    table[br_q1_hash(v >> 8, shift, 4)] = (TT)(ip - 2 - base);
    table[br_q1_hash(first ? v : v >> 16, shift, 4)] = (TT)(ip - 1 - base);
  } else {
    u64 v = M::ld64(d, ip - 5);
    table[br_q1_hash(v, shift, 6)] = (TT)(ip - 5 - base);
    table[br_q1_hash(v >> 8, shift, 6)] = (TT)(ip - 4 - base);
    table[br_q1_hash(v >> 16, shift, 6)] = (TT)(ip - 3 - base);
    v = M::ld64(d, ip - 2);
    cur = br_q1_hash(v >> 16, shift, 6);
    table[br_q1_hash(v, shift, 6)] = (TT)(ip - 2 - base);
    table[br_q1_hash(v >> 8, shift, 6)] = (TT)(ip - 1 - base);
  }
  const u32 cand = base + (u32)table[cur];
  table[cur] = (TT)(ip - base);
  return cand;
}

#ifndef BR_Q1_PREFETCH
#define BR_Q1_PREFETCH 1
#endif
// Behind a copy that ends at ip: lane 0's slot is the one the refresh reads (:358), lanes 1.. are the
// first probes of the trawl that follows if no copy starts at ip.  L2 prefetch hints only.
template <class M>
BR_DEV void br_q1_prefetch_ahead(const u8* d, u32 ip, u32 ip_limit, const typename M::TT* table, u32 shift, u32 mm) {
#if BR_Q1_PREFETCH
  const u32 pos = ip + (u32)br_lane();
  if (pos <= ip_limit) M::prefetch(table + br_q1_hash(M::ld64(d, pos), shift, mm));
#endif
}

// lanes copy n literal bytes
template <class M>
BR_DEV void br_q1_copy_literals(const u8* d, u32 from, u8* to, u32 n) {
  for (u32 i = (u32)br_lane(); i < n; i += BR_WARP) to[i] = M::ld8(d + from + i);
}

// :228 CreateCommands for one block; warp-uniform.
template <class M>
BR_DEV void br_q1_parse_block(const BrQ1& q, const u8* d, const BrQ1Frag& fr, u32 bi, typename M::TT* table, u64 in_off) {
  typedef typename M::TT TT;
  const int lane = br_lane();
  BrQ1Block& blk = q.blocks[bi];
  const u32 start = blk.start, ip_end = start + blk.size, base = fr.start;
  const u32 remaining = fr.start + fr.size - start;
  const u32 mm = fr.table_bits <= 15 ? 4u : 6u, shift = 64u - fr.table_bits;
  u32* cw = q.cmds + in_off + start;
  u8* lw = q.lits + in_off + start;
  u32 ncmd = 0, nlit = 0;
  u32 ip = start, next_emit = start;
  u32 last_distance = 0;                     // 0 = none yet (the reference's -1 never matches, :291)
  if (blk.size >= 16) {
    const u32 ip_limit = start + br_min(blk.size - mm, remaining - 16u);
    ++ip;
    for (;;) {
      // ---- trawl (:262-304), BR_WARP probes per step
      u32 skip = 32, cand = 0;
      bool hit = false;
      // Right behind a copy the next match is usually close: the first step probes fewer positions,
      // so fewer table / candidate sectors are fetched for nothing.
      u32 width = br_min(q.first_width, (u32)BR_WARP);
      for (;;) {
        const u32 m1 = skip + (u32)lane;
        const u32 pos = ip + (br_q1_skip_sum(m1) - br_q1_skip_sum(skip));
        const u32 nxt = pos + (m1 >> 5);
        const bool act = (u32)lane < width;
        const bool valid = act && nxt <= ip_limit;       // else the reference leaves for emit_remainder first (:283)
#if BR_Q1_PREFETCH
        {
          // Table slots of the NEXT step's probes are pulled into L2 now: if this step finds nothing,
          // the next one reads them at L2 instead of HBM latency.  A hint only: no value is consumed.
          const u32 m2 = skip + width + (u32)lane;
          const u32 pos2 = ip + (br_q1_skip_sum(m2) - br_q1_skip_sum(skip));
          if (pos2 + (m2 >> 5) <= ip_limit) M::prefetch(table + br_q1_hash(M::ld64(d, pos2), shift, mm));
        }
#endif
        u64 v = 0; u32 h = 0xFFFFFFFFu - (u32)lane; u32 t = 0;
        if (valid) { v = M::ld64(d, pos); h = br_q1_hash(v, shift, mm); t = (u32)table[h]; }
        const u32 peers = br_match_any(h);
        const u32 earlier = peers & br_lanemask_lt();
        const int src = earlier ? 31 - br_clz(earlier) : lane;
        const u32 ppos = br_shfl(pos, src);
        const u32 ctab = earlier ? ppos : base + t;
        bool m_last = false, m_tab = false;
        if (valid) {
          if (last_distance) m_last = br_q1_is_match<M>(d, v, pos - last_distance, mm);
          if (!m_last) m_tab = br_q1_is_match<M>(d, v, ctab, mm) && pos - ctab <= BR_Q1_MAX_DISTANCE;
        }
        const u32 hits = br_ballot(valid && (m_last || m_tab));
        const u32 inval = br_ballot(act && !valid);
        // lanes up to and including `lim` performed their probe: they file their position
        const int lim = hits ? br_ffs(hits) - 1 : inval ? br_ffs(inval) - 2 : (int)width - 1;
        const u32 upto = lim >= 31 ? 0xFFFFFFFFu : ((1u << (lim + 1)) - 1u);
        const u32 mine = peers & upto;
        if (valid && lane <= lim && 31 - br_clz(mine) == lane) table[h] = (TT)(pos - base);
        br_syncwarp();
        if (hits) {
          const int f = br_ffs(hits) - 1;
          ip = br_shfl(pos, f);
          cand = br_shfl(m_last ? pos - last_distance : ctab, f);
          hit = true; break;
        }
        if (inval) break;
        ip = br_shfl(nxt, (int)width - 1);
        skip += width;
        width = BR_WARP;
      }
      if (!hit) break;
      // ---- first copy of the run, with its literals (:309-360)
      {
        const u32 matched = mm + br_q1_match_len<M>(d, cand + mm, ip + mm, ip_end - ip - mm);
        const u32 distance = ip - cand, insert = ip - next_emit;
        br_q1_copy_literals<M>(d, next_emit, lw + nlit, insert);
        nlit += insert;
        const u32 m2 = matched - 2u, cc = br_copy_code(m2), cx = (m2 - br_copy_base(cc)) << 8;
        if (lane == 0) {
          u32 k = ncmd;
          cw[k++] = br_q1_insert_word(insert);
          cw[k++] = distance == last_distance ? 64u : br_q1_distance_word(distance);
          if (cc < 16) cw[k++] = (cc + 24u) | cx;
          else { cw[k++] = (cc + 40u) | cx; cw[k++] = 64u; }
        }
        ncmd += cc < 16 ? 3u : 4u;
        last_distance = distance;
        ip += matched; next_emit = ip;
        if (ip >= ip_limit) break;
        br_q1_prefetch_ahead<M>(d, ip, ip_limit, table, shift, mm);
        u32 c0 = 0;
        if (lane == 0) c0 = br_q1_refresh<M>(d, ip, base, table, shift, mm, true);
        cand = br_shfl(c0, 0);
        br_syncwarp();
      }
      // ---- further copies that start right here (:377-440)
      bool out = false;
      while (ip - cand <= BR_Q1_MAX_DISTANCE && br_q1_is_match<M>(d, M::ld64(d, ip), cand, mm)) {
        const u32 matched = mm + br_q1_match_len<M>(d, cand + mm, ip + mm, ip_end - ip - mm);
        last_distance = ip - cand;
        if (lane == 0) { cw[ncmd] = br_q1_copy_word(matched); cw[ncmd + 1] = br_q1_distance_word(last_distance); }
        ncmd += 2;
        ip += matched; next_emit = ip;
        if (ip >= ip_limit) { out = true; break; }
        br_q1_prefetch_ahead<M>(d, ip, ip_limit, table, shift, mm);
        u32 c0 = 0;
        if (lane == 0) c0 = br_q1_refresh<M>(d, ip, base, table, shift, mm, false);
        cand = br_shfl(c0, 0);
        br_syncwarp();
      }
      if (out) break;
      ++ip;
    }
  }
  if (next_emit < ip_end) {                  // :444 emit_remainder
    const u32 insert = ip_end - next_emit;
    br_q1_copy_literals<M>(d, next_emit, lw + nlit, insert);
    if (lane == 0) cw[ncmd] = br_q1_insert_word(insert);
    ++ncmd; nlit += insert;
  }
  if (lane == 0) { blk.ncmd = ncmd; blk.nlit = nlit; }
  br_syncwarp();
}

// One fragment: zero the table (encode.c:156 GetHashTable), then its blocks in order (:563).
BR_DEV void br_q1_parse_fragment(const BrQ1& q, u32 fi, int* table) {
  const BrQ1Frag fr = q.frags[fi];
  const BrQ1Stream& st = q.streams[fr.stream];
  for (u32 i = (u32)br_lane(); i < (1u << fr.table_bits); i += BR_WARP) table[i] = 0;
  br_syncwarp();
  for (u32 b = 0; b < fr.nblocks; ++b) br_q1_parse_block<BrQ1Glob>(q, q.in + st.in_off, fr, fr.first_block + b, table, st.in_off);
}
// The same with table and input on chip.  `buf` holds the bytes [fr.start & ~15, ...) of the stream (16-byte aligned
// copy: see k_q1_parse_shm), so buf - (fr.start & ~15) is a 4-byte aligned base that is indexed by stream positions.
BR_DEV void br_q1_parse_fragment_shm(const BrQ1& q, u32 fi, u16* table, const u8* buf) {
  const BrQ1Frag fr = q.frags[fi];
  const BrQ1Stream& st = q.streams[fr.stream];
  const u8* d = buf - (fr.start & ~15u);
  for (u32 b = 0; b < fr.nblocks; ++b) br_q1_parse_block<BrQ1Shm>(q, d, fr, fr.first_block + b, table, st.in_off);
}

// ------------------------------------------------------------------ prep
// entropy_encode.h:82 SortHuffmanTreeItems under brotli_bit_stream.c:398's count-only comparator.
// That is not a total order, so the reference's exact insertion / shell sequence is reproduced.
BR_DEV void br_q1_sort_by_count(BrHTree* it, u32 n) {
  if (n < 13) {
    for (u32 i = 1; i < n; ++i) {
      BrHTree t = it[i]; u32 k = i;
      while (k > 0 && t.count < it[k - 1].count) { it[k] = it[k - 1]; --k; }
      it[k] = t;
    }
    return;
  }
  for (int g = n < 57 ? 2 : 0; g < 6; ++g) {
    const u32 gap = g == 0 ? 132u : g == 1 ? 57u : g == 2 ? 23u : g == 3 ? 10u : g == 4 ? 4u : 1u;
    for (u32 i = gap; i < n; ++i) {
      BrHTree t = it[i]; u32 j = i;
      for (; j >= gap && t.count < it[j - gap].count; j -= gap) it[j] = it[j - gap];
      it[j] = t;
    }
  }
}
// The static code-length code of entropy_encode_static.h:20: depths 4 for symbols 0..12, 16, 17,
// 5 for 13 and 14, none for 15.  Canonical codes, bit-reversed (:82 kCodeLengthBits).
BR_DEV u32 br_q1_cl_depth(u32 s) { return s == 13 || s == 14 ? 5u : s == 15 ? 0u : 4u; }
BR_DEV u32 br_q1_cl_bits(u32 s) {
  if (s == 13) return 15u;
  if (s == 14) return 31u;
  const u32 rank = s < 13 ? s : s - 3u;      // position among the 15 four-bit codes
  return br_reverse_bits(4, rank);
}
// a run of sym 16 (2 extra bits) or 17 (3 extra bits), entropy_encode.c:160/198 digit order
BR_DEV void br_q1_put_run(BrBitW& w, u32 sym, u32 reps) {
  const u32 xb = sym == 16 ? 2u : 3u;
  u32 digits[12]; int nd = 0;
  for (;;) {
    digits[nd++] = reps & ((1u << xb) - 1u);
    reps >>= xb;
    if (reps == 0) break;
    --reps;
  }
  while (nd--) { br_put_bits(w, 4, br_q1_cl_bits(sym)); br_put_bits(w, xb, digits[nd]); }
}
// brotli_bit_stream.c:404 BrotliBuildAndStoreHuffmanTreeFast (serial; lane 0 of the caller)
BR_DEV void br_q1_fast_tree(const u32* histo, u32 total, u32 max_bits, BrHTree* tree, u8* depth, u16* bits, BrBitW& w) {
  u32 count = 0, symbols[4] = {0, 0, 0, 0}, length = 0, left = total;
  while (left != 0) {
    if (histo[length]) { if (count < 4) symbols[count] = length; ++count; left -= histo[length]; }
    ++length;
  }
  if (count <= 1) {
    br_put_bits(w, 4, 1); br_put_bits(w, max_bits, symbols[0]);
    depth[symbols[0]] = 0; bits[symbols[0]] = 0;
    return;
  }
  for (u32 i = 0; i < length; ++i) depth[i] = 0;
  BrHTree sentinel; sentinel.count = 0xFFFFFFFFu; sentinel.left = -1; sentinel.right_or_value = -1;
  for (u32 limit = 1;; limit *= 2) {
    u32 n = 0;
    for (u32 i = length; i != 0;) {
      --i;
      if (histo[i]) { tree[n].count = histo[i] >= limit ? histo[i] : limit; tree[n].left = -1; tree[n].right_or_value = (short)i; ++n; }
    }
    br_q1_sort_by_count(tree, n);
    tree[n] = sentinel; tree[n + 1] = sentinel;
    u32 a = 0, b = n + 1;
    for (u32 k = n - 1; k > 0; --k) {
      u32 l, r; const u32 parent = 2 * n - k;
      if (tree[a].count <= tree[b].count) l = a++; else l = b++;
      if (tree[a].count <= tree[b].count) r = a++; else r = b++;
      tree[parent].count = tree[l].count + tree[r].count;
      tree[parent].left = (short)l; tree[parent].right_or_value = (short)r;
      tree[parent + 1] = sentinel;
    }
    if (br_set_depth((int)(2 * n - 1), tree, depth, 14)) break;
  }
  br_depths_to_symbols(depth, length, bits);
  if (count <= 4) {
    br_put_bits(w, 2, 1); br_put_bits(w, 2, count - 1);
    for (u32 i = 0; i < count; i++)
      for (u32 j = i + 1; j < count; j++)
        if (depth[symbols[j]] < depth[symbols[i]]) { u32 t = symbols[j]; symbols[j] = symbols[i]; symbols[i] = t; }
    for (u32 i = 0; i < count; ++i) br_put_bits(w, max_bits, symbols[i]);
    if (count == 4) br_put_bits(w, 1, depth[symbols[0]] == 1 ? 1 : 0);
    return;
  }
  // entropy_encode_static.h:86 StoreStaticCodeLengthCode = brotli_bit_stream.c:165 applied to the
  // static depths: HSKIP 0, fifteen "length 4" (2 bits, value 1), two "length 5" (4 bits, 15)
  br_put_bits(w, 32, 0x55555554u); br_put_bits(w, 8, 0xFFu);
  u32 prev = 8;
  for (u32 i = 0; i < length;) {
    const u32 v = depth[i]; u32 reps = 1;
    for (u32 k = i + 1; k < length && depth[k] == v; ++k) ++reps;
    i += reps;
    if (v == 0) {      // :93 kZeroRepsBits = the generic zero-run writer under the static code
      if (reps == 11) { br_put_bits(w, 4, br_q1_cl_bits(0)); --reps; }
      if (reps < 3) { while (reps--) br_put_bits(w, 4, br_q1_cl_bits(0)); }
      else br_q1_put_run(w, 17, reps - 3);
    } else {
      if (prev != v) { br_put_bits(w, br_q1_cl_depth(v), br_q1_cl_bits(v)); --reps; }
      if (reps < 3) { while (reps--) br_put_bits(w, br_q1_cl_depth(v), br_q1_cl_bits(v)); }
      else br_q1_put_run(w, 16, reps - 3);
      prev = v;
    }
  }
}
// the 64 insert/copy words in the order of their symbols in the 704-symbol alphabet (:74-79), and
// that symbol (:92-101)
BR_DEV u32 br_q1_perm_code(u32 k) { return k < 24 ? k + 24 : k < 32 ? k - 24 : k < 40 ? k + 16 : k < 48 ? k - 32 : k < 56 ? k + 8 : k - 40; }
BR_DEV u32 br_q1_sym704(u32 code) {
  if (code < 8) return 128 + 8 * code;
  if (code < 16) return 256 + 8 * (code - 8);
  if (code < 24) return 448 + 8 * (code - 16);
  if (code < 32) return code - 24;
  if (code < 40) return 64 + (code - 32);
  if (code < 48) return 128 + (code - 40);
  if (code < 56) return 192 + (code - 48);
  return 384 + (code - 56);
}
// :58 BuildAndStoreCommandPrefixCode (serial)
BR_DEV void br_q1_command_code(BrQ1Smem* sm, BrBitW& w) {
  for (u32 i = 0; i < 128; ++i) { sm->cmd_depth[i] = 0; sm->cmd_bits[i] = 0; }
  br_create_huffman_tree(sm->cmd_histo, 64, 15, sm->tree, sm->cmd_depth);
  br_create_huffman_tree(sm->cmd_histo + 64, 64, 14, sm->tree, sm->cmd_depth + 64);
  for (u32 k = 0; k < 64; ++k) { sm->perm_depth[k] = sm->cmd_depth[br_q1_perm_code(k)]; sm->perm_bits[k] = 0; }
  br_depths_to_symbols(sm->perm_depth, 64, sm->perm_bits);
  for (u32 k = 0; k < 64; ++k) sm->cmd_bits[br_q1_perm_code(k)] = sm->perm_bits[k];
  br_depths_to_symbols(sm->cmd_depth + 64, 64, sm->cmd_bits + 64);
  for (u32 i = 0; i < 704; ++i) sm->full[i] = 0;
  for (u32 k = 24; k < 64; ++k) sm->full[br_q1_sym704(k)] = sm->cmd_depth[k];
  for (u32 k = 0; k < 24; ++k) sm->full[br_q1_sym704(k)] = sm->cmd_depth[k];
  br_store_huffman_tree(sm->full, 704, sm, w);
  br_store_huffman_tree(sm->cmd_depth + 64, 64, sm, w);
}
// :197 BrotliStoreMetaBlockHeader
BR_DEV u32 br_q1_mb_header_bits(u32 len) { return 4u + 4u * (len <= (1u << 16) ? 4u : len <= (1u << 20) ? 5u : 6u); }
BR_DEV void br_q1_put_mb_header(u32* out, u32 ix, u32 len, u32 uncompressed) {
  const u32 nib = len <= (1u << 16) ? 4u : len <= (1u << 20) ? 5u : 6u;
  // ISLAST 0 | MNIBBLES-4 (2) | MLEN-1 (4 nib) | ISUNCOMPRESSED
  const u64 v = ((u64)(nib - 4u) << 1) | ((u64)(len - 1u) << 3) | ((u64)uncompressed << (3u + 4u * nib));
  br_put_bits_at(out, ix, 4u + 4u * nib, v);
}

// One block: ShouldCompress (:526), histograms, codes, header, bit counts.  CTA-cooperative.
BR_DEV void br_q1_prep_block(const BrQ1& q, u32 bi, BrQ1Smem* sm) {
  const u32 tid = BR_CTA_TID, nt = BR_CTA_N;
  BrQ1Block& blk = q.blocks[bi];
  const BrQ1Frag& fr = q.frags[blk.frag];
  const BrQ1Stream& st = q.streams[fr.stream];
  const u8* d = q.in + st.in_off;
  const u32* cw = q.cmds + st.in_off + blk.start;
  const u8* lw = q.lits + st.in_off + blk.start;
  const u32 size = blk.size, nlit = blk.nlit, ncmd = blk.ncmd;
  for (u32 i = tid; i < 256; i += nt) sm->lit_histo[i] = 0;
  for (u32 i = tid; i < 128; i += nt) sm->cmd_histo[i] = 0;
  for (u32 i = tid; i < BR_Q1_HDR_WORDS; i += nt) sm->hdr[i] = 0;
  br_cta_sync();
  const double corpus = (double)size;
  bool compress = (double)nlit < br_dmul(0.98, corpus);
  if (!compress) {
    // sampled entropy, every 43rd byte (:534)
    for (u32 i = tid * 43u; i < size; i += nt * 43u) br_smem_add(&sm->lit_histo[br_ldg(d + blk.start + i)], 1);
    br_cta_sync();
    if (tid == 0) {
      const double max_cost = br_ddiv(br_dmul(br_dmul(corpus, 8.0), 0.98), 43.0);
      u32 sum = 0; double r = 0;
      for (u32 i = 0; i < 256; ++i) {      // bit_cost.c:18 BrotliBitsEntropy, sequential
        const u32 p = sm->lit_histo[i];
        sum += p;
        if (p) r = br_dsub(r, br_dmul((double)p, br_ldg(q.log2tab + (p < q.log2tab_n ? p : q.log2tab_n - 1))));
      }
      if (sum) r = br_dadd(r, br_dmul((double)sum, br_ldg(q.log2tab + (sum < q.log2tab_n ? sum : q.log2tab_n - 1))));
      if (r < (double)sum) r = (double)sum;
      sm->flag[0] = r < max_cost ? 1u : 0u;
    }
    br_cta_sync();
    compress = sm->flag[0] != 0;
    br_cta_sync();
    for (u32 i = tid; i < 256; i += nt) sm->lit_histo[i] = 0;
    br_cta_sync();
  }
  if (!compress) {
    if (tid == 0) { blk.compress = 0; blk.hdr_bits = 0; blk.body_bits = 0; }
    return;
  }
  for (u32 i = tid; i < nlit; i += nt) br_smem_add(&sm->lit_histo[lw[i]], 1);
  for (u32 i = tid; i < ncmd; i += nt) br_smem_add(&sm->cmd_histo[cw[i] & 0xFFu], 1);
  br_cta_sync();
  if (tid == 0) {
    BrBitW w; w.out = sm->hdr; w.ix = 0; w.per_thread = 0;
    br_q1_put_mb_header(sm->hdr, 0, size, 0); w.ix = br_q1_mb_header_bits(size);
    br_put_bits(w, 13, 0);                       // :581 no block splits, no contexts
    for (u32 i = 0; i < 256; ++i) { sm->lit_depth[i] = 0; sm->lit_bits[i] = 0; }
    br_q1_fast_tree(sm->lit_histo, nlit, 8, sm->tree, sm->lit_depth, sm->lit_bits, w);
    sm->cmd_histo[1] += 1; sm->cmd_histo[2] += 1; sm->cmd_histo[64] += 1; sm->cmd_histo[84] += 1;   // :496
    br_q1_command_code(sm, w);
    sm->cmd_histo[1] -= 1; sm->cmd_histo[2] -= 1; sm->cmd_histo[64] -= 1; sm->cmd_histo[84] -= 1;
    u32 body = 0;
    for (u32 i = 0; i < 256; ++i) body += sm->lit_histo[i] * sm->lit_depth[i];
    for (u32 i = 0; i < 128; ++i) body += sm->cmd_histo[i] * (sm->cmd_depth[i] + br_q1_word_extra_bits(i));
    blk.compress = 1; blk.hdr_bits = w.ix; blk.body_bits = body;
  }
  br_cta_sync();
  BrQ1Codes& c = q.codes[bi];
  for (u32 i = tid; i < 256; i += nt) { c.lit_bits[i] = sm->lit_bits[i]; c.lit_depth[i] = sm->lit_depth[i]; }
  for (u32 i = tid; i < 128; i += nt) { c.cmd_bits[i] = sm->cmd_bits[i]; c.cmd_depth[i] = sm->cmd_depth[i]; }
  for (u32 i = tid; i < BR_Q1_HDR_WORDS; i += nt) q.hdr[(size_t)bi * BR_Q1_HDR_WORDS + i] = sm->hdr[i];
}

// ------------------------------------------------------------------ chain
// One stream: bit offsets of its fragments and blocks (:563-:644 seen from the output side).
BR_DEV void br_q1_chain_stream(const BrQ1& q, u32 si) {
  BrQ1Stream& st = q.streams[si];
  u32* out = q.out + (st.out_off >> 2);
  u32 ix = st.start_bits;
  if (st.hdr_lgwin) {      // encode.c:203 EncodeWindowBits for lgwin >= 18 (a header segment starts at bit 0)
    br_put_bits_at(out, 0, 4, (u64)(((st.hdr_lgwin - 17u) << 1) | 1u));
    ix = 4;
  }
  for (u32 f = st.first_frag; f < st.first_frag + st.nfrags; ++f) {
    BrQ1Frag& fr = q.frags[f];
    const u32 start_ix = ix;
    for (u32 b = fr.first_block; b < fr.first_block + fr.nblocks; ++b) {
      BrQ1Block& blk = q.blocks[b];
      blk.out_bit = ix; blk.emit = 1;
      if (blk.compress) ix += blk.hdr_bits + blk.body_bits;
      else ix = ((ix + br_q1_mb_header_bits(blk.size) + 7u) & ~7u) + (blk.size << 3);     // :548
    }
    fr.raw = 0; fr.out_bit = start_ix;
    if (ix - start_ix > 31u + (fr.size << 3)) {      // :635
      fr.raw = 1;
      for (u32 b = fr.first_block; b < fr.first_block + fr.nblocks; ++b) q.blocks[b].emit = 0;
      ix = ((start_ix + br_q1_mb_header_bits(fr.size) + 7u) & ~7u) + (fr.size << 3);
    }
    fr.end_bit = ix;
    if (fr.is_last) { br_put_bits_at(out, ix, 2, 3); ix = (ix + 2u + 7u) & ~7u; }   // :641 ISLAST, ISEMPTY
  }
  if (st.flush_end && (ix & 7u)) {
    // encode.c:1356 InjectBytePaddingBlock: ISLAST 0, MNIBBLES 11 (metadata), reserved 0, MSKIPBYTES 00
    br_put_bits_at(out, ix, 6, 6);
    ix = (ix + 6u + 7u) & ~7u;
  }
  st.out_bytes = (ix + 7u) >> 3;
  st.end_bit = ix;
}

// ------------------------------------------------------------------ emit
// raw bytes [from, from+n) of the stream to byte offset `to` of its output (atomic OR, 4 bytes per step)
BR_DEV void br_q1_copy_raw(const u8* d, u32 from, u32* out, u32 to, u32 n, u32 tid, u32 nt) {
  for (u32 i = tid * 4u; i < n; i += nt * 4u) {
    const u32 k = br_min(4u, n - i);
    u32 v = br_ld32u(d, from + i);
    if (k < 4) v &= (1u << (8u * k)) - 1u;
    br_put_bits_at(out, (to + i) << 3, 8u * k, v);
  }
}
// CTA-wide exclusive scan of one value per thread; returns the exclusive prefix, *total = CTA sum.
// scratch: one u32 per warp + 1.
BR_DEV u32 br_q1_cta_scan(u32 v, u32* total, u32* scratch) {
#if BR_GPU
  const u32 lane = threadIdx.x & 31u, wid = threadIdx.x >> 5, nw = (blockDim.x + 31u) >> 5;
  u32 wt; const u32 ex = br_warp_excl_scan(v, &wt);
  __syncthreads();
  if (lane == 0) scratch[wid] = wt;
  __syncthreads();
  u32 before = 0, all = 0;
  for (u32 i = 0; i < nw; ++i) { const u32 s = scratch[i]; if (i < wid) before += s; all += s; }
  *total = all;
  return before + ex;
#else
  (void)scratch; *total = v; return 0;
#endif
}

BR_DEV void br_q1_emit_block(const BrQ1& q, u32 bi, u32* scratch) {
  const u32 tid = BR_CTA_TID, nt = BR_CTA_N;
  const int lane = br_lane();
  const BrQ1Block blk = q.blocks[bi];
  const BrQ1Frag fr = q.frags[blk.frag];
  const BrQ1Stream& st = q.streams[fr.stream];
  const u8* d = q.in + st.in_off;
  u32* out = q.out + (st.out_off >> 2);
  if (fr.raw) {                                   // :637 the whole fragment as one raw meta-block
    const u32 data_byte = (fr.out_bit + br_q1_mb_header_bits(fr.size) + 7u) >> 3;
    if (bi == fr.first_block && tid == 0) br_q1_put_mb_header(out, fr.out_bit, fr.size, 1);
    br_q1_copy_raw(d, blk.start, out, data_byte + (blk.start - fr.start), blk.size, tid, nt);
    return;
  }
  if (!blk.compress) {                            // :548 EmitUncompressedMetaBlock
    if (tid == 0) br_q1_put_mb_header(out, blk.out_bit, blk.size, 1);
    br_q1_copy_raw(d, blk.start, out, (blk.out_bit + br_q1_mb_header_bits(blk.size) + 7u) >> 3, blk.size, tid, nt);
    return;
  }
  const u32* hdr = q.hdr + (size_t)bi * BR_Q1_HDR_WORDS;
  for (u32 i = tid; i * 32u < blk.hdr_bits; i += nt)
    br_put_bits_at(out, blk.out_bit + 32u * i, br_min(32u, blk.hdr_bits - 32u * i), hdr[i]);
  const BrQ1Codes& c = q.codes[bi];
  const u32* cw = q.cmds + st.in_off + blk.start;
  const u8* lw = q.lits + st.in_off + blk.start;
  const u32 body = blk.out_bit + blk.hdr_bits;
  u32 carry_l = 0, carry_p = 0;                   // literals / bits before the current tile
  for (u32 t0 = 0; t0 < blk.ncmd; t0 += nt) {
    const u32 ci = t0 + tid;
    const bool act = ci < blk.ncmd;
    const u32 word = act ? cw[ci] : 0u, code = word & 0xFFu, extra = word >> 8;
    const u32 dep = act ? c.cmd_depth[code] : 0u, xb = act ? br_q1_word_extra_bits(code) : 0u;
    const u32 ins = act && code < 24 ? br_ins_base(code) + extra : 0u;
    u32 tot_l; const u32 l0 = carry_l + br_q1_cta_scan(ins, &tot_l, scratch);
    // literal bits of every insert word of the tile: the warp walks its insert words
    u32 lb = 0;
    for (u32 m = br_ballot(ins != 0); m; m &= m - 1) {
      const int j = br_ffs(m) - 1;
      const u32 n = br_shfl(ins, j), lj = br_shfl(l0, j);
      u32 s = 0;
      for (u32 i = (u32)lane; i < n; i += BR_WARP) s += c.lit_depth[lw[lj + i]];
      s = br_warp_sum(s);
      if (lane == j) lb = s;
    }
    u32 tot_p; const u32 p = body + carry_p + br_q1_cta_scan(dep + xb + lb, &tot_p, scratch);
    if (act) br_put_bits_at(out, p, dep + xb, (u64)c.cmd_bits[code] | ((u64)extra << dep));   // :506
    for (u32 m = br_ballot(ins != 0); m; m &= m - 1) {
      const int j = br_ffs(m) - 1;
      const u32 n = br_shfl(ins, j), lj = br_shfl(l0, j);
      u32 at = br_shfl(p + dep + xb, j);
      for (u32 i0 = 0; i0 < n; i0 += BR_WARP) {
        const u32 i = i0 + (u32)lane;
        const u32 lit = i < n ? lw[lj + i] : 0u;
        const u32 ld = i < n ? c.lit_depth[lit] : 0u;
        u32 tot; const u32 ex = br_warp_excl_scan(ld, &tot);
        if (i < n) br_put_bits_at(out, at + ex, ld, c.lit_bits[lit]);
        at += tot;
      }
    }
    carry_l += tot_l; carry_p += tot_p;
  }
}
