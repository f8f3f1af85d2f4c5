// br_entropy.h -- per-metablock entropy pipeline, one warp per metablock:
//   literal context-model decision   (c/enc/encode.c:258-455)
//   greedy block splitting           (c/enc/metablock.c:708 BrotliBuildMetaBlockGreedy,
//                                     metablock_inc.h, metablock.c:463 ContextBlockSplitter)
//   histogram smoothing              (c/enc/entropy_encode.c:241)
//   Huffman construction + storage   (c/enc/entropy_encode.c:68, brotli_bit_stream.c:349)
//   symbol emission                  (c/enc/brotli_bit_stream.c:947 BrotliStoreMetaBlock)
// All decisions that the reference takes in double precision are replayed with the same
// operation order and without FMA contraction (br_dmul/br_dadd), log2 through the
// host-generated table.  Wide steps (histogram adds, entropy sums of independent histograms,
// literal runs) are spread over the lanes; the decision chain itself is warp-uniform.
#pragma once
#include "br_cmd.h"

// ------------------------------------------------------------------ bit writer
// per_thread = 0: the cursor is warp-uniform and lane 0 writes; 1: the writer belongs to ONE thread (parallel tree
// storing in br_code_build / br_code_store).  out = nullptr: count bits only.
struct BrBitW { u32* out; u32 ix; u32 per_thread; };
// LSB-first append (write_bits.h:33).  The buffer is pre-zeroed and every write is an atomic
// OR (RED at L2), so lane-0 serial writes and lane-parallel writes can interleave freely.
BR_DEV void br_put_bits_at(u32* out, u32 ix, u32 n, u64 bits) {  // n <= 56
  if (!n) return;
  u32 wi = ix >> 5, sh = ix & 31;
  u64 lo = bits << sh;
  if ((u32)lo) br_atomic_or(out + wi, (u32)lo);
  if ((u32)(lo >> 32)) br_atomic_or(out + wi + 1, (u32)(lo >> 32));
  if (sh && n + sh > 64) { u32 hi = (u32)(bits >> (64 - sh)); if (hi) br_atomic_or(out + wi + 2, hi); }
}
// warp-uniform call: lane 0 writes, every lane advances its copy of the cursor
BR_DEV void br_put_bits(BrBitW& w, u32 n, u64 bits) {
  if (w.out && (w.per_thread || br_lane() == 0)) br_put_bits_at(w.out, w.ix, n, bits);
  w.ix += n;
}
// Serial sections run on lane 0 only; afterwards the cursor is re-broadcast.
#define BR_LANE0_BEGIN if (br_lane() == 0) {
#define BR_LANE0_END(w) } (w).ix = br_shfl((w).ix, 0); br_syncwarp();

// ------------------------------------------------------------------ Huffman
struct BrHTree { short left, right_or_value; u32 count; };

// entropy_encode.c:20 BrotliSetDepth
BR_DEV int br_set_depth(int p0, BrHTree* pool, u8* depth, int max_depth) {
  int stack[16]; int level = 0; int p = p0;
  stack[0] = -1;
  for (;;) {
    if (pool[p].left >= 0) {
      level++;
      if (level > max_depth) return 0;
      stack[level] = pool[p].right_or_value;
      p = pool[p].left;
      continue;
    } else {
      depth[pool[p].right_or_value] = (u8)level;
    }
    while (level >= 0 && stack[level] == -1) level--;
    if (level < 0) return 1;
    p = stack[level];
    stack[level] = -1;
  }
}
BR_DEV int br_htree_less(const BrHTree& a, const BrHTree& b) {
  if (a.count != b.count) return a.count < b.count;
  return a.right_or_value > b.right_or_value;
}
// entropy_encode.c:68 BrotliCreateHuffmanTree.  Executed by lane 0 (callers guard); the sort
// key (count, symbol descending) is a strict total order, so a plain shell sort gives the
// same permutation as entropy_encode.h:82 SortHuffmanTreeItems.
BR_DEV void br_create_huffman_tree(const u32* data, u32 length, int tree_limit, BrHTree* tree, u8* depth) {
  BrHTree sentinel; sentinel.count = 0xFFFFFFFFu; sentinel.left = -1; sentinel.right_or_value = -1;
  for (u32 count_limit = 1;; count_limit *= 2) {
    u32 n = 0;
    for (u32 i = length; i != 0;) {
      --i;
      if (data[i]) {
        tree[n].count = data[i] > count_limit ? data[i] : count_limit;
        tree[n].left = -1; tree[n].right_or_value = (short)i; ++n;
      }
    }
    if (n == 1) { depth[tree[0].right_or_value] = 1; break; }
    for (u32 gap = n >> 1; gap > 0; gap = gap == 2 ? 1 : (gap * 5) / 11) {
      for (u32 i = gap; i < n; ++i) {
        BrHTree t = tree[i]; u32 q = i;
        while (q >= gap && br_htree_less(t, tree[q - gap])) { tree[q] = tree[q - gap]; q -= gap; }
        tree[q] = t;
      }
    }
    tree[n] = sentinel; tree[n + 1] = sentinel;
    u32 i = 0, j = n + 1;
    for (u32 k = n - 1; k != 0; --k) {
      u32 left, right;
      if (tree[i].count <= tree[j].count) { left = i; ++i; } else { left = j; ++j; }
      if (tree[i].count <= tree[j].count) { right = i; ++i; } else { right = j; ++j; }
      u32 j_end = 2 * n - k;
      tree[j_end].count = tree[left].count + tree[right].count;
      tree[j_end].left = (short)left;
      tree[j_end].right_or_value = (short)right;
      tree[j_end + 1] = sentinel;
    }
    if (br_set_depth((int)(2 * n - 1), tree, depth, tree_limit)) break;
  }
}
// entropy_encode.c:474 BrotliConvertBitDepthsToSymbols
BR_DEV u16 br_reverse_bits(u32 nbits, u32 bits) {
  u32 r = 0;
  for (u32 i = 0; i < nbits; ++i) { r = (r << 1) | (bits & 1); bits >>= 1; }
  return (u16)r;
}
BR_DEV void br_depths_to_symbols(const u8* depth, u32 len, u16* bits) {
  u16 bl_count[16], next_code[16];
  for (int i = 0; i < 16; ++i) bl_count[i] = 0;
  for (u32 i = 0; i < len; ++i) ++bl_count[depth[i]];
  bl_count[0] = 0; next_code[0] = 0;
  int code = 0;
  for (int i = 1; i < 16; ++i) { code = (code + bl_count[i - 1]) << 1; next_code[i] = (u16)code; }
  for (u32 i = 0; i < len; ++i)
    if (depth[i]) bits[i] = br_reverse_bits(depth[i], next_code[depth[i]]++);
}

// entropy_encode.c:241 BrotliOptimizeHuffmanCountsForRle (lane 0); the 32-bit products are
// the reference's: `256 * counts[i]` is evaluated in unsigned int.
BR_DEV void br_optimize_counts_for_rle(u32 length, u32* counts, u8* good_for_rle) {
  u32 nonzero_count = 0;
  const u64 streak_limit = 1240;
  for (u32 i = 0; i < length; i++) if (counts[i]) ++nonzero_count;
  if (nonzero_count < 16) return;
  while (length != 0 && counts[length - 1] == 0) --length;
  if (length == 0) return;
  {
    u32 nonzeros = 0, smallest_nonzero = 1u << 30;
    for (u32 i = 0; i < length; ++i)
      if (counts[i] != 0) { ++nonzeros; if (smallest_nonzero > counts[i]) smallest_nonzero = counts[i]; }
    if (nonzeros < 5) return;
    if (smallest_nonzero < 4) {
      u32 zeros = length - nonzeros;
      if (zeros < 6)
        for (u32 i = 1; i + 1 < length; ++i)
          if (counts[i - 1] != 0 && counts[i] == 0 && counts[i + 1] != 0) counts[i] = 1;
    }
    if (nonzeros < 28) return;
  }
  for (u32 i = 0; i < length; ++i) good_for_rle[i] = 0;
  {
    u32 symbol = counts[0], step = 0;
    for (u32 i = 0; i <= length; ++i) {
      if (i == length || counts[i] != symbol) {
        if ((symbol == 0 && step >= 5) || (symbol != 0 && step >= 7))
          for (u32 k = 0; k < step; ++k) good_for_rle[i - k - 1] = 1;
        step = 1;
        if (i != length) symbol = counts[i];
      } else ++step;
    }
  }
  u64 stride = 0, sum = 0;
  u64 limit = (u32)(256u * (counts[0] + counts[1] + counts[2]) / 3u + 420u);
  for (u32 i = 0; i <= length; ++i) {
    if (i == length || good_for_rle[i] || (i != 0 && good_for_rle[i - 1]) ||
        ((u64)(u32)(256u * counts[i]) - limit + streak_limit) >= 2 * streak_limit) {
      if (stride >= 4 || (stride >= 3 && sum == 0)) {
        u64 count = (sum + stride / 2) / stride;
        if (count == 0) count = 1;
        if (sum == 0) count = 0;
        for (u64 k = 0; k < stride; ++k) counts[i - k - 1] = (u32)count;
      }
      stride = 0; sum = 0;
      if (i + 2 < length) limit = (u32)(256u * (counts[i] + counts[i + 1] + counts[i + 2]) / 3u + 420u);
      else if (i < length) limit = (u32)(256u * counts[i]);
      else limit = 0;
    }
    ++stride;
    if (i != length) {
      sum += counts[i];
      if (stride >= 4) limit = (256 * sum + stride / 2) / stride;
      if (stride == 4) limit += 120;
    }
  }
}

// entropy_encode.c:160-239, :372 DecideOverRleUse, :402 BrotliWriteHuffmanTree
BR_DEV void br_rev(u8* v, u32 s, u32 e) { --e; while (s < e) { u8 t = v[s]; v[s] = v[e]; v[e] = t; ++s; --e; } }
BR_DEV void br_write_reps(u8 prev, u8 value, u32 reps, u32* ts, u8* tree, u8* extra) {
  if (prev != value) { tree[*ts] = value; extra[*ts] = 0; ++(*ts); --reps; }
  if (reps == 7) { tree[*ts] = value; extra[*ts] = 0; ++(*ts); --reps; }
  if (reps < 3) {
    for (u32 i = 0; i < reps; ++i) { tree[*ts] = value; extra[*ts] = 0; ++(*ts); }
  } else {
    u32 start = *ts;
    reps -= 3;
    for (;;) {
      tree[*ts] = 16; extra[*ts] = (u8)(reps & 0x3); ++(*ts);
      reps >>= 2;
      if (reps == 0) break;
      --reps;
    }
    br_rev(tree, start, *ts); br_rev(extra, start, *ts);
  }
}
BR_DEV void br_write_reps_zeros(u32 reps, u32* ts, u8* tree, u8* extra) {
  if (reps == 11) { tree[*ts] = 0; extra[*ts] = 0; ++(*ts); --reps; }
  if (reps < 3) {
    for (u32 i = 0; i < reps; ++i) { tree[*ts] = 0; extra[*ts] = 0; ++(*ts); }
  } else {
    u32 start = *ts;
    reps -= 3;
    for (;;) {
      tree[*ts] = 17; extra[*ts] = (u8)(reps & 0x7); ++(*ts);
      reps >>= 3;
      if (reps == 0) break;
      --reps;
    }
    br_rev(tree, start, *ts); br_rev(extra, start, *ts);
  }
}
BR_DEV void br_write_huffman_tree(const u8* depth, u32 length, u32* ts, u8* tree, u8* extra) {
  u8 prev = 8; u32 new_length = length;
  int rle_nz = 0, rle_z = 0;
  for (u32 i = 0; i < length; ++i) { if (depth[length - i - 1] == 0) --new_length; else break; }
  if (length > 50) {
    u32 tz = 0, tnz = 0, cz = 1, cnz = 1;
    for (u32 i = 0; i < new_length;) {
      u8 v = depth[i]; u32 reps = 1;
      for (u32 k = i + 1; k < new_length && depth[k] == v; ++k) ++reps;
      if (reps >= 3 && v == 0) { tz += reps; ++cz; }
      if (reps >= 4 && v != 0) { tnz += reps; ++cnz; }
      i += reps;
    }
    rle_nz = tnz > cnz * 2; rle_z = tz > cz * 2;
  }
  for (u32 i = 0; i < new_length;) {
    u8 v = depth[i]; u32 reps = 1;
    if ((v != 0 && rle_nz) || (v == 0 && rle_z))
      for (u32 k = i + 1; k < new_length && depth[k] == v; ++k) ++reps;
    if (v == 0) br_write_reps_zeros(reps, ts, tree, extra);
    else { br_write_reps(prev, v, reps, ts, tree, extra); prev = v; }
    i += reps;
  }
}

// Scratch every metablock task owns (global memory).
struct BrMbScratch {
  BrHTree tree[2 * 704 + 2];
  u8 ht[704], hx[704];       // RLE-coded code lengths
  u8 good_for_rle[704];
  u32 small_histo[272];
  u8 small_depth[272];
  u16 small_bits[272];
  double ent[3 * 13];        // entropies of the split decision
  u32 rle_syms[256 * 64];    // context map run-length symbols
};

// What one thread needs to store one prefix code (br_store_huffman_tree): the RLE-coded code lengths and the tree of
// the 18-symbol code-length code.
struct BrTreeSc { BrHTree tree[2 * 18 + 2]; u8 ht[704], hx[704]; };

// brotli_bit_stream.c:165 + :283 BrotliStoreHuffmanTree
template <class SC> BR_DEV void br_store_huffman_tree(const u8* depths, u32 num, SC* sc, BrBitW& w) {
  const u8 kOrder[18] = {1, 2, 3, 4, 0, 5, 17, 6, 16, 7, 8, 9, 10, 11, 12, 13, 14, 15};
  const u8 kSym[6] = {0, 7, 3, 2, 1, 15};
  const u8 kLen[6] = {2, 4, 3, 2, 2, 4};
  u8 cl_depth[18]; u16 cl_bits[18]; u32 histo[18];
  u32 hs = 0; int num_codes = 0; u32 code = 0;
  for (int i = 0; i < 18; ++i) { cl_depth[i] = 0; histo[i] = 0; cl_bits[i] = 0; }
  br_write_huffman_tree(depths, num, &hs, sc->ht, sc->hx);
  for (u32 i = 0; i < hs; ++i) ++histo[sc->ht[i]];
  for (u32 i = 0; i < 18; ++i) {
    if (histo[i]) {
      if (num_codes == 0) { code = i; num_codes = 1; }
      else if (num_codes == 1) { num_codes = 2; break; }
    }
  }
  br_create_huffman_tree(histo, 18, 5, sc->tree, cl_depth);
  br_depths_to_symbols(cl_depth, 18, cl_bits);
  {
    u32 skip = 0, to_store = 18;
    if (num_codes > 1)
      for (; to_store > 0; --to_store) if (cl_depth[kOrder[to_store - 1]] != 0) break;
    if (cl_depth[kOrder[0]] == 0 && cl_depth[kOrder[1]] == 0) {
      skip = 2;
      if (cl_depth[kOrder[2]] == 0) skip = 3;
    }
    br_put_bits(w, 2, skip);
    for (u32 i = skip; i < to_store; ++i) { u32 l = cl_depth[kOrder[i]]; br_put_bits(w, kLen[l], kSym[l]); }
  }
  if (num_codes == 1) cl_depth[code] = 0;
  for (u32 i = 0; i < hs; ++i) {
    u32 ix = sc->ht[i];
    br_put_bits(w, cl_depth[ix], cl_bits[ix]);
    if (ix == 16) br_put_bits(w, 2, sc->hx[i]);
    else if (ix == 17) br_put_bits(w, 3, sc->hx[i]);
  }
}
// brotli_bit_stream.c:349 BuildAndStoreHuffmanTree, split in two so that the construction of
// all prefix codes of a metablock can run in parallel and only the (cheap) storing is serial.
// Build: depth[] and bits[] (count <= 1 leaves depth 0 at the only symbol).
BR_DEV void br_build_tree(const u32* histo, u32 histo_len, BrHTree* tree, u8* depth, u16* bits) {
  u32 count = 0, first = 0;
  for (u32 i = 0; i < histo_len; i++) {
    if (histo[i]) { if (count == 0) first = i; if (++count > 1) break; }
  }
  if (count <= 1) { depth[first] = 0; bits[first] = 0; return; }
  for (u32 i = 0; i < histo_len; ++i) depth[i] = 0;
  br_create_huffman_tree(histo, histo_len, 15, tree, depth);
  br_depths_to_symbols(depth, histo_len, bits);
}
// Store (+ :242 StoreSimpleHuffmanTree / :283 BrotliStoreHuffmanTree)
template <class SC> BR_DEV void br_store_tree(const u32* histo, u32 histo_len, u32 alphabet_size, SC* sc,
                          const u8* depth, BrBitW& w) {
  u32 count = 0, s4[4] = {0, 0, 0, 0}, max_bits = 0;
  for (u32 i = 0; i < histo_len; i++) {
    if (histo[i]) {
      if (count < 4) s4[count] = i; else if (count > 4) break;
      count++;
    }
  }
  { u32 c = alphabet_size - 1; while (c) { c >>= 1; ++max_bits; } }
  if (count <= 1) {
    br_put_bits(w, 4, 1);
    br_put_bits(w, max_bits, s4[0]);
    return;
  }
  if (count <= 4) {
    br_put_bits(w, 2, 1);
    br_put_bits(w, 2, count - 1);
    for (u32 i = 0; i < count; i++)
      for (u32 j = i + 1; j < count; j++)
        if (depth[s4[j]] < depth[s4[i]]) { u32 t = s4[j]; s4[j] = s4[i]; s4[i] = t; }
    for (u32 i = 0; i < count; ++i) br_put_bits(w, max_bits, s4[i]);
    if (count == 4) br_put_bits(w, 1, depth[s4[0]] == 1 ? 1 : 0);
  } else {
    br_store_huffman_tree(depth, histo_len, sc, w);
  }
}
BR_DEV void br_build_and_store_tree(const u32* histo, u32 histo_len, u32 alphabet_size,
                                    BrMbScratch* sc, u8* depth, u16* bits, BrBitW& w) {
  br_build_tree(histo, histo_len, sc->tree, depth, bits);
  br_store_tree(histo, histo_len, alphabet_size, sc, depth, w);
}

BR_DEV void br_store_varlen_uint8(u32 n, BrBitW& w) {
  if (n == 0) br_put_bits(w, 1, 0);
  else { u32 nb = br_log2floor(n); br_put_bits(w, 1, 1); br_put_bits(w, 3, nb); br_put_bits(w, nb, n - (1u << nb)); }
}
// RFC 7932 section 6 block count codes (common/constants.c:10); closed form per code.
BR_DEV u32 br_block_len_offset(u32 c) {
  const u16 t[26] = {1, 5, 9, 13, 17, 25, 33, 41, 49, 65, 81, 97, 113, 145, 177, 209, 241, 305,
                     369, 497, 753, 1265, 2289, 4337, 8433, 16625};
  return t[c];
}
BR_DEV u32 br_block_len_nbits(u32 c) {
  const u8 t[26] = {2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 6, 6, 7, 8, 9, 10, 11, 12, 13, 24};
  return t[c];
}
BR_DEV u32 br_block_len_code(u32 len) {
  u32 code = (len >= 177) ? (len >= 753 ? 20 : 14) : (len >= 41 ? 7 : 0);
  while (code < 25 && len >= br_block_len_offset(code + 1)) ++code;
  return code;
}
// brotli_bit_stream.c:70 BrotliEncodeMlen
BR_DEV void br_store_mlen(u32 length, BrBitW& w) {
  u32 lg = (length == 1) ? 1 : br_log2floor(length - 1) + 1;
  u32 mnibbles = (lg < 16 ? 16 : (lg + 3)) / 4;
  br_put_bits(w, 2, mnibbles - 4);
  br_put_bits(w, mnibbles * 4, length - 1);
}

// ------------------------------------------------------------------ greedy block splitter
struct BrSplit { u32 num_types, num_blocks; u8* types; u32* lengths; };

#define BR_CTX_UTF8(st, p1, p2) ((u32)(br_ldg((st).ctx_lut + 1024 + (p1)) | br_ldg((st).ctx_lut + 1280 + (p2))))

BR_DEV u32 br_static_ctx_map(int which, u32 ctx) {
  // encode.c:283 (continuation), :289 (simple UTF8), :343 (complex UTF8)
  if (which == 3) return ctx < 2 ? 1 : ctx < 4 ? 2 : 0;
  if (which == 2) return (ctx == 2 || ctx == 3) ? 1 : 0;
  const u8 c13[64] = {11, 11, 12, 12, 0, 0, 0, 0, 1, 1, 9, 9, 2, 2, 2, 2, 1, 1, 1, 1, 8, 3, 3, 3,
                      1, 1, 1, 1, 2, 2, 2, 2, 8, 4, 4, 4, 8, 7, 4, 4, 8, 0, 0, 0, 3, 3, 3, 3,
                      5, 5, 10, 5, 5, 5, 10, 5, 6, 6, 6, 6, 6, 6, 6, 6};
  return c13[ctx];
}
// the byte `back` positions in front of pos; zero in front of the stream's first byte (base)
BR_DEV u8 br_data_or_zero(const BrStream& st, u32 pos, u32 back, u32 base) { return pos - base >= back ? st.data[pos - back] : 0; }

// A CTA's threads (one in the CPU simulation) and its barrier.
#if BR_GPU
#define BR_CTA_TID ((u32)threadIdx.x)
#define BR_CTA_N ((u32)blockDim.x)
BR_DEV void br_cta_sync() { __syncthreads(); }
BR_DEV u32 br_smem_add(u32* p, u32 v) { return atomicAdd(p, v); }
#else
#define BR_CTA_TID 0u
#define BR_CTA_N 1u
BR_DEV void br_cta_sync() {}
BR_DEV u32 br_smem_add(u32* p, u32 v) { u32 o = *p; *p = o + v; return o; }
#endif

// encode.c:258 EstimateEntropy
BR_DEV double br_estimate_entropy(const BrStream& st, const u32* pop, u32 size) {
  u32 total = 0; double result = 0;
  for (u32 i = 0; i < size; ++i) {
    u32 p = pop[i];
    total += p;
    result = br_dadd(result, br_dmul((double)p, br_fast_log2(st, p)));
  }
  return br_dsub(br_dmul((double)total, br_fast_log2(st, total)), result);
}
// encode.c:424 DecideOverLiteralContextModeling; returns number of contexts (1, 2, 3 or 13).  Run by a whole CTA (one
// thread in the CPU simulation), the strides spread over its threads; the counts are integers, so the order in which
// the threads add them does not matter.  scratch: >= 14*32 words, shared memory in k_mb_setup.
BR_DEV u32 br_decide_context_modeling(const BrStream& st, u32 start_pos, u32 length, u32* scratch) {
  const BrParams& P = st.P;
  const u32 tid = BR_CTA_TID, nt = BR_CTA_N;
  if (P.quality < 5 || length < 64) return 1;
  const u32 end_pos = start_pos + length;
  if (P.size_hint >= (1u << 20)) {
    u32* combined = scratch; u32* ctxh = scratch + 32;
    for (u32 i = tid; i < 14 * 32; i += nt) scratch[i] = 0;
    br_cta_sync();
    u32 nstrides = (length >= 64) ? (length - 64) / 4096 + 1 : 0;
    for (u32 si = tid; si < nstrides; si += nt) {
      u32 sp = start_pos + si * 4096;
      u8 prev2 = st.data[sp], prev1 = st.data[sp + 1];
      for (u32 pos = sp + 2; pos < sp + 64; ++pos) {
        u8 lit = st.data[pos];
        u32 ctx = br_static_ctx_map(13, BR_CTX_UTF8(st, prev1, prev2));
        br_smem_add(combined + (lit >> 3), 1);
        br_smem_add(ctxh + (ctx << 5) + (lit >> 3), 1);
        prev2 = prev1; prev1 = lit;
      }
    }
    br_cta_sync();
    u32 total = nstrides * 62;
    double e1 = br_estimate_entropy(st, combined, 32), e2 = 0;
    for (u32 i = 0; i < 13; ++i) e2 = br_dadd(e2, br_estimate_entropy(st, ctxh + (i << 5), 32));
    double e0 = br_ddiv(1.0, (double)total);
    e1 = br_dmul(e1, e0); e2 = br_dmul(e2, e0);
    if (!(e2 > 3.0 || br_dsub(e1, e2) < 0.2)) return 13;
    br_cta_sync();   // (every thread has read `combined` before bigram, which overlaps it, is cleared)
  }
  {
    u32* bigram = scratch;
    for (u32 i = tid; i < 16; i += nt) bigram[i] = 0;
    br_cta_sync();
    u32 nstrides = (length - 64) / 4096 + 1;
    for (u32 si = tid; si < nstrides; si += nt) {
      u32 sp = start_pos + si * 4096;
      const u8 lut[4] = {0, 0, 1, 2};
      u32 prev = lut[st.data[sp] >> 6] * 3u;
      for (u32 pos = sp + 1; pos < sp + 64; ++pos) {
        u8 lit = st.data[pos];
        br_smem_add(bigram + prev + lut[lit >> 6], 1);
        prev = lut[lit >> 6] * 3u;
      }
    }
    br_cta_sync();
    (void)end_pos;
    // encode.c:277 ChooseContextMap
    u32 mono[3] = {0, 0, 0}, two[6] = {0, 0, 0, 0, 0, 0};
    for (u32 i = 0; i < 9; ++i) { mono[i % 3] += bigram[i]; two[i % 6] += bigram[i]; }
    double entropy[4];
    entropy[1] = br_estimate_entropy(st, mono, 3);
    entropy[2] = br_dadd(br_estimate_entropy(st, two, 3), br_estimate_entropy(st, two + 3, 3));
    entropy[3] = 0;
    for (u32 i = 0; i < 3; ++i) entropy[3] = br_dadd(entropy[3], br_estimate_entropy(st, bigram + 3 * i, 3));
    u32 total = mono[0] + mono[1] + mono[2];
    entropy[0] = br_ddiv(1.0, (double)total);
    entropy[1] = br_dmul(entropy[1], entropy[0]);
    entropy[2] = br_dmul(entropy[2], entropy[0]);
    entropy[3] = br_dmul(entropy[3], entropy[0]);
    if (P.quality < 7) entropy[3] = br_dmul(entropy[1], 10.0);
    if (br_dsub(entropy[1], entropy[2]) < 0.2 && br_dsub(entropy[1], entropy[3]) < 0.2) return 1;
    if (br_dsub(entropy[2], entropy[3]) < 0.02) return 2;
    return 3;
  }
}

// ------------------------------------------------------------------ metablock memory map
// Fixed-size part of the per-metablock global scratch (worst case over block types).
struct BrBlockCode {   // brotli_bit_stream.c:95 BlockSplitCode
  u8 type_depths[258]; u16 type_bits[258];
  u8 len_depths[26]; u16 len_bits[26];
};
struct BrMbMem {
  BrMbScratch sc;
  BrBlockCode code[3];
  u32 lit_H[256 * 256];
  u32 cmd_H[256 * 704];
  u32 dist_H[256 * 64];
  u32 lit_comb[2 * 13 * 256];
  u32 cmd_comb[2 * 704];
  u32 dist_comb[2 * 64];
  u8 lit_depth[256 * 256]; u16 lit_bits[256 * 256];
  u8 cmd_depth[256 * 704]; u16 cmd_bits[256 * 704];
  u8 dist_depth[256 * 64]; u16 dist_bits[256 * 64];
  u32 cmap[256 * 64];
};
// variable part follows: literal split (types, lengths), command split, distance split
BR_HD u32 br_align8(u32 x) { return (x + 7u) & ~7u; }

// brotli_bit_stream.c:879 BlockEncoder state (warp-uniform registers)
struct BrBlockEnc {
  u32 hist_len, num_types, num_blocks;
  const u8* types; const u32* lengths;
  u32 last_type, second_last_type;
  BrBlockCode* code;
  u32 block_ix, block_len, entropy_ix;
  const u8* depths; const u16* bits;
};
BR_DEV u32 br_next_type_code(u32* last, u32* second, u32 type) {
  u32 code = (type == *last + 1) ? 1u : (type == *second) ? 0u : type + 2u;
  *second = *last; *last = type;
  return code;
}
// brotli_bit_stream.c:736 StoreBlockSwitch
BR_DEV void br_store_block_switch(BrBlockEnc& b, u32 block_len, u32 block_type, int is_first, BrBitW& w) {
  u32 typecode = br_next_type_code(&b.last_type, &b.second_last_type, block_type);
  if (!is_first) br_put_bits(w, b.code->type_depths[typecode], b.code->type_bits[typecode]);
  u32 lencode = br_block_len_code(block_len);
  br_put_bits(w, b.code->len_depths[lencode], b.code->len_bits[lencode]);
  br_put_bits(w, br_block_len_nbits(lencode), block_len - br_block_len_offset(lencode));
}
// brotli_bit_stream.c:760 BuildAndStoreBlockSplitCode (lane-0 section inside)
BR_DEV void br_build_and_store_block_split_code(BrBlockEnc& b, BrMbScratch* sc, BrBitW& w) {
  br_store_varlen_uint8(b.num_types - 1, w);
  if (b.num_types > 1) {
    BR_LANE0_BEGIN
      u32* type_histo = sc->small_histo;   // num_types + 2 <= 258
      u32 length_histo[26];
      u32 last = 1, second = 0;
      for (u32 i = 0; i < b.num_types + 2; ++i) type_histo[i] = 0;
      for (u32 i = 0; i < 26; ++i) length_histo[i] = 0;
      for (u32 i = 0; i < b.num_blocks; ++i) {
        u32 tc = br_next_type_code(&last, &second, b.types[i]);
        if (i != 0) ++type_histo[tc];
        ++length_histo[br_block_len_code(b.lengths[i])];
      }
      br_build_and_store_tree(type_histo, b.num_types + 2, b.num_types + 2, sc, b.code->type_depths, b.code->type_bits, w);
      br_build_and_store_tree(length_histo, 26, 26, sc, b.code->len_depths, b.code->len_bits, w);
    BR_LANE0_END(w)
    br_store_block_switch(b, b.lengths[0], b.types[0], 1, w);
  }
}
BR_DEV void br_block_enc_init(BrBlockEnc& b, u32 hist_len, const BrSplit& s, BrBlockCode* code) {
  b.hist_len = hist_len; b.num_types = s.num_types; b.types = s.types; b.lengths = s.lengths;
  b.num_blocks = s.num_blocks; b.last_type = 1; b.second_last_type = 0; b.code = code;
  b.block_ix = 0; b.block_len = s.num_blocks == 0 ? 0 : s.lengths[0]; b.entropy_ix = 0;
  b.depths = 0; b.bits = 0;
}
// brotli_bit_stream.c:794 StoreTrivialContextMap (lane-0 section)
BR_DEV void br_store_trivial_context_map(u32 num_types, u32 context_bits, BrMbScratch* sc, BrBitW& w) {
  br_store_varlen_uint8(num_types - 1, w);
  if (num_types > 1) {
    BR_LANE0_BEGIN
      u32 repeat_code = context_bits - 1u, repeat_bits = (1u << repeat_code) - 1u;
      u32 alphabet = num_types + repeat_code;
      u32* histo = sc->small_histo; u8* depths = sc->small_depth; u16* bits = sc->small_bits;
      for (u32 i = 0; i < alphabet; ++i) histo[i] = 0;
      br_put_bits(w, 1, 1); br_put_bits(w, 4, repeat_code - 1);
      histo[repeat_code] = num_types;
      histo[0] = 1;
      for (u32 i = context_bits; i < alphabet; ++i) histo[i] = 1;
      br_build_and_store_tree(histo, alphabet, alphabet, sc, depths, bits, w);
      for (u32 i = 0; i < num_types; ++i) {
        u32 code = (i == 0 ? 0 : i + context_bits - 1);
        br_put_bits(w, depths[code], bits[code]);
        br_put_bits(w, depths[repeat_code], bits[repeat_code]);
        br_put_bits(w, repeat_code, repeat_bits);
      }
      br_put_bits(w, 1, 1);
    BR_LANE0_END(w)
  }
}
// brotli_bit_stream.c:683 EncodeContextMap with :592 MoveToFrontTransform, :624 RunLengthCodeZeros
BR_DEV void br_encode_context_map(const u32* cmap, u32 cmap_size, u32 num_clusters, BrMbScratch* sc, BrBitW& w) {
  br_store_varlen_uint8(num_clusters - 1, w);
  if (num_clusters == 1) return;
  BR_LANE0_BEGIN
    u32* rle = sc->rle_syms; u32 max_prefix = 6, n_rle = 0;
    u32* histo = sc->small_histo; u8* depths = sc->small_depth; u16* bits = sc->small_bits;
    {
      u8 mtf[256]; u32 maxv = cmap[0];
      for (u32 i = 1; i < cmap_size; ++i) if (cmap[i] > maxv) maxv = cmap[i];
      for (u32 i = 0; i <= maxv; ++i) mtf[i] = (u8)i;
      u32 sz = maxv + 1;
      for (u32 i = 0; i < cmap_size; ++i) {
        u32 idx = 0;
        while (idx < sz && mtf[idx] != (u8)cmap[i]) ++idx;
        rle[i] = idx;
        u8 v = mtf[idx];
        for (u32 k = idx; k != 0; --k) mtf[k] = mtf[k - 1];
        mtf[0] = v;
      }
    }
    {
      u32 max_reps = 0;
      for (u32 i = 0; i < cmap_size;) {
        u32 reps = 0;
        for (; i < cmap_size && rle[i] != 0; ++i) ;
        for (; i < cmap_size && rle[i] == 0; ++i) ++reps;
        if (reps > max_reps) max_reps = reps;
      }
      u32 mp = max_reps > 0 ? br_log2floor(max_reps) : 0;
      if (mp < max_prefix) max_prefix = mp;
      for (u32 i = 0; i < cmap_size;) {
        if (rle[i] != 0) { rle[n_rle++] = rle[i] + max_prefix; ++i; }
        else {
          u32 reps = 1;
          for (u32 k = i + 1; k < cmap_size && rle[k] == 0; ++k) ++reps;
          i += reps;
          while (reps != 0) {
            if (reps < (2u << max_prefix)) {
              u32 pfx = br_log2floor(reps);
              rle[n_rle++] = pfx + ((reps - (1u << pfx)) << 9);
              break;
            } else {
              rle[n_rle++] = max_prefix + (((1u << max_prefix) - 1u) << 9);
              reps -= (2u << max_prefix) - 1u;
            }
          }
        }
      }
    }
    for (u32 i = 0; i < 272; ++i) histo[i] = 0;
    for (u32 i = 0; i < n_rle; ++i) ++histo[rle[i] & 511];
    {
      int use_rle = max_prefix > 0;
      br_put_bits(w, 1, (u64)use_rle);
      if (use_rle) br_put_bits(w, 4, max_prefix - 1);
    }
    br_build_and_store_tree(histo, num_clusters + max_prefix, num_clusters + max_prefix, sc, depths, bits, w);
    for (u32 i = 0; i < n_rle; ++i) {
      u32 sym = rle[i] & 511, extra = rle[i] >> 9;
      br_put_bits(w, depths[sym], bits[sym]);
      if (sym > 0 && sym <= max_prefix) br_put_bits(w, sym, extra);
    }
    br_put_bits(w, 1, 1);
  BR_LANE0_END(w)
}
