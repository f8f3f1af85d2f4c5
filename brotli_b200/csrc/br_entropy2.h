// br_entropy2.h -- data-parallel formulation of the per-metablock entropy pipeline.
//
// The serial restatement in br_entropy.h (one warp per metablock) stays as the reference the
// sim checks against; this file decomposes the same computation:
//
//   E0  prefix sums over commands      literal ordinal / input position / distance ordinal
//   E1  br_expand_cmd                   literal ordinal -> input position, compact distance symbols
//   E2  br_decide_context_modeling      (br_entropy.h; one CTA per metablock, shared-memory counts)
//   E3  br_split_syms / br_split_cta    greedy block split: every symbol's histogram row as a u16
//                                       array, then the decision CHAIN of metablock_inc.h:86, serial,
//                                       each link executed by a whole CTA (16-byte symbol loads counted
//                                       with shared-memory atomics, the 3 x contexts entropy sums on
//                                       separate threads)
//   E4  br_code_build / br_mb_header    smoothing + Huffman construction of every prefix code of the job
//       / br_code_store                 in parallel, the header by one warp per metablock, then every
//                                       code stored at its offset in parallel
//   E5  br_lit_bits / br_cmd_bits       per-symbol bit counts; prefix sums give every symbol its
//                                       absolute bit offset (the north-star "prefix-sum packing")
//   E6  br_emit_lit / br_emit_cmd       scatter of the code words with atomic OR
#pragma once
#include "br_entropy.h"

// per-metablock results of the parallel stages
struct BrMbAux {
  u32 which;                 // 1, 2, 3 or 13 literal contexts (static map id)
  u32 num_types[3], num_blocks[3];   // literal, command, distance
  u32 nsym[3];
  u32 lit_base, dist_base;   // global ordinals of the first literal / distance symbol
  u32 hdr_bits;
  u32 var_off[3];            // byte offsets of the per-category block arrays inside the scratch
  u32 cmap_size;
};
// per block of a split (stored after E4): where it starts and what precedes its first symbol
struct BrBlockInfo { u32 start; u32 sw_nbits; u64 sw_bits; u32 type; u32 pad; };

BR_HD u32 br_mb2_var_bytes(u32 nblk) { return br_align8(nblk * ((u32)sizeof(BrBlockInfo) + 4) + nblk) + 8; }
#define BR_CODE_BITS_WORDS (3 * 256 + 8)
BR_HD u32 br_mb2_scratch_bytes(u32 nlit, u32 ncmd) {
  u32 lb = nlit / 512 + 2, cb = ncmd / 1024 + 2, db = ncmd / 512 + 2;
  return br_align8((u32)sizeof(BrMbMem)) + br_mb2_var_bytes(lb) + br_mb2_var_bytes(cb) + br_mb2_var_bytes(db) +
         BR_CODE_BITS_WORDS * 4;   // + sizes / offsets of the stored codes
}
// [nl + ncm + nd + 1]: the stored size of every prefix code of the metablock, then (br_mb_header) its bit offset
BR_DEV u32* br_mb2_code_bits(u8* scratch, const BrMetaBlock& mb) {
  return (u32*)(scratch + br_mb2_scratch_bytes(mb.nlit, mb.ncmd) - BR_CODE_BITS_WORDS * 4);
}
// Most prefix codes a metablock can have: a literal code per (block type, context) and a command and a distance code per
// block type.  A split has at most one type per block and at most 256 / contexts types (up to 13 contexts).
BR_HD u32 br_mb2_code_bound(u32 nlit, u32 ncmd) {
  const u32 lb = nlit / 512 + 2, cb = ncmd / 1024 + 2, db = ncmd / 512 + 2;
  return (13 * lb < 256 ? 13 * lb : 256) + (cb < 256 ? cb : 256) + (db < 256 ? db : 256);
}
// Prefix codes of a job (E4) are built and stored either by a warp each, on a copy in shared memory (BrCodeSmem), when
// the job has at most BR_CODE_WARP_MAX of them, or else by a thread each.  A thread worker's tree area (the Huffman tree
// of the largest alphabet, which the store reuses as its BrTreeSc) comes from a pool of the job: BR_CODE_TREE_NODES each,
// for at most BR_CODE_THREADS_MAX workers.
#define BR_CODE_TREE_NODES (2 * 704 + 2)
#define BR_CODE_WARP_MAX 8192u
#define BR_CODE_THREADS_MAX 65536u
struct BrCodeSmem {
  BrHTree tree[BR_CODE_TREE_NODES];
  u32 H[704];
  u16 bits[704];
  u8 depth[704], good[704];
};
BR_DEV BrBlockInfo* br_mb2_blocks(u8* scratch, const BrMbAux& a, int cat) { return (BrBlockInfo*)(scratch + a.var_off[cat]); }
BR_DEV u32* br_mb2_lengths(u8* scratch, const BrMbAux& a, int cat, u32 nblk) {
  return (u32*)(scratch + a.var_off[cat] + nblk * (u32)sizeof(BrBlockInfo));
}
BR_DEV u8* br_mb2_types(u8* scratch, const BrMbAux& a, int cat, u32 nblk) {
  return scratch + a.var_off[cat] + nblk * ((u32)sizeof(BrBlockInfo) + 4);
}
BR_HD u32 br_mb2_nblk(int cat, u32 nlit, u32 ncmd) { return cat == 0 ? nlit / 512 + 2 : cat == 1 ? ncmd / 1024 + 2 : ncmd / 512 + 2; }

// Qualities 2 and 3 (BrParams::mb_kind != 0): one prefix code per category, no block splits, no contexts
// (br_entropy_flat.h).  This is the whole per-metablock scratch of such a job.
struct BrMbFlat {
  u32 lit_H[256], cmd_H[704], dist_H[64];
  u8 lit_depth[256], cmd_depth[704], dist_depth[64];
  u16 lit_bits[256], cmd_bits[704], dist_bits[64];
  BrHTree tree[2 * 704 + 2];
  BrTreeSc tsc;
};
BR_HD u32 br_mb_scratch_bytes(const BrParams& P, u32 nlit, u32 ncmd) {
  return P.mb_kind ? br_align8((u32)sizeof(BrMbFlat)) : br_mb2_scratch_bytes(nlit, ncmd);
}

// stream-wide arrays of the parallel entropy stage
struct BrEnt {
  const BrCmd* cmds;       // compacted commands of the stream
  u32 total_cmds, total_lits, total_dist;
  const u32* lit_ord;      // [total_cmds + 1] exclusive scan of insert_len
  const u32* cmd_pos;      // [total_cmds + 1] exclusive scan of insert_len + copy_len (absolute input position)
  const u32* dist_ord;     // [total_cmds + 1] exclusive scan of "has explicit distance"
  u32* lit_pos;            // [total_lits] input position of every literal
  u32* lit_cmd;            // [total_lits] command owning the literal
  u16* dist_sym;           // [total_dist + 16]
  u16* lit_sym;            // [total_lits + 16] E3's histogram row of every literal: context * 256 + byte (br_split_syms)
  u16* cmd_sym;            // [total_cmds + 16] command prefix of every command
  u32* lit_len;            // [total_lits + 1] bit counts, then (in place) their exclusive scan
  u32* cmd_len;            // [total_cmds + 1] likewise for command + distance parts
  u32* lit_bit_base;       // [total_cmds] add the scanned lit_len of a literal to get its bit offset
  u32* cmd_mb;             // [total_cmds] metablock of every command
  BrMbAux* aux;            // [n_mbs]
  u8* scratch; const u64* scratch_off;   // per-metablock scratch
  u32* outbits; const u64* out_off;      // per-metablock bit buffers (u32 words)
};

// largest i in [0, n) with a[i] <= x  (a is non-decreasing, a[0] <= x)
BR_DEV u32 br_upper_index(const u32* a, u32 n, u32 x) {
  u32 lo = 0, hi = n;
  while (hi - lo > 1) { u32 mid = (lo + hi) >> 1; if (br_ldg(a + mid) <= x) lo = mid; else hi = mid; }
  return lo;
}

// ---------------------------------------------------------------------------------- E0 inputs
BR_DEV void br_cmd_scan_inputs(const BrCmd& c, u32* ins, u32* span, u32* hasd) {
  u32 cl = br_cmd_copy_len(c);
  *ins = c.insert_len; *span = c.insert_len + cl; *hasd = (cl && c.cmd_prefix >= 128) ? 1u : 0u;
}
// ---------------------------------------------------------------------------------- E1
// one warp handles 32 consecutive commands: literal ordinal -> position / owner, distance symbols
BR_DEV void br_expand_cmds(const BrEnt& e, u32 first_cmd) {
  const int lane = br_lane();
  u32 i = first_cmd + (u32)lane;
  u32 ord = 0, pos = 0, len = 0;
  if (i < e.total_cmds) {
    const BrCmd c = e.cmds[i];
    ord = e.lit_ord[i]; pos = e.cmd_pos[i]; len = c.insert_len;
    if (br_cmd_copy_len(c) && c.cmd_prefix >= 128) e.dist_sym[e.dist_ord[i]] = (u16)(c.dist_prefix & 0x3FF);
  }
  u32 cnt = e.total_cmds - first_cmd < BR_WARP ? e.total_cmds - first_cmd : BR_WARP;
  for (u32 t = 0; t < cnt; ++t) {
    u32 o = br_shfl(ord, (int)t), p = br_shfl(pos, (int)t), l = br_shfl(len, (int)t);
    for (u32 k = (u32)lane; k < l; k += BR_WARP) { e.lit_pos[o + k] = p + k; e.lit_cmd[o + k] = first_cmd + t; }
  }
}

// ---------------------------------------------------------------------------------- E2 / E3 setup
// What k_mb_setup records for a compressed metablock once E2 has chosen `which`: its first literal and distance ordinals,
// its symbol counts and where its block arrays lie in the scratch.
BR_DEV void br_mb_aux_init(BrMbAux& a, const BrMetaBlock& mb, const BrEnt& e, u32 which) {
  memset(&a, 0, sizeof(a));
  a.which = which;
  a.lit_base = e.lit_ord[mb.cmd_off]; a.dist_base = e.dist_ord[mb.cmd_off];
  a.nsym[0] = mb.nlit; a.nsym[1] = mb.ncmd; a.nsym[2] = e.dist_ord[mb.cmd_off + mb.ncmd] - a.dist_base;
  u32 off = br_align8((u32)sizeof(BrMbMem));
  for (int cat = 0; cat < 3; ++cat) { a.var_off[cat] = off; off += br_mb2_var_bytes(br_mb2_nblk(cat, mb.nlit, mb.ncmd)); }
}
// The greedy splitter's constants of a category (metablock.c:708): alphabet, histogram contexts (literals, cat 0, have
// the metablock's `which`; commands and distances one), shortest block and split threshold.  Macros, so that k_split
// reads `which` only for literals, as it always has; br_split_cat gathers them for the CPU simulation.
#define BR_SPLIT_ALPHABET(cat) ((cat) == 0 ? 256u : (cat) == 1 ? 704u : 64u)
#define BR_SPLIT_CONTEXTS(cat, which) ((cat) == 0 ? (which) : 1u)
#define BR_SPLIT_MIN_BLOCK(cat) ((cat) == 1 ? 1024u : 512u)
#define BR_SPLIT_THR(cat) ((cat) == 0 ? 400.0 : (cat) == 1 ? 500.0 : 100.0)
#define BR_SPLIT_HIST(M, cat) ((cat) == 0 ? (M)->lit_H : (cat) == 1 ? (M)->cmd_H : (M)->dist_H)
struct BrSplitCat { u32 A, nc, min_block; double thr; };
BR_HD BrSplitCat br_split_cat(int cat, u32 which) {
  BrSplitCat k;
  k.A = BR_SPLIT_ALPHABET(cat); k.nc = BR_SPLIT_CONTEXTS(cat, which);
  k.min_block = BR_SPLIT_MIN_BLOCK(cat); k.thr = BR_SPLIT_THR(cat);
  return k;
}

// ---------------------------------------------------------------------------------- E3
struct BrSplitState {
  u32 target, block_size, num_blocks, num_types, last_ix[2], merge_last_count, action;
  double last_entropy[26];
};
// symbol `o` (metablock-relative ordinal) of category cat: value and histogram row (context)
BR_DEV void br_symbol_at(const BrStream& st, const BrEnt& e, const BrMetaBlock& mb, const BrMbAux& a, int cat, u32 o,
                         u32* sym, u32* ctx) {
  *ctx = 0;
  if (cat == 0) {
    u32 p = e.lit_pos[a.lit_base + o];
    *sym = st.data[p];
    if (a.which != 1) *ctx = br_static_ctx_map((int)a.which, BR_CTX_UTF8(st, br_data_or_zero(st, p, 1, mb.base), br_data_or_zero(st, p, 2, mb.base)));
  } else if (cat == 1) {
    *sym = e.cmds[mb.cmd_off + o].cmd_prefix;
  } else {
    *sym = e.dist_sym[a.dist_base + o];
  }
}
// the histogram row of symbol `o` of category cat: context * 256 + byte for a literal, the symbol itself otherwise
BR_DEV u16 br_split_row(const BrStream& st, const BrEnt& e, const BrMetaBlock& mb, const BrMbAux& a, int cat, u32 o) {
  u32 sym, ctx;
  br_symbol_at(st, e, mb, a, cat, o, &sym, &ctx);
  return (u16)(ctx * 256 + sym);
}
// E3's symbols of compressed metablock mb as coalesced u16 arrays, element i of its literals and of its commands (E2 has
// chosen a.which): their histogram rows.  Distances are dist_sym.
BR_DEV void br_split_syms(const BrStream& st, const BrEnt& e, const BrMetaBlock& mb, const BrMbAux& a, u32 i) {
  if (i < mb.nlit) e.lit_sym[a.lit_base + i] = br_split_row(st, e, mb, a, 0, i);
  if (i < mb.ncmd) e.cmd_sym[mb.cmd_off + i] = br_split_row(st, e, mb, a, 1, i);
}
// 8 u16 from p (16-byte aligned) as 4 words
BR_DEV void br_load_u16x8(const u16* p, u32 w[4]) {
#if BR_GPU
  const uint4 q = __ldg((const uint4*)p);
  w[0] = q.x; w[1] = q.y; w[2] = q.z; w[3] = q.w;
#else
  memcpy(w, p, 16);
#endif
}
// Counts the rows syms[b .. b + n) into cur.  Each thread reads whole 16-byte groups of 8 symbols, up to 4 groups before
// it counts any, so that its loads are in flight together; of the groups at either end only what lies inside is counted
// (the arrays are 16-byte aligned and padded by 16 symbols).  The counts are integers: their order does not matter.
BR_DEV void br_split_count(const u16* syms, u32 b, u32 n, u32* cur) {
  const u32 tid = BR_CTA_TID, nt = BR_CTA_N, end = b + n;
  for (u32 g = (b & ~7u) + tid * 8; g < end; g += 32 * nt) {
    u32 w[4][4] = {};
#pragma unroll
    for (u32 j = 0; j < 4; ++j)
      if (g + j * 8 * nt < end) br_load_u16x8(syms + g + j * 8 * nt, w[j]);
#pragma unroll
    for (u32 j = 0; j < 4; ++j)
#pragma unroll
      for (u32 k = 0; k < 8; ++k) {
        const u32 x = g + j * 8 * nt + k;
        if (x >= b && x < end) br_smem_add(cur + ((w[j][k >> 1] >> (16 * (k & 1))) & 0xFFFFu), 1);
      }
  }
}
// Counts symbols [o, o + n) of category cat of metablock mb into cur.  On the GPU from the arrays br_split_syms has
// written (k_split_syms); the CPU simulation, which has no such arrays, stages the same rows (br_split_row) in pieces that
// keep the arrays' alignment and counts them with the same br_split_count.
BR_DEV void br_split_take(const BrStream& st, const BrEnt& e, const BrMetaBlock& mb, const BrMbAux& a, int cat, u32 o,
                          u32 n, u32* cur) {
  const u32 base = cat == 0 ? a.lit_base : cat == 1 ? mb.cmd_off : a.dist_base;
#if BR_GPU
  br_split_count(cat == 0 ? e.lit_sym : cat == 1 ? e.cmd_sym : e.dist_sym, base + o, n, cur);
#else
  for (u32 k = 0; k < n;) {
    u16 buf[1024 + 16] = {};
    const u32 lead = (base + o + k) & 7u, m = br_min(n - k, 1024u);
    for (u32 j = 0; j < m; ++j) buf[lead + j] = br_split_row(st, e, mb, a, cat, o + k + j);
    br_split_count(buf, lead, m, cur);
    k += m;
  }
#endif
}
// shared memory plan (u32 words): cur[nc*A] | comb[2*nc*A] | (8-aligned) terms[3*nc*(A|1)] doubles | ent[3*nc] | state
BR_HD u32 br_split_smem_bytes(u32 A, u32 nc) {
  return (3 * nc * A) * 4 + 8 + (3 * nc * (A | 1) + 3 * nc) * 8 + (u32)sizeof(BrSplitState) + 16;
}
// -(sum of terms[0 .. A)) from 0.0, in index order, as the reference's BitsEntropy accumulates it, and *sum = the sum of
// the counts p[0 .. A).  The zero terms (counts of 0 and 1) are subtracted too: r - (+0.0) is r bit for bit, -0.0
// included, so the result is the reference's without a branch, and the loads of 8 entries go out before their
// subtractions.
BR_DEV double br_split_neg_sum(const double* terms, const u32* p, u32 A, u32* sum) {
  double r = 0;
  u32 s = 0, i = 0;
  for (; i + 8 <= A; i += 8) {
    double v[8];
#pragma unroll
    for (u32 k = 0; k < 8; ++k) { v[k] = terms[i + k]; s += p[i + k]; }
#pragma unroll
    for (u32 k = 0; k < 8; ++k) r = br_dsub(r, v[k]);
  }
  for (; i < A; ++i) { r = br_dsub(r, terms[i]); s += p[i]; }
  *sum = s;
  return r;
}
// One CTA = one (metablock, category).  H: [256/nc * nc][A] finished histograms (global).
BR_DEV void br_split_cta(const BrStream& st, const BrEnt& e, const BrMetaBlock& mb, BrMbAux& a, int cat,
                         u32 A, u32 nc, u32 min_block, double thr, u32 nsym,
                         u8* types, u32* lengths, u32* H, u32* smem) {
  const u32 tid = BR_CTA_TID, nt = BR_CTA_N;
  const u32 NA = nc * A, AS = A | 1u, max_types = 256 / nc;
  u32* cur = smem; u32* comb = smem + NA;
  double* terms = (double*)(((uintptr_t)(smem + 3 * NA) + 7) & ~(uintptr_t)7);
  double* ent = terms + 3 * nc * AS;
  BrSplitState* S = (BrSplitState*)(ent + 3 * nc);
  for (u32 x = tid; x < NA; x += nt) cur[x] = 0;
  if (tid == 0) {
    S->target = min_block; S->block_size = 0; S->num_blocks = 0; S->num_types = 0;
    S->last_ix[0] = S->last_ix[1] = 0; S->merge_last_count = 0; S->action = 0;
  }
  br_cta_sync();
  u32 o = 0;
  for (;;) {
    const bool final_call = (o >= nsym);
    u32 take = 0;
    if (!final_call) {
      take = br_min(nsym - o, S->target - S->block_size);
      br_split_take(st, e, mb, a, cat, o, take, cur);
      o += take;
    }
    br_cta_sync();
    u32 bsz = S->block_size + take;
    if (!final_call && bsz != S->target) {   // input exhausted inside a block: the final call follows
      br_cta_sync();
      if (tid == 0) S->block_size = bsz;
      br_cta_sync();
      continue;
    }
    // ---------------- BlockSplitterFinishBlock (metablock_inc.h:86 / metablock.c:524)
    if (bsz < min_block) bsz = min_block;
    const u32 nb_now = S->num_blocks;
    if (nb_now == 0) {
      for (u32 x = tid; x < nc * A; x += nt) { u32 t = x / A, i = x - t * A; u32 p = cur[x]; terms[t * AS + i] = p ? br_dmul((double)p, br_fast_log2(st, p)) : 0.0; }
      br_cta_sync();
      for (u32 t = tid; t < nc; t += nt) {
        u32 sum;
        double r = br_split_neg_sum(terms + t * AS, cur + t * A, A, &sum);
        if (sum) r = br_dadd(r, br_dmul((double)sum, br_fast_log2(st, sum)));
        if (r < (double)sum) r = (double)sum;
        ent[t] = r;
      }
      br_cta_sync();
      if (tid == 0) {
        lengths[0] = bsz; types[0] = 0;
        for (u32 i = 0; i < nc; ++i) { S->last_entropy[i] = ent[i]; S->last_entropy[nc + i] = ent[i]; }
        S->num_blocks = 1; S->num_types = 1; S->block_size = 0;
      }
      for (u32 x = tid; x < NA; x += nt) { H[x] = cur[x]; cur[x] = 0; }
      br_cta_sync();
    } else if (bsz > 0) {
      const u32 l0 = S->last_ix[0], l1 = S->last_ix[1];
      for (u32 x = tid; x < 2 * NA; x += nt) {
        u32 j = x / NA, r = x - j * NA;
        comb[x] = cur[r] + H[(j ? l1 : l0) * A + r];
      }
      br_cta_sync();
      for (u32 x = tid; x < 3 * NA; x += nt) {
        u32 t = x / A, i = x - t * A;
        u32 p = t < nc ? cur[x] : comb[x - NA];
        terms[t * AS + i] = p ? br_dmul((double)p, br_fast_log2(st, p)) : 0.0;
      }
      br_cta_sync();
      for (u32 t = tid; t < 3 * nc; t += nt) {
        const u32* src = t < nc ? cur + t * A : comb + (t - nc) * A;
        u32 sum;
        double r = br_split_neg_sum(terms + t * AS, src, A, &sum);
        if (sum) r = br_dadd(r, br_dmul((double)sum, br_fast_log2(st, sum)));
        if (r < (double)sum) r = (double)sum;
        ent[t] = r;
      }
      br_cta_sync();
      if (tid == 0) {
        double diff[2] = {0.0, 0.0};
        for (u32 i = 0; i < nc; ++i)
          for (u32 j = 0; j < 2; ++j) {
            u32 jx = j * nc + i;
            diff[j] = br_dadd(diff[j], br_dsub(br_dsub(ent[nc + jx], ent[i]), S->last_entropy[jx]));
          }
        u32 nbk = S->num_blocks;
        if (S->num_types < max_types && diff[0] > thr && diff[1] > thr) {
          lengths[nbk] = bsz; types[nbk] = (u8)S->num_types;
          S->last_ix[1] = S->last_ix[0]; S->last_ix[0] = S->num_types * nc;
          for (u32 i = 0; i < nc; ++i) { S->last_entropy[nc + i] = S->last_entropy[i]; S->last_entropy[i] = ent[i]; }
          ++S->num_blocks; ++S->num_types;
          S->merge_last_count = 0; S->target = min_block; S->action = 1;
        } else if (diff[1] < br_dsub(diff[0], 20.0)) {
          lengths[nbk] = bsz; types[nbk] = types[nbk - 2];
          u32 t = S->last_ix[0]; S->last_ix[0] = S->last_ix[1]; S->last_ix[1] = t;
          for (u32 i = 0; i < nc; ++i) { S->last_entropy[nc + i] = S->last_entropy[i]; S->last_entropy[i] = ent[2 * nc + i]; }
          ++S->num_blocks;
          S->merge_last_count = 0; S->target = min_block; S->action = 2;
        } else {
          lengths[nbk - 1] += bsz;
          for (u32 i = 0; i < nc; ++i) {
            S->last_entropy[i] = ent[nc + i];
            if (S->num_types == 1) S->last_entropy[nc + i] = S->last_entropy[i];
          }
          if (++S->merge_last_count > 1) S->target += min_block;
          S->action = 3;
        }
        S->block_size = 0;
      }
      br_cta_sync();
      {
        const u32 act = S->action, dst = S->last_ix[0];
        for (u32 x = tid; x < NA; x += nt) {
          H[dst * A + x] = act == 1 ? cur[x] : act == 2 ? comb[NA + x] : comb[x];
          cur[x] = 0;
        }
      }
      br_cta_sync();
    }
    if (final_call) break;
  }
  if (tid == 0) { a.num_types[cat] = S->num_types; a.num_blocks[cat] = S->num_blocks; }
}

// ---------------------------------------------------------------------------------- E4
// Three job-wide phases (brotli_bit_stream.c:947-1060 and :349 BuildAndStoreHuffmanTree).  Every prefix code of the job
// is built by one worker, which also measures how many bits its serialised form takes (the store, run against a counting
// writer).  Then one warp per metablock writes the header in front of the codes, turns the code sizes into bit offsets
// and fills the block tables used by E5/E6.  Then the workers store their codes at those offsets: all writes are atomic
// ORs.  A code's global index t maps to (metablock, code) through code_base, the exclusive scan of br_mb_code_count.
BR_DEV u32 br_mb_code_count(const BrMbAux& a) { return a.num_types[0] * a.which + a.num_types[1] + a.num_types[2]; }
// code x of a metablock: literal codes (type * contexts + context), then command codes, then distance codes
BR_DEV u32 br_code_ref(BrMbMem* M, const BrMbAux& a, u32 x, u32** H, u8** dep, u16** bits) {
  const u32 nl = a.num_types[0] * a.which, ncm = a.num_types[1];
  if (x < nl) { *H = M->lit_H + x * 256; *dep = M->lit_depth + x * 256; *bits = M->lit_bits + x * 256; return 256; }
  if (x < nl + ncm) { x -= nl; *H = M->cmd_H + x * 704; *dep = M->cmd_depth + x * 704; *bits = M->cmd_bits + x * 704; return 704; }
  x -= nl + ncm;
  *H = M->dist_H + x * 64; *dep = M->dist_depth + x * 64; *bits = M->dist_bits + x * 64; return 64;
}
// Smoothing, Huffman construction and the counting store of code x; tree: BR_CODE_TREE_NODES of the worker's own.
BR_DEV void br_code_build(const BrMetaBlock& mb, const BrMbAux& a, u8* scratch, u32 x, BrHTree* tree) {
  BrMbMem* M = (BrMbMem*)scratch;
  u32* H; u8* dep; u16* bits;
  const u32 len = br_code_ref(M, a, x, &H, &dep, &bits);
  u8 good[704];
  br_optimize_counts_for_rle(len, H, good);
  br_build_tree(H, len, tree, dep, bits);
  BrBitW cw; cw.out = nullptr; cw.ix = 0; cw.per_thread = 1;
  br_store_tree(H, len, len, (BrTreeSc*)tree, dep, cw);   // (the big tree is done: its memory is the store's scratch)
  br_mb2_code_bits(scratch, mb)[x] = cw.ix;
}
// One warp: MapStaticContexts, the metablock header up to the codes, the code offsets and the block tables.
BR_DEV void br_mb_header(const BrStream& st, const BrMetaBlock& mb, BrMbAux& a, u8* scratch, u32* out) {
  BrMbMem* M = (BrMbMem*)scratch;
  const int lane = br_lane();
  const u32 nctx = a.which;
  const u32 nl = a.num_types[0] * nctx, nd = a.num_types[2], ntrees = br_mb_code_count(a);
  u32* code_bits = br_mb2_code_bits(scratch, mb);
  // metablock.c:677 MapStaticContexts
  if (nctx > 1)
    for (u32 x = (u32)lane; x < (a.num_types[0] << 6); x += BR_WARP) M->cmap[x] = (x >> 6) * nctx + br_static_ctx_map((int)nctx, x & 63);
  br_syncwarp();
  BrMbScratch* sc = &M->sc;
  const u32 cmap_size = nctx > 1 ? (a.num_types[0] << 6) : 0;
  BrBitW w; w.out = out; w.ix = 0; w.per_thread = 0;
  br_put_bits(w, 1, (u64)mb.is_last);
  if (mb.is_last) br_put_bits(w, 1, 0);
  br_store_mlen(mb.end - mb.start, w);
  if (!mb.is_last) br_put_bits(w, 1, 0);
  for (int cat = 0; cat < 3; ++cat) {
    const u32 hist_len = cat == 0 ? 256u : cat == 1 ? 704u : 64u;
    u32 nblk = br_mb2_nblk(cat, mb.nlit, mb.ncmd);
    BrSplit sp; sp.num_types = a.num_types[cat]; sp.num_blocks = a.num_blocks[cat];
    sp.types = br_mb2_types(scratch, a, cat, nblk); sp.lengths = br_mb2_lengths(scratch, a, cat, nblk);
    BrBlockEnc be;
    br_block_enc_init(be, hist_len, sp, &M->code[cat]);
    br_build_and_store_block_split_code(be, sc, w);
  }
  br_put_bits(w, 2, 0);
  br_put_bits(w, 4, 0);
  for (u32 i = 0; i < a.num_types[0]; ++i) br_put_bits(w, 2, 2);
  if (cmap_size == 0) br_store_trivial_context_map(nl, 6, sc, w);
  else br_encode_context_map(M->cmap, cmap_size, nl, sc, w);
  br_store_trivial_context_map(nd, 2, sc, w);
  // code sizes -> bit offsets: a warp-wide exclusive scan, 32 codes at a time
  u32 acc = w.ix;
  for (u32 t0 = 0; t0 < ntrees; t0 += BR_WARP) {
    const u32 t = t0 + (u32)lane;
    u32 total;
    const u32 ex = br_warp_excl_scan(t < ntrees ? code_bits[t] : 0u, &total);
    if (t < ntrees) code_bits[t] = acc + ex;
    acc += total;
  }
  if (lane == 0) code_bits[ntrees] = acc;
  w.ix = acc;
  // ---- block tables: start ordinal of every block and the block-switch bits that precede it
  for (int cat = 0; cat < 3; ++cat) {
    u32 nblk = br_mb2_nblk(cat, mb.nlit, mb.ncmd);
    const u8* types = br_mb2_types(scratch, a, cat, nblk);
    const u32* lengths = br_mb2_lengths(scratch, a, cat, nblk);
    BrBlockInfo* bi = br_mb2_blocks(scratch, a, cat);
    const BrBlockCode* code = &M->code[cat];
    const u32 nb = a.num_blocks[cat];
    if (lane == 0) { u32 acc = 0; for (u32 b = 0; b < nb; ++b) { bi[b].start = acc; acc += lengths[b]; } }
    for (u32 b = (u32)lane; b < nb; b += BR_WARP) {
      u32 type = types[b];
      u64 bits = 0; u32 n = 0;
      if (b > 0 && a.num_types[cat] > 1) {
        // brotli_bit_stream.c:58 NextBlockTypeCode: last = types[b-1], second last = types[b-2]
        // (the calculator starts at last = 1, second last = 0 and block 0 is fed first)
        u32 prev1 = types[b - 1], prev2 = b >= 2 ? types[b - 2] : 1u;
        u32 tc = (type == prev1 + 1) ? 1u : (type == prev2) ? 0u : type + 2u;
        u32 lc = br_block_len_code(lengths[b]);
        bits = code->type_bits[tc]; n = code->type_depths[tc];
        bits |= (u64)code->len_bits[lc] << n; n += code->len_depths[lc];
        bits |= (u64)(lengths[b] - br_block_len_offset(lc)) << n; n += br_block_len_nbits(lc);
      }
      bi[b].type = type; bi[b].sw_nbits = n; bi[b].sw_bits = bits; bi[b].pad = 0;
    }
  }
  br_syncwarp();
  if (lane == 0) { a.hdr_bits = w.ix; a.cmap_size = cmap_size; }
}
// Code x stored at the offset br_mb_header gave it.
BR_DEV void br_code_store(const BrMetaBlock& mb, const BrMbAux& a, u8* scratch, u32 x, BrHTree* tree, u32* out) {
  BrMbMem* M = (BrMbMem*)scratch;
  u32* H; u8* dep; u16* bits;
  const u32 len = br_code_ref(M, a, x, &H, &dep, &bits);
  BrBitW tw; tw.out = out; tw.ix = br_mb2_code_bits(scratch, mb)[x]; tw.per_thread = 1;
  br_store_tree(H, len, len, (BrTreeSc*)tree, dep, tw);
}

// ---- the same two steps by one warp, on a copy of the code in shared memory
// entropy_encode.c:68 BrotliCreateHuffmanTree with the sort spread over the lanes: every node's place is the number of
// nodes before it in the order of br_htree_less, a strict total order on (count, symbol), so this is the permutation the
// serial sort gives.  The merge and BrotliSetDepth run on lane 0.
BR_DEV u64 br_htree_key(const BrHTree& t) { return ((u64)t.count << 16) | (u32)(0xFFFF - t.right_or_value); }
BR_DEV void br_create_huffman_tree_warp(const u32* data, u32 length, int tree_limit, BrHTree* tree, u8* depth) {
  const int lane = br_lane();
  BrHTree* src = tree + 704;   // the unsorted nodes (n <= 704: tree[0, n) and src[0, n) are apart)
  for (u32 count_limit = 1;; count_limit *= 2) {
    u32 n = 0;
    for (u32 base = 0; base < length; base += BR_WARP) {   // nonzero symbols, from the last down
      const u32 k = base + (u32)lane, i = length - 1 - k;
      const u32 v = k < length ? data[i] : 0u;
      const u32 m = br_ballot(v != 0);
      if (v) {
        BrHTree t; t.count = v > count_limit ? v : count_limit; t.left = -1; t.right_or_value = (short)i;
        src[n + (u32)br_popc(m & br_lanemask_lt())] = t;
      }
      n += (u32)br_popc(m);
    }
    br_syncwarp();
    if (n == 1) { if (lane == 0) depth[src[0].right_or_value] = 1; br_syncwarp(); break; }
    for (u32 g0 = 0; g0 < n; g0 += 8 * BR_WARP) {
      u64 key[8]; u32 rk[8];
      for (int r = 0; r < 8; ++r) {
        const u32 ix = g0 + (u32)r * BR_WARP + (u32)lane;
        key[r] = ix < n ? br_htree_key(src[ix]) : ~0ull; rk[r] = 0;
      }
      for (u32 j = 0; j < n; ++j) {
        const u64 kj = br_htree_key(src[j]);
        for (int r = 0; r < 8; ++r) rk[r] += kj < key[r] ? 1u : 0u;
      }
      for (int r = 0; r < 8; ++r) {
        const u32 ix = g0 + (u32)r * BR_WARP + (u32)lane;
        if (ix < n) tree[rk[r]] = src[ix];
      }
    }
    br_syncwarp();
    int ok = 0;
    if (lane == 0) {
      BrHTree sentinel; sentinel.count = 0xFFFFFFFFu; sentinel.left = -1; sentinel.right_or_value = -1;
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
      ok = br_set_depth((int)(2 * n - 1), tree, depth, tree_limit);
    }
    ok = br_shfl(ok, 0);
    br_syncwarp();
    if (ok) break;
  }
}
// br_code_build by one warp.  S->depth and S->bits start zeroed.
BR_DEV void br_code_build_warp(const BrMetaBlock& mb, const BrMbAux& a, u8* scratch, u32 x, BrCodeSmem* S) {
  BrMbMem* M = (BrMbMem*)scratch;
  const int lane = br_lane();
  u32* H; u8* dep; u16* bits;
  const u32 len = br_code_ref(M, a, x, &H, &dep, &bits);
  for (u32 i = (u32)lane; i < len; i += BR_WARP) { S->H[i] = H[i]; S->depth[i] = 0; S->bits[i] = 0; }
  br_syncwarp();
  if (lane == 0) br_optimize_counts_for_rle(len, S->H, S->good);
  br_syncwarp();
  u32 count = 0;   // br_build_tree: a code of one symbol (or none) keeps depth 0
  for (u32 base = 0; base < len && count <= 1; base += BR_WARP) count += (u32)br_popc(br_ballot(base + (u32)lane < len && S->H[base + lane]));
  if (count > 1) {
    br_create_huffman_tree_warp(S->H, len, 15, S->tree, S->depth);
    if (lane == 0) br_depths_to_symbols(S->depth, len, S->bits);
    br_syncwarp();
  }
  if (lane == 0) {
    BrBitW cw; cw.out = nullptr; cw.ix = 0; cw.per_thread = 1;
    br_store_tree(S->H, len, len, (BrTreeSc*)S->tree, S->depth, cw);
    br_mb2_code_bits(scratch, mb)[x] = cw.ix;
  }
  for (u32 i = (u32)lane; i < len; i += BR_WARP) { H[i] = S->H[i]; dep[i] = S->depth[i]; bits[i] = S->bits[i]; }
  br_syncwarp();
}
// br_code_store by one warp (lane 0 writes, from the shared copy)
BR_DEV void br_code_store_warp(const BrMetaBlock& mb, const BrMbAux& a, u8* scratch, u32 x, BrCodeSmem* S, u32* out) {
  BrMbMem* M = (BrMbMem*)scratch;
  const int lane = br_lane();
  u32* H; u8* dep; u16* bits;
  const u32 len = br_code_ref(M, a, x, &H, &dep, &bits);
  for (u32 i = (u32)lane; i < len; i += BR_WARP) { S->H[i] = H[i]; S->depth[i] = dep[i]; }
  br_syncwarp();
  if (lane == 0) {
    BrBitW tw; tw.out = out; tw.ix = br_mb2_code_bits(scratch, mb)[x]; tw.per_thread = 1;
    br_store_tree(S->H, len, len, (BrTreeSc*)S->tree, S->depth, tw);
  }
  br_syncwarp();
}
#if !BR_GPU
// E4 of one metablock, for the CPU simulation (tests/sim), which runs the entropy stage metablock by metablock: every
// code built, the header, every code stored, by the warp workers' functions.  The job-wide phase order of the device
// gives the same bytes: each phase of a metablock reads and writes only that metablock's scratch and bit buffer.
BR_DEV void br_prep_codes(const BrStream& st, const BrMetaBlock& mb, BrMbAux& a, u8* scratch, u32* out) {
  BrCodeSmem S;
  for (u32 x = 0; x < br_mb_code_count(a); ++x) br_code_build_warp(mb, a, scratch, x, &S);
  br_mb_header(st, mb, a, scratch, out);
  for (u32 x = 0; x < br_mb_code_count(a); ++x) br_code_store_warp(mb, a, scratch, x, &S, out);
}
#endif

// ---------------------------------------------------------------------------------- E5 / E6
BR_DEV u32 br_block_of(const BrBlockInfo* bi, u32 nb, u32 o) {
  u32 lo = 0, hi = nb;
  while (hi - lo > 1) { u32 mid = (lo + hi) >> 1; if (bi[mid].start <= o) lo = mid; else hi = mid; }
  return lo;
}
// code word of literal `o` (global ordinal): returns its length; *sw / *swn: block switch before it
BR_DEV u32 br_lit_code(const BrStream& st, const BrEnt& e, u32 o, u32* code, u64* sw, u32* swn, u32* mb_out) {
  const u32 cmd = e.lit_cmd[o], m = e.cmd_mb[cmd];
  *mb_out = m; *swn = 0; *sw = 0; *code = 0;
  if (!st.mbs[m].compress) return 0;
  const BrMbAux& a = e.aux[m];
  u8* scratch = e.scratch + e.scratch_off[m];
  if (st.P.mb_kind) {   // qualities 2, 3: one literal code
    const BrMbFlat* F = (const BrMbFlat*)scratch;
    const u32 lit = st.data[e.lit_pos[o]];
    *code = F->lit_bits[lit];
    return F->lit_depth[lit];
  }
  const BrMbMem* M = (const BrMbMem*)scratch;
  const BrBlockInfo* bi = br_mb2_blocks(scratch, a, 0);
  const u32 orel = o - a.lit_base;
  const u32 b = br_block_of(bi, a.num_blocks[0], orel);
  const u32 p = e.lit_pos[o], lit = st.data[p], type = bi[b].type;
  u32 hix;
  const u32 base = st.mbs[m].base;
  if (a.cmap_size) hix = M->cmap[(type << 6) + BR_CTX_UTF8(st, br_data_or_zero(st, p, 1, base), br_data_or_zero(st, p, 2, base))] * 256 + lit;
  else hix = type * 256 + lit;
  if (bi[b].start == orel) { *swn = bi[b].sw_nbits; *sw = bi[b].sw_bits; }
  *code = M->lit_bits[hix];
  return M->lit_depth[hix];
}
BR_DEV void br_lit_bits(const BrStream& st, const BrEnt& e, u32 o) {
  u32 code, swn, m; u64 sw;
  u32 n = br_lit_code(st, e, o, &code, &sw, &swn, &m);
  e.lit_len[o] = n + swn;
}
// The seven pieces a command contributes, in stream order (brotli_bit_stream.c:1062-1106):
// [cmd block switch] cmd symbol, insert/copy extra bits, <literals>, [dist block switch] dist symbol, dist extra
struct BrCmdCode { u64 csw, extra, dsw; u32 cswn, csym, cn, en, dswn, dsym, dn, xbits, xn; };
BR_DEV void br_cmd_code(const BrStream& st, const BrEnt& e, u32 i, BrCmdCode* k) {
  const u32 m = e.cmd_mb[i];
  const BrMetaBlock& mb = st.mbs[m];
  k->csw = k->extra = k->dsw = 0;
  k->cswn = k->csym = k->cn = k->en = k->dswn = k->dsym = k->dn = k->xbits = k->xn = 0;
  if (!mb.compress) return;
  const BrMbAux& a = e.aux[m];
  u8* scratch = e.scratch + e.scratch_off[m];
  const BrMbMem* M = (const BrMbMem*)scratch;
  const BrCmd c = e.cmds[i];
  if (st.P.mb_kind) {   // qualities 2, 3: one command code, one distance code (brotli_bit_stream.c:1159 StoreDataWithHuffmanCodes)
    const BrMbFlat* F = (const BrMbFlat*)scratch;
    k->cn = F->cmd_depth[c.cmd_prefix]; k->csym = F->cmd_bits[c.cmd_prefix];
    const u32 clc = br_cmd_copy_len_code(c);
    const u32 ic = br_ins_code(c.insert_len), cc = br_copy_code(clc);
    const u32 insn = br_ins_extra(ic);
    const u64 insv = c.insert_len - br_ins_base(ic), copyv = clc - br_copy_base(cc);
    k->extra = (copyv << insn) | insv; k->en = insn + br_copy_extra(cc);
    if (br_cmd_copy_len(c) && c.cmd_prefix >= 128) {
      const u32 ds = c.dist_prefix & 0x3FF;
      k->dn = F->dist_depth[ds]; k->dsym = F->dist_bits[ds];
      k->xn = c.dist_prefix >> 10; k->xbits = c.dist_extra;
    }
    return;
  }
  {
    const BrBlockInfo* bi = br_mb2_blocks(scratch, a, 1);
    const u32 orel = i - mb.cmd_off, b = br_block_of(bi, a.num_blocks[1], orel);
    if (bi[b].start == orel) { k->cswn = bi[b].sw_nbits; k->csw = bi[b].sw_bits; }
    const u32 ix = bi[b].type * 704 + c.cmd_prefix;
    k->cn = M->cmd_depth[ix]; k->csym = M->cmd_bits[ix];
    // brotli_bit_stream.c:82 StoreCommandExtra
    u32 clc = br_cmd_copy_len_code(c);
    u32 ic = br_ins_code(c.insert_len), cc = br_copy_code(clc);
    u32 insn = br_ins_extra(ic);
    u64 insv = c.insert_len - br_ins_base(ic), copyv = clc - br_copy_base(cc);
    k->extra = (copyv << insn) | insv; k->en = insn + br_copy_extra(cc);
  }
  if (br_cmd_copy_len(c) && c.cmd_prefix >= 128) {
    const BrBlockInfo* bi = br_mb2_blocks(scratch, a, 2);
    const u32 orel = e.dist_ord[i] - a.dist_base, b = br_block_of(bi, a.num_blocks[2], orel);
    if (bi[b].start == orel) { k->dswn = bi[b].sw_nbits; k->dsw = bi[b].sw_bits; }
    const u32 ix = bi[b].type * 64 + (c.dist_prefix & 0x3FF);
    k->dn = M->dist_depth[ix]; k->dsym = M->dist_bits[ix];
    k->xn = c.dist_prefix >> 10; k->xbits = c.dist_extra;
  }
}
BR_DEV void br_cmd_bits(const BrStream& st, const BrEnt& e, u32 i) {
  BrCmdCode k;
  br_cmd_code(st, e, i, &k);
  e.cmd_len[i] = k.cswn + k.cn + k.en + k.dswn + k.dn + k.xn;
}
// after the exclusive scans of lit_len / cmd_len: place the command's own pieces
BR_DEV void br_emit_cmd(const BrStream& st, const BrEnt& e, u32 i) {
  const u32 m = e.cmd_mb[i];
  const BrMetaBlock& mb = st.mbs[m];
  if (!mb.compress) return;
  const BrMbAux& a = e.aux[m];
  BrCmdCode k;
  br_cmd_code(st, e, i, &k);
  u32* out = e.outbits + e.out_off[m];
  const u32 lo = e.lit_ord[i], ins = e.cmds[i].insert_len;
  u32 off = a.hdr_bits + (e.cmd_len[i] - e.cmd_len[mb.cmd_off]) + (e.lit_len[lo] - e.lit_len[a.lit_base]);
  br_put_bits_at(out, off, k.cswn, k.csw); off += k.cswn;
  br_put_bits_at(out, off, k.cn, k.csym); off += k.cn;
  br_put_bits_at(out, off, k.en, k.extra); off += k.en;
  e.lit_bit_base[i] = off - e.lit_len[lo];
  off += e.lit_len[lo + ins] - e.lit_len[lo];
  br_put_bits_at(out, off, k.dswn, k.dsw); off += k.dswn;
  br_put_bits_at(out, off, k.dn, k.dsym); off += k.dn;
  br_put_bits_at(out, off, k.xn, k.xbits); off += k.xn;
  if (i + 1 == mb.cmd_off + mb.ncmd) st.mbs[m].out_bits = off;
}
BR_DEV void br_emit_lit(const BrStream& st, const BrEnt& e, u32 o) {
  u32 code, swn, m; u64 sw;
  u32 n = br_lit_code(st, e, o, &code, &sw, &swn, &m);
  if (!st.mbs[m].compress) return;
  u32* out = e.outbits + e.out_off[m];
  u32 off = e.lit_bit_base[e.lit_cmd[o]] + e.lit_len[o];
  br_put_bits_at(out, off, swn, sw);
  br_put_bits_at(out, off + swn, n, code);
}

#include <vector>
// Host: where every metablock's scratch (bytes) and bit buffer (words) start -- only compressed metablocks take room --
// and how many bytes the assembled stream may take.
struct BrMbLayout {
  std::vector<u64> scratch_off, out_off;
  size_t scratch_bytes, out_words, out_cap;
  u32 code_warps;     // warp workers for the prefix codes of the job (E4): one per code, when there are few enough
  u32 code_workers;   // thread workers for the prefix codes of the job (E4), each with BR_CODE_TREE_NODES of tree area
};
static inline void br_mb_layout(const BrParams& P, const BrMetaBlock* mbs, u32 n_mbs, BrMbLayout& L) {
  L.scratch_off.assign(n_mbs, 0); L.out_off.assign(n_mbs, 0);
  L.scratch_bytes = L.out_words = 0;
  u64 codes = 0;
  for (u32 i = 0; i < n_mbs; ++i) {
    L.scratch_off[i] = L.scratch_bytes; L.out_off[i] = L.out_words;
    if (mbs[i].compress) {
      L.scratch_bytes += ((size_t)br_mb_scratch_bytes(P, mbs[i].nlit, mbs[i].ncmd) + 255) & ~(size_t)255;
      L.out_words += (2 * (size_t)(mbs[i].end - mbs[i].start) + 503) / 4 + 16;
      codes += br_mb2_code_bound(mbs[i].nlit, mbs[i].ncmd);
    }
  }
  // (a job that may have no more codes than the warps take never needs the thread workers)
  L.code_warps = P.mb_kind ? 0u : (u32)(codes < BR_CODE_WARP_MAX ? codes : BR_CODE_WARP_MAX);
  L.code_workers = P.mb_kind || codes <= BR_CODE_WARP_MAX ? 0u : (u32)(codes < BR_CODE_THREADS_MAX ? codes : BR_CODE_THREADS_MAX);
  L.out_cap = (size_t)P.n + ((size_t)P.n >> 3) + 4096 + 8ull * n_mbs;
}

// Host: n synthetic metablocks for E4 alone (the test hooks br_debug_codes and tests/sim sim_debug_codes).  counts[3 i ..
// 3 i + 2]: the literal, command and distance codes of metablock i, 1 to 256 each, with one literal context; all three 0:
// the metablock is stored raw.  histos: the counts of every code in code order (256, 704 or 64 words each).  Every split
// has one block per type, so the header is valid, and every metablock is sized for 256 blocks of each category.  Fills
// mbs, aux (as k_mb_setup and k_split leave them), the layout, and the image of the whole scratch: the histograms and the
// splits in place and every other byte `fill`, as a reused arena leaves it.  Returns false on a count out of range.
#define BR_SYNTH_MB_BYTES (1u << 20)
static inline bool br_codes_synth(const u32* counts, u32 n, const u32* histos, u8 fill, std::vector<BrMetaBlock>& mbs,
                                  std::vector<BrMbAux>& aux, BrMbLayout& L, std::vector<u8>& scratch) {
  BrParams P; memset(&P, 0, sizeof(P));
  P.n = n * BR_SYNTH_MB_BYTES;
  mbs.assign(n, BrMetaBlock()); aux.assign(n, BrMbAux());
  for (u32 i = 0; i < n; ++i) {
    const u32* c = counts + 3 * i;
    const bool raw = c[0] == 0 && c[1] == 0 && c[2] == 0;
    for (int cat = 0; cat < 3; ++cat) if (!raw && (c[cat] < 1 || c[cat] > 256)) return false;
    BrMetaBlock& mb = mbs[i]; memset(&mb, 0, sizeof(mb));
    mb.start = i * BR_SYNTH_MB_BYTES; mb.end = mb.start + BR_SYNTH_MB_BYTES;
    mb.nlit = 254 * 512; mb.ncmd = 254 * 1024;   // br_mb2_nblk: 256, 256 and 510 blocks
    mb.is_last = i + 1 == n; mb.compress = raw ? 0u : 1u;
    BrMbAux& a = aux[i]; memset(&a, 0, sizeof(a));
    if (raw) continue;
    a.which = 1;
    u32 off = br_align8((u32)sizeof(BrMbMem));
    for (int cat = 0; cat < 3; ++cat) {
      a.num_types[cat] = a.num_blocks[cat] = c[cat];
      a.var_off[cat] = off; off += br_mb2_var_bytes(br_mb2_nblk(cat, mb.nlit, mb.ncmd));
    }
  }
  br_mb_layout(P, mbs.data(), n, L);
  scratch.assign(L.scratch_bytes + 256, fill);
  const u32* h = histos;
  for (u32 i = 0; i < n; ++i) {
    if (!mbs[i].compress) continue;
    const BrMetaBlock& mb = mbs[i]; const BrMbAux& a = aux[i];
    u8* sc = scratch.data() + L.scratch_off[i];
    BrMbMem* M = (BrMbMem*)sc;
    const u32 A[3] = {256, 704, 64};
    u32* H[3] = {M->lit_H, M->cmd_H, M->dist_H};
    for (int cat = 0; cat < 3; ++cat) {
      memcpy(H[cat], h, (size_t)a.num_types[cat] * A[cat] * 4); h += (size_t)a.num_types[cat] * A[cat];
      const u32 nblk = br_mb2_nblk(cat, mb.nlit, mb.ncmd);
      u8* types = sc + a.var_off[cat] + nblk * ((u32)sizeof(BrBlockInfo) + 4);
      u32* lengths = (u32*)(sc + a.var_off[cat] + nblk * (u32)sizeof(BrBlockInfo));
      for (u32 b = 0; b < a.num_blocks[cat]; ++b) { types[b] = (u8)b; lengths[b] = 1 + 37 * b; }
    }
  }
  return true;
}
// Host: what E4 left in the scratch image of br_codes_synth's metablocks.  Per code, in code order: H, depth and bits (256,
// 704 or 64 entries each).  offsets: per compressed metablock the bit offset of each of its codes (br_mb2_code_bits), then
// the end of its last code; per raw metablock one 0.
static inline void br_codes_collect(const std::vector<BrMetaBlock>& mbs, const std::vector<BrMbAux>& aux, const BrMbLayout& L,
                                    const u8* scratch, u32* H, u8* depth, u16* bits, u32* offsets) {
  for (size_t i = 0; i < mbs.size(); ++i) {
    if (!mbs[i].compress) { *offsets++ = 0; continue; }
    const u8* sc = scratch + L.scratch_off[i];
    const BrMbMem* M = (const BrMbMem*)sc;
    const u32 A[3] = {256, 704, 64};
    const u32* Hs[3] = {M->lit_H, M->cmd_H, M->dist_H};
    const u8* Ds[3] = {M->lit_depth, M->cmd_depth, M->dist_depth};
    const u16* Bs[3] = {M->lit_bits, M->cmd_bits, M->dist_bits};
    u32 ntrees = 0;
    for (int cat = 0; cat < 3; ++cat) {
      const size_t k = (size_t)aux[i].num_types[cat] * A[cat];
      memcpy(H, Hs[cat], k * 4); memcpy(depth, Ds[cat], k); memcpy(bits, Bs[cat], k * 2);
      H += k; depth += k; bits += k; ntrees += aux[i].num_types[cat];
    }
    const u32* code_bits = (const u32*)(sc + br_mb2_scratch_bytes(mbs[i].nlit, mbs[i].ncmd) - BR_CODE_BITS_WORDS * 4);
    memcpy(offsets, code_bits, (ntrees + 1) * 4ull); offsets += ntrees + 1;
  }
}

// Host: metablocks for E2..E4 described by the caller (the test hooks br_debug_split and tests/sim sim_debug_split).
// mbw: BR_SPLIT_MB_WORDS words per metablock: start, end, first command, command count, is_last, compress (0: stored
// raw) and base, the first byte of its stream (literal contexts see zeros in front of it).  The metablocks and their
// commands must cover the n input bytes in order, as the compacted commands of a job do.  Fills mbs (nlit from the
// commands) and the layout; returns false on a description that does not hold together.
#define BR_SPLIT_MB_WORDS 7
static inline bool br_split_synth(const BrParams& P, const u32* mbw, u32 n_mbs, const BrCmd* cmds, u32 ncmd,
                                  std::vector<BrMetaBlock>& mbs, BrMbLayout& L) {
  mbs.assign(n_mbs, BrMetaBlock());
  u32 pos = 0, c = 0;
  for (u32 i = 0; i < n_mbs; ++i) {
    const u32* w = mbw + (size_t)i * BR_SPLIT_MB_WORDS;
    BrMetaBlock& mb = mbs[i]; memset(&mb, 0, sizeof(mb));
    mb.start = w[0]; mb.end = w[1]; mb.cmd_off = w[2]; mb.ncmd = w[3]; mb.is_last = w[4]; mb.compress = w[5]; mb.base = w[6];
    if (mb.start != pos || mb.end <= mb.start || mb.cmd_off != c || mb.ncmd == 0 || (u64)c + mb.ncmd > ncmd || mb.base > mb.start)
      return false;
    u64 span = 0;
    for (u32 k = c; k < c + mb.ncmd; ++k) { mb.nlit += cmds[k].insert_len; span += (u64)cmds[k].insert_len + (cmds[k].copy_len & 0x1FFFFFF); }
    if (span != mb.end - mb.start) return false;
    pos = mb.end; c += mb.ncmd;
  }
  if (pos != P.n || c != ncmd) return false;
  br_mb_layout(P, mbs.data(), n_mbs, L);
  return true;
}
// Host: the record of a compressed metablock that the split hooks return, from the image of its scratch after E3 (before
// E4 smooths the histograms in place): which, num_types[3], num_blocks[3], a word for the bit count (br_split_record_bits),
// then per category types[num_blocks] and lengths[num_blocks] (a word each), then the histograms: literal (num_types *
// which rows of 256), command (rows of 704) and distance (rows of 64).
#define BR_SPLIT_REC_HEAD 8
static inline void br_split_record(const BrMetaBlock& mb, const BrMbAux& a, const u8* sc, std::vector<u32>& rec) {
  rec.assign({a.which, a.num_types[0], a.num_types[1], a.num_types[2], a.num_blocks[0], a.num_blocks[1], a.num_blocks[2], 0u});
  for (int cat = 0; cat < 3; ++cat) {
    const u32 nblk = br_mb2_nblk(cat, mb.nlit, mb.ncmd);
    const u8* types = sc + a.var_off[cat] + nblk * ((u32)sizeof(BrBlockInfo) + 4);
    const u32* lengths = (const u32*)(sc + a.var_off[cat] + nblk * (u32)sizeof(BrBlockInfo));
    for (u32 b = 0; b < a.num_blocks[cat]; ++b) rec.push_back(types[b]);
    rec.insert(rec.end(), lengths, lengths + a.num_blocks[cat]);
  }
  const BrMbMem* M = (const BrMbMem*)sc;
  rec.insert(rec.end(), M->lit_H, M->lit_H + (size_t)a.num_types[0] * a.which * 256);
  rec.insert(rec.end(), M->cmd_H, M->cmd_H + (size_t)a.num_types[1] * 704);
  rec.insert(rec.end(), M->dist_H, M->dist_H + (size_t)a.num_types[2] * 64);
}
// ... then, after E4, the metablock's bit buffer from bit 0 to the end of its last prefix code: the header, the block-split
// codes, the context maps and every code (nbits bits, (nbits + 31) / 32 words).
static inline void br_split_record_bits(std::vector<u32>& rec, const u32* bits, u32 nbits) {
  rec[7] = nbits;
  rec.insert(rec.end(), bits, bits + (nbits + 31) / 32);
}
// The offset in the scratch of a metablock's code bit offsets (br_mb2_code_bits); entry br_mb_code_count(a) is the end of
// its last code.
static inline size_t br_split_code_end_off(const BrMetaBlock& mb, const BrMbAux& a) {
  return br_mb2_scratch_bytes(mb.nlit, mb.ncmd) - BR_CODE_BITS_WORDS * 4 + 4ull * (a.num_types[0] * a.which + a.num_types[1] + a.num_types[2]);
}
// The records of every compressed metablock, one after another, into out (cap words).  Returns the words they take.
static inline size_t br_split_put(const std::vector<std::vector<u32>>& recs, u32* out, size_t cap) {
  size_t k = 0;
  for (const auto& r : recs) {
    for (size_t j = 0; j < r.size(); ++j, ++k) if (k < cap) out[k] = r[j];
  }
  return k;
}
