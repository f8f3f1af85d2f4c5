// br_entropy_flat.h -- qualities 2 and 3: metablocks without block splits and contexts.
//
// What it replaces: BrotliStoreMetaBlockTrivial (c/enc/brotli_bit_stream.c:1196, quality 3) and BrotliStoreMetaBlockFast
// (:1243, quality 2), chosen in WriteMetaBlockInternal (c/enc/encode.c:543-556).  One prefix code per category:
//   quality 3  BuildAndStoreHuffmanTree (:349) over the three histograms -- the same builder / serialiser pair the block
//              codes of quality 4..9 use (br_entropy.h br_build_tree / br_store_tree), without OptimizeHistograms;
//   quality 2  BrotliBuildAndStoreHuffmanTreeFast (:404; br_q1.h br_q1_fast_tree, shared with quality 1), or -- for at
//              most 128 commands -- the static command / distance codes of entropy_encode_static.h with their
//              pre-serialised forms (:524 StoreStaticCommandHuffmanTree, :538 StoreStaticDistanceHuffmanTree).
// The GPU shape: one CTA per metablock (k_prep_flat) builds the three histograms with atomics, one thread builds and
// stores the codes behind the header; the symbols themselves go through the shared, fully data-parallel
// stages E5 / E6 (br_entropy2.h: per-symbol bit counts -> prefix sums -> atomic-OR scatter), which read this
// metablock's codes from BrMbFlat.
#pragma once
#include "br_q1.h"

BR_DEV void br_prep_flat(const BrStream& st, const BrEnt& e, const BrMetaBlock& mb, BrMbAux& a, u8* scratch, u32* out) {
  const u32 tid = BR_CTA_TID, nt = BR_CTA_N;
  BrMbFlat* F = (BrMbFlat*)scratch;
  for (u32 i = tid; i < 256; i += nt) { F->lit_H[i] = 0; F->lit_depth[i] = 0; F->lit_bits[i] = 0; }
  for (u32 i = tid; i < 704; i += nt) { F->cmd_H[i] = 0; F->cmd_depth[i] = 0; F->cmd_bits[i] = 0; }
  for (u32 i = tid; i < 64; i += nt) { F->dist_H[i] = 0; F->dist_depth[i] = 0; F->dist_bits[i] = 0; }
#if BR_GPU
  __threadfence_block();
#endif
  br_cta_sync();
  // brotli_bit_stream.c:1133 BuildHistograms
  for (u32 i = tid; i < mb.ncmd; i += nt) {
    const BrCmd c = e.cmds[mb.cmd_off + i];
    br_smem_add(F->cmd_H + c.cmd_prefix, 1);
    if (br_cmd_copy_len(c) && c.cmd_prefix >= 128) br_smem_add(F->dist_H + (c.dist_prefix & 0x3FF), 1);
  }
  for (u32 o = tid; o < mb.nlit; o += nt) br_smem_add(F->lit_H + st.data[e.lit_pos[a.lit_base + o]], 1);
#if BR_GPU
  __threadfence_block();
#endif
  br_cta_sync();
  if (tid != 0) return;
  // ---- one thread: header and the three codes (a writer of its own: every write is an atomic OR into the zeroed buffer)
  BrBitW w; w.out = out; w.ix = 0; w.per_thread = 1;
  br_put_bits(w, 1, (u64)mb.is_last);          // :120 StoreCompressedMetaBlockHeader
  if (mb.is_last) br_put_bits(w, 1, 0);
  br_store_mlen(mb.end - mb.start, w);
  if (!mb.is_last) br_put_bits(w, 1, 0);
  br_put_bits(w, 13, 0);                        // one block type per category, NPOSTFIX / NDIRECT 0, context mode, trivial maps
  const u32 ndist = a.nsym[2];
  if (st.P.mb_kind == 1) {
    br_build_tree(F->lit_H, 256, F->tree, F->lit_depth, F->lit_bits);
    br_store_tree(F->lit_H, 256, 256, &F->tsc, F->lit_depth, w);
    br_build_tree(F->cmd_H, 704, F->tree, F->cmd_depth, F->cmd_bits);
    br_store_tree(F->cmd_H, 704, 704, &F->tsc, F->cmd_depth, w);
    br_build_tree(F->dist_H, 64, F->tree, F->dist_depth, F->dist_bits);
    br_store_tree(F->dist_H, 64, 64, &F->tsc, F->dist_depth, w);
  } else if (mb.ncmd <= 128) {
    br_q1_fast_tree(F->lit_H, mb.nlit, 8, F->tree, F->lit_depth, F->lit_bits, w);
    // entropy_encode_static.h: kStaticCommandCodeDepth = 9 for symbols < 448, 11 behind; kStaticDistanceCodeDepth = 6;
    // the code words are the canonical ones of those depths
    for (u32 i = 0; i < 704; ++i) F->cmd_depth[i] = i < 448 ? 9 : 11;
    for (u32 i = 0; i < 64; ++i) F->dist_depth[i] = 6;
    br_depths_to_symbols(F->cmd_depth, 704, F->cmd_bits);
    br_depths_to_symbols(F->dist_depth, 64, F->dist_bits);
    br_put_bits(w, 56, 0x0092624416307003ull); br_put_bits(w, 3, 0);
    br_put_bits(w, 28, 0x0369DC03u);
  } else {
    br_q1_fast_tree(F->lit_H, mb.nlit, 8, F->tree, F->lit_depth, F->lit_bits, w);
    br_q1_fast_tree(F->cmd_H, mb.ncmd, 10, F->tree, F->cmd_depth, F->cmd_bits, w);
    br_q1_fast_tree(F->dist_H, ndist, 6, F->tree, F->dist_depth, F->dist_bits, w);
  }
  a.hdr_bits = w.ix; a.cmap_size = 0;
  a.num_types[0] = a.num_types[1] = a.num_types[2] = 1; a.num_blocks[0] = a.num_blocks[1] = a.num_blocks[2] = 1;
}
