// br_params.h -- host-side parameter derivation: what SanitizeParams / ComputeLgBlock /
// ChooseHasher / ComputeRbBits / MaxMetablockSize (c/enc/quality.h:59-225) decide for a
// given (quality, lgwin, size_hint).  Host only.
#pragma once
#include <vector>
#include "br_types.h"

// Returns 0 if the combination is outside what this library implements (the BrotliEncoder*
// entry points then fail instead of silently doing something else).
// lgblock_user: BROTLI_PARAM_LGBLOCK (0 = let the encoder choose, quality.h:76 ComputeLgBlock).
static inline int br_derive_params(int quality, int lgwin, u32 size_hint, u32 n, BrParams* P, int lgblock_user = 0) {
  memset(P, 0, sizeof(*P));
  if (quality >= 2 && quality <= 4) {
    // Qualities 2..4: the one-position-per-slot hashers (quality.h:172 ChooseHasher, hash.h:251-338), window 10..24 bits.
    if (lgwin < 10 || lgwin > 24) return 0;
    P->quality = quality; P->lgwin = lgwin;
    P->lgblock = quality < 4 ? 14 : 16;          // quality.h:81 (below MIN_QUALITY_FOR_BLOCK_SPLIT the parameter is ignored)
    if (quality == 4 && lgblock_user != 0) P->lgblock = lgblock_user > 24 ? 24 : lgblock_user < 16 ? 16 : lgblock_user;
    P->quick = 1; P->qk_hash_len = 5;
    if (quality == 2) { P->qk_bits = 16; P->qk_sweep_bits = 0; P->qk_dict = 1; }            // H2
    else if (quality == 3) { P->qk_bits = 16; P->qk_sweep_bits = 1; P->qk_dict = 0; }       // H3
    else if (size_hint >= (1u << 20)) { P->qk_bits = 20; P->qk_sweep_bits = 2; P->qk_dict = 0; P->qk_hash_len = 7; }   // H54
    else { P->qk_bits = 17; P->qk_sweep_bits = 2; P->qk_dict = 1; }                         // H4
    P->mb_kind = quality == 2 ? 2u : quality == 3 ? 1u : 0u;
    P->htl = 8;                                   // HashTypeLength == StoreLookahead == 8
    const int rbq = 1 + (lgwin > P->lgblock ? lgwin : P->lgblock);
    P->rmask = (1u << rbq) - 1;
    P->max_backward = (1u << lgwin) - 16;
    P->spree = 64;
    P->max_mb = 1u << (rbq < 24 ? rbq : 24);
    P->size_hint = size_hint; P->n = n;
    P->nbuckets = 1u << P->qk_bits;
    P->chunk_bits = n < BR_SMALL_STREAM ? BR_CHUNK_BITS_SMALL : BR_CHUNK_BITS;
    P->heavy_min = 0xffffffffu; P->step_cap = 4096;
    P->sweep_epoch = 3; P->force_epoch = 64; P->pilot = 0;
    P->sweep_blocks = P->lgblock >= 21 ? 1u : (1u << (21 - P->lgblock));
    return 1;
  }
  if (quality < 5 || quality > 9) return 0;   // q0: one-pass fragment coder; q10-11: Zopfli path
  if (lgwin < 17 || lgwin > 24) return 0;      // <=16: forgetful-chain hashers; >24: large window
  P->quality = quality; P->lgwin = lgwin;
  P->lgblock = 16;                              // quality.h:86
  if (quality >= 9 && lgwin > 16) P->lgblock = lgwin < 18 ? lgwin : 18;
  if (lgblock_user != 0) P->lgblock = lgblock_user > 24 ? 24 : lgblock_user < 16 ? 16 : lgblock_user;   // quality.h:88
  P->hash64 = (size_hint >= (1u << 20) && lgwin >= 19) ? 1 : 0;   // quality.h:182
  P->block_bits = quality - 1;
  P->bucket_bits = P->hash64 ? 15 : (quality < 7 ? 14 : 15);
  P->ndist = quality < 7 ? 4 : quality < 9 ? 10 : 16;
  P->htl = P->hash64 ? 8 : 4;
  int rb = 1 + (lgwin > P->lgblock ? lgwin : P->lgblock);        // quality.h:99
  P->rmask = (1u << rb) - 1;
  P->max_backward = (1u << lgwin) - 16;
  P->spree = quality < 9 ? 64 : 512;                              // quality.h:116
  P->max_mb = 1u << (rb < 24 ? rb : 24);                          // quality.h:103
  P->size_hint = size_hint;
  P->n = n;
  P->nbuckets = 1u << P->bucket_bits;
  P->chunk_bits = n < BR_SMALL_STREAM ? BR_CHUNK_BITS_SMALL : BR_CHUNK_BITS;
  P->heavy_min = 65536;
  P->step_cap = 4096;
  P->sweep_epoch = 3;    // text / web input settles in 3 launches; what is still dirty then is swept run by run
  P->force_epoch = 64;
  // pilot launch (BrParams::pilot): pays where a chunk walk is expensive (the deep rings of quality 7-9: a quarter fewer
  // chunk walks on config C4); at quality 5-6 the extra launch costs more than the saved walks
  P->pilot = (n >= BR_SMALL_STREAM && P->block_bits >= 6) ? 1u : 0u;
  P->sweep_blocks = P->lgblock >= 21 ? 1u : (1u << (21 - P->lgblock));   // sweeps are at most 2 MiB of input long
  return 1;
}

// Chunk size of a BATCH of streams (BrParams::multi): the fine chunks of a small stream buy latency with extra warm-up
// work (256 bytes re-parsed in front of every chunk); a batch that fills the GPU anyway takes the 2 KiB chunks.
static inline u32 br_batch_chunk_bits(u32 n_total) { return n_total < (8u << 20) ? BR_CHUNK_BITS_SMALL : BR_CHUNK_BITS; }

// The reference's input blocks (one EncodeData call each, c/enc/encode.c:1665-1719) and their 2 KiB chunks for a stream
// of n bytes.  `cuts` (sorted, each in (0, n]) are the positions where a FLUSH / EMIT_METADATA operation ended the input
// of a CompressStream call: the running block ends there with force_flush set (encode.c:1700) and the next one starts
// with a full 1 << lgblock budget again (encode.c:1016 UpdateLastProcessedPos).  is_final: FINISH has been seen (the
// last block carries is_last); otherwise the stream simply stops behind its last block.
// kinds (nullable) = what each cut is: 1 FLUSH, 2 EMIT_METADATA, 3 = END OF A STREAM (a batch of independent streams laid
// end to end, BrParams::multi): the block in front of the cut carries is_last, the blocks behind it belong to a new stream.
// chunks == nullptr: only the block table (the CUDA pipeline fills the chunk table on the device, k_build_chunks).
static inline void br_build_blocks(const BrParams& P, u32 n, const u32* cuts, u32 ncuts, bool is_final,
                                   std::vector<BrBlockIn>* chunks, std::vector<BrBlk>& blks, u32* nchunks_total = nullptr,
                                   const u32* kinds = nullptr) {
  const u32 bs = 1u << P.lgblock, ch = 1u << P.chunk_bits;
  u32 ci = 0, total = 0;
  u64 bstart = 0, base = 0;
  u32 stream = 0;
  while (bstart < n) {
    while (ci < ncuts && cuts[ci] <= bstart) ++ci;
    u64 bend = bstart + bs < n ? bstart + bs : n;
    bool forced = false, stream_end = false;
    if (ci < ncuts && cuts[ci] <= bend) { bend = cuts[ci]; forced = true; stream_end = kinds && kinds[ci] == 3; }
    BrBlk B; memset(&B, 0, sizeof(B));
    B.start = (u32)bstart; B.end = (u32)bend; B.is_last = ((is_final && bend == n) || stream_end) ? 1u : 0u;
    B.base = (u32)base; B.stream = stream;
    B.force_flush = forced && !B.is_last ? 1u : 0u; B.changed_epoch = -1;
    B.first_chunk = total;
    B.nchunks = (u32)((bend - bstart + ch - 1) / ch);
    if (chunks)
      for (u64 c = bstart; c < bend; c += ch) {
        BrBlockIn k; memset(&k, 0, sizeof(k));
        k.pos = (u32)c; k.end = (u32)(c + ch < bend ? c + ch : bend); k.blk_start = (u32)bstart; k.blk_end = (u32)bend;
        k.first = (c == bstart); k.last = (k.end == bend); k.is_last = B.is_last; k.force_flush = B.force_flush; k.blk = (u32)blks.size();
        k.base = B.base;
        chunks->push_back(k);
      }
    total += B.nchunks;
    blks.push_back(B);
    bstart = bend;
    if (stream_end) { base = bend; ++stream; }
  }
  { u32 send = n; for (size_t i = blks.size(); i-- > 0;) { if (blks[i].is_last) send = blks[i].end; blks[i].send = send; } }
  if (nchunks_total) *nchunks_total = total;
}
