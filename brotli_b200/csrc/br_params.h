// br_params.h -- host-side parameter derivation: what SanitizeParams / ComputeLgBlock /
// ChooseHasher / ComputeRbBits / MaxMetablockSize (c/enc/quality.h:59-225) decide for a
// given (quality, lgwin, size_hint), and the plan of one stream built from them.  Host only.
#pragma once
#include <type_traits>
#include <vector>
#include "br_types.h"
#include "br_pipeline.h"

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
// chunks == nullptr: only the block table (the CUDA pipeline fills the chunk table on the device: k_build_chunks, by
// br_chunk_in, the entry of chunk c of input block B, block index b, chunks of ch bytes).
BR_HD BrBlockIn br_chunk_in(const BrBlk& B, u32 b, u32 c, u32 ch) {
  BrBlockIn k; memset(&k, 0, sizeof(k));
  k.pos = B.start + c * ch; k.end = k.pos + ch < B.end ? k.pos + ch : B.end; k.blk_start = B.start; k.blk_end = B.end;
  k.first = c == 0; k.last = k.end == B.end; k.is_last = B.is_last; k.force_flush = B.force_flush; k.blk = b; k.base = B.base;
  return k;
}
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
    if (chunks) for (u32 c = 0; c < B.nchunks; ++c) chunks->push_back(br_chunk_in(B, (u32)blks.size(), c, ch));
    total += B.nchunks;
    blks.push_back(B);
    bstart = bend;
    if (stream_end) { base = bend; ++stream; }
  }
  { u32 send = n; for (size_t i = blks.size(); i-- > 0;) { if (blks[i].is_last) send = blks[i].end; blks[i].send = send; } }
  if (nchunks_total) *nchunks_total = total;
}

// Everything the host decides about one stream (or batch of streams) before its first kernel runs.
struct BrStreamPlan {
  BrParams P;                    // with the cuts, the knobs, the batch rules, finish_empty, nblocks and max_epochs applied
  std::vector<BrBlk> blk;        // the input blocks (br_build_blocks)
  std::vector<u32> slot_blk;     // BrStream::slot_blk
  std::vector<u32> stream_blk;   // BrStream::stream_blk: [nstreams + 1], the first input block of every stream
  u32 nstreams;
  u32 cmd_stride;                // commands one chunk may emit (BrStream::cmd_stride)
  u32 ran_cap;                   // entries of ran_list
  u32 max_rounds;                // late-fallback rounds after which the stream fails
  bool is_final;
  int with_header;
};

// Plans a stream of n bytes: false where the combination is outside what the pipeline implements.  cuts, knobs (nullable):
// br_pipeline.h.  batch_chunk_bits (the sim's schedules): the chunk size of a batch of streams instead of
// br_batch_chunk_bits.  chunks (nullable): also the chunk table (the CUDA pipeline builds it on the device, k_build_chunks).
static inline bool br_plan_stream(int quality, int lgwin, u32 size_hint, u32 n, const BrCuts* cuts, const BrSchedKnobs* knobs,
                                  BrStreamPlan* plan, u32 batch_chunk_bits = BR_KNOB_KEEP,
                                  std::vector<BrBlockIn>* chunks = nullptr) {
  BrParams& P = plan->P;
  if (n == 0 || !br_derive_params(quality, lgwin, size_hint, n, &P, cuts ? cuts->lgblock : 0)) return false;
  P.disable_ctx = cuts && cuts->disable_ctx ? 1u : 0u;
  P.stream_offset = cuts ? (cuts->stream_offset < P.max_backward ? cuts->stream_offset : P.max_backward) : 0u;   // encode.c:680
  if (knobs) {
    if (knobs->sweep_epoch != BR_KNOB_KEEP) P.sweep_epoch = knobs->sweep_epoch;
    if (knobs->force_epoch != BR_KNOB_KEEP) P.force_epoch = knobs->force_epoch;
    if (knobs->step_cap != BR_KNOB_KEEP) P.step_cap = knobs->step_cap;
    if (knobs->heavy_min != BR_KNOB_KEEP) P.heavy_min = knobs->heavy_min;
    if (knobs->pilot != BR_KNOB_KEEP) P.pilot = knobs->pilot;
    if (knobs->sweep_blocks != BR_KNOB_KEEP) {
      if (knobs->sweep_blocks == 0 || (knobs->sweep_blocks & (knobs->sweep_blocks - 1))) return false;   // (a power of two)
      P.sweep_blocks = knobs->sweep_blocks;
    }
  }
  const u32 ncuts = cuts ? cuts->n : 0;
  u32 nstreams = 1;
  for (u32 i = 0; i < ncuts; ++i) if (cuts->kind[i] == 3) ++nstreams;
  if (nstreams > 1) {
    // a batch of independent streams (each below BR_SMALL_STREAM, size_hint = the largest): no FLUSH cuts, all finished
    if (nstreams != ncuts + 1 || !cuts->is_final || !cuts->with_header || cuts->finish_empty || cuts->stream_offset ||
        cuts->pos[ncuts - 1] >= n || size_hint >= BR_SMALL_STREAM) return false;
    P.multi = nstreams; P.pilot = 0;
    P.chunk_bits = batch_chunk_bits != BR_KNOB_KEEP ? batch_chunk_bits : br_batch_chunk_bits(n);
  }
  if (P.quick && P.stream_offset) return false;   // (STREAM_OFFSET: quality 5..9)
  plan->is_final = cuts ? cuts->is_final != 0 : true;
  plan->with_header = cuts ? cuts->with_header : 1;
  P.finish_empty = cuts && cuts->finish_empty ? 1u : 0u;
  if (!plan->is_final && (ncuts == 0 || cuts->pos[ncuts - 1] != n)) return false;   // an unfinished stream ends at a cut
  if (P.finish_empty && (!plan->is_final || (ncuts && cuts->pos[ncuts - 1] == n))) return false;
  std::vector<BrBlk>& blk = plan->blk;
  blk.clear();
  if (chunks) chunks->clear();
  u32 nb = 0;
  br_build_blocks(P, n, cuts ? cuts->pos : nullptr, ncuts, plan->is_final && !P.finish_empty, chunks, blk, &nb,
                  cuts ? cuts->kind : nullptr);
  const u32 nblk = (u32)blk.size();
  plan->slot_blk.assign(((size_t)n >> P.lgblock) + 2, 0);
  for (size_t i = 0, b = 0; i < plan->slot_blk.size(); ++i) {
    while (b + 1 < nblk && blk[b].end <= ((u64)i << P.lgblock)) ++b;
    plan->slot_blk[i] = (u32)b;
  }
  plan->stream_blk.assign(nstreams + 1, nblk);
  for (u32 bi = nblk; bi-- > 0;) plan->stream_blk[blk[bi].stream] = bi;
  plan->nstreams = nstreams;
  P.nblocks = nb;
  // Launch bound: in forced mode every launch finalises at least one input block (at most two launches per block with
  // the conservative block-level re-marks), and a late uncompressed fallback restarts the count at most once per metablock.
  P.max_epochs = 4 * nb + 4096;
  plan->cmd_stride = (1u << P.chunk_bits) / 2 + 2;
  // ran_list: every chunk is walked at most once per launch -- by its own scheduled walker or by the one sweep that chases
  // into it, and in a forced launch the walkers scheduled behind the forced one in its input block stand down
  // (br_walk_block) -- so a launch appends at most nb entries
  plan->ran_cap = nb + 16;
  plan->max_rounds = nblk + 8;   // (every round stores at least one more metablock raw)
  return true;
}

// Points s at the constant tables: brotli_tables.bin (oracle/gen_tables.c) at `blob` and the log2 table.
static inline void br_bind_tables(BrStream& s, const u8* blob, const double* log2tab, u32 log2tab_n) {
  const u8* p = blob + 8;
  s.dict_size_bits = p; p += 32;
  s.dict_offsets = (const u32*)p; p += 128;
  s.dict = p; p += 122784;
  s.dict_hash_words = (const u16*)p; p += 65536;
  s.dict_hash_lengths = p; p += 32768;
  s.ctx_lut = p;
  s.log2tab = log2tab; s.log2tab_n = log2tab_n;
}

// G = bucket-ring rows the walker fetches together (br_lz77.h): 1 for the 16/32-entry rings of quality 5-6 (throughput
// bound, 8 CTAs per SM), 4 for the 64-256-entry rings of quality 7-9 (more registers, fewer resident warps).
#ifndef BR_WALK_G_DEEP
#define BR_WALK_G_DEEP 4    /* rows fetched together for the 256-entry rings of quality 9: 8 (the whole ring, 125 registers,
                               16 warps per SM) walks one chunk faster, 4 (96 registers, 20 warps per SM) won on the whole
                               job of config C4 when the two were timed against each other */
#endif
#ifndef BR_WALK_G_SMALL
#define BR_WALK_G_SMALL 1   /* rows fetched together for the 16/32-entry rings */
#endif
// Calls f(F, M) with the walker's template arguments for P as std::integral_constants: F the walker form (br_walk_form:
// the row grouping, 0 for the quick search of qualities 2..4, and the ring size where it is fixed), M a batch of streams.
// Quality 5 (16-entry ring) gets a form with the ring fixed; qualities 6..9 read it from P.  (A fixed 32-entry form for
// quality 6 compiled with less spilling but walked 100 MB of text 5 % slower on an H100, DESIGN.md section 5.)
template <int F, class Fn> static inline void br_walk_dispatch_m(const BrParams& P, Fn& f) {
  if (P.multi) f(std::integral_constant<int, F>(), std::true_type());
  else f(std::integral_constant<int, F>(), std::false_type());
}
template <class Fn> static inline void br_walk_dispatch(const BrParams& P, Fn&& f) {
  if (P.quick) br_walk_dispatch_m<0>(P, f);
  else if (P.block_bits >= 6) br_walk_dispatch_m<BR_WALK_G_DEEP>(P, f);
  else if (P.block_bits == 4) br_walk_dispatch_m<br_walk_form(BR_WALK_G_SMALL, 4)>(P, f);
  else br_walk_dispatch_m<BR_WALK_G_SMALL>(P, f);
}
