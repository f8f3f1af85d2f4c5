// br_types.h -- plain-old-data shared by host driver, CUDA kernels and the test sim.
#pragma once
#include "br_port.h"

// One Brotli command, same 16-byte layout as the reference's Command (c/enc/command.h:108).
struct BrCmd {
  u32 insert_len;
  u32 copy_len;    // low 25 bits: copy length; high 7 bits: copy_len_code - copy_len
  u32 dist_extra;
  u16 cmd_prefix;
  u16 dist_prefix; // low 10 bits: distance symbol; high 6: number of extra bits
};

// Encoder parameters after the reference's sanitising (c/enc/quality.h, c/enc/encode.c:642).
struct BrParams {
  int quality, lgwin, lgblock;
  int hash64;       // 1: 5-byte hash H6/H68 (quality.h:182), 0: 4-byte hash H5/H58
  int bucket_bits;  // 14 or 15
  int block_bits;   // quality - 1: bucket ring holds 1 << block_bits positions
  int ndist;        // 4, 10 or 16 distance-cache probes
  u32 htl;          // HashTypeLength == StoreLookahead: 8 (hash64) or 4
  u32 rmask;        // ring buffer mask of the reference: (1 << (1 + max(lgwin, lgblock))) - 1
  u32 max_backward; // (1 << lgwin) - 16
  u32 spree;        // LiteralSpreeLengthForSparseSearch: 64 (q < 9) or 512
  u32 max_mb;       // MaxMetablockSize
  u32 size_hint;
  u32 n;            // input bytes
  u32 nblocks;      // number of chunks (speculation units); input blocks are groups of them
  u32 nbuckets;     // 1 << bucket_bits (+1 overflow bucket for the unhashable tail positions)
  u32 chunk_bits;   // the unit of speculation is a chunk of 1 << chunk_bits bytes (see BR_CHUNK_BITS below)
  u32 sweep_epoch;  // from this launch on: only the HEAD of every run of consecutive dirty chunks is scheduled; its walker
                    // sweeps the run serially, seeing its own fresh stored-bits (Gauss-Seidel inside a run, Jacobi across runs)
  u32 force_epoch;  // from this launch on the first scheduled walker also runs to the end of its input block whatever the
                    // flags say: every launch then finalises at least one block, which bounds the number of launches
  u32 stream_offset; // BROTLI_PARAM_STREAM_OFFSET (encode.h:231), clamped to the window: the stream continues another one -- no window
                    // bits, poisoned distance cache (encode.c:656), dictionary distances count from the virtual start
  u32 disable_ctx;  // BROTLI_PARAM_DISABLE_LITERAL_CONTEXT_MODELING: one literal context (encode.c:561)
  u32 finish_empty; // FINISH arrived without input right behind a full input block: that block was encoded as a non-last one
                    // (encode.c:1700), the stream is closed by whatever is still pending or by an empty last metablock
  u32 sweep_blocks; // power of two: a sweep crosses input-block boundaries except into blocks whose index is a multiple of this
  u32 max_epochs;   // size of the per-launch arrays (a bound no input reaches: see br_kernels.cu)
  u32 step_cap;     // successor-walk budget per flipped bit in the dependency marking; beyond it the block-level rule
  u32 heavy_min;    // buckets with at least this many positions take the counter-wrap path (65536; tests lower it)
  u32 pilot;        // != 0: the first launch walks only the stream's first chunk: the static-dictionary gate (hash.h:186) nearly
                    // always closes inside it, and then every other chunk starts with the exact (closed) counters -- no dictionary
                    // probes in the big launch, no re-walk of chunks that found dictionary words under an open-gate guess
  u32 multi;        // != 0: the job is a BATCH of this many independent streams laid end to end in `data` (cuts of kind 3,
                    // br_params.h): every position-dependent rule counts from the stream's first byte (BrBlk::base)
  // ---- qualities 2..4: the one-position-per-slot hashers H2 / H3 / H4 / H54 (hash_longest_match_quickly_inc.h, hash.h:251-338)
  u32 quick;        // != 0: the index is sorted by SLOT (the table entry a position is filed in), searches consult
                    // 1 << qk_sweep_bits slots and see the latest stored position of each (br_find_quick)
  u32 qk_bits;      // BUCKET_BITS: 16 (H2, H3), 17 (H4), 20 (H54)
  u32 qk_sweep_bits;  // BUCKET_SWEEP_BITS: 0 (H2), 1 (H3), 2 (H4, H54)
  u32 qk_hash_len;  // HASH_LEN: 5, or 7 (H54)
  u32 qk_dict;      // USE_DICTIONARY (H2, H4): one shallow probe of the static dictionary when nothing else matched
  u32 mb_kind;      // how a metablock is stored: 0 BrotliStoreMetaBlock after the greedy block split (quality >= 4),
                    // 1 BrotliStoreMetaBlockTrivial (quality 3), 2 BrotliStoreMetaBlockFast (quality 2) (encode.c:543-556)
};

// The unit of speculation is a CHUNK: a slice (1 << BR_CHUNK_BITS bytes) of one of the
// reference's input blocks.  Per chunk: what the chain hands to the chunk's walker.
// 2 KiB chunks for streams of a megabyte and more; 512-byte chunks below that: a small stream has few chunks and its
// latency is the serial walk of ONE chunk per launch, so finer chunks cut it four-fold (a 64 KiB stream: 12.7 -> see DESIGN.md).
#define BR_CHUNK_BITS 11
#define BR_CHUNK_BITS_SMALL 9
#define BR_SMALL_STREAM (1u << 20)
// The walker's compile-time form F (br_lz77.h, br_walk_dispatch): the row grouping G in the low byte (0: the quick search
// of qualities 2..4) and above it the bucket ring's size as block_bits where it is fixed at compile time (0: P.block_bits,
// read at run time).  A fixed ring lets quality 5 get a walker that holds only its own search paths.
constexpr int br_walk_form(int G, int ring_bits) { return G | ring_bits << 8; }
#define BR_FORM_G(F) ((F) & 0xff)
#define BR_FORM_RB(F) ((F) >> 8)
struct BrBlockIn {
  u32 pos, end;          // nominal slice [pos, end) of the input
  u32 blk_start, blk_end;  // the reference input block (one EncodeData call) that contains it
  u32 first, last;       // first / last chunk of that block
  u32 blk;               // index of that block
  u32 start_pos;         // where the parse resumes (first chunk: blk_start)
  u32 last_insert_len;   // pending literals at start_pos (informational: walkers count from zero)
  int dc[4];             // distance cache at start_pos
  u32 ext_dist;          // first chunk, != 0: ExtendLastCommand applies with this distance (encode.c:905)
  u32 apply_rh;          // apply_random_heuristics (backward_references_inc.h:29) carried into the chunk
  u32 store_end;         // store_end of the block (backward_references_inc.h:24); set by its first chunk
  u32 dict_l_lo, dict_l_hi, dict_m_lo, dict_m_hi;  // dict_num_lookups / dict_num_matches (hash.h:49)
  u32 is_last;           // block flags (copied to all its chunks)
  u32 force_flush;       // BROTLI_OPERATION_FLUSH ended the input here (encode.c:1700)
  u32 warm;              // != 0: the state above is a guess; walk this many bytes before `pos` first to refine it
  u32 base;              // first byte of the stream the block belongs to (0 unless BrParams::multi)
};
#define BR_WARM_BYTES 256
// What the walker reports back.
struct BrBlockOut {
  u32 ncmd, nlit;        // commands emitted, literals covered by them (without the carried-in literals)
  u32 out_pos;           // where the parse stands when the walker leaves the chunk
  u32 last_insert_len;   // pending literals there, counted from the chunk start if it emitted no command
  int dc[4];
  u32 apply_rh, store_end;
  u32 ext_len;           // bytes swallowed by ExtendLastCommand
  u32 dl, dm;            // static-dictionary counter deltas
  u32 gate_checks, gate_fail;
  u32 min_wrap_dist;     // see br_lz77.h (bucket counter wrap sensitivity)
  u32 valid;
  u32 epoch;             // walker launch that produced this record
  u32 head;              // first chunk of the sweep (one warp walking consecutive chunks) this run belongs to
  u32 own_par;           // which of the two bits_cur bitmaps the run wrote (the parity of the sweep's head)
#ifdef BR_DEBUG_KNOBS
  u32 dbg_kcycles, dbg_searches, dbg_rows, dbg_mlsteps;   // profile of the latest run (debug build)
#endif
};

// Per reference input block (one EncodeData call): static layout, aggregates over its chunks and
// what the block-level chain derives for it.
struct BrBlk {
  u32 start, end, first_chunk, nchunks, is_last, force_flush;
  // aggregates (chain phase 2)
  u32 ncmd, nlit_rel, has_cmd, lil_head, lil_tail, last_cmd_chunk, dl, dm, ext_len, valid;
  int out_dc[4];
  u32 lc_copy_len, lc_dist_prefix, lc_dist_extra;   // the block's last command
  int changed_epoch;
  u32 state_dirty;   // br_chain_c: the block holds a chunk whose in-state is off (a sweep starts in it)
  u32 base, send;    // [base, send): the stream the block belongs to ([0, n) unless BrParams::multi)
  u32 stream;        // index of that stream
};
// What the block-to-block recurrence derives for an input block (br_chain_b -> br_chain_c).
struct BrBlkIn {
  int in_dc[4];
  u32 in_ext_dist, lil_in, dict_l_lo, dict_l_hi, dict_m_lo, dict_m_hi, cmd_base, mb;
};

// Per metablock record produced by the chain kernel.
struct BrMetaBlock {
  u32 start, end;        // input range
  u32 first_block, last_block;
  u32 cmd_off, ncmd;     // commands in the compacted array (incl. trailing insert-only command)
  u32 nlit;
  u32 is_last;
  u32 compress;          // 0: stored uncompressed (ShouldCompress said no or late fallback)
  u8 prev_byte, prev_byte2;
  u8 flushed;            // the metablock ends at a FLUSH / EMIT_METADATA cut (BrBlk::force_flush)
  u8 empty_last;         // an empty last metablock (ISLAST, ISLASTEMPTY) follows this one (BrParams::finish_empty)
  u32 tail_insert;       // insert-only command appended at flush (0 if none)
  u32 out_bits;          // bits produced by the compressed encoder (relative, from bit 0)
  u32 scratch_off;
  u32 base;              // first byte of the metablock's stream (literal contexts see zeros in front of it)
};

// BrStream::dirty[] values: 0 clean; reason (1..5) = scheduled for the next walker launch; with a BR_DEFER_* bit the
// chunk is dirty but left to the walker of the chunk before it (br_walk_block):
//   BR_DEFER_STATE  its in-state is off and the chunk before it is walked anyway (chase);
//   BR_DEFER_SWEEP  it lies behind a state-dirty chunk of its input block: the sweep that starts there walks it if it
//                   arrives with another state than the chunk consumed, otherwise the chunk is scheduled next time;
//   BR_DEFER_FULL   full sweep: the walker of the run's head walks it whatever the state.
#define BR_DEFER_STATE 0x100u
#define BR_DEFER_SWEEP 0x200u
#define BR_DEFER_FULL 0x400u
#define BR_DEFER (BR_DEFER_STATE | BR_DEFER_SWEEP | BR_DEFER_FULL)
#define BR_SAW_NONE 0xffffffffu
#define BR_SAW_SKIP 0xfffffffeu
#define BR_BATCH_HEAD_CHUNKS 16u   // batch of streams: chunks the walker of a stream's first chunk covers in the first launch (br_chain_c)

// Device-resident view of one stream (all pointers are device pointers).
struct BrStream {
  BrParams P;
  const u8* data;        // n bytes + >= 16 zero bytes
  const u32* S;          // positions sorted by (bucket key, position)
  const u32* rank;       // rank[S[j]] = j
  const u32* seg;        // seg[key] = first index of bucket key in S; nbuckets + 2 entries
  u32* bits_latest;      // stored-position bitmap, latest run of every block
  u32* bits_cur;         // written by the walkers of this iteration: TWO bitmaps of bits_words words each; a run writes the
                         // one of its chunk's parity, so the ranges of neighbouring chunks can overlap without mixing
  u32 bits_words;
  const u32* bits_prev;  // copy of bits_latest taken before the commits of this iteration
  u32* srch_latest;      // positions FindLongestMatch was called on (latest run of their owner) ...
  u32* srch_cur;         // ... and in this iteration
  u32* cover_cur;        // positions covered by a run of this launch (br_cover_run): what br_commit_bits may count as "stored in
                         // everybody's view" is a position stored before the launch AND, where a run of this launch covers it, after it
  const u32* storedS;    // bits_latest permuted into S order ...
  const u32* prefS;      // ... with exclusive popcount prefix every 1024 bits
  BrBlockIn* bin;        // [nblocks]   chain state handed to walkers
  BrBlockIn* bin_used;   // [nblocks]   state the latest run of each block consumed
  BrBlockOut* bout;      // [nblocks]
  BrCmd* cmd_blocks;     // per block command buffers, stride cmd_stride
  u32 cmd_stride;
  u32* dirty;            // [nblocks] run this block in the next walker launch
  u32* changed_bits;     // [nblocks] popcount of bitmap changes of the latest run
  int* changed_epoch;    // [nblocks] last walker launch whose commit changed this chunk's bits (-1: never)
  int* bitdep_epoch;     // [nblocks] last launch that changed a stored-bit this chunk's searches may consult
  const u16* skeys;      // bucket key of S[j]
  const u16* tagS;       // 16-bit hash of the first four bytes at S[j]: a candidate whose tag differs from the search position's
                         // cannot match four bytes, so its bytes are never fetched (the reference's H58 / H68 keep 8-bit tags
                         // for the same reason, hash_longest_match64_simd_inc.h:26)
  u32* epoch_cum;        // [max_epochs + 1] epoch_cum[t] = sum over launches <= t of the largest number of stored-bit flips
                         // any single heavy bucket saw in that launch (bucket counter wrap rule)
  u32 epoch;             // current walker launch number (1-based)
  u32 forced;            // this launch: the first scheduled walker runs to the end of its input block (BrParams::force_epoch)
  u32* ext_total;        // [nblocks] bytes added to the chunk's last command by ExtendLastCommand
  u32* lil_in;           // [nblocks] true pending-literal count at the chunk start (added to its first command)
  const u32* slot_blk;   // [(n >> lgblock) + 1] index of the input block that holds position i << lgblock (streams cut by FLUSH
                         // have irregular blocks; see br_chunk_of)
  BrBlk* blk;            // [nblk] reference input blocks
  BrBlkIn* blkin;        // [nblk]
  u32* key_flips;        // [nbuckets + 1] stored-bit flips per heavy bucket in the current launch
  const u32* qpred;      // BrParams::quick: [n << qk_sweep_bits] for position p and slot i of its search: first index of that slot's
                         // segment of S whose position is >= p (br_lz77.h br_quick_pred_fill)
  u32* saw;              // BrParams::quick: [n << qk_sweep_bits] what the latest search at a position read from each of its slots
                         // (index into S of the candidate, BR_SAW_NONE: the slot was empty, BR_SAW_SKIP: not read) -- br_verify_run
  u32 nblk;
  u32* dirty_list;       // [nblocks] chunks scheduled for the next walker launch (counters[5] entries)
  u32* ran_list;         // [nblocks] chunks walked in the current launch (counters[4] entries)
  u32* block_mb;         // [nblocks] metablock of every chunk
  u32* cmd_off;          // [nblocks] offset of the block's commands in the compacted array
  BrMetaBlock* mbs;      // [max_mbs]
  u32* force_unc;        // [max_mbs] late fallback: store this metablock uncompressed
  u32* counters;         // [8]: 0 n_dirty, 1 n_mbs, 2 total cmds, 3 error flags, 4 chunks walked this launch, 5 chunks scheduled, 6 first scheduled chunk, 7 last launch entered in epoch_cum (+1), 8.. dirty reasons
  u32* hist_scratch;     // [256] (batch of streams: 256 per stream)
  // batch of streams (BrParams::multi): the chain runs per stream (br_chain_b1..b3)
  const u32* stream_blk; // [multi + 1] first input block of every stream
  u32* stream_nmb;       // [multi + 1] metablocks of every stream, then (exclusive scan) the number of its first metablock
  u32* stream_ncmd;      // [multi + 1] likewise for commands
  BrMetaBlock* mbs_stage;  // [nblk] metablock records of stream k at [stream_blk[k] ..), before they are numbered
  // tables
  const u8* dict;        // RFC 7932 dictionary
  const u32* dict_offsets;  // [32]
  const u8* dict_size_bits; // [32]
  const u16* dict_hash_words;   // [32768]
  const u8* dict_hash_lengths;  // [32768]
  const u8* ctx_lut;     // [2048]
  const double* log2tab; // [log2tab_n]
  u32 log2tab_n;
};
