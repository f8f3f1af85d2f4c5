// br_lz77.h -- LZ77 backward-reference search for one input block, one warp per block.
//
// What it replaces: BrotliCreateBackwardReferences (c/enc/backward_references_inc.h:10) with
// the bucket-ring hashers H5/H6/H58/H68 (c/enc/hash_longest_match*_inc.h), plus
// ExtendLastCommand (c/enc/encode.c:905).
//
// Why it looks nothing like the reference: the reference keeps ONE mutable hash table per
// stream, so every block depends on the complete history of the parse before it.  Here the
// table is replaced by two immutable, position-ordered structures built by sorting kernels:
//
//   S[]     all positions sorted by (bucket key, position)   -> "the bucket ring at time p"
//           is the run of STORED positions just before rank[p] in S;
//   bits[]  one "was this position ever inserted" bit per position, produced by the parse
//           itself (every FindLongestMatch / StoreRange / Stitch call site sets bits).
//
// A block's walker only needs (a) the small serial state at its start (distance cache,
// pending literals, dictionary counters: BrBlockIn) and (b) the stored-bits of earlier
// positions.  All blocks of a stream therefore run CONCURRENTLY from speculated inputs, and a
// serial-but-tiny chain kernel (br_chain below) re-derives the true inputs from the outputs;
// blocks whose inputs changed are re-run until a fixpoint.  By induction over blocks a
// fixpoint equals the sequential parse, so the commands are bit-identical to the reference.
#pragma once
#include "br_cmd.h"

struct BrSR { u32 len, distance, score; int delta; };
#ifdef BR_SIM_DEBUG
static u64 br_sim_w[12];   // tests/sim: 0 searches, 1 ring rows, 2 heavy-path searches, 3 heavy own-scan rows, 4 countS calls, 5 own_set, 6 set_range, 7 dict searches, 8 ring groups, 9 candidates taken, 10 match_len beyond 16 bytes
#define BR_W(i, n) (br_sim_w[i] += (n))
static u64 br_sim_bnd[2];  // tests/sim: block boundaries a sweep reached where br_predict_next_block 0 accepted, 1 refused
#else
#define BR_W(i, n)
#endif

#define BR_SCORE_BASE 1920u  /* hash.h:102: 30 * 8 * sizeof(size_t) */
#define BR_MIN_SCORE (BR_SCORE_BASE + 100u)

BR_DEV u32 br_match_len(const u8* d, u32 a, u32 b, u32 limit) {
  u32 len = 0;
  while (len + 8 <= limit) {
    u64 x = br_ld64u(d, a + len) ^ br_ld64u(d, b + len);
    if (x) return len + (u32)(br_ctz64(x) >> 3);
    len += 8;
  }
  while (len < limit && br_ldg(d + a + len) == br_ldg(d + b + len)) ++len;
  return len;
}

// Same, with the first 16 bytes at `b` (the search position, identical for all candidates of one
// search) already in registers.
BR_DEV u32 br_match_len_c(const u8* d, u32 a, u32 b, u32 limit, u64 c0, u64 c1) {
  if (limit >= 8) {
    u64 x = br_ld64u(d, a) ^ c0;
    if (x) return (u32)(br_ctz64(x) >> 3);
    if (limit >= 16) {
      x = br_ld64u(d, a + 8) ^ c1;
      if (x) return 8u + (u32)(br_ctz64(x) >> 3);
      return 16u + br_match_len(d, a + 16, b + 16, limit - 16);
    }
    return 8u + br_match_len(d, a + 8, b + 8, limit - 8);
  }
  return br_match_len(d, a, b, limit);
}

// Same, with the first 8 bytes at `a` (the candidate) already loaded as well.
BR_DEV u32 br_match_len_d0(const u8* d, u32 a, u32 b, u32 limit, u64 c0, u64 c1, u64 a0) {
  if (limit >= 8) {
    u64 x = a0 ^ c0;
    if (x) return (u32)(br_ctz64(x) >> 3);
    if (limit >= 16) {
      x = br_ld64u(d, a + 8) ^ c1;
      if (x) return 8u + (u32)(br_ctz64(x) >> 3);
      return 16u + br_match_len(d, a + 16, b + 16, limit - 16);
    }
    return 8u + br_match_len(d, a + 8, b + 8, limit - 8);
  }
  return br_match_len(d, a, b, limit);
}

// hash_longest_match64_inc.h:23 / hash_longest_match_inc.h:23 HashBytes
BR_DEV u32 br_hash_key(const BrParams& P, const u8* d, u32 pos) {
  if (P.hash64) {
    u64 v = br_ld64u(d, pos);
    return (u32)((v * (0x1FE35A7BD3579BD3ull << 24)) >> (64 - 15));
  }
  return (br_ld32u(d, pos) * 0x1E35A7BDu) >> (32 - P.bucket_bits);
}

// tag of a position: 16 bits of a hash of its first four bytes (BrStream::tagS)
BR_DEV u32 br_tag4(u32 first4) { return (first4 * 0x9E3779B1u) >> 16; }
// same, from the 8 bytes at the position
BR_DEV u32 br_hash_key_v(const BrParams& P, u64 v) {
  if (P.hash64) return (u32)((v * (0x1FE35A7BD3579BD3ull << 24)) >> (64 - 15));
  return ((u32)v * 0x1E35A7BDu) >> (32 - P.bucket_bits);
}
struct BrWalk {
  const BrStream* s;
  const u8* d;
  u32 p0, pend;    // p0: first position this walker owns; pend: end of the reference input block
  u32 base;        // first byte of the stream (BrBlockIn::base): ring-buffer positions and distance limits count from it
  int dc[4];       // distance cache; entries 4..15 of the reference (hash.h:80) are derived on the fly
  // the static-dictionary counters dict_num_lookups / dict_num_matches (hash.h:49) are dict0 + dl / dict0 + dm: dict0 points
  // at their values where the walk starts (lo, hi, lo, hi as in BrBlockIn), so that no 64-bit copy rides in registers
  const u32* dict0;
  u32 dl, dm, gate_checks, gate_fail;
  u32 min_wrap;
  u32 stale;       // the byte the reference finds just past the block end (see oracle)
  bool warming;    // warm-up (state refinement before the chunk proper): reads the snapshot, records nothing
  u32* own;        // the bits_cur bitmap of this run (parity of the sweep's head chunk)
  bool fence_due;  // own bits were written to memory since the last fence (see br_own_sync)
  u32 acc_wi, acc_own, acc_srch;   // the word of the own / searched bitmaps the parse stands in, gathered in registers
#ifdef BR_DEBUG_KNOBS
  u32 dbg_searches, dbg_rows, dbg_mlsteps;
#endif
};

// Stored-bits of the walker's own range [p0, ...) live in bits_cur (global): written with
// atomic OR (other walkers own neighbouring bits of the same words), read around L1.
BR_DEV u32 br_ld_cur(const u32* p) {
#if BR_GPU
  return __ldcg(p);
#else
  return *p;
#endif
}
// The walker's writes are gathered per 32-position word: the parse moves forward, so the bits it sets (stored, searched)
// cluster in the word that holds its position.  `acc_*` is that word -- warp-uniform registers, visible to every lane
// at once -- and it goes to memory (one atomic OR each) only when the parse leaves the word.  Reads of own bits merge it in.
BR_DEV int br_own_get(const BrWalk& w, u32 q) {
  u32 v = br_ld_cur(w.own + (q >> 5));
  if ((q >> 5) == w.acc_wi) v |= w.acc_own;
  return (v >> (q & 31)) & 1;
}
// Writers (one lane per word) and readers (any lane) of the own bits in MEMORY are different threads of the warp: a
// fence + warp barrier must lie between a write and the next read.  The fence is not paid at the write -- it would wait
// for the atomic's round trip to L2 -- but right before the next read, several memory round trips later.
BR_DEV void br_own_sync(BrWalk& w) {
  if (w.fence_due) {
#if BR_GPU
    __threadfence_block();
#endif
    w.fence_due = false;
    br_syncwarp();
  }
}
BR_DEV void br_own_flush(BrWalk& w) {
  if (w.acc_wi != 0xffffffffu) {
    if (br_lane() == 0) {
      if (w.acc_own) br_atomic_or(w.own + w.acc_wi, w.acc_own);
      if (w.acc_srch) br_atomic_or(w.s->srch_cur + w.acc_wi, w.acc_srch);
    }
    w.fence_due = true;
    w.acc_wi = 0xffffffffu; w.acc_own = 0; w.acc_srch = 0;
  }
}
BR_DEV void br_own_word(BrWalk& w, u32 wi) {   // make wi the gathered word
  if (wi != w.acc_wi) { br_own_flush(w); w.acc_wi = wi; }
}
BR_DEV void br_own_set(BrWalk& w, u32 q) {
  BR_W(5, 1);
  if (w.warming) return;   // warm-up: the snapshot is read, nothing is recorded
  br_own_word(w, q >> 5);
  w.acc_own |= 1u << (q & 31);
}
BR_DEV void br_srch_set(BrWalk& w, u32 q) {
  if (w.warming) return;
  br_own_word(w, q >> 5);
  w.acc_srch |= 1u << (q & 31);
}
BR_DEV void br_own_set_range(BrWalk& w, u32 a, u32 b) {
  BR_W(6, 1);
  if (a >= b) return;
  if (w.warming) return;
  const u32 wa = a >> 5, wb = (b - 1) >> 5;
  const u32 ma = 0xffffffffu << (a & 31), mb = 0xffffffffu >> (31 - ((b - 1) & 31));
  if (wa == wb) { br_own_word(w, wa); w.acc_own |= ma & mb; return; }
  // several words: the gathered word may be the first one; the middle goes straight to memory, the last becomes the gathered word
  if (w.acc_wi == wa) w.acc_own |= ma;
  else if (br_lane() == 0) br_atomic_or(w.own + wa, ma);
  for (u32 x = wa + 1 + (u32)br_lane(); x < wb; x += BR_WARP) br_atomic_or(w.own + x, 0xffffffffu);
  w.fence_due = true;
  br_own_word(w, wb);
  w.acc_own |= mb;
}
BR_DEV int br_is_stored(const BrWalk& w, u32 q) {
  if (q >= w.p0) return br_own_get(w, q);
  return (br_ldg(w.s->bits_latest + (q >> 5)) >> (q & 31)) & 1;
}
// Number of stored positions (latest snapshot) among S[a .. b).
BR_DEV u32 br_countS_upto(const BrStream& s, u32 x) {
  BR_W(4, 1);
  u32 base = br_ldg(s.prefS + (x >> 10));
  u32 w0 = (x >> 10) << 5, w1 = x >> 5, acc = 0;
  for (u32 wi = w0 + (u32)br_lane(); wi < w1; wi += BR_WARP) acc += (u32)br_popc(br_ldg(s.storedS + wi));
  acc = br_warp_sum(acc);
  if (x & 31) acc += (u32)br_popc(br_ldg(s.storedS + w1) & ((1u << (x & 31)) - 1u));
  return base + acc;
}

// hash.h:186: the dictionary is searched only while dict_num_matches >= dict_num_lookups >> 7
BR_DEV bool br_dict_gate_closed(const BrWalk& w) {
  const u64 l = (((u64)w.dict0[1] << 32) | w.dict0[0]) + w.dl, m = (((u64)w.dict0[3] << 32) | w.dict0[2]) + w.dm;
  return m < (l >> 7);
}
// hash.h:140 TestStaticDictionaryItem
BR_DEV int br_test_dict_item(const BrWalk& w, u32 len, u32 word_idx, u32 cur, u32 max_length,
                             u32 max_backward, BrSR& out) {
  const BrStream& s = *w.s;
  if (len > max_length) return 0;
  u32 offset = br_ldg(s.dict_offsets + len) + len * word_idx;
  u32 matchlen = 0;
  while (matchlen < len && br_ldg(w.d + cur + matchlen) == br_ldg(s.dict + offset + matchlen)) ++matchlen;
  if (matchlen + 10 <= len || matchlen == 0) return 0;
  u32 cut = len - matchlen;
  u32 transform_id = (cut << 2) + (u32)((0x071B520ADA2D3200ull >> (cut * 6)) & 0x3F);
  u32 backward = max_backward + 1 + word_idx + (transform_id << br_ldg(s.dict_size_bits + len));
  if (backward > 0x3FFFFFCu) return 0;
  u32 score = BR_SCORE_BASE + 135u * matchlen - 30u * br_log2floor(backward);
  if (score < out.score) return 0;
  out.len = matchlen;
  out.delta = (int)len - (int)matchlen;
  out.distance = backward;
  out.score = score;
  return 1;
}
// hash.h:179 SearchInStaticDictionary (warp-uniform)
BR_DEV void br_search_static_dict(BrWalk& w, u32 cur, u32 max_length, u32 max_backward, BrSR& out) {
  const BrStream& s = *w.s;
  BR_W(7, 1);
  ++w.gate_checks;
  if (br_dict_gate_closed(w)) { ++w.gate_fail; return; }
  u32 key = ((br_ld32u(w.d, cur) * 0x1E35A7BDu) >> (32 - 14)) << 1;
  for (int i = 0; i < 2; ++i, ++key) {
    ++w.dl;
    u32 len = br_ldg(s.dict_hash_lengths + key);
    if (len != 0) {
      if (br_test_dict_item(w, len, br_ldg(s.dict_hash_words + key), cur, max_length, max_backward, out)) {
        ++w.dm;
      }
    }
  }
}

// Entries of the bucket ring at search position `cur` (rank j) of a heavy bucket (slice [lo, hi) of S, hi - lo >= heavy_min).
// The reference's per-bucket counter is a uint16 (hash_longest_match64_inc.h:52): after 65536 insertions it wraps and the
// ring looks empty again.  c = insertions so far (of this stream).  Returns the number of entries the ring holds
// (1 << block_bits unless the counter has wrapped to below that).
// (Not skipped while the stream is shorter than 65536 bytes, although c cannot wrap there: the sensitivity this path
// records -- min_wrap = 0 while the ring is not full -- also re-walks chunks whose view reached through their own freshly
// unstored positions into a range that flipped in the same launch, which the successor count of br_commit_bits, taken over
// the previous snapshot, could miss before it learnt to count with the runs' own fresh bits (k_cover): DESIGN.md
// section 3, "the marking gap".  Kept: it costs nothing and is the net under that rule.)
BR_DEV u32 br_ring_heavy(BrWalk& w, u32 j, u32 lo) {
  const BrStream& s = *w.s;
  const int lane = br_lane();
  const u32 block_size = 1u << s.P.block_bits;
  u32 lo_s = lo;
  if (w.base) {   // batch of streams: the bucket's slice starts with the positions of the streams in front
    u32 a = lo, b = j;
    while (a < b) { const u32 mid = (a + b) >> 1; if (br_ldg(s.S + mid) < w.base) a = mid + 1; else b = mid; }
    lo_s = a;
  }
  u32 own_cnt = 0, jj = j, n_own = 0;
  BR_W(2, 1);
  br_own_sync(w);
  while (jj > lo) {
    BR_W(3, 1);
    u32 idx = jj - 1 - (u32)lane;
    bool has = (jj >= lo + 1 + (u32)lane);
    u32 q = has ? br_ldg(s.S + idx) : 0;
    bool mine = has && q >= w.p0;
    u32 mm = br_ballot(mine);
    own_cnt += (u32)br_popc(br_ballot(mine && br_own_get(w, q)));
    n_own += (u32)br_popc(mm);
    if (mm != (BR_WARP == 32 ? 0xffffffffu : 1u)) break;
    jj -= BR_WARP;
  }
  u32 jb = j - n_own;
  u32 prev_cnt = br_countS_upto(s, jb) - br_countS_upto(s, lo_s);
  u32 c = (prev_cnt + own_cnt) & 0xFFFFu;
  if (c < block_size) { w.min_wrap = 0; return c; }
  u32 sd = c - block_size, su = 65535u - c;
  u32 m = sd < su ? sd : su;
  if (m < w.min_wrap) w.min_wrap = m;
  return block_size;
}

// Lookahead of the quality 5 search (the shared pass below): L2 prefetch hints for the searches still to come, issued
// while the current search waits on its own loads.  A search waits on three dependent round trips -- (bytes at cur, rank)
// -> (row of S, its snapshot bits) -> candidates' first bytes -- and the last two are random reads of 400 MB and of the
// 4 MB window that miss L2.  Their addresses for the next searches do not depend on the current search's result, only on
// their positions, which the walker predicts (br_walk_one).  So:
//   stage 1, BR_WALK1_LOOKAHEAD searches ahead: prefetch the row of S and its snapshot words;
//   stage 2 (lookahead >= 2), the next search: load its row (now from L2) and prefetch the first bytes of its newest
//   block_size entries inside the window.
// Nothing loaded here reaches a search: every search still does all its own loads, which then hit L2.  A wrong prediction
// costs memory traffic only.  0 turns the lookahead off; the one-lane CPU build (tests/sim) has none.
// The walk is as much issue bound as latency bound (DESIGN.md section 3), so every instruction added here has to pay for
// itself.  Timed on 100 MB of text at quality 5 (H100, section 5): lookahead 1 walks about 5 % faster than none; 2 and 3
// (stage 2, in either of two forms) were slower than 1, and a prefetch of the bucket bounds seg[key] (a table L2 already
// holds) cost more than it saved.
#ifndef BR_WALK1_LOOKAHEAD
#define BR_WALK1_LOOKAHEAD 1
#endif
struct BrLook {
  u32 next;     // stage 2: the next search's position (~0u: none)
  u32 f0, nf;   // stage 1: the rows of positions f0 .. f0 + nf - 1 (nf <= BR_WALK1_LOOKAHEAD)
};
// Position of the search that follows a FAILED search at x (br_walk_one's rule: x + 1, or the random-heuristics jump
// past the literals; its clamp at the block end is left out, a prediction only has to be right most of the time).
BR_DEV u32 br_next_search(u32 x, u32 apply_rh, u32 window) {
  const u32 p = x + 1;
  if (p <= apply_rh) return p;
  return p + (p > apply_rh + 4 * window ? 16u : 8u);
}

// FindLongestMatch (hash_longest_match64_inc.h:157, hash_longest_match_inc.h:156), lane-parallel:
// every candidate's full match length is computed by its own lane, then the reference's
// sequential "better than the best so far" rule is replayed with ballots.  The reference's
// quick reject (4 bytes ending at best_len) passes exactly when the candidate is longer than
// best_len, or -- only when best_len already equals max_length -- when the byte just past the
// block end compares equal (w.stale).  Candidates that pass it by coincidence with a shorter
// length can never beat the running score, so they are dropped here without side effects.
//
// G = rows (32 candidates each) of the bucket's slice of S that are fetched TOGETHER.  A deep bucket ring
// (quality 7-9: 64-256 entries) is several rows; fetching row by row puts three dependent memory round trips
// (S row -> stored bits -> candidate bytes) on the search's critical path PER ROW.  With G > 1 the G rows are
// loaded back to back, then their stored bits and the first 8 bytes of every candidate (speculatively, before the
// stored bit is known), and only then the rows are folded in order: three round trips per G rows.  This is what a
// latency-bound walker (a sweep, br_walk_block) needs; the fold itself is unchanged.
//
// G == 1 (quality 5-6: 4 distance-cache probes, 16- or 32-entry rings): a separate pass for the four distance-cache
// candidates leaves 28 of 32 lanes idle.  So at quality 5 the first pass runs over 32 candidate slots
// [distance cache ++ the newest 28 entries of the ring] -- the reference's order (hash.h:80 first, then the ring newest
// first) -- with one match-length computation and one fold; further ring rows (32 entries each) follow from j - 28.
//
// F = the walker form (br_walk_form): G, and the ring size where it is fixed at compile time.  Quality 5's form (16
// entries) compiles the shared pass alone, with the four distance-cache probes as a constant; the forms that read
// block_bits at run time hold every path.
template <int F>
BR_DEV void br_find_longest_match(BrWalk& w, u32 cur, u32 max_length, u32 max_backward,
                                  u32 dict_distance, BrSR& out, BrLook look = {~0u, 0u, 0u}) {
  constexpr int G = BR_FORM_G(F), RB = BR_FORM_RB(F);
  const BrStream& s = *w.s;
  const BrParams& P = s.P;
  const u8* d = w.d;
  const int lane = br_lane();
  const u32 rmask = P.rmask;
  const u32 cur_m = (cur - w.base) & rmask;
  const u32 min_score = out.score;
  u32 best_score = out.score, best_len = out.len;
  out.len = 0; out.delta = 0;
  BR_W(0, 1);
#ifdef BR_DEBUG_KNOBS
  ++w.dbg_searches;
#endif
  // the bytes at the search position, shared by every candidate comparison below
  const u64 c0 = br_ld64u(d, cur), c1 = br_ld64u(d, cur + 8);
  // Load order = latency plan.  (1) the index entry of `cur` (bucket bounds, rank) and the first bytes of the
  // distance-cache candidates are requested together; (2) the first G rows of the bucket's slice of S go out as soon
  // as the rank is there (G > 1: the distance-cache fold runs while they are in flight; quality 5: the first row shares
  // the distance cache's pass, and its snapshot bits go out with it); (3) stored bits + candidate bytes; (4) fold.
  // Three dependent round trips per search instead of one per step.
  const u32 key = br_hash_key_v(P, c0);
  const u32 lo = br_ldg(s.seg + key), hi = br_ldg(s.seg + key + 1);
  const u32 j = br_ldg(s.rank + cur);
  const u32 block_size = RB ? 1u << RB : 1u << P.block_bits;
  const u32 ndist = RB ? 4u : P.ndist;   // (qualities 5-6 probe the four last distances: br_derive_params)
  u32 V = block_size;   // ring entries the reference holds (fewer only in a heavy bucket whose counter wrapped)
  u32 collected = 0, jj = j;   // stored ring entries seen so far; the ring's slice of S still to read is [lo, jj)
  bool done = false;           // the ring ends (window, stream start, ring-buffer stop)
  const u32 tag_cur = br_tag4((u32)c0);
  u32 q[G] = {}; bool has[G] = {}, tagok[G] = {};   // the ring rows in flight (G > 1: the first G are loaded up front)
  // The shared pass only where the whole ring fits in it (quality 5: 16 entries).  The 32-entry ring of quality 6 would
  // need a second, dependent row after it: timed on 100 MB of text, that made the walk 22 % slower than a distance-cache
  // pass that runs while the first full row is in flight.
  if (G == 1 && block_size <= 28u) {
    // ---- one pass over the 32 candidate slots k = [distance cache (hash.h:80, qualities 5-6 probe 4) ++ the newest
    // 28 ring entries].  On the GPU lane k owns slot k; in the one-lane build (tests/sim) the same code is a loop over k.
    constexpr int NDC = 4, NC = 32 / BR_WARP;
    // slot's candidate position; its first 8 bytes (distance cache); valid / has; the word of the S-ordered snapshot bits
    // that holds the entry's bit (ring)
    u32 ca[NC]; u64 ca0[NC]; bool cv[NC]; u32 csw[NC];
#if BR_GPU && BR_WALK1_LOOKAHEAD > 0
    // lookahead loads, requested with this search's own first round trip (the ranks share its sectors)
    const u32 lrk = (u32)(lane - NDC);   // lane's row entry (lanes >= NDC)
    // (a position is searched only while it lies more than htl bytes before the block end: rank exists there)
    u32 jf[BR_WALK1_LOOKAHEAD];
#pragma unroll
    for (int i = 0; i < BR_WALK1_LOOKAHEAD; ++i) {
      const u32 t = look.f0 + (u32)i;
      jf[i] = (u32)i < look.nf && t < w.pend && w.pend - t > P.htl ? br_ldg(s.rank + t) : 0u;
    }
#if BR_WALK1_LOOKAHEAD >= 2
    const u32 jn = look.next < w.pend && w.pend - look.next > P.htl ? br_ldg(s.rank + look.next) : 0u;
    const u32 qn = lane >= NDC && lrk < block_size && jn > lrk ? br_ldg(s.S + (jn - 1 - lrk)) : 0u;
#endif
#endif
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      const int k = i * BR_WARP + lane;
      csw[i] = 0;
      if (k < NDC) {
        const int back = k == 0 ? w.dc[0] : k == 1 ? w.dc[1] : k == 2 ? w.dc[2] : w.dc[3];
        cv[i] = back > 0 && (u32)back <= max_backward;
        ca[i] = cur - (u32)back;
        ca0[i] = cv[i] ? br_ld64u(d, ca[i]) : 0;
      } else {
        // The row of S and its snapshot bits are requested as soon as the rank is there, not after the bucket bounds: the
        // row's address depends on j only, and the slots in front of the bucket's slice (entries of other buckets) are
        // dropped once lo arrives.  The snapshot word is needed only when the row lies in front of the walker's own range
        // (decided below from the row's positions), but requesting it now takes a memory round trip off the search.
        const u32 rk = (u32)(k - NDC);   // ring entry rk, newest first
        const u32 idx = j - 1 - rk;
        u32 qs = 0;
        if (j > rk) { qs = br_ldg(s.S + idx); csw[i] = br_ldg(s.storedS + (idx >> 5)); }
        cv[i] = j >= lo + 1 + rk;
        ca[i] = cv[i] ? qs : 0;
        ca0[i] = 0;
      }
    }
#if BR_GPU && BR_WALK1_LOOKAHEAD > 0
    // stage 1: the rows of S and their snapshot words, each lane its own entry (the row is one or two lines)
#pragma unroll
    for (int i = 0; i < BR_WALK1_LOOKAHEAD; ++i) {
      if (lane >= NDC && jf[i] > lrk) {
        br_prefetch_l2(s.S + (jf[i] - 1 - lrk));
        br_prefetch_l2(s.storedS + ((jf[i] - 1 - lrk) >> 5));
      }
    }
#if BR_WALK1_LOOKAHEAD >= 2
    // stage 2: the first bytes of the next search's candidates
    if (qn != 0 && qn < look.next && look.next - qn <= max_backward) br_prefetch_l2(d + qn);
#endif
#endif
    if (hi - lo >= P.heavy_min) V = br_ring_heavy(w, j, lo);
    br_own_sync(w);
    BR_W(8, 1); BR_W(1, 1);
#ifdef BR_DEBUG_KNOBS
    ++w.dbg_rows;
#endif
    bool brk = false;
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      const int k = i * BR_WARP + lane;
      const bool isdc = k < NDC;
      const u32 a = ca[i];
      // ring slots: stored bits as in the rows below (the newest ring entry is slot NDC's); rank among the stored ring
      // entries, then the ring ends at the first entry outside the window or the slice
      const bool inwin = !isdc && cv[i] && cur - a <= max_backward;
      bool st;
      if (br_shfl(a, NDC % BR_WARP) < w.p0) {
        const u32 idx = j - 1 - (u32)(k - NDC);
        st = inwin && ((csw[i] >> (idx & 31)) & 1u);
      } else st = inwin && br_is_stored(w, a);
      const u32 m = br_ballot(st);
      const bool take = st && (collected + (u32)br_popc(m & br_lanemask_lt()) < V);
      if (br_ballot(!isdc && !inwin) != 0) done = true;
      collected += (u32)br_popc(m);
      // one match length for every probed slot
      u32 len = 0; int eqmax = 0;
      if (isdc ? cv[i] : take) {
        BR_W(9, isdc ? 0 : 1);
        len = br_match_len_d0(d, a, cur, max_length, c0, c1, isdc ? ca0[i] : br_ld64u(d, a));
        if (!isdc && len < 4) len = 0;
        if (len == max_length) eqmax = (w.stale == (u32)br_ldg(d + a + max_length));
      }
      const u32 dist = cur - a;
      u32 score;
      if (isdc) {
        score = 135u * len + BR_SCORE_BASE + 15u;
        if (k != 0) score -= 39u + ((0x1CA10u >> (k & 0xE)) & 0xEu);
      } else score = len ? BR_SCORE_BASE + 135u * len - 30u * br_log2floor(dist) : 0;
      const bool lenok = isdc ? cv[i] && (len >= 3 || (len == 2 && k < 2)) : take && len != 0;
      const u32 pm = (a - w.base) & rmask;
      int last = -1;
      while (!brk) {
        // a distance-cache candidate still to come ends the whole search once cur_m + best_len passes the ring buffer
        if (br_ballot(isdc && cv[i] && lane > last) != 0 && cur_m + best_len > rmask) { brk = done = true; break; }
        // the ring compares against a best length of at least 3, and the same test with it ends the ring only
        const u32 bl3 = best_len < 3 ? 3u : best_len, bl = isdc ? best_len : bl3;
        const bool rstop = cur_m + bl3 > rmask;
        if (rstop) done = true;
        const bool ok = lenok && lane > last && !(!isdc && rstop) && !(pm + bl > rmask) &&
                        (len > bl || (len == bl && bl == max_length && eqmax)) && score > best_score;
        const u32 mm = br_ballot(ok);
        if (!mm) break;
        const int f = br_ffs(mm) - 1;
        best_len = br_shfl(len, f); best_score = br_shfl(score, f);
        out.len = best_len; out.distance = br_shfl(dist, f); out.score = best_score;
        last = f;
      }
    }
    jj = j > 32u - NDC ? j - (32u - NDC) : 0u;
  } else {
    // ---- distance cache probes: lane k owns candidate k (hash.h:80 PrepareDistanceCache layout)
    constexpr int ND = (16 + BR_WARP - 1) / BR_WARP;
    u32 dback[ND]; u64 da0[ND]; bool dvalid[ND];
#pragma unroll
    for (int i = 0; i < ND; ++i) {
      const int k = i * BR_WARP + lane;
      int back_i = 0;
      if (k < 4) back_i = k == 0 ? w.dc[0] : k == 1 ? w.dc[1] : k == 2 ? w.dc[2] : w.dc[3];
      else if (k < 16) {   // dc[4..15] = last -1, +1, -2, +2, -3, +3; second last likewise (hash.h:83-97)
        int mag = (int)((0xE79u >> (2 * ((k - 4) >> 1))) & 3u);
        back_i = (k < 10 ? w.dc[0] : w.dc[1]) + ((k & 1) ? mag : -mag);
      }
      dvalid[i] = ((u32)k < ndist) && back_i > 0 && (u32)back_i <= max_backward;
      dback[i] = (u32)back_i;
      da0[i] = dvalid[i] ? br_ld64u(d, cur - (u32)back_i) : 0;
    }
    // first G rows of the bucket ring (consumed by the loop further down), with their tags (deep rings only, see k_tags)
#pragma unroll
    for (int r = 0; r < G; ++r) {
      const u32 jr = j > (u32)(r * BR_WARP) ? j - (u32)(r * BR_WARP) : 0u;
      has[r] = jr >= lo + 1 + (u32)lane;
      q[r] = has[r] ? br_ldg(s.S + (jr - 1 - (u32)lane)) : 0;
      tagok[r] = has[r] && (G == 1 || (u32)br_ldg(s.tagS + (jr - 1 - (u32)lane)) == tag_cur);
    }
    bool brk = false;
#pragma unroll
    for (int i = 0; i < ND; ++i) {
      if ((u32)(i * BR_WARP) >= ndist || brk) break;
      const int k = i * BR_WARP + lane;
      const bool valid = dvalid[i];
      const u32 back = dback[i];
      u32 len = 0; int eqmax = 0;
      if (valid) {
        len = br_match_len_d0(d, cur - back, cur, max_length, c0, c1, da0[i]);
        if (len == max_length) eqmax = (w.stale == (u32)br_ldg(d + (cur - back) + max_length));
      }
      u32 score = 135u * len + BR_SCORE_BASE + 15u;
      if (k != 0) score -= 39u + ((0x1CA10u >> (k & 0xE)) & 0xEu);
      const bool lenok = valid && (len >= 3 || (len == 2 && k < 2));
      const u32 pm = (cur - back - w.base) & rmask;
      int last = -1;
      for (;;) {
        // candidates are examined in order; everything up to `last` has been decided
        u32 pending = br_ballot(valid && lane > last);
        if (!pending) break;
        if (cur_m + best_len > rmask) { brk = true; break; }
        bool ok = lenok && lane > last && !(pm + best_len > rmask) &&
                  (len > best_len || (len == best_len && best_len == max_length && eqmax)) && score > best_score;
        u32 mm = br_ballot(ok);
        if (!mm) break;
        int f = br_ffs(mm) - 1;
        best_len = br_shfl(len, f); best_score = br_shfl(score, f);
        out.len = best_len; out.distance = br_shfl(back, f); out.score = best_score;
        last = f;
      }
    }
    if (hi - lo >= P.heavy_min) V = br_ring_heavy(w, j, lo);
  }
  if (best_len < 3) best_len = 3;
  // ---- bucket ring (for G == 1: the rows after the first pass)
  {
    br_own_sync(w);
    while (!done && collected < V && jj > lo) {
      u64 d0[G]; bool inwin[G], st[G];
      BR_W(8, 1);
      // ---- fetch: G rows of S (the first G are already here unless the shared pass took the first row), then their
      // stored bits and (G > 1) the candidates' first bytes
      if (jj != j) {
#pragma unroll
        for (int r = 0; r < G; ++r) {
          const u32 jr = jj > (u32)(r * BR_WARP) ? jj - (u32)(r * BR_WARP) : 0u;
          has[r] = jr >= lo + 1 + (u32)lane;
          q[r] = has[r] ? br_ldg(s.S + (jr - 1 - (u32)lane)) : 0;
          tagok[r] = has[r] && (G == 1 || (u32)br_ldg(s.tagS + (jr - 1 - (u32)lane)) == tag_cur);
        }
      }
#pragma unroll
      for (int r = 0; r < G; ++r) {
        inwin[r] = has[r] && cur - q[r] <= max_backward;
        // Stored bits.  A row that lies entirely before this walker's own range (its newest entry, lane 0's, does) reads the
        // S-ordered copy of the snapshot: the row's 32 bits sit in one or two words.  Otherwise every lane reads the bit of
        // its position (own bitmap or snapshot): 32 scattered sectors.
        const u32 jr = jj > (u32)(r * BR_WARP) ? jj - (u32)(r * BR_WARP) : 0u;
        const u32 q0 = br_shfl(q[r], 0);
        if (q0 < w.p0) {
          const u32 idx = jr - 1 - (u32)lane;
          st[r] = inwin[r] && ((br_ldg(s.storedS + (idx >> 5)) >> (idx & 31)) & 1u);
        } else st[r] = inwin[r] && br_is_stored(w, q[r]);
      }
      if (G > 1) {
#pragma unroll
        for (int r = 0; r < G; ++r) d0[r] = (inwin[r] && tagok[r]) ? br_ld64u(d, q[r]) : 0;
      }
      // ---- fold, row by row, newest first
#pragma unroll
      for (int r = 0; r < G; ++r) {
        if (r > 0) {
          const u32 jr = jj > (u32)(r * BR_WARP) ? jj - (u32)(r * BR_WARP) : 0u;
          if (done || collected >= V || jr <= lo) break;
        }
        const u32 backward = cur - q[r];
        BR_W(1, 1);
#ifdef BR_DEBUG_KNOBS
        ++w.dbg_rows;
#endif
        const u32 m = br_ballot(st[r]);
        const u32 rnk = (u32)br_popc(m & br_lanemask_lt());
        const bool take = st[r] && (collected + rnk < V);
        if (br_ballot(has[r] && !inwin[r]) != 0 || br_ballot(!has[r]) != 0) done = true;
        collected += (u32)br_popc(m);
        // full match length of every taken candidate
        // (H6: the first four bytes must agree, then the length counts on; H5: length >= 4.  Same thing.)
        u32 len = 0; int eqmax = 0;
        if (take && tagok[r]) {
          BR_W(9, 1);
          len = G > 1 ? br_match_len_d0(d, q[r], cur, max_length, c0, c1, d0[r]) : br_match_len_c(d, q[r], cur, max_length, c0, c1);
          if (len < 4) len = 0;
          if (len == max_length) eqmax = (w.stale == (u32)br_ldg(d + q[r] + max_length));
        }
        const u32 score = len ? BR_SCORE_BASE + 135u * len - 30u * br_log2floor(backward) : 0;
        const u32 pm = (q[r] - w.base) & rmask;
        int last = -1;
        for (;;) {
          if (cur_m + best_len > rmask) { done = true; break; }
          bool ok = take && len != 0 && lane > last && !(pm + best_len > rmask) &&
                    (len > best_len || (len == best_len && best_len == max_length && eqmax)) &&
                    score > best_score;
          u32 mm = br_ballot(ok);
          if (!mm) break;
          int f = br_ffs(mm) - 1;
          best_len = br_shfl(len, f);
          best_score = br_shfl(score, f);
          out.len = best_len; out.distance = br_shfl(backward, f); out.score = best_score;
          last = f;
        }
      }
      jj = jj > (u32)(G * BR_WARP) ? jj - (u32)(G * BR_WARP) : 0;
    }
    br_own_set(w, cur);  // the insertion at hash_longest_match64_inc.h:268
    br_srch_set(w, cur);
  }
  if (min_score == out.score) br_search_static_dict(w, cur, max_length, dict_distance, out);
}

// ---------------------------------------------------------------------------------------------------------------------
// Qualities 2..4: HashLongestMatchQuickly (hash_longest_match_quickly_inc.h; H2, H3, H4, H54 of hash.h:251-338).
// The reference's table holds ONE position per slot; a position p is filed in slot (key(p) + (p & SWEEP_MASK)) & MASK
// (Store, :96) and a search reads the 1 << BUCKET_SWEEP_BITS slots key, key + 8, ... (:231).  Here the index S is sorted by
// (slot, position), so "the content of slot s at time p" is the latest STORED position in front of p in the slot's
// segment of S (position 0 when there is none: the table starts zeroed, :76).  Every slot read is recorded in
// BrStream::saw (index into S of the position read, or BR_SAW_ABSENT | the index the backward walk stopped at), and
// br_verify_run (br_chain.h) checks the records of every run against the committed stored-bits after each launch.
// The code below is warp-UNIFORM: every lane executes the same scalar search (the loads are broadcasts); a search is a
// handful of candidates, and a uniform formulation is what the one-lane CPU sim (tests/sim) validates completely.
#define BR_SAW_ABSENT 0x80000000u
// hash_longest_match_quickly_inc.h:27 HashBytes: HASH_LEN bytes, kHashMul64, the top BUCKET_BITS bits
BR_DEV u32 br_quick_key_v(const BrParams& P, u64 v) {
  return (u32)(((v << (64 - 8 * P.qk_hash_len)) * 0x1FE35A7BD3579BD3ull) >> (64 - P.qk_bits));
}
// the slot position `pos` (counted from the first byte of its stream) is filed in (Store, :96)
BR_DEV u32 br_quick_slot(const BrParams& P, u64 v, u32 pos) {
  return (br_quick_key_v(P, v) + (pos & (((1u << P.qk_sweep_bits) - 1u) << 3))) & ((1u << P.qk_bits) - 1u);
}
// data[cur_ix_masked + off] as the reference reads it (:162, :185): at off == max_length that byte lies just past the
// input block (w.stale, see the oracle's stale_byte)
BR_DEV u32 br_cur_byte(const BrWalk& w, u32 cur, u32 off, u32 max_length) {
  return off < max_length ? (u32)br_ldg(w.d + cur + off) : w.stale;
}
// hash.h:179 SearchInStaticDictionary with shallow == TRUE: one probe
BR_DEV void br_search_static_dict_shallow(BrWalk& w, u32 cur, u32 max_length, u32 max_backward, BrSR& out) {
  const BrStream& s = *w.s;
  BR_W(7, 1);
  ++w.gate_checks;
  if (br_dict_gate_closed(w)) { ++w.gate_fail; return; }
  const u32 key = ((br_ld32u(w.d, cur) * 0x1E35A7BDu) >> (32 - 14)) << 1;
  ++w.dl;
  const u32 len = br_ldg(s.dict_hash_lengths + key);
  if (len != 0) {
    if (br_test_dict_item(w, len, br_ldg(s.dict_hash_words + key), cur, max_length, max_backward, out)) ++w.dm;
  }
}
// First index of slot `slot`'s segment of S whose position is >= p (p itself is not in that segment): where a search at p
// starts looking for the slot's content.  Computed once per position and slot by k_slot_pred (BrStream::qpred), outside
// the fixpoint -- in the walker it would be ~10 dependent memory round trips per foreign slot and search.
BR_DEV u32 br_quick_lower_bound(const BrStream& s, u32 slot, u32 p) {
  u32 a = br_ldg(s.seg + slot), b = br_ldg(s.seg + slot + 1);
  while (a < b) {
    const u32 mid = (a + b) >> 1;
    if (br_ldg(s.S + mid) < p) a = mid + 1; else b = mid;
  }
  return a;
}
// qpred entries of position p (thread task; `base`: first byte of p's stream)
BR_DEV void br_quick_pred_fill(const BrStream& s, u32 p, u32 base, u32* out) {
  const BrParams& P = s.P;
  const u32 sweep = 1u << P.qk_sweep_bits, mask = (1u << P.qk_bits) - 1u;
  if (p + P.htl > P.n) { for (u32 i = 0; i < sweep; ++i) out[i] = 0; return; }   // (never searched: the parse stops htl bytes before a block end)
  const u32 key = br_quick_key_v(P, br_ld64u(s.data, p));
  const u32 i_own = ((p - base) >> 3) & (sweep - 1u);
  for (u32 i = 0; i < sweep; ++i)
    out[i] = i == i_own ? br_ldg(s.rank + p) : br_quick_lower_bound(s, (key + (i << 3)) & mask, p);
}
// hash_longest_match_quickly_inc.h:147 FindLongestMatch.  out.len carries best_len_in (backward_references_inc.h:127).
// Load plan (every step = one memory round trip for all slots together): (1) the bytes at cur; (2) segment starts,
// qpred entries, the last-distance candidate's bytes; (3) the newest entry in front of cur in every slot; (4) their
// stored bits; (5) the candidates' first bytes and pre-check bytes; then the reference's sequential fold.
BR_DEV void br_find_quick(BrWalk& w, u32 cur, u32 max_length, u32 max_backward, u32 dict_distance, BrSR& out) {
  const BrStream& s = *w.s;
  const BrParams& P = s.P;
  const u8* d = w.d;
  const u32 sweep = 1u << P.qk_sweep_bits, mask = (1u << P.qk_bits) - 1u;
  const u32 best_len_in = out.len;
  const u32 min_score = out.score;
  u32 best_score = out.score, best_len = best_len_in;
  const u64 c0 = br_ld64u(d, cur), c1 = br_ld64u(d, cur + 8);
  const u32 key = br_quick_key_v(P, c0);
  u32 compare_char = br_cur_byte(w, cur, best_len_in, max_length);
  const bool rec = !w.warming && br_lane() == 0;
  u32* saw = s.saw + ((size_t)cur << P.qk_sweep_bits);
  const u32 base = w.base;   // first byte of the stream (0 unless the job is a batch of streams): the table's positions count from it
  BR_W(0, 1);
  out.delta = 0;
  u32 lo[4], ja[4];
#pragma unroll
  for (u32 i = 0; i < 4; ++i) {
    lo[i] = ja[i] = 0;
    if (i < sweep) {
      lo[i] = br_ldg(s.seg + ((key + (i << 3)) & mask));
      ja[i] = br_ldg(s.qpred + ((size_t)cur << P.qk_sweep_bits) + i);
    }
  }
  bool early = false;
  {
    const int cached = w.dc[0];
    if (cached > 0 && (u32)cached <= max_backward) {   // (:168: prev_ix < cur_ix && cached_backward <= max_backward)
      const u32 prev = cur - (u32)cached;
      if (compare_char == (u32)br_ldg(d + prev + best_len)) {
        const u32 len = br_match_len_c(d, prev, cur, max_length, c0, c1);
        if (len >= 4) {
          const u32 score = 135u * len + BR_SCORE_BASE + 15u;   // BackwardReferenceScoreUsingLastDistance
          if (best_score < score) {
            out.len = len; out.distance = (u32)cached; out.score = score;
            if (sweep == 1) early = true;   // (:178: the slot is overwritten unread)
            else { best_len = len; best_score = score; compare_char = br_cur_byte(w, cur, len, max_length); }
          }
        }
      }
    }
  }
  if (early) {
    if (rec) saw[0] = BR_SAW_SKIP;
    br_own_set(w, cur); br_srch_set(w, cur);
    return;
  }
  br_own_sync(w);
  // ---- (3) the newest entry in front of cur in every slot, (4) its stored bit (own fresh bits inside the walker's range,
  // the snapshot in front of it), inside the window and the stream
  u32 q0[4]; bool has0[4], inw[4], st0[4];
#pragma unroll
  for (u32 i = 0; i < 4; ++i) { has0[i] = i < sweep && ja[i] > lo[i]; q0[i] = has0[i] ? br_ldg(s.S + (ja[i] - 1)) : 0u; }
#pragma unroll
  for (u32 i = 0; i < 4; ++i) {
    inw[i] = has0[i] && q0[i] >= base && cur - q0[i] <= max_backward;
    st0[i] = inw[i] && br_is_stored(w, q0[i]);
  }
  // ---- the slot's content as this walker sees it: the latest stored position in front of cur.  Absent: the stream's
  // first position (the zeroed table holds 0) while the window still reaches it; otherwise the slot holds something the
  // reference rejects (backward > max_backward) whatever its first byte.
  u32 prev[4]; bool valid[4]; u64 f8[4]; u32 cb[4];
#pragma unroll
  for (u32 i = 0; i < 4; ++i) {
    prev[i] = 0; valid[i] = false;
    if (i >= sweep) continue;
    u32 j = ja[i];
    bool found = false, at_start = true;
    if (st0[i]) { found = true; j = ja[i] - 1; prev[i] = q0[i]; }
    else if (has0[i] && q0[i] >= base) {
      if (!inw[i]) at_start = false;
      else {   // in the window but not stored: walk on (short: most positions are stored)
        j = ja[i] - 1;
        while (j > lo[i]) {
          const u32 q = br_ldg(s.S + (j - 1));
          if (q < base) break;                                // (batch of streams: positions of the streams in front)
          if (cur - q > max_backward) { at_start = false; break; }
          --j;
          if (br_is_stored(w, q)) { found = true; prev[i] = q; break; }
        }
      }
    }
    if (rec) saw[i] = found ? j : (BR_SAW_ABSENT | j);
    BR_W(1, 1);
    if (!found) prev[i] = base;
    const u32 backward = cur - prev[i];
    valid[i] = (found || (at_start && cur - base <= max_backward)) && backward != 0 && backward <= max_backward;
  }
  // ---- (5) first bytes and pre-check byte (data[prev + best_len], :191 / :236) of every candidate
#pragma unroll
  for (u32 i = 0; i < 4; ++i) {
    f8[i] = valid[i] ? br_ld64u(d, prev[i]) : 0ull;
    cb[i] = valid[i] ? (u32)br_ldg(d + prev[i] + best_len) : 0u;
  }
  const u32 bl0 = best_len;
  bool h2_return = false;
#pragma unroll
  for (u32 i = 0; i < 4; ++i) {
    if (i >= sweep) break;
    if (!valid[i]) { if (sweep == 1) h2_return = true; continue; }   // (:191-196: a rejected candidate ends H2's search)
    const u32 pc = best_len == bl0 ? cb[i] : (u32)br_ldg(d + prev[i] + best_len);
    if (compare_char != pc) { if (sweep == 1) h2_return = true; continue; }
    const u32 backward = cur - prev[i];
    const u32 len = br_match_len_d0(d, prev[i], cur, max_length, c0, c1, f8[i]);
    if (len >= 4) {
      const u32 score = BR_SCORE_BASE + 135u * len - 30u * br_log2floor(backward);
      if (best_score < score) {
        best_len = len; best_score = score;
        out.len = len; out.distance = backward; out.score = score;
        compare_char = br_cur_byte(w, cur, len, max_length);
        if (sweep == 1) h2_return = true;   // (:217)
      }
    }
  }
  br_own_set(w, cur);   // buckets[key_out] = cur_ix (:208, :265)
  br_srch_set(w, cur);
  if (h2_return) return;
  if (P.qk_dict && min_score == out.score) br_search_static_dict_shallow(w, cur, max_length, dict_distance, out);
}

// backward_references.c:87 ComputeDistanceCode
BR_DEV u32 br_compute_distance_code(u32 distance, u32 max_distance, const int* dc) {
  if (distance <= max_distance) {
    u32 d3 = distance + 3;
    u32 o0 = d3 - (u32)dc[0], o1 = d3 - (u32)dc[1];
    if (distance == (u32)dc[0]) return 0;
    if (distance == (u32)dc[1]) return 1;
    if (o0 < 7) return (0x9750468u >> (4 * o0)) & 0xF;
    if (o1 < 7) return (0xFDB1ACEu >> (4 * o1)) & 0xF;
    if (distance == (u32)dc[2]) return 2;
    if (distance == (u32)dc[3]) return 3;
  }
  return distance + 15;
}

// One chunk (see br_types.h).  The walker resumes the parse of its input block at
// in.start_pos with the carried state and leaves when the position reaches the chunk end
// (the last chunk of a block runs to the block end like the reference loop).
// `head` is the first chunk of the sweep this run belongs to (== b when the walker starts here), `sweep_p0` the
// first position the sweep owns (0xffffffff on entry for the head, which sets it): a walker that continues into the
// chunks behind its own keeps writing the head's bitmap and reads its own fresh bits from sweep_p0 on.
// F: the walker form (br_walk_form).  M: the job is a batch of streams (BrParams::multi); with M = false the stream base
// is the constant 0 and folds away.
// The chunk records -- `in`, `o` and `used` (the state this run really starts from, refined by the warm-up; the caller's
// `used_rec`, else a local) -- are read and written before and after the per-position loop and at the warm-up crossing
// only.  The loop carries the parse state alone (position, pending literals, the random-heuristics mark, the distance
// cache, the counts, the gathered bit word) and one precomputed bound: on the GPU the records sit in the warp's shared
// memory (br_walk_block), so that none of them holds registers across the search, which needs every register there is
// at 8 blocks of 4 warps per SM (quality 5).
template <int F, bool M = false>
BR_DEV void br_walk_one(const BrStream& s, u32 b, const BrBlockIn& in, BrBlockOut& o, u32 head, u32& sweep_p0,
                        BrBlockIn* used_rec = nullptr) {
  constexpr int G = BR_FORM_G(F);
  const BrParams& P = s.P;
  const int lane = br_lane();
  BrBlockIn used_local;
  BrBlockIn& used = used_rec ? *used_rec : used_local;
  BrWalk w;
  w.s = &s; w.d = s.data; w.p0 = head == b ? in.start_pos : sweep_p0; w.pend = in.blk_end;
  w.own = s.bits_cur + (size_t)(head & 1u) * s.bits_words;
  w.dict0 = &in.dict_l_lo;
  w.dl = w.dm = w.gate_checks = w.gate_fail = 0;
  w.min_wrap = 0xffffffffu;
  w.fence_due = false;
  w.acc_wi = 0xffffffffu; w.acc_own = 0; w.acc_srch = 0;
#ifdef BR_DEBUG_KNOBS
  w.dbg_searches = w.dbg_rows = w.dbg_mlsteps = 0;
  const long long dbg_t0 = clock64();
#endif
  const u32 base = M ? in.base : 0u;
  w.base = base;
  w.stale = in.blk_end - base <= P.rmask ? 0u : (u32)s.data[in.blk_end - (P.rmask + 1)];
  for (int i = 0; i < 4; ++i) w.dc[i] = in.dc[i];
  const u32 pos_end = in.blk_end;
  u32 position = in.start_pos;
  u32 ext = 0;
  u32 apply_random_heuristics = in.apply_rh;
  used = in;
  used.warm = 0;
  w.warming = false;
  u32 cross_at = 0xffffffffu;   // warm-up: where the parse crosses into the chunk
  if (in.warm && !in.first && in.pos >= in.blk_start + in.warm) {
    // State refinement: parse the last `warm` bytes before the chunk from a neutral state; by the
    // time the parse crosses into the chunk it has usually synchronised with the true parse.
    w.warming = true;
    position = in.pos - in.warm;
    w.p0 = 0xffffffffu;
    apply_random_heuristics = position + P.spree;
    cross_at = in.pos;
  }
  const u32 window = P.spree;
  u32 store_end;
  if (in.first) {
    u32 bytes = pos_end - position;
    // ---- ExtendLastCommand (encode.c:941): grow the previous block's final copy.
    if (in.ext_dist) {
      while (bytes) {
        u32 chunk = bytes < BR_WARP ? bytes : BR_WARP;
        bool eq = (u32)lane < chunk && s.data[position + lane] == s.data[position + lane - in.ext_dist];
        u32 m = br_ballot(eq);
        u32 run = (u32)br_ffs(~m) - 1u;  // leading equal lanes
        if (run > chunk) run = chunk;
        ext += run; position += run; bytes -= run;
        if (run < chunk) break;
      }
    }
    apply_random_heuristics = position + window;
  }
  o.ext_len = ext;
  if (in.first) {
    u32 bytes = pos_end - position;   // what CreateBackwardReferences receives after the extension
    store_end = bytes >= P.htl ? pos_end - P.htl + 1 : position;
  } else {
    store_end = in.store_end;
  }
  // Pending literals are carried as an OFFSET: the parse does not depend on how many literals
  // are pending at the chunk start, only the first command's insert length does.  The walker
  // counts from zero and the chain / compaction add the true carry (BrStream::lil_in).
  u32 insert_length = 0;
  u32 ncmd = 0, nlit = 0;
  // the warm-up's crossing into the chunk: from here on this is the chunk's own run
  auto cross = [&]() {
    w.warming = false; w.p0 = position;
    used.start_pos = position; used.apply_rh = apply_random_heuristics;
    for (int i = 0; i < 4; ++i) used.dc[i] = w.dc[i];
    insert_length = 0; ncmd = 0; nlit = 0;
    w.dl = w.dm = w.gate_checks = w.gate_fail = 0;
    w.min_wrap = 0xffffffffu;
  };
  // The parse goes on while position + htl < pos_end and, but in the block's last chunk, position < in.end: one bound.
  // (So a crossing always lies inside the chunk proper: the warm-up ends inside the loop or, jumping over it, behind it.)
  u32 bound = pos_end > P.htl ? pos_end - P.htl : 0u;
  if (!in.last && in.end < bound) bound = in.end;
  BrCmd* cmds = s.cmd_blocks + (size_t)b * s.cmd_stride;
  while (position < bound) {
    if (position >= cross_at) { cross(); cross_at = 0xffffffffu; }
    // One search call site for the primary search and the (up to 4) lazy ones at position + 1
    // (backward_references_inc.h:58-101): the walker's code is dominated by the inlined search.
    u32 max_length = pos_end - position;
    BrSR sr; sr.len = 0; sr.delta = 0; sr.distance = 0; sr.score = BR_MIN_SCORE;
    bool have = false;
    int delayed = 0;
    for (;;) {
      const u32 sp = position + (have ? 1u : 0u);
      const u32 md = br_min(sp - base, P.max_backward);
      const u32 dd = P.stream_offset ? br_min(sp + P.stream_offset, P.max_backward) : md;   // backward_references_inc.h:94 dictionary_start
      BrSR cur; cur.len = 0; cur.delta = 0; cur.distance = 0; cur.score = BR_MIN_SCORE;
      if constexpr (G == 0) {   // qualities 2..4 (k_walk<0>): best_len_in of the lazy search, backward_references_inc.h:127
        if (have) cur.len = br_min(sr.len - 1u, max_length);
        br_find_quick(w, sp, max_length, md, dd, cur);
      } else {
        BrLook look = {~0u, 0u, 0u};
#if BR_GPU && BR_WALK1_LOOKAHEAD > 0
        if (G == 1) {   // (the search uses it in the shared pass of quality 5 only)
          if (have) {
            // a lazy search: predicted to lose, so the parse goes on at position + sr.len.  That row was not prefetched
            // (sr.len was not known), so only stage 1 runs for it and the positions behind it: loading it here for stage 2
            // would put a round trip to HBM on this search.
            look.f0 = position + sr.len; look.nf = BR_WALK1_LOOKAHEAD;
          } else {
            // predicted to fail (the parse goes on one position later, or jumps in a literal spree)
            u32 n = br_next_search(sp, apply_random_heuristics, window);
            if (BR_WALK1_LOOKAHEAD >= 2) look.next = n;
            for (int i = 1; i < BR_WALK1_LOOKAHEAD; ++i) n = br_next_search(n, apply_random_heuristics, window);
            look.f0 = n; look.nf = 1;
          }
        }
#endif
        br_find_longest_match<F>(w, sp, max_length, md, dd, cur, look);
      }
      if (!have) {
        sr = cur;
        if (!(sr.score > BR_MIN_SCORE)) break;
        have = true; --max_length;
        continue;
      }
      if (cur.score >= sr.score + 175u) {
        ++position; ++insert_length; sr = cur;
        if (++delayed < 4 && position + P.htl < pos_end) { --max_length; continue; }
      }
      break;
    }
    if (have) {
      apply_random_heuristics = position + 2 * sr.len + window;
      u32 dictionary_start = br_min(position - base + P.stream_offset, P.max_backward);
      u32 dcode = br_compute_distance_code(sr.distance, dictionary_start, w.dc);
      if (sr.distance <= dictionary_start && dcode > 0) {
        w.dc[3] = w.dc[2]; w.dc[2] = w.dc[1]; w.dc[1] = w.dc[0]; w.dc[0] = (int)sr.distance;
      }
      if (lane == 0 && !w.warming) cmds[ncmd] = br_init_cmd(insert_length, sr.len, sr.delta, dcode);
      ++ncmd;
      nlit += insert_length;
      insert_length = 0;
      {
        u32 range_start = position + 2;
        u32 range_end = br_min(position + sr.len, store_end);
        if (sr.distance < (sr.len >> 2)) {
          u32 t = position + sr.len - (sr.distance << 2);
          range_start = br_min(range_end, br_max(range_start, t));
        }
        br_own_set_range(w, range_start, range_end);
      }
      position += sr.len;
    } else {
      ++insert_length;
      ++position;
      if (position > apply_random_heuristics) {
        u32 step, reach, margin;
        if (position > apply_random_heuristics + 4 * window) {
          step = 4; reach = 16; margin = br_max(P.htl - 1, 4);
        } else {
          step = 2; reach = 8; margin = br_max(P.htl - 1, 2);
        }
        u32 pos_jump = br_min(position + reach, pos_end - margin);
        for (; position < pos_jump; position += step) {
          br_own_set(w, position);
          insert_length += step;
        }
      }
    }
  }
  if (w.warming) cross();   // the warm-up parse jumped over the whole chunk (or the block ended)
  br_own_flush(w);
  br_own_sync(w);   // a sweep's next chunk starts with a fresh BrWalk: nothing may stay pending
  if (in.last) {
    insert_length += pos_end - position;
    position = pos_end;
  }
  {
    o.ncmd = ncmd; o.nlit = nlit; o.out_pos = position; o.last_insert_len = insert_length;
    for (int i = 0; i < 4; ++i) o.dc[i] = w.dc[i];
    o.apply_rh = apply_random_heuristics; o.store_end = store_end;
    o.dl = w.dl; o.dm = w.dm;
    o.gate_checks = w.gate_checks; o.gate_fail = w.gate_fail;
    o.min_wrap_dist = w.min_wrap; o.valid = 1; o.epoch = s.epoch;
    o.head = head; o.own_par = head & 1u;
#ifdef BR_DEBUG_KNOBS
    o.dbg_kcycles = (u32)((clock64() - dbg_t0) >> 10); o.dbg_searches = w.dbg_searches; o.dbg_rows = w.dbg_rows; o.dbg_mlsteps = w.dbg_mlsteps;
#endif
  }
  if (head == b) sweep_p0 = used.start_pos;
  if (lane == 0) {
    s.bout[b] = o;
    s.bin_used[b] = used;
    u32 slot = br_atomic_add(s.counters + 4, 1);   // list of chunks to commit
    s.ran_list[slot] = b;
  }
  br_syncwarp();
}

// A sweep that reaches the end of its input block goes on into the next one.  What EncodeData does between two blocks
// (encode.c:985: StitchToPreviousBlock, ExtendLastCommand eligibility, merge-or-flush) is the chain's business, but
// the walker can PREDICT the in-state of the next block's first chunk from its own out-state and the metablock layout
// of the last chain run; the chain verifies it like any other in-state (a wrong prediction leaves that chunk dirty).
// Returns false at a boundary the walker cannot see through (metablock stored raw: distance cache restored; a block
// swallowed whole by ExtendLastCommand; chunk records it cannot trust).
BR_DEV bool br_predict_next_block(const BrStream& s, u32 b, const BrBlockIn& in, const BrBlockOut& o, BrBlockIn& ni) {
  const BrParams& P = s.P;
  const u32 nb = b + 1;
  ni = s.bin[nb];
  const bool flush = s.block_mb[nb] != s.block_mb[b];   // (layout of the last chain run)
  if (flush && !s.mbs[s.block_mb[b]].compress) return false;
  // (lane 0 reads what lane 0 wrote -- this sweep's own chunk records and commands -- and broadcasts the verdict)
  u32 ext_dist = 0, fail = 0;
  if (!flush && br_lane() == 0) {
    // pending literals behind the block's last command, and that command
    u32 lil = 0, c = b;
    const u32 first = s.blk[in.blk].first_chunk;
    bool found = false;
    for (;;) {
      const BrBlockOut oc = c == b ? o : s.bout[c];
      if (!oc.valid) { fail = 1; break; }
      lil += oc.last_insert_len;
      if (oc.ncmd > 0) { found = true; break; }
      if (c == first) break;
      --c;
    }
    if (!fail && !found && lil == 0) fail = 1;   // no command and nothing pending: swallowed by ExtendLastCommand
    if (!fail && found && lil == 0) {
      const BrCmd lc = s.cmd_blocks[(size_t)c * s.cmd_stride + (c == b ? o.ncmd : s.bout[c].ncmd) - 1];
      const u32 dcode = br_cmd_restore_dcode(lc.dist_prefix, lc.dist_extra);
      const int cmd_dist = o.dc[0];
      if (dcode < 16 || (cmd_dist > 0 && dcode - 15 == (u32)cmd_dist)) {
        const u32 lpp = in.blk_end - (lc.copy_len & 0x1FFFFFF);
        const u32 maxd = br_min(lpp - in.base, P.max_backward);
        if (cmd_dist > 0 && (u32)cmd_dist <= maxd) ext_dist = (u32)cmd_dist;
      }
    }
  }
  ext_dist = br_shfl(ext_dist, 0); fail = br_shfl(fail, 0);
  if (fail) return false;
  ni.start_pos = ni.blk_start; ni.ext_dist = ext_dist; ni.apply_rh = 0; ni.store_end = 0; ni.warm = 0;
  for (int i = 0; i < 4; ++i) ni.dc[i] = o.dc[i];
  return true;
}

// Walk chunk b, then go on into the chunks behind it (same input block) while nobody else runs the next chunk in this
// launch and
//   * the state this walker leaves differs from what the next chunk consumed on its latest run (CHASE; the chain leaves
//     such chunks to this walker: BR_DEFER_STATE, BR_DEFER_SWEEP), or
//   * the next chunk was handed to this walker unconditionally (BR_DEFER_FULL, full-sweep launches).
// The walker sees its own fresh stored-bits from the sweep's first position on, so a sweep over consecutive chunks is
// the sequential parse of that stretch: serial ripples (the position phase of the sparse search running through
// incompressible data, a distance-cache change flowing through match-free data) cost one launch per input block, not
// one launch per chunk.
//
// A forced launch (BrStream::forced): the walker of the first scheduled chunk runs to the end of its input block
// (`to_block_end`) through every chunk behind it, so the walkers scheduled behind it in that block stand down.  Were they to
// walk too, those chunks would be walked twice in one launch by walkers that share one chunk record (bout, bin_used,
// cmd_blocks) and, at equal head parity, one bits_cur bitmap: each walk would read the other's fresh stored-bits as its own,
// the commit would store their union, and the fixpoint could settle on bits no walk of the chunk produced (DESIGN.md
// section 3).  So every chunk is walked at most once per launch, and a launch appends at most nblocks entries to ran_list.
//
// The chunk records of the walk (br_walk_one) are kept in the warp's shared memory on the GPU: every lane writes the same
// values, and a warp barrier lies between a record's last read and the next write over it.
#define BR_WALK_WARPS 4   /* warps per block of k_walk */
struct BrWalkRecs { BrBlockIn in, ni, used; BrBlockOut o; };
template <int F, bool M = false>
BR_DEV void br_walk_block(const BrStream& s, u32 b, bool to_block_end) {
  if (s.forced && !to_block_end && s.bin[b].blk == s.bin[s.counters[6]].blk) return;
#if BR_GPU
  __shared__ BrWalkRecs recs[BR_WALK_WARPS];
  BrWalkRecs& R = recs[threadIdx.x >> 5];
#else
  BrWalkRecs R;
#endif
  BrBlockIn& in = R.in;
  BrBlockIn& ni = R.ni;
  BrBlockOut& o = R.o;
  in = s.bin[b];
  const u32 head = b;
  u32 sweep_p0 = 0xffffffffu;
  for (;;) {
    br_walk_one<F, M>(s, b, in, o, head, sweep_p0, &R.used);
    if (br_lane() == 0) br_atomic_max((int*)s.counters + 16, (int)(b - head + 1));   // longest sweep of this launch (diagnostic)
    const u32 nb = b + 1;
    if (in.last) {
      // block boundary: crossed by the sweeps of a sweep-mode launch, inside a group of sweep_blocks blocks
      const bool full_sweep = s.epoch > s.P.sweep_epoch + 9 && (s.epoch - 1 - s.P.sweep_epoch) % 3 == 0;   // (as br_chain_c decided it)
      if (to_block_end || in.is_last || nb >= s.P.nblocks || s.epoch <= s.P.sweep_epoch || full_sweep || ((in.blk + 1) & (s.P.sweep_blocks - 1u)) == 0) return;
      const bool crossed = br_predict_next_block(s, b, in, o, ni);
#ifdef BR_SIM_DEBUG
      ++br_sim_bnd[crossed ? 0 : 1];
#endif
      if (!crossed) return;
    } else {
      ni = s.bin[nb];
      ni.start_pos = o.out_pos; ni.apply_rh = o.apply_rh; ni.store_end = o.store_end; ni.ext_dist = 0; ni.warm = 0;
      for (int i = 0; i < 4; ++i) ni.dc[i] = o.dc[i];
    }
    const u32 df = s.dirty[nb];
    bool go = to_block_end;
    if (!go) {
      if (df != 0 && !(df & BR_DEFER)) return;   // scheduled: another walker runs it in this launch
      go = (df & BR_DEFER_FULL) != 0;   // (BR_DEFER_STATE / BR_DEFER_SWEEP: only if the state differs, below)
    }
    const u64 dl = (((u64)in.dict_l_hi << 32) | in.dict_l_lo) + o.dl, dm = (((u64)in.dict_m_hi << 32) | in.dict_m_lo) + o.dm;   // (a closed gate reports dl = dm = 0)
    if (!go && !s.bout[nb].valid) { if (!(df & BR_DEFER)) return; go = true; }   // (a deferred chunk that never ran)
    if (!go) {
      const BrBlockIn u = s.bin_used[nb];
      bool same = u.start_pos == ni.start_pos && u.apply_rh == ni.apply_rh && u.store_end == ni.store_end && u.ext_dist == ni.ext_dist &&
                  u.dc[0] == ni.dc[0] && u.dc[1] == ni.dc[1] && u.dc[2] == ni.dc[2] && u.dc[3] == ni.dc[3];
      if (same) {
        const BrBlockOut uo = s.bout[nb];
        const u64 ul = ((u64)u.dict_l_hi << 32) | u.dict_l_lo, um = ((u64)u.dict_m_hi << 32) | u.dict_m_lo;
        u32 edl, edm;
        if (ul != dl || um != dm) same = br_dict_gate_valid(dl, dm, uo.dl, uo.dm, uo.gate_checks, uo.gate_fail, &edl, &edm, s.P.quick ? 1u : 2u) != 0;
      }
      if (same) return;
    }
    ni.dict_l_lo = (u32)dl; ni.dict_l_hi = (u32)(dl >> 32); ni.dict_m_lo = (u32)dm; ni.dict_m_hi = (u32)(dm >> 32);
    if (in.last && ni.blk_end - ni.blk_start >= s.P.htl - 1 && ni.blk_start - ni.base >= 3) {
      // StitchToPreviousBlock (hash_longest_match64_inc.h:127) of the block the sweep enters: the last three positions of
      // the block it leaves.  br_commit_bits adds them for their owner; the sweep reads its own bitmap from sweep_p0 on.
      u32* own = s.bits_cur + (size_t)(head & 1u) * s.bits_words;
      if (br_lane() == 0)
        for (u32 q = ni.blk_start - 3; q < ni.blk_start; ++q) if (q >= sweep_p0) br_atomic_or(own + (q >> 5), 1u << (q & 31));
#if BR_GPU
      __threadfence_block();
#endif
      br_syncwarp();
    }
    br_syncwarp();
    in = ni; b = nb;
    br_syncwarp();
  }
}
