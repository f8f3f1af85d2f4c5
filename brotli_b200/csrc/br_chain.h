// br_chain.h -- the serial glue of one stream: replays what EncodeData (c/enc/encode.c:985)
// does between input blocks -- carrying distance cache / pending literals / dictionary counters,
// ExtendLastCommand eligibility, the merge-or-flush policy (encode.c:1141-1166), ShouldCompress
// (encode.c:457) -- over the walkers' per-chunk summaries, and hands every chunk the state it must
// start from.  Inside an input block the state simply flows from one chunk to the next.  It also
// decides which chunks must be re-run: a chunk is dirty when the state it consumed differs from the
// state the chain now derives for it, or when stored-bits it may have consulted were changed by a
// later commit.
#pragma once
#include "br_cmd.h"
#include "br_lz77.h"
#ifdef BR_SIM_DEBUG
#include <stdio.h>
static u32 br_sim_watch = 0xffffffffu;   // tests/sim: report commits that flip this position
static u64 br_sim_cnt[8];                // tests/sim: marks by source (0 successor, 1 overlap, 2 cap hits, 3 flips, 4 steps)
#endif

// First byte of the stream that holds position p (0 unless the job is a batch of streams, BrParams::multi).
BR_DEV u32 br_stream_base_of(const BrStream& s, u32 p) {
  if (!s.P.multi) return 0u;
  u32 b = s.slot_blk[p >> s.P.lgblock];
  while (p >= s.blk[b].end) ++b;
  return s.blk[b].base;
}
// Chunk whose nominal slice holds position p.  Input blocks are at most 1 << lgblock bytes long but need not be aligned
// (a FLUSH cuts one short): slot_blk gives the block at the aligned position below p, a short scan finds p's block.
BR_DEV u32 br_chunk_of(const BrStream& s, u32 p) {
  u32 b = s.slot_blk[p >> s.P.lgblock];
  while (p >= s.blk[b].end) ++b;
  return s.blk[b].first_chunk + ((p - s.blk[b].start) >> s.P.chunk_bits);
}

// Initial speculation for input block bi: every hashable position of the block is stored (true for > 99.8 % of text
// positions, SURVEY.md appendix E).  Lane `lane` of `stride` ORs its words of the block into a zeroed bits_latest (words
// shared by two blocks are ORed by both).
BR_DEV void br_init_bits(const BrStream& s, u32 bi, u32 lane, u32 stride) {
  const BrBlk B = s.blk[bi];
  const u32 htl = s.P.htl;
  // positions of this block that the parse stores: those with a full hash load inside the block ...
  u32 lo = B.start, hi = B.end - B.start >= htl ? B.end - htl + 1 : B.start;
  // ... and the last three, stored by StitchToPreviousBlock of the next block (hash_longest_match64_inc.h:127)
  u32 s_lo = 0, s_hi = 0;
  if (bi + 1 < s.nblk) {
    const BrBlk N = s.blk[bi + 1];
    if (N.end - N.start >= htl - 1 && N.start >= 3) { s_lo = N.start - 3 > B.start ? N.start - 3 : B.start; s_hi = N.start; }
  }
  const u32 w0 = B.start >> 5, w1 = (B.end - 1) >> 5;
  for (u32 wi = w0 + lane; wi <= w1; wi += stride) {
    u32 v = 0;
    for (u32 b = 0; b < 32; ++b) {
      const u32 p = wi * 32 + b;
      if ((p >= lo && p < hi) || (p >= s_lo && p < s_hi)) v |= 1u << b;
    }
    if (v) br_atomic_or(s.bits_latest + wi, v);
  }
}

// Compare and commit the stored-bits a walker just produced for chunk k (warp task).  The
// walker owns the positions [start_pos, out_pos).  StitchToPreviousBlock of the FOLLOWING input
// block (hash_longest_match64_inc.h:127) stores the last three positions of a block after its
// parse; that set is static, so it is added here, by whoever owns those positions.
// Marks the positions [start_pos, out_pos) of run k in cover_cur (warp task; runs before the commits of the launch).
BR_DEV void br_cover_run(const BrStream& s, u32 k) {
  const u32 a = s.bin_used[k].start_pos, b = s.bout[k].out_pos;
  if (b <= a) return;
  const u32 w0 = a >> 5, w1 = (b - 1) >> 5;
  for (u32 x = w0 + (u32)br_lane(); x <= w1; x += BR_WARP) {
    u32 m = 0xffffffffu;
    if (x == w0) m &= 0xffffffffu << (a & 31);
    if (x == w1) m &= 0xffffffffu >> (31 - ((b - 1) & 31));
    br_atomic_or(s.cover_cur + x, m);
  }
}
BR_DEV void br_commit_bits(const BrStream& s, u32 k) {
  const BrBlockIn in = s.bin_used[k];
  const u32 a = in.start_pos, b = s.bout[k].out_pos;
  u32 diff = 0;
  // Ranges of different runs must not overlap: where they do, one of the two runs is stale (it started
  // from a guessed position, or a predecessor's last copy / ExtendLastCommand reaches into it), the later
  // commit overwrites the earlier one, and two runs of the same parity in one launch even share their
  // bits_cur bitmap.  The stale run is walked again anyway (its in-state changes); the other one is not --
  // so every chunk whose latest range intersects mine is told to walk again.  Ranges of one input block
  // are disjoint at the fixpoint, so this stops.
  if (b > a) {
    const u32 k0 = s.blk[in.blk].first_chunk, k1 = k0 + s.blk[in.blk].nchunks;
    for (u32 c = k0 + (u32)br_lane(); c < k1; c += BR_WARP) {
      if (c == k || !s.bout[c].valid) continue;
      const u32 ca = s.bin_used[c].start_pos, cb = s.bout[c].out_pos;
      if (ca < cb && ca < b && a < cb) {
        br_atomic_max(s.bitdep_epoch + c, (int)s.epoch);
#ifdef BR_SIM_DEBUG
        ++br_sim_cnt[1];
#endif
      }
    }
  }
  const u32* mine = s.bits_cur + (size_t)(s.bout[k].own_par & 1u) * s.bits_words;
  const u32 my_head = s.bout[k].head;
  const u32 send = s.blk[in.blk].send;   // (batch of streams: nobody behind the end of my stream looks at my positions)
  if (b > a) {
    // stitch positions inside [a, b): the next block(s) starting at or shortly after blk_end
    u32 st_lo = 0, st_hi = 0;   // [st_lo, st_hi) of stitch-stored positions (at most one run here)
    // (any owner of one of the block's last three positions, not only the block's last chunk: a copy
    // that runs to the block end makes an earlier chunk the owner)
    if (b + 3 > in.blk_end) {
      for (u32 nb = k + 1; nb < s.P.nblocks; ++nb) {
        if (!s.bin[nb].first) continue;
        u32 np = s.bin[nb].blk_start, ne = s.bin[nb].blk_end;
        if (np >= in.blk_end + 3) break;
        // (a block shorter than HashTypeLength - 1 does not stitch -- a FLUSH one or two bytes behind a block boundary makes
        // such a block -- but the block behind it may, and its three positions then reach back into this one)
        if (ne - np >= s.P.htl - 1 && np - s.bin[nb].base >= 3) { st_lo = np - 3; st_hi = np; break; }
      }
    }
    u32 w0 = a >> 5, w1 = (b - 1) >> 5;
    for (u32 x = w0 + (u32)br_lane(); x <= w1; x += BR_WARP) {
      u32 m = 0xffffffffu;
      if (x == w0) m &= 0xffffffffu << (a & 31);
      if (x == w1) m &= 0xffffffffu >> (31 - ((b - 1) & 31));
      u32 nv = mine[x];
      for (u32 q = st_lo; q < st_hi; ++q) if ((q >> 5) == x) nv |= 1u << (q & 31);
      nv &= m;
      u32 ov = s.bits_latest[x] & m;
      u32 flips = nv ^ ov;
      {  // searched-positions bitmap of this run
        u32 sv = s.srch_cur[x] & m, so = s.srch_latest[x] & m;
        if (sv != so) {
          if (m == 0xffffffffu) s.srch_latest[x] = sv;
          else { br_atomic_and(s.srch_latest + x, ~m); br_atomic_or(s.srch_latest + x, sv); }
        }
      }
      diff += (u32)br_popc(flips);
#ifdef BR_SIM_DEBUG
      if (br_sim_watch != 0xffffffffu && (br_sim_watch >> 5) == x && ((flips >> (br_sim_watch & 31)) & 1))
        fprintf(stderr, "watch %u: epoch %u chunk %u range [%u,%u) flips it to %u\n", br_sim_watch, s.epoch, k, a, b,
                (nv >> (br_sim_watch & 31)) & 1);
#endif
      if (flips) {
        if (m == 0xffffffffu) s.bits_latest[x] = nv;
        else { br_atomic_and(s.bits_latest + x, ~m); br_atomic_or(s.bits_latest + x, nv); }
        // Who may have consulted a flipped bit?  Position q sits in the bucket ring seen from a later
        // position p of the same key until block_size stored positions lie between them.
        const u32 reach = (1u << s.P.block_bits) + 2;
        if (s.P.quick) flips = 0;   // qualities 2..4: every run is checked against the committed bits instead (br_verify_run)
        while (flips) {
          const u32 q = (x << 5) + (u32)br_ffs(flips) - 1u;
          flips &= flips - 1;
          const u32 jq = s.rank[q];
#ifdef BR_SIM_DEBUG
          ++br_sim_cnt[3];
#endif
          const u16 key = s.skeys[jq];
          if (s.seg[key + 1] - s.seg[key] >= s.P.heavy_min) br_atomic_add(s.key_flips + key, 1);   // uint16 bucket counter may wrap
          // cnt: stored (snapshot the walkers read) strictly between q and pp -> is q inside pp's view
          u32 cnt = 0, steps = 0;
          for (u32 j = jq + 1; j < s.P.n && s.skeys[j] == key && cnt < reach; ++j) {
#ifdef BR_SIM_DEBUG
            ++br_sim_cnt[4];
#endif
            if (++steps > s.P.step_cap) {
#ifdef BR_SIM_DEBUG
              ++br_sim_cnt[2];
#endif  // pathological bucket (long runs of unstored positions): give up precision,
              br_atomic_max(&s.blk[in.blk].changed_epoch, (int)s.epoch);   // block-level window rule (br_chain_c)
              break;
            }
            const u32 pp = s.S[j];
            if (pp - q > s.P.max_backward || pp >= send) break;
            {
              // A position shields q from pp only if it is stored in EVERY view a dependent run may have had: the snapshot
              // before this launch and, where a run of this launch covers it, that run's fresh bits (a walker reads its
              // own bits inside its range: a stretch it has just left unstored lets its searches see further back than
              // the snapshot count says -- into a range that flips in the same launch; fuzz case (35, 22)).
              const u32 wi = pp >> 5, sh = pp & 31;
              const u32 prev = (s.bits_prev[wi] >> sh) & 1u, cov = (s.cover_cur[wi] >> sh) & 1u;
              const u32 cur = ((s.bits_cur[wi] | s.bits_cur[s.bits_words + wi]) >> sh) & 1u;
              if (prev && (!cov || cur)) ++cnt;
            }
            if (pp >= a && pp < b) continue;            // my own run is consistent with my own bits
            if (!(((s.srch_cur[pp >> 5] | s.srch_latest[pp >> 5]) >> (pp & 31)) & 1)) continue;   // never searched there
            u32 c = br_chunk_of(s, pp);
#ifdef BR_SIM_DEBUG
            ++br_sim_cnt[0];
#endif
            // (its owner may be the chunk before.)  Not marked: this run itself, and the runs that the same walker
            // made AFTER this one in this launch -- a sweep reads its own fresh bits (br_walk_block).
            for (u32 xc = c > 0 ? c - 1 : 0; xc <= c; ++xc) {
              if (xc == k) continue;
              if (xc > k && s.bout[xc].valid && s.bout[xc].epoch == s.epoch && s.bout[xc].head == my_head) continue;
              br_atomic_max(s.bitdep_epoch + xc, (int)s.epoch);
            }
          }
        }
      }
    }
  }
  diff = br_warp_sum(diff);
  if (br_lane() == 0) {
    s.changed_bits[k] = diff;
    if (diff) s.changed_epoch[k] = (int)s.epoch;
  }
}

// Qualities 5..9: carries the commits of a launch into the S-ordered snapshot the walkers read.  Between launches storedS
// is bits_latest permuted into S order and cntS[b] counts its set bits in [1024 b, 1024 b + 1024) (prefS is the exclusive
// scan of cntS).  bits_latest changes only in br_commit_bits, against the copy bits_prev taken before the commits, so the
// bits q of word x that differ from bits_prev are exactly the entries rank[q] of storedS to flip.
BR_DEV void br_snapshot_update(const BrStream& s, u32 x, u32* storedS, u32* cntS) {
  u32 f = s.bits_latest[x] ^ s.bits_prev[x];
  while (f) {
    const u32 j = s.rank[(x << 5) + (u32)br_ffs(f) - 1u];
    f &= f - 1;
    const u32 b = 1u << (j & 31);
    const u32 old = br_atomic_xor(storedS + (j >> 5), b);
    br_atomic_add(cntS + (j >> 10), (old & b) ? 0xFFFFFFFFu : 1u);
  }
}

// Qualities 2..4 (BrParams::quick): is the latest run of chunk k consistent with the committed stored-bits?  A slot of the
// reference's table holds one position, so the run recorded what every search read from each slot (BrStream::saw,
// br_find_quick): the index in S of the stored position it took, or BR_SAW_ABSENT | the index its backward walk
// stopped at (everything in front of that index lies outside the window).  The record still holds iff that position is
// stored and nothing between it and the search position is.  Runs after the commits of every launch, over ALL chunks:
// a run that read a bit another run flipped -- in this launch or any earlier one -- is walked again (reason 4).  This
// is an exact check, not a conservative marking: no successor counting, no view mismatch (DESIGN.md section 3).
// Warp task; the lanes take the words of the run's range independently and meet in one ballot at the end.
BR_DEV void br_verify_run(const BrStream& s, u32 k) {
  const BrParams& P = s.P;
  const BrBlockOut o = s.bout[k];
  const u32 a = s.bin_used[k].start_pos, b = o.out_pos;
  u32 bad = 0;
  if (o.valid && b > a) {
    const u32 sweep = 1u << P.qk_sweep_bits, mask = (1u << P.qk_bits) - 1u;
    const u32 w0 = a >> 5, w1 = (b - 1) >> 5;
    for (u32 x = w0 + (u32)br_lane(); x <= w1 && !bad; x += BR_WARP) {
      u32 m = s.srch_latest[x];
      if (x == w0) m &= 0xffffffffu << (a & 31);
      if (x == w1) m &= 0xffffffffu >> (31 - ((b - 1) & 31));
      while (m && !bad) {
        const u32 p = (x << 5) + (u32)br_ffs(m) - 1u;
        m &= m - 1;
        const u32 key = br_quick_key_v(P, br_ld64u(s.data, p));
        const u32* saw = s.saw + ((size_t)p << P.qk_sweep_bits);
        for (u32 i = 0; i < sweep && !bad; ++i) {
          const u32 v = saw[i];
          if (v == BR_SAW_SKIP) continue;
          const u32 hi = s.seg[((key + (i << 3)) & mask) + 1];
          u32 j = v & ~BR_SAW_ABSENT;
          if (j > hi) { bad = 1; break; }
          if (!(v & BR_SAW_ABSENT)) {
            if (j >= hi) { bad = 1; break; }
            const u32 q = s.S[j];
            if (q >= p || !((s.bits_latest[q >> 5] >> (q & 31)) & 1u)) { bad = 1; break; }
            ++j;
          }
          for (; j < hi; ++j) {
            const u32 q = s.S[j];
            if (q >= p) break;
            if ((s.bits_latest[q >> 5] >> (q & 31)) & 1u) { bad = 1; break; }
          }
        }
      }
    }
  }
  if (br_ballot(bad != 0) != 0 && br_lane() == 0) br_atomic_max(s.bitdep_epoch + k, (int)s.epoch);
}

// encode.c:457 ShouldCompress
BR_DEV int br_should_compress(const BrStream& s, u32* h, u32 start, u32 bytes, u32 num_literals, u32 num_commands) {
  if (bytes <= 2) return 0;
  if (num_commands < (bytes >> 8) + 2) {
    if ((double)num_literals > br_dmul(0.99, (double)bytes)) {
      for (u32 i = (u32)br_lane(); i < 256; i += BR_WARP) h[i] = 0;
      br_syncwarp();
      u32 t = (bytes + 12) / 13;
      for (u32 i = (u32)br_lane(); i < t; i += BR_WARP) br_atomic_add(h + s.data[start + 13 * i], 1);
#if BR_GPU
      __threadfence_block();
#endif
      br_syncwarp();
      const double thr = br_dmul(br_dmul((double)bytes, 7.92), 1.0 / 13.0);
      if (br_bits_entropy(s, h, 256) > thr) return 0;
    }
  }
  return 1;
}

// ---- The chain, three kernels per walker launch ------------------------------------------
//   br_chain_a  (thread per input block)  state flow through the block's chunks + aggregates
//   br_chain_b  (one warp)                block-to-block recurrence of encode.c:985
//   br_chain_c  (thread per input block)  final in-state of every chunk, dirty decision, offsets

BR_DEV void br_chain_a(const BrStream& s, u32 bi) {
  const BrParams& P = s.P;
  BrBlk B = s.blk[bi];
  u32 ncmd = 0, nlit_rel = 0, has_cmd = 0, lil_run = 0, lil_head = 0, last_cmd_chunk = 0, dl = 0, dm = 0;
  u32 flow_pos = 0, flow_rh = 0, flow_se = 0; int fdc[4] = {0, 0, 0, 0};
  bool all_valid = true;
  for (u32 c = 0; c < B.nchunks; ++c) {
    const u32 k = B.first_chunk + c;
    const BrBlockOut out = s.bout[k];
    s.ext_total[k] = 0;
    if (c > 0) {
      BrBlockIn ni = s.bin[k];
      ni.start_pos = flow_pos; ni.apply_rh = flow_rh; ni.store_end = flow_se; ni.ext_dist = 0;
      for (int i = 0; i < 4; ++i) ni.dc[i] = fdc[i];
      ni.warm = out.valid ? 0u : (u32)BR_WARM_BYTES;
      s.bin[k] = ni;
    }
    // pending literals relative to the block start (true value = + block lil_in while no command seen)
    s.lil_in[k] = lil_run | (has_cmd ? 0u : 0x80000000u);
    if (out.valid) {
      if (out.ncmd > 0) {
        nlit_rel += out.nlit + lil_run;
        if (!has_cmd) lil_head = lil_run;
        has_cmd = 1; lil_run = out.last_insert_len; last_cmd_chunk = k;
      } else lil_run += out.last_insert_len;
      ncmd += out.ncmd; dl += out.dl; dm += out.dm;
      flow_pos = out.out_pos; flow_rh = out.apply_rh; flow_se = out.store_end;
      for (int i = 0; i < 4; ++i) fdc[i] = out.dc[i];
    } else {
      // never ran: pretend it emitted nothing and stopped at its nominal end
      all_valid = false;
      const BrBlockIn cur = s.bin[k];
      u32 sp = c == 0 ? cur.blk_start : cur.start_pos;
      u32 from = sp > cur.pos ? sp : cur.pos, to = cur.last ? cur.blk_end : cur.end;
      if (to > from) lil_run += to - from;
      flow_pos = to > from ? to : sp; flow_rh = flow_pos + P.spree;
      flow_se = cur.blk_end - cur.blk_start >= P.htl ? cur.blk_end - P.htl + 1 : cur.blk_start;
      if (c == 0) { fdc[0] = 4; fdc[1] = 11; fdc[2] = 15; fdc[3] = 16; if (P.stream_offset) fdc[0] = fdc[1] = fdc[2] = fdc[3] = -16; }
    }
  }
  B.ncmd = ncmd; B.nlit_rel = nlit_rel; B.has_cmd = has_cmd; B.lil_head = lil_head; B.lil_tail = lil_run;
  B.last_cmd_chunk = last_cmd_chunk; B.dl = dl; B.dm = dm; B.valid = all_valid ? 1u : 0u;
  B.ext_len = 0;
  if (s.bout[B.first_chunk].valid && s.bin_used[B.first_chunk].ext_dist) B.ext_len = s.bout[B.first_chunk].ext_len;
  for (int i = 0; i < 4; ++i) B.out_dc[i] = fdc[i];
  B.lc_copy_len = B.lc_dist_prefix = B.lc_dist_extra = 0;
  if (has_cmd) {
    const BrCmd c = s.cmd_blocks[(size_t)last_cmd_chunk * s.cmd_stride + s.bout[last_cmd_chunk].ncmd - 1];
    B.lc_copy_len = c.copy_len; B.lc_dist_prefix = c.dist_prefix; B.lc_dist_extra = c.dist_extra;
  }
  s.blk[bi] = B;
}

BR_DEV void br_chain_prologue(const BrStream& s) {
  const BrParams& P = s.P;
  const u32 t_now = s.epoch;
  const int lane = br_lane();
  // counter-wrap rule: per launch, the largest number of stored-bit flips any single (heavy) bucket saw
  {
    u32 mx = 0;
    if (!P.quick)   // (no bucket counters in the one-position-per-slot hashers of quality 2..4, and up to 2^20 slots)
    for (u32 k = (u32)lane; k <= P.nbuckets; k += BR_WARP) { u32 v = s.key_flips[k]; if (v > mx) mx = v; s.key_flips[k] = 0; }
    mx = br_warp_max(mx);
    if (lane == 0) {
      if (t_now <= P.max_epochs) {   // (the chain runs again for the same launch when a metablock falls back late)
        if (s.counters[7] == t_now + 1) s.epoch_cum[t_now] += mx;
        else { s.epoch_cum[t_now] = (t_now ? s.epoch_cum[t_now - 1] : 0u) + mx; s.counters[7] = t_now + 1; }
      }
      s.counters[0] = 0; s.counters[5] = 0; s.counters[6] = 0xffffffffu; s.counters[17] = 0; s.counters[18] = 0;
      for (int i = 8; i < 16; ++i) s.counters[i] = 0;
    }
  }
}

// The block-to-block recurrence over the input blocks [bi0, bi1) (a whole stream: every stream of a batch is independent of
// the others).  Command offsets (BrBlkIn::cmd_base, BrMetaBlock::cmd_off) and metablock numbers (BrBlkIn::mb) count from
// the first block of the range; metablock records go to mbs_out[0..].  hist: 256 words of scratch (br_should_compress).
BR_DEV void br_chain_blocks(const BrStream& s, u32 bi0, u32 bi1, BrMetaBlock* mbs_out, u32* hist, u32* n_mbs_out, u32* cmd_total_out,
                            u32* dbg_slow_out) {
  const BrParams& P = s.P;
  const int lane = br_lane();
  u32 num_cmds = 0, num_lits = 0, last_insert_len = 0;
  int dc[4] = {4, 11, 15, 16}, saved_dc[4] = {4, 11, 15, 16};
  if (P.stream_offset) for (int i = 0; i < 4; ++i) dc[i] = saved_dc[i] = -16;   // encode.c:656: poisoned distance cache
  u32 last_flush_pos = s.blk[bi0].start, first_blk = bi0, cmd_total = 0, n_mbs = 0;
  u64 dict_l = 0, dict_m = 0;
  bool have_last = false;
  u32 lc_copy_len = 0, lc_dist_prefix = 0, lc_dist_extra = 0, lc_chunk = 0, first_blk_chunk = 0, first_blk_cmd_base = 0;
  u32 dbg_slow = 0;
  bool mb_valid = true;
  const u32 blocksize = 1u << P.lgblock;
  // The recurrence is serial, but its loads need not be: every lane fetches the summary of one of the next BR_WARP
  // blocks, and the loop takes them out of the lanes' registers with shuffles (the loop-carried state is in registers
  // only, so a block costs arithmetic latency instead of a memory round trip).
  BrBlk mine; memset(&mine, 0, sizeof(mine));
  for (u32 bi = bi0; bi < bi1; ++bi) {
    if (((bi - bi0) % BR_WARP) == 0) { const u32 mi = bi + (u32)lane; if (mi < bi1) mine = s.blk[mi]; }
    BrBlk B;
    {
      const int src = (int)((bi - bi0) % BR_WARP);
      B.start = br_shfl(mine.start, src); B.end = br_shfl(mine.end, src); B.first_chunk = br_shfl(mine.first_chunk, src);
      B.nchunks = br_shfl(mine.nchunks, src); B.is_last = br_shfl(mine.is_last, src); B.force_flush = br_shfl(mine.force_flush, src);
      B.ncmd = br_shfl(mine.ncmd, src); B.nlit_rel = br_shfl(mine.nlit_rel, src); B.has_cmd = br_shfl(mine.has_cmd, src);
      B.lil_head = br_shfl(mine.lil_head, src); B.lil_tail = br_shfl(mine.lil_tail, src); B.last_cmd_chunk = br_shfl(mine.last_cmd_chunk, src);
      B.dl = br_shfl(mine.dl, src); B.dm = br_shfl(mine.dm, src); B.ext_len = br_shfl(mine.ext_len, src); B.valid = br_shfl(mine.valid, src);
      for (int i = 0; i < 4; ++i) B.out_dc[i] = br_shfl(mine.out_dc[i], src);
      B.lc_copy_len = br_shfl(mine.lc_copy_len, src); B.lc_dist_prefix = br_shfl(mine.lc_dist_prefix, src); B.lc_dist_extra = br_shfl(mine.lc_dist_extra, src);
      B.changed_epoch = br_shfl(mine.changed_epoch, src); B.state_dirty = br_shfl(mine.state_dirty, src);
      B.base = br_shfl(mine.base, src); B.send = br_shfl(mine.send, src);
    }
    if (bi > bi0 && B.start == B.base) {
      // a new stream of the batch begins (the block before carried is_last, so nothing is pending): fresh encoder state
      for (int i = 0; i < 4; ++i) dc[i] = saved_dc[i] = (i == 0 ? 4 : i == 1 ? 11 : i == 2 ? 15 : 16);
      dict_l = dict_m = 0; last_insert_len = 0; have_last = false;
    }
    u32 ext_dist = 0;
    if (num_cmds > 0 && last_insert_len == 0 && have_last) {
      u32 dcode = br_cmd_restore_dcode(lc_dist_prefix, lc_dist_extra);
      int cmd_dist = dc[0];
      if (dcode < 16 || (cmd_dist > 0 && dcode - 15 == (u32)cmd_dist)) {
        u32 lpp = B.start - (lc_copy_len & 0x1FFFFFF);
        u32 maxd = br_min(lpp - B.base, P.max_backward);
        if (cmd_dist > 0 && (u32)cmd_dist <= maxd) ext_dist = (u32)cmd_dist;
      }
    }
    if (lane == 0) {
      BrBlkIn W;
      for (int i = 0; i < 4; ++i) W.in_dc[i] = dc[i];
      W.in_ext_dist = ext_dist; W.lil_in = last_insert_len;
      W.dict_l_lo = (u32)dict_l; W.dict_l_hi = (u32)(dict_l >> 32);
      W.dict_m_lo = (u32)dict_m; W.dict_m_hi = (u32)(dict_m >> 32);
      W.cmd_base = cmd_total; W.mb = n_mbs;
      s.blkin[bi] = W;
    }
    if (bi == first_blk) { first_blk_chunk = B.first_chunk; first_blk_cmd_base = cmd_total; mb_valid = true; }
    if (!B.valid) mb_valid = false;
    // carry on with the block's latest (possibly stale) summary
    if (B.ext_len && have_last && ext_dist) {
      lc_copy_len += B.ext_len;
      if (lane == 0) s.ext_total[lc_chunk] += B.ext_len;
    }
    if (B.has_cmd) {
      lc_copy_len = B.lc_copy_len; lc_dist_prefix = B.lc_dist_prefix; lc_dist_extra = B.lc_dist_extra;
      lc_chunk = B.last_cmd_chunk; have_last = true;
      num_lits += B.nlit_rel + last_insert_len;
      last_insert_len = B.lil_tail;
    } else last_insert_len += B.lil_tail;
    num_cmds += B.ncmd;
    for (int i = 0; i < 4; ++i) dc[i] = B.out_dc[i];
    // dictionary counters: chunk by chunk only around the (single) point where the gate closes
    if (!(dict_m < (dict_l >> 7))) {
      if (dict_m >= ((dict_l + B.dl) >> 7)) { dict_l += B.dl; dict_m += B.dm; }
      else {
        ++dbg_slow;
        for (u32 c = 0; c < B.nchunks; ++c) {
          const BrBlockOut o = s.bout[B.first_chunk + c];
          if (!o.valid || dict_m < (dict_l >> 7)) continue;
          u32 edl = o.dl, edm = o.dm;
          const BrBlockIn u = s.bin_used[B.first_chunk + c];
          const u64 ul = ((u64)u.dict_l_hi << 32) | u.dict_l_lo, um = ((u64)u.dict_m_hi << 32) | u.dict_m_lo;
          if (ul != dict_l || um != dict_m) {
            if (!br_dict_gate_valid(dict_l, dict_m, o.dl, o.dm, o.gate_checks, o.gate_fail, &edl, &edm, s.P.quick ? 1u : 2u)) { edl = o.dl; edm = o.dm; }
          }
          dict_l += edl; dict_m += edm;
        }
      }
    }
    cmd_total += B.ncmd;
    bool closes_stream = false, empty_last = false;
    // merge-or-flush (encode.c:1141)
    const u32 end = B.end;
    {
      const u32 processed = end - last_flush_pos;
      const bool next_fits = processed + blocksize <= P.max_mb;
      // (encode.c:1152: without block splitting -- qualities 2, 3 -- at most MAX_NUM_DELAYED_SYMBOLS literals + commands are buffered)
      const bool should_flush = P.mb_kind != 0 && num_lits + num_cmds >= 0x2FFFu;
      if (!B.is_last && !B.force_flush && !should_flush && next_fits && num_lits < P.max_mb / 8 && num_cmds < P.max_mb / 8) {
        if (!(P.finish_empty && bi + 1 == s.nblk)) continue;
        closes_stream = true;    // merged, and the FINISH call that brought nothing flushes it as the last metablock
      } else if (P.finish_empty && bi + 1 == s.nblk) empty_last = true;
    }
    u32 tail = 0;
    if (last_insert_len > 0) { tail = last_insert_len; ++num_cmds; num_lits += tail; last_insert_len = 0; ++cmd_total; }
    const u32 bytes = end - last_flush_pos;
    // (summaries of chunks that never ran are placeholders: do not sample the input for them)
    int compress = mb_valid ? br_should_compress(s, hist, last_flush_pos, bytes, num_lits, num_cmds) : 1;
    if (compress && s.force_unc[first_blk_chunk]) compress = 0;   // (late fallback of an earlier round: br_assemble_scan)
    if (!compress) for (int i = 0; i < 4; ++i) dc[i] = saved_dc[i];
    if (lane == 0) {
      BrMetaBlock m;
      m.start = last_flush_pos; m.end = end;
      m.first_block = first_blk_chunk; m.last_block = B.first_chunk + B.nchunks - 1;
      m.cmd_off = first_blk_cmd_base; m.ncmd = num_cmds; m.nlit = num_lits;
      m.is_last = (B.is_last || closes_stream) ? 1u : 0u; m.compress = (u32)compress;
      m.prev_byte = last_flush_pos > B.base ? s.data[last_flush_pos - 1] : 0;
      m.prev_byte2 = last_flush_pos > B.base + 1 ? s.data[last_flush_pos - 2] : 0;
      m.base = B.base;
      m.flushed = (u8)B.force_flush; m.empty_last = empty_last ? 1 : 0; m.tail_insert = tail; m.out_bits = 0; m.scratch_off = 0;
      mbs_out[n_mbs] = m;
    }
    br_syncwarp();
    ++n_mbs;
    last_flush_pos = end; num_cmds = 0; num_lits = 0; have_last = false; first_blk = bi + 1;
    for (int i = 0; i < 4; ++i) saved_dc[i] = dc[i];
  }
  *n_mbs_out = n_mbs; *cmd_total_out = cmd_total; *dbg_slow_out = dbg_slow;
}

// one stream: the whole recurrence in one warp
BR_DEV void br_chain_b(const BrStream& s) {
#if BR_GPU
  long long t_begin = clock64();
#endif
  br_chain_prologue(s);
  br_syncwarp();
#if BR_GPU
  long long t_phase0 = clock64();
#endif
  u32 n_mbs, cmd_total, dbg_slow;
  br_chain_blocks(s, 0, s.nblk, s.mbs, s.hist_scratch, &n_mbs, &cmd_total, &dbg_slow);
  if (br_lane() == 0) {
    s.counters[1] = n_mbs; s.counters[2] = cmd_total;
#if BR_GPU
    long long t_end = clock64();
    s.counters[20] = (u32)((t_phase0 - t_begin) >> 10); s.counters[21] = (u32)((t_end - t_phase0) >> 10); s.counters[22] = dbg_slow;
#endif
  }
}
// A batch of streams (BrParams::multi): the recurrence runs per stream, a warp each (b1); metablock numbers and command
// offsets are made global by a scan over the streams' totals (b2) and added to what b1 left (b3, thread per input block).
BR_DEV void br_chain_b1(const BrStream& s, u32 st) {
  const u32 fb = s.stream_blk[st], lb = s.stream_blk[st + 1];
  u32 n_mbs, cmd_total, dbg_slow;
  br_chain_blocks(s, fb, lb, s.mbs_stage + fb, s.hist_scratch + 256u * st, &n_mbs, &cmd_total, &dbg_slow);
  if (br_lane() == 0) { s.stream_nmb[st] = n_mbs; s.stream_ncmd[st] = cmd_total; }
}
BR_DEV void br_chain_b2(const BrStream& s) {   // one warp
  br_chain_prologue(s);
  br_syncwarp();
  const u32 ns = s.P.multi;
  u32 mb_run = 0, cmd_run = 0;
  for (u32 st0 = 0; st0 < ns; st0 += BR_WARP) {
    const u32 st = st0 + (u32)br_lane();
    const u32 a = st < ns ? s.stream_nmb[st] : 0u, c = st < ns ? s.stream_ncmd[st] : 0u;
    u32 ta, tc;
    const u32 ea = br_warp_excl_scan(a, &ta), ec = br_warp_excl_scan(c, &tc);
    if (st < ns) { s.stream_nmb[st] = mb_run + ea; s.stream_ncmd[st] = cmd_run + ec; }
    mb_run += ta; cmd_run += tc;
  }
  if (br_lane() == 0) { s.stream_nmb[ns] = mb_run; s.stream_ncmd[ns] = cmd_run; s.counters[1] = mb_run; s.counters[2] = cmd_run; }
}
BR_DEV void br_chain_b3(const BrStream& s, u32 bi) {
  const u32 st = s.blk[bi].stream, fb = s.stream_blk[st];
  const u32 mb0 = s.stream_nmb[st], c0 = s.stream_ncmd[st];
  s.blkin[bi].cmd_base += c0; s.blkin[bi].mb += mb0;
  const u32 j = bi - fb;
  if (j < s.stream_nmb[st + 1] - mb0) { BrMetaBlock m = s.mbs_stage[bi]; m.cmd_off += c0; s.mbs[mb0 + j] = m; }
}

BR_DEV void br_chain_c(const BrStream& s, u32 bi) {
  const BrBlk B = s.blk[bi];
  const BrBlkIn W = s.blkin[bi];
  u64 dict_l = ((u64)W.dict_l_hi << 32) | W.dict_l_lo, dict_m = ((u64)W.dict_m_hi << 32) | W.dict_m_lo;
  u32 cmd_off = W.cmd_base;
  const u32 t_now = s.epoch;
  // conservative fallback for buckets where the precise tracking gave up: newest such commit among the
  // blocks inside this block's window (including itself)
  int ovf = B.changed_epoch;
  {
    const u32 lowpos = B.start - B.base > s.P.max_backward ? B.start - s.P.max_backward : B.base;
    for (u32 j = bi; j-- > 0;) {
      if (s.blk[j].end <= lowpos) break;
      int ce = s.blk[j].changed_epoch;
      if (ce > ovf) ovf = ce;
    }
  }
  bool prev_dirty = false, sweeping = false;
  u32 blk_state_dirty = 0;
  for (u32 c = 0; c < B.nchunks; ++c) {
    const u32 k = B.first_chunk + c;
    BrBlockIn ni = s.bin[k];
    if (c == 0) {
      ni.start_pos = B.start; ni.ext_dist = W.in_ext_dist; ni.apply_rh = 0; ni.store_end = 0;
      for (int i = 0; i < 4; ++i) ni.dc[i] = W.in_dc[i];
    }
    ni.dict_l_lo = (u32)dict_l; ni.dict_l_hi = (u32)(dict_l >> 32);
    ni.dict_m_lo = (u32)dict_m; ni.dict_m_hi = (u32)(dict_m >> 32);
    if (s.P.multi && !s.bout[k].valid && !(c == 0 && B.start == B.base)) {
      // Batch of streams, first walk of a chunk that is not the first of its stream: the counters in front of it are not
      // known yet.  Guess the static-dictionary gate (hash.h:186) CLOSED: it closes within the first kilobytes of a
      // stream and stays closed, and a walk made with the gate closed is valid for every closed state -- with the gate
      // guessed open, every chunk that finds a dictionary word has to be walked again once the true (closed) state is
      // known (44% of the chunks of 64 KiB web payloads).  The chunks where it really is open are chased from the
      // stream's first chunk (`defer` below).
      ni.dict_l_lo = 0; ni.dict_l_hi = 1u; ni.dict_m_lo = 0; ni.dict_m_hi = 0;
    }
    u32 rel = s.lil_in[k];
    u32 lil_true = (rel & 0x7fffffffu) + ((rel & 0x80000000u) ? W.lil_in : 0u);
    ni.last_insert_len = lil_true;
    const BrBlockOut out = s.bout[k];
    u32 dirty = out.valid ? 0u : 1u;  // reason: 1 never ran, 2 state, 3 dict gate, 4 stored-bits, 5 counter wrap
    u32 edl = out.valid ? out.dl : 0, edm = out.valid ? out.dm : 0;
    if (!dirty) {
      const BrBlockIn u = s.bin_used[k];
      if (u.ext_dist != ni.ext_dist || u.start_pos != ni.start_pos || u.apply_rh != ni.apply_rh ||
          u.store_end != ni.store_end || u.dc[0] != ni.dc[0] || u.dc[1] != ni.dc[1] || u.dc[2] != ni.dc[2] ||
          u.dc[3] != ni.dc[3]) dirty = 2;
      u64 ul = ((u64)u.dict_l_hi << 32) | u.dict_l_lo, um = ((u64)u.dict_m_hi << 32) | u.dict_m_lo;
      if (!dirty && (ul != dict_l || um != dict_m) &&
          !br_dict_gate_valid(dict_l, dict_m, out.dl, out.dm, out.gate_checks, out.gate_fail, &edl, &edm, s.P.quick ? 1u : 2u)) dirty = 3;
      if (!dirty && out.out_pos > ni.start_pos) {
        int seen = (int)out.epoch;
        if (s.bitdep_epoch[k] >= seen || ovf >= seen) dirty = 4;
        // flips in heavy buckets committed by launches >= seen (this run read the snapshot before launch `seen`)
        u32 unseen = s.epoch_cum[t_now] - (seen > 0 ? s.epoch_cum[seen - 1] : 0u);
        if (!dirty && unseen > out.min_wrap_dist) dirty = 5;
      }
    }
    // From the third launch on, a chunk whose only problem is the state handed over by a dirty
    // predecessor is not scheduled: the predecessor's walker chases into it (br_walk_block), which
    // resolves a serial ripple in one launch instead of one launch per chunk.
    bool defer = (dirty == 2 && prev_dirty && t_now >= 2) || (s.P.multi && dirty == 3 && prev_dirty && t_now >= 1);
    // Sweep mode (from launch sweep_epoch on).  Two kinds of dirt need opposite treatment:
    //  * STATE (reason 2, 3): the parse really arrives here in another state (position phase of the sparse search on
    //    incompressible data, distance cache).  Everything behind it in the input block is suspect, and only a walker
    //    that carries the true state can settle it: the chunk becomes the head of a SWEEP and every later dirty chunk of
    //    the block is left to that walker (it walks on while chunks are deferred or its out-state differs from what the
    //    next chunk consumed).  Scheduling those later chunks on their own would stop the sweep in front of each of them
    //    and the settled front would advance one chunk per launch.
    //  * BITS only (reason 4, 5): a stored-bit this chunk may have consulted flipped.  The marking rule is conservative
    //    (br_commit_bits: megabytes of input behind every flip), most such chunks come out unchanged, and they are
    //    independent of each other: each is walked on its own, all in parallel.
    // Safety net for inputs whose stored-bits truly chase each other from chunk to chunk: after sweep_epoch + 9 launches
    // every third launch sweeps every run of dirty chunks whatever the reason.
    const bool sweep_mode = t_now >= s.P.sweep_epoch;
    const bool full_sweep = sweep_mode && t_now >= s.P.sweep_epoch + 9 && (t_now - s.P.sweep_epoch) % 3 == 0;
    u32 defer_sweep = 0;
    if (sweep_mode && dirty) {
      if (full_sweep && prev_dirty) defer_sweep = BR_DEFER_FULL;
      else if (dirty == 2 || dirty == 3) sweeping = true;   // head of a sweep (or chased by the walker of the chunk before it: `defer`)
      else if (sweeping) defer_sweep = BR_DEFER_SWEEP;
    }
    // Batch of streams, first launch: the walker of a stream's first chunk (the one chunk whose in-state is exact) goes
    // on through the next BR_BATCH_HEAD_CHUNKS - 1 chunks: the head of a stream is where guesses are worst (the
    // dictionary gate is still open, the window is empty), and 2 000 long-running warps next to 60 000 one-chunk walkers
    // cost the launch nothing, while the same chunks chased one launch later cost a whole latency-bound launch.
    if (s.P.multi && t_now == 0 && dirty == 1 && B.start == B.base && c >= 1 && c < BR_BATCH_HEAD_CHUNKS) defer_sweep = BR_DEFER_FULL;
    if (sweep_mode && !full_sweep && (dirty == 2 || dirty == 3)) blk_state_dirty = 1;
    prev_dirty = dirty != 0;
    s.bin[k] = ni;
    s.dirty[k] = defer_sweep ? (defer_sweep | dirty) : defer ? (BR_DEFER_STATE | dirty) : dirty;   // br_chain_d schedules
    s.cmd_off[k] = cmd_off;
    s.lil_in[k] = lil_true;
    s.block_mb[k] = W.mb;
    if (dirty) { br_atomic_add(s.counters + 0, 1); br_atomic_add(s.counters + 8 + (dirty < 6 ? dirty : 6), 1); }
    if (out.valid) {
      cmd_off += out.ncmd;
      if (!(dict_m < (dict_l >> 7))) { dict_l += edl; dict_m += edm; }
    }
  }
  s.blk[bi].state_dirty = blk_state_dirty;
}

// Scheduling (thread per chunk, after br_chain_c has flagged every chunk): builds the list of walkers of the next launch.
//   * VERIFY launch: in sweep mode, when far more chunks are dirty than the last launch walked, most of them were only
//     marked by the conservative dependency rule of br_commit_bits (a flipped stored-bit marks every searched position of
//     its bucket within the ring's reach, i.e. megabytes of input).  Sweeping them serially run by run would cost a full
//     serial launch for chunks that come out unchanged; instead every dirty chunk is walked on its own, in parallel, from
//     the snapshot: unchanged ones are clean afterwards, the others flip bits and are swept in the next launch.
BR_DEV void br_chain_d(const BrStream& s, u32 k) {
  u32 d = s.dirty[k];
  if (!d) return;
  const u32 t_now = s.epoch;
  const bool sweep_mode = t_now >= s.P.sweep_epoch;
  const bool verify = sweep_mode && s.counters[4] != 0 && s.counters[0] > 4u * s.counters[4] && s.counters[0] > 64u;
  if (verify) d &= ~(BR_DEFER_SWEEP | BR_DEFER_FULL);
  else if (sweep_mode && ((t_now - s.P.sweep_epoch) & 1u) == 0 && (d == 4 || d == 5) && s.bout[k].valid) {
    // a sweep that starts in an earlier block of this group of sweep_blocks blocks may arrive here (br_walk_block crosses
    // block boundaries): leave the chunk to it, like the chunks behind a state-dirty chunk of its own block.  Every
    // second launch only: a sweep that stops early (its state fell in step again) leaves these chunks unwalked, and
    // they must not wait behind ever new sweeps of the blocks before them.
    const u32 bi = s.bin[k].blk, g0 = bi & ~(s.P.sweep_blocks - 1u);
    for (u32 j = g0; j < bi; ++j) if (s.blk[j].state_dirty && s.blk[j].base == s.blk[bi].base) { d |= BR_DEFER_SWEEP; break; }
  }
  s.dirty[k] = d;
  if (s.P.pilot && t_now == 0 && k != 0) return;   // pilot launch: chunk 0 only (the others stay dirty, unscheduled)
  if (!(d & BR_DEFER)) {
    // Sweep heads (state-dirty chunks) go to the FRONT of the list, the rest is filled from the back: CTAs start in list
    // order, so the long serial sweeps begin with the launch instead of trailing behind thousands of one-chunk walkers.
    const bool stream_head = s.P.multi && t_now == 0 && s.bin[k].first && s.bin[k].blk_start == s.bin[k].base;
    if ((sweep_mode && (d == 2 || d == 3)) || stream_head) { u32 slot = br_atomic_add(s.counters + 17, 1); s.dirty_list[slot] = k; }
    else { u32 slot = br_atomic_add(s.counters + 18, 1); s.dirty_list[s.P.nblocks - 1u - slot] = k; }
    br_atomic_add(s.counters + 5, 1);
    br_atomic_min(s.counters + 6, k);
  }
}
// entry t of the schedule built above (t < counters[5])
BR_DEV u32 br_sched_entry(const BrStream& s, u32 t) {
  const u32 nfront = s.counters[17];
  return t < nfront ? s.dirty_list[t] : s.dirty_list[s.P.nblocks - 1u - (t - nfront)];
}

// sequential driver for the CPU sim / single-thread use
BR_DEV void br_chain(const BrStream& s) {
  for (u32 bi = 0; bi < s.nblk; ++bi) br_chain_a(s, bi);
  if (s.P.multi) {
    for (u32 st = 0; st < s.P.multi; ++st) br_chain_b1(s, st);
    br_chain_b2(s);
    for (u32 bi = 0; bi < s.nblk; ++bi) br_chain_b3(s, bi);
  } else br_chain_b(s);
  for (u32 bi = 0; bi < s.nblk; ++bi) br_chain_c(s, bi);
  for (u32 k = 0; k < s.P.nblocks; ++k) br_chain_d(s, k);
}

// Gather one chunk's commands into the stream-wide compacted array, applying the
// ExtendLastCommand growth (encode.c:961) and the trailing insert-only command
// (encode.c:1169).  Warp task per chunk.
BR_DEV void br_compact_block(const BrStream& s, u32 k, BrCmd* cmds_all, const u32* block_mb) {
  const BrBlockOut out = s.bout[k];
  const BrCmd* src = s.cmd_blocks + (size_t)k * s.cmd_stride;
  BrCmd* dst = cmds_all + s.cmd_off[k];
  for (u32 i = (u32)br_lane(); i < out.ncmd; i += BR_WARP) {
    BrCmd c = src[i];
    if (i == 0 && s.lil_in[k]) {   // literals pending when the chunk started belong to its first command
      c.insert_len += s.lil_in[k];
      c.cmd_prefix = br_length_code(c.insert_len, br_cmd_copy_len_code(c), (c.dist_prefix & 0x3FF) == 0);
    }
    if (i + 1 == out.ncmd && s.ext_total[k]) {
      c.copy_len += s.ext_total[k];
      c.cmd_prefix = br_length_code(c.insert_len,
          (u32)((int)(c.copy_len & 0x1FFFFFF) + (int)(c.copy_len >> 25)),
          (c.dist_prefix & 0x3FF) == 0);
    }
    dst[i] = c;
  }
  const BrMetaBlock mb = s.mbs[block_mb[k]];
  if (mb.last_block == k && mb.tail_insert && br_lane() == 0)
    dst[out.ncmd] = br_init_insert_cmd(mb.tail_insert);
}
