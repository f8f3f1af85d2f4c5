// br_probe.h -- test hook (tests/test_search_probe.py): one match search from a fully specified state, set up the way
// br_walk_one sets up its walker.  Shared by the CUDA hook br_debug_search (br_kernels.cu) and the one-lane sim
// (tests/sim/search_probe.cc), so that both run the same search on the same state.  No pipeline code includes it.
#pragma once
#include "br_lz77.h"

// A probe, BR_PROBE_WORDS words: cur, p0, base, pend, max_backward, dict_distance, dc[0..3], len_in, score_in,
// dict_l (lo, hi), dict_m (lo, hi).  max_length is pend - cur.
// Its result, as many words: len, distance, score, delta, dl, dm, gate_checks, gate_fail, the own bit and the searched bit
// the search set at cur, saw[0..3] (qualities 2..4; the slots a search does not read keep what the caller put there), 0, 0.
// own: the walker's own bitmap (positions >= p0); the snapshot is s.bits_latest with its S-ordered copy s.storedS / s.prefS.
// F: the walker form (br_walk_form), as br_walk_dispatch picks it; F == 0: the quick search of qualities 2..4.  Nothing is written to own or to the searched bitmap: a search's own writes
// stay in the walker's gathered word, which is where the result reads them.
#define BR_PROBE_WORDS 16
template <int F>
BR_DEV void br_probe_search(const BrStream& s, u32* own, const u32* pr, u32* res) {
  const BrParams& P = s.P;
  BrWalk w;
  w.s = &s; w.d = s.data; w.p0 = pr[1]; w.base = pr[2]; w.pend = pr[3];
  w.own = own;
  w.dict0 = pr + 12;
  w.dl = w.dm = w.gate_checks = w.gate_fail = 0;
  w.min_wrap = 0xffffffffu;
  w.fence_due = false;
  w.acc_wi = 0xffffffffu; w.acc_own = 0; w.acc_srch = 0;
  w.warming = false;
#ifdef BR_DEBUG_KNOBS
  w.dbg_searches = w.dbg_rows = w.dbg_mlsteps = 0;
#endif
  w.stale = w.pend - w.base <= P.rmask ? 0u : (u32)s.data[w.pend - (P.rmask + 1)];
  for (int i = 0; i < 4; ++i) w.dc[i] = (int)pr[6 + i];
  const u32 cur = pr[0];
  BrSR sr; sr.len = pr[10]; sr.delta = 0; sr.distance = 0; sr.score = pr[11];
  if constexpr (F == 0) br_find_quick(w, cur, w.pend - cur, pr[4], pr[5], sr);
  else br_find_longest_match<F>(w, cur, w.pend - cur, pr[4], pr[5], sr, BrLook{cur + 1, cur + 2, 1});   // (with a lookahead, which must not change the result)
  if (br_lane() == 0) {
    const bool here = w.acc_wi == (cur >> 5);
    res[0] = sr.len; res[1] = sr.distance; res[2] = sr.score; res[3] = (u32)sr.delta;
    res[4] = w.dl; res[5] = w.dm; res[6] = w.gate_checks; res[7] = w.gate_fail;
    res[8] = here ? (w.acc_own >> (cur & 31)) & 1u : 0u;
    res[9] = here ? (w.acc_srch >> (cur & 31)) & 1u : 0u;
    for (u32 i = 0; i < 4; ++i) res[10 + i] = P.quick && i < (1u << P.qk_sweep_bits) ? s.saw[((size_t)cur << P.qk_sweep_bits) + i] : 0u;
    res[14] = res[15] = 0;
  }
}
