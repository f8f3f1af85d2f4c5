// tests/sim/snapshot_check.cc -- TEST INFRASTRUCTURE (tests/test_gpu_index.py).  The LZ77 fixpoint of br_sim.cc's
// sim_lz77_fixpoint, with the S-ordered snapshot of the stored bits kept the way the product keeps it: gathered once, then
// carried along by br_snapshot_update after every launch's commits (k_snapshot_update).  The walkers read the kept snapshot;
// before every launch it is compared with one gathered from scratch (sim_build_storedS).  Qualities 5..9.
#include "br_sim.cc"

// stats[0] launches checked, [1] launches whose kept snapshot or prefix differed, [2] stored bits flipped by the commits.
// cut_pos / cut_kind / ncuts: the stream's cuts (br_pipeline.h BrCuts: kind 1 FLUSH, 3 the end of one stream of a batch).
extern "C" int snap_check_lz77(int q, int lgwin, const u8* in, u32 n, u32 size_hint, const u32* cut_pos, const u32* cut_kind,
                               u32 ncuts, u64* stats) {
  const BrCuts c = {cut_pos, cut_kind, ncuts, 1, 1, 0, nullptr, 0, 0, 0, nullptr};
  SimStream* m = sim_setup(q, lgwin, size_hint, in, n, ncuts ? &c : nullptr);
  if (!m) return 0;
  BrStream& s = m->s;
  if (s.P.quick) { delete m; return 0; }   // (qualities 2..4 read no snapshot)
  stats[0] = stats[1] = stats[2] = 0;
  sim_build_storedS(*m);
  std::vector<u32> kept = m->storedS, cnt(m->prefS.size(), 0), kept_pref(m->prefS.size(), 0);
  for (size_t w = 0; w < kept.size() && w / 32 < cnt.size(); ++w) cnt[w / 32] += __builtin_popcount(kept[w]);
  s.storedS = kept.data(); s.prefS = kept_pref.data();
  const u32 nsnap = (n + 1023) / 1024 + 1;   // the prefix entries sim_build_storedS writes
  const u32 round_epoch0 = s.epoch;
  for (;;) {
    br_chain(s);
    if (s.counters[0] == 0) break;
    ++s.epoch;
    for (u32 b = 0, acc = 0; b < nsnap; ++b) { kept_pref[b] = acc; acc += cnt[b]; }
    sim_build_storedS(*m);
    ++stats[0];
    if (kept != m->storedS || !std::equal(kept_pref.begin(), kept_pref.begin() + nsnap, m->prefS.begin())) ++stats[1];
    std::fill(m->bits_cur.begin(), m->bits_cur.end(), 0); std::fill(m->srch_cur.begin(), m->srch_cur.end(), 0);
    s.counters[4] = 0; s.counters[16] = 0;
    s.forced = s.epoch - round_epoch0 >= s.P.force_epoch;
    { u32 nd = s.counters[5]; std::vector<u32> dl(nd); for (u32 t = 0; t < nd; ++t) dl[t] = br_sched_entry(s, t); for (u32 k : dl) { const bool f = s.forced && k == s.counters[6];
      br_walk_dispatch(s.P, [&](auto g, auto mm) { br_walk_block<decltype(g)::value, decltype(mm)::value>(s, k, f); }); } }
    m->bits_prev = m->bits_latest; s.bits_prev = m->bits_prev.data();
    std::fill(m->cover_cur.begin(), m->cover_cur.end(), 0);
    for (u32 i = 0; i < s.counters[4]; ++i) br_cover_run(s, s.ran_list[i]);
    for (u32 i = 0; i < s.counters[4]; ++i) br_commit_bits(s, s.ran_list[i]);
    for (u32 x = 0; x < s.bits_words; ++x) {
      stats[2] += __builtin_popcount(m->bits_latest[x] ^ m->bits_prev[x]);
      br_snapshot_update(s, x, kept.data(), cnt.data());
    }
    if (s.epoch + 2 >= s.P.max_epochs) break;
  }
  delete m;
  return 1;
}
