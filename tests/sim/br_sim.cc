// tests/sim/br_sim.cc -- TEST INFRASTRUCTURE.  Compiles the product's warp-task device code
// (brotli_b200/csrc/br_lz77.h, br_chain.h, br_entropy.h) for the CPU with a one-lane "warp"
// (BR_SIM) so that the bit-exact logic can be debugged against the oracle in a container
// without a GPU.  The data-parallel kernels (hash, sort, scans, packing) have trivial
// sequential stand-ins here; their CUDA versions are checked on the GPU (tests -m gpu).
#define BR_SIM 1
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <algorithm>
#include <vector>
#include "../../brotli_b200/csrc/br_params.h"
#include "../../brotli_b200/csrc/br_lz77.h"
#include "../../brotli_b200/csrc/br_chain.h"
#ifdef BR_SIM_ENTROPY
#include "../../brotli_b200/csrc/br_entropy.h"
#include "../../brotli_b200/csrc/br_entropy2.h"
#include "../../brotli_b200/csrc/br_assemble.h"
#include "../../brotli_b200/csrc/br_entropy_flat.h"
#endif

struct SimTables {
  std::vector<u8> blob;
  std::vector<double> log2tab;
};
static SimTables g_t;

extern "C" int sim_init(const u8* blob, size_t len, u32 log2n) {
  g_t.blob.assign(blob, blob + len);
  g_t.log2tab.resize(log2n);
  g_t.log2tab[0] = 0;
  for (u32 i = 1; i < log2n; ++i)
    g_t.log2tab[i] = i < 256 ? (double)(float)log2((double)i) : log2((double)i);
  return 1;
}

// An explicit schedule of the LZ77 fixpoint (sim_compress_sched): the knobs of BrParams that decide which chunks a launch
// walks and when the safety nets take over, and the order in which the sim runs a launch's walks and commits (on the GPU
// they run concurrently, in no fixed order).  BR_KNOB_KEEP keeps the value the plan chose.
enum { SIM_ORDER_SCHEDULED = 0, SIM_ORDER_REVERSED = 1, SIM_ORDER_SHUFFLED = 2 };
struct SimSched {
  BrSchedKnobs knobs;               // as br_debug_compress_sched takes them (br_pipeline.h)
  u32 batch_chunk_bits;             // chunk size of a batch of streams (log2; br_plan_stream)
  u32 walk_order, commit_order;     // SIM_ORDER_*; commit_order applies to the br_cover_run and the br_commit_bits loops
  u32 walk_seed, commit_seed;       // SIM_ORDER_SHUFFLED
  u32 verify;                       // != 0: re-walk every chunk at the fixpoint (SIM_ST_VERIFY_DIFF); the output is unchanged
};
// stats words of sim_compress_sched (the first five as sim_compress reports them)
enum {
  SIM_ST_LAUNCHES = 0, SIM_ST_WALKS = 1, SIM_ST_CHUNKS = 2, SIM_ST_ROUNDS = 3, SIM_ST_MODEL_COST = 4,
  SIM_ST_FULL_SWEEP = 5,        // launches that follow a full-sweep chain decision (br_chain_c)
  SIM_ST_FORCED = 6,            // launches with a forced walker (BrStream::forced)
  SIM_ST_STEP_CAP = 7,          // step-cap hits of br_commit_bits (BR_SIM_DEBUG builds only)
  SIM_ST_PREDICT_OK = 8,        // block boundaries a sweep crossed (br_predict_next_block true; BR_SIM_DEBUG builds only)
  SIM_ST_PREDICT_NO = 9,        // block boundaries where the prediction refused (BR_SIM_DEBUG builds only)
  SIM_ST_MAX_WALKS = 10,        // the largest number of chunk walks of one launch (counters[4])
  SIM_ST_RAN_CAP = 11,          // capacity of ran_list (BrStreamPlan::ran_cap)
  SIM_ST_VERIFY_DIFF = 12,      // chunks whose re-walk at the fixpoint gives other bits or another out-state (SimSched::verify)
  SIM_ST_WORDS = 16
};
#define SIM_ERR_CAPACITY (-5)   // a launch appended more entries than an array holds (the call fails, nothing is corrupted)
#define SIM_ERR_NO_FIXPOINT (-6)   // the launch bound (BrParams::max_epochs) was reached

struct SimStream {
  BrStream s;
  std::vector<u8> data;
  std::vector<u32> S, rank, seg, bits_latest, bits_cur, bits_prev, srch_latest, srch_cur, cover_cur, storedS, prefS, dirty, changed_bits,
      epoch_cum, ext_total, lil_in, cmd_off, force_unc, counters, hist, block_mb;
  std::vector<int> changed_epoch, bitdep_epoch;
  std::vector<u16> skeys, tagS;
  std::vector<BrBlockIn> bin, bin_used;
  std::vector<BrBlockOut> bout;
  std::vector<BrCmd> cmd_blocks, cmds_all;
  std::vector<BrMetaBlock> mbs;
  BrStreamPlan plan;                // the block, slot and stream tables and the sizes, as the product plans them
  std::vector<BrBlkIn> blkin;
  std::vector<u32> key_flips, saw, qpred;
  std::vector<u32> dirty_list, ran_list, stream_nmb, stream_ncmd;
  std::vector<BrMetaBlock> mbs_stage;
  int iterations = 0;
  u64 block_runs = 0;
  double model_cost = 0;
  SimSched sched;
  u32 st[SIM_ST_WORDS] = {};
};

static void sim_build_sorted(SimStream& m) {
  BrStream& s = m.s; const BrParams& P = s.P; u32 n = P.n;
  std::vector<u32> key(n);
  u32 hashable = n >= P.htl ? n - P.htl + 1 : 0;  // positions with a full hash load
  for (u32 p = 0; p < n; ++p) key[p] = p >= hashable ? P.nbuckets : P.quick ? br_quick_slot(P, br_ld64u(s.data, p), p - br_stream_base_of(s, p)) : br_hash_key(P, s.data, p);
  m.seg.assign(P.nbuckets + 2, 0);
  for (u32 p = 0; p < n; ++p) m.seg[key[p] + 1]++;
  for (u32 k = 0; k <= P.nbuckets; ++k) m.seg[k + 1] += m.seg[k];
  std::vector<u32> cur(m.seg.begin(), m.seg.end() - 1);
  m.S.resize(n); m.rank.resize(n);
  m.skeys.resize(n + 1);
  for (u32 p = 0; p < n; ++p) { u32 j = cur[key[p]]++; m.S[j] = p; m.rank[p] = j; m.skeys[j] = (u16)key[p]; }
  s.skeys = m.skeys.data();
  m.tagS.resize(n + 1);
  for (u32 j = 0; j < n; ++j) m.tagS[j] = (u16)br_tag4(br_ld32u(s.data, m.S[j]));
  s.tagS = m.tagS.data();
  s.S = m.S.data(); s.rank = m.rank.data(); s.seg = m.seg.data();
}
static void sim_build_storedS(SimStream& m) {
  u32 n = m.s.P.n;
  std::fill(m.storedS.begin(), m.storedS.end(), 0);
  for (u32 j = 0; j < n; ++j) {
    u32 q = m.S[j];
    if ((m.bits_latest[q >> 5] >> (q & 31)) & 1) m.storedS[j >> 5] |= 1u << (j & 31);
  }
  u32 acc = 0;
  for (u32 b = 0; b * 1024 < n + 1024; ++b) {
    m.prefS[b] = acc;
    for (u32 w = b * 32; w < b * 32 + 32 && w < m.storedS.size(); ++w) acc += __builtin_popcount(m.storedS[w]);
  }
}

// the schedule of the tools' environment switches (BR_SIM_*): everything else as planned, walks and commits in list order
static SimSched sim_sched_from_env() {
  SimSched c;
  auto env = [](const char* name) { const char* v = getenv(name); return v ? (u32)atoi(v) : BR_KNOB_KEEP; };
  c.knobs.heavy_min = env("BR_SIM_HEAVY_MIN"); c.knobs.step_cap = env("BR_SIM_STEP_CAP"); c.knobs.sweep_epoch = env("BR_SIM_SWEEP_EPOCH");
  c.knobs.sweep_blocks = env("BR_SIM_SWEEP_BLOCKS"); c.knobs.pilot = env("BR_SIM_PILOT"); c.knobs.force_epoch = env("BR_SIM_FORCE_EPOCH");
  c.batch_chunk_bits = env("BR_SIM_BATCH_CHUNK_BITS");
  c.walk_order = c.commit_order = SIM_ORDER_SCHEDULED; c.walk_seed = c.commit_seed = 0;
  c.verify = getenv("BR_SIM_VERIFY") ? 1u : 0u;
  return c;
}

// The stream planned by br_plan_stream (nullptr where the product refuses it), with the sim's own memory.
static SimStream* sim_setup(int q, int lgwin, u32 size_hint, const u8* in, u32 n, const BrCuts* cuts = nullptr,
                            const SimSched* sched = nullptr) {
  SimStream* m = new SimStream();
  m->sched = sched ? *sched : sim_sched_from_env();
  BrStreamPlan& plan = m->plan;
  if (!br_plan_stream(q, lgwin, size_hint, n, cuts, &m->sched.knobs, &plan, m->sched.batch_chunk_bits, &m->bin)) {
    delete m; return nullptr;
  }
  BrStream& s = m->s;
  memset(&s, 0, sizeof(s));
  s.P = plan.P;
  const BrParams& P = s.P;
  const u32 nb = P.nblocks, words = (n + 31) / 32 + 2;
  s.blk = plan.blk.data(); s.nblk = (u32)plan.blk.size(); s.slot_blk = plan.slot_blk.data(); s.stream_blk = plan.stream_blk.data();
  m->data.assign(in, in + n); m->data.resize(n + 64, 0);
  s.data = m->data.data();
  m->bin_used.resize(nb); m->bout.resize(nb);
  memset(m->bin_used.data(), 0, nb * sizeof(BrBlockIn));
  memset(m->bout.data(), 0, nb * sizeof(BrBlockOut));
  m->bits_latest.assign(words, 0); m->bits_cur.assign(2 * words, 0); m->srch_latest.assign(words, 0); m->srch_cur.assign(words, 0); m->cover_cur.assign(words, 0);
  s.bits_latest = m->bits_latest.data();
  for (u32 bi = 0; bi < s.nblk; ++bi) br_init_bits(s, bi, 0, 1);   // k_init_bits
  m->storedS.assign(words + 32, 0); m->prefS.assign(n / 1024 + 4, 0);
  m->dirty.assign(nb, 0); m->changed_bits.assign(nb, 0); m->changed_epoch.assign(nb, -1); m->bitdep_epoch.assign(nb + 1, -1);
  m->epoch_cum.assign(P.max_epochs + 2, 0);
  m->ext_total.assign(nb, 0); m->lil_in.assign(nb, 0); m->cmd_off.assign(nb, 0); m->force_unc.assign(nb + 1, 0);
  m->counters.assign(64, 0); m->hist.assign(256 * (size_t)plan.nstreams, 0); m->mbs.resize(nb + 1);
  m->stream_nmb.assign(plan.nstreams + 1, 0); m->stream_ncmd.assign(plan.nstreams + 1, 0); m->mbs_stage.resize(s.nblk);
  s.stream_nmb = m->stream_nmb.data(); s.stream_ncmd = m->stream_ncmd.data(); s.mbs_stage = m->mbs_stage.data();
  s.cmd_stride = plan.cmd_stride;
  m->cmd_blocks.resize((size_t)(nb + 1) * s.cmd_stride);   // (+ a guard slice behind the last chunk's: see sim_lz77_fixpoint)
  s.bits_cur = m->bits_cur.data(); s.bits_words = words;
  s.srch_latest = m->srch_latest.data(); s.srch_cur = m->srch_cur.data(); s.cover_cur = m->cover_cur.data();
  s.storedS = m->storedS.data(); s.prefS = m->prefS.data();
  s.bin = m->bin.data(); s.bin_used = m->bin_used.data(); s.bout = m->bout.data();
  s.cmd_blocks = m->cmd_blocks.data(); s.dirty = m->dirty.data();
  s.changed_bits = m->changed_bits.data(); s.changed_epoch = m->changed_epoch.data(); s.bitdep_epoch = m->bitdep_epoch.data();
  s.epoch_cum = m->epoch_cum.data();
  s.ext_total = m->ext_total.data(); s.lil_in = m->lil_in.data(); s.cmd_off = m->cmd_off.data();
  s.mbs = m->mbs.data(); s.force_unc = m->force_unc.data(); s.counters = m->counters.data();
  s.hist_scratch = m->hist.data();
  m->blkin.resize(s.nblk); s.blkin = m->blkin.data();
  m->key_flips.assign(P.nbuckets + 2, 0); s.key_flips = m->key_flips.data();
  if (P.quick) { m->saw.assign(((size_t)n << P.qk_sweep_bits) + 4, 0xdeadbeefu); s.saw = m->saw.data(); }
  m->dirty_list.assign(nb + 1, 0); m->block_mb.assign(nb + 1, 0);
  s.dirty_list = m->dirty_list.data(); s.block_mb = m->block_mb.data();
  // ran_list followed by a guard as long again: a launch that appends more walks than the product holds writes into the
  // guard, and the fixpoint fails the call (SIM_ERR_CAPACITY)
  m->ran_list.assign(2 * (size_t)plan.ran_cap, 0); s.ran_list = m->ran_list.data();
  br_bind_tables(s, g_t.blob.data(), g_t.log2tab.data(), (u32)g_t.log2tab.size());
  sim_build_sorted(*m);
  if (P.quick) {   // k_slot_pred
    m->qpred.assign(((size_t)n << P.qk_sweep_bits) + 4, 0);
    for (u32 p = 0; p < n; ++p) br_quick_pred_fill(s, p, br_stream_base_of(s, p), m->qpred.data() + ((size_t)p << P.qk_sweep_bits));
    s.qpred = m->qpred.data();
  }
  return m;
}

// The order in which the sim runs the n entries of a launch's list (SimSched::walk_order / commit_order).  The shuffle is a
// Fisher-Yates draw from a 64-bit LCG seeded by (seed, launch, pass): reproducible on every platform.
static std::vector<u32> sim_order(u32 n, u32 order, u32 seed, u32 launch, u32 pass) {
  std::vector<u32> o(n);
  for (u32 i = 0; i < n; ++i) o[i] = order == SIM_ORDER_REVERSED ? n - 1 - i : i;
  if (order == SIM_ORDER_SHUFFLED) {
    u64 x = ((u64)seed << 32) ^ ((u64)launch << 8) ^ pass ^ 0x9E3779B97F4A7C15ull;
    for (u32 i = n; i > 1; --i) {
      x = x * 6364136223846793005ull + 1442695040888963407ull;
      std::swap(o[i - 1], o[(u32)((x >> 33) % i)]);
    }
  }
  return o;
}

// Is the fixpoint self-consistent?  Re-walks every chunk from its final in-state against the final stored-bits and returns
// the number of chunks whose bits or out-state come out differently.  Everything the re-walk writes is restored afterwards,
// so the output is that of the fixpoint.
static u32 sim_verify_fixpoint(SimStream& m);

// Runs the LZ77 fixpoint; 0, or SIM_ERR_CAPACITY when a launch appended more entries than an array of the product holds.
static int sim_lz77_fixpoint(SimStream& m) {
  BrStream& s = m.s; u32 nb = s.P.nblocks;
#ifdef BR_SIM_DEBUG
  if (getenv("BR_SIM_WATCH")) br_sim_watch = (u32)atoi(getenv("BR_SIM_WATCH"));
#endif
  const SimSched& K = m.sched;
  // (the launch counter runs on through the rounds of a late fallback, as in br_job_compress_device: runs are stamped with
  // it -- BrBlockOut::epoch -- and the marks of br_commit_bits / br_verify_run are compared with those stamps)
  const u32 round_epoch0 = s.epoch;
  for (;;) {
    br_chain(s);
    if (getenv("BR_SIM_TRACE")) { u32 h[6] = {0}; u32 first = nb; for (u32 k = 0; k < nb; ++k) { h[s.dirty[k] & 7]++; if (s.dirty[k] && first == nb) first = k; }
      fprintf(stderr, "epoch %u dirty %u first %u: never %u state %u dict %u window %u wrap %u | flipped bits %u\n", s.epoch, s.counters[0], first, h[1], h[2], h[3], h[4], h[5], s.epoch_cum[s.epoch] - (s.epoch ? s.epoch_cum[s.epoch - 1] : 0));
#ifdef BR_SIM_DEBUG
      fprintf(stderr, "   last commit: flips %llu successor steps %llu marks %llu overlap marks %llu cap hits %llu\n", (unsigned long long)br_sim_cnt[3],
              (unsigned long long)br_sim_cnt[4], (unsigned long long)br_sim_cnt[0], (unsigned long long)br_sim_cnt[1], (unsigned long long)br_sim_cnt[2]);
      memset(br_sim_cnt, 0, sizeof(br_sim_cnt));
#endif
    }
    if (s.counters[0] == 0) break;
    // (the rule of br_chain_c, at the launch number the chain ran with)
    if (s.epoch >= s.P.sweep_epoch + 9 && (s.epoch - s.P.sweep_epoch) % 3 == 0) ++m.st[SIM_ST_FULL_SWEEP];
    ++s.epoch; ++m.iterations;
    sim_build_storedS(m);
    std::fill(m.bits_cur.begin(), m.bits_cur.end(), 0); std::fill(m.srch_cur.begin(), m.srch_cur.end(), 0);
    s.counters[4] = 0; s.counters[16] = 0;
    s.forced = s.epoch - round_epoch0 >= s.P.force_epoch;
    if (s.forced) ++m.st[SIM_ST_FORCED];
    { u32 nd = s.counters[5]; std::vector<u32> dl(nd); for (u32 t = 0; t < nd; ++t) dl[t] = br_sched_entry(s, t);
      for (u32 t : sim_order(nd, K.walk_order, K.walk_seed, s.epoch, 0)) { const u32 k = dl[t]; const bool f = s.forced && k == s.counters[6];
        br_walk_dispatch(s.P, [&](auto g, auto mm) { br_walk_block<decltype(g)::value, decltype(mm)::value>(s, k, f); }); } }
    m.block_runs += s.counters[4];
    if (s.counters[4] > m.st[SIM_ST_MAX_WALKS]) m.st[SIM_ST_MAX_WALKS] = s.counters[4];
    if (s.counters[4] > m.plan.ran_cap) {
      fprintf(stderr, "sim: launch %u walked %u chunks, ran_list holds %u\n", s.epoch, s.counters[4], m.plan.ran_cap);
      return SIM_ERR_CAPACITY;
    }
    for (u32 i = 0; i < s.counters[4]; ++i)
      if (s.bout[s.ran_list[i]].ncmd > s.cmd_stride) {
        fprintf(stderr, "sim: chunk %u made %u commands, its slice of cmd_blocks holds %u\n", s.ran_list[i], s.bout[s.ran_list[i]].ncmd, s.cmd_stride);
        return SIM_ERR_CAPACITY;
      }
#ifdef BR_SIM_DEBUG
    if (getenv("BR_SIM_TRACE")) { fprintf(stderr, "   work: searches %llu rows %llu groups %llu taken %llu | heavy %llu own-scan rows %llu countS %llu | own_set %llu set_range %llu dict %llu\n",
      (unsigned long long)br_sim_w[0], (unsigned long long)br_sim_w[1], (unsigned long long)br_sim_w[8], (unsigned long long)br_sim_w[9], (unsigned long long)br_sim_w[2], (unsigned long long)br_sim_w[3],
      (unsigned long long)br_sim_w[4], (unsigned long long)br_sim_w[5], (unsigned long long)br_sim_w[6], (unsigned long long)br_sim_w[7]); memset(br_sim_w, 0, sizeof(br_sim_w)); }
#endif
    { // cost model of a launch on the GPU, in chunk-walk times: the longest sweep (serial) or the whole work over ~2000 resident warps
      double c = (double)s.counters[16] > s.counters[4] / 2000.0 ? (double)s.counters[16] : s.counters[4] / 2000.0;
      m.model_cost += c;
      if (getenv("BR_SIM_TRACE")) fprintf(stderr, "   launch %u: sched %u ran %u longest sweep %u  (model cost %.1f, total %.1f)\n", s.epoch, s.counters[5], s.counters[4], s.counters[16], c, m.model_cost);
    }
    m.bits_prev = m.bits_latest; s.bits_prev = m.bits_prev.data();
    std::fill(m.cover_cur.begin(), m.cover_cur.end(), 0);
    // (every run is covered before any commit, as k_cover runs before k_commit on the GPU)
    for (u32 i : sim_order(s.counters[4], K.commit_order, K.commit_seed, s.epoch, 1)) br_cover_run(s, s.ran_list[i]);
#ifdef BR_SIM_DEBUG
    const u64 cap_hits0 = br_sim_cnt[2];
#endif
    for (u32 i : sim_order(s.counters[4], K.commit_order, K.commit_seed, s.epoch, 2)) br_commit_bits(s, s.ran_list[i]);
#ifdef BR_SIM_DEBUG
    m.st[SIM_ST_STEP_CAP] += (u32)(br_sim_cnt[2] - cap_hits0);
#endif
    if (s.P.quick) for (u32 k = 0; k < nb; ++k) br_verify_run(s, k);
    if (s.epoch + 2 >= s.P.max_epochs) { fprintf(stderr, "sim: no fixpoint\n"); return SIM_ERR_NO_FIXPOINT; }
  }
  if (K.verify) m.st[SIM_ST_VERIFY_DIFF] += sim_verify_fixpoint(m);
  if (getenv("BR_SIM_TRACE")) {   // the static-dictionary gate (hash.h:186) at the fixpoint: chunks that start with it closed
    u32 closed = 0, hits = 0; for (u32 k = 0; k < nb; ++k) { const u64 l = ((u64)s.bin[k].dict_l_hi << 32) | s.bin[k].dict_l_lo, mm = ((u64)s.bin[k].dict_m_hi << 32) | s.bin[k].dict_m_lo; if (mm < (l >> 7)) ++closed; if (s.bout[k].dm) ++hits; }
    fprintf(stderr, "dictionary gate: %u of %u chunks start with the gate closed; %u chunks found dictionary matches\n", closed, nb, hits);
  }
  m.cmds_all.resize(s.counters[2] + 1);
  for (u32 k = 0; k < nb; ++k) br_compact_block(s, k, m.cmds_all.data(), m.block_mb.data());
  return 0;
}

static u32 sim_verify_fixpoint(SimStream& m) {
  BrStream& s = m.s; const u32 nb = s.P.nblocks;
  const char* show = getenv("BR_SIM_VERIFY");   // (the tools: print what differs; "2" also the positions)
  // what the re-walk and its commits write
  const u32 epoch0 = s.epoch;
  const std::vector<BrBlockOut> old(m.bout);
  const std::vector<BrBlockIn> used0(m.bin_used);
  const std::vector<BrCmd> old_cmds(m.cmd_blocks);
  const std::vector<u32> latest0(m.bits_latest), srch0(m.srch_latest), counters0(m.counters), key_flips0(m.key_flips), saw0(m.saw), changed_bits0(m.changed_bits);
  const std::vector<int> bitdep0(m.bitdep_epoch), changed_epoch0(m.changed_epoch);
  const std::vector<BrBlk> blks0(m.plan.blk);
  ++s.epoch;
  sim_build_storedS(m);   // (the S-ordered snapshot of the final bits: the last launch's commits are not in it yet)
  std::fill(m.bits_cur.begin(), m.bits_cur.end(), 0); std::fill(m.srch_cur.begin(), m.srch_cur.end(), 0);
  s.counters[4] = 0;
  for (u32 k = 0; k < nb; ++k) {
    BrBlockOut o; u32 sp0 = 0xffffffffu;
    br_walk_dispatch(s.P, [&](auto g, auto mm) { br_walk_one<decltype(g)::value, decltype(mm)::value>(s, k, s.bin[k], o, k, sp0); });
  }
  m.bits_prev = m.bits_latest; s.bits_prev = m.bits_prev.data();
  std::fill(m.cover_cur.begin(), m.cover_cur.end(), 0);
  for (u32 k = 0; k < nb; ++k) br_cover_run(s, k);
  u32 ndiff = 0;
  for (u32 k = 0; k < nb; ++k) {
    br_commit_bits(s, k);
    const BrBlockOut& a = old[k]; const BrBlockOut& b = s.bout[k];
    const bool same = a.ncmd == b.ncmd && a.nlit == b.nlit && a.out_pos == b.out_pos && a.last_insert_len == b.last_insert_len &&
                      !memcmp(a.dc, b.dc, sizeof(a.dc)) && a.apply_rh == b.apply_rh;
    const bool same_cmds = same && !memcmp(&old_cmds[(size_t)k * s.cmd_stride], &m.cmd_blocks[(size_t)k * s.cmd_stride], (size_t)a.ncmd * sizeof(BrCmd));
    if (s.changed_bits[k] || !same_cmds) ++ndiff;
    if (!show) continue;
    if (s.changed_bits[k] && show[0] == '2') {
      u32 shown = 0;
      for (u32 q = s.bin_used[k].start_pos; q < s.bout[k].out_pos && shown < 12; ++q) {
        u32 o = (m.bits_prev[q >> 5] >> (q & 31)) & 1, n2 = (m.bits_latest[q >> 5] >> (q & 31)) & 1;
        if (o != n2) { fprintf(stderr, "  pos %u: fixpoint %u rewalk %u\n", q, o, n2); ++shown; }
      }
    }
    if (!same_cmds) {
      // first command that differs: where it starts in the input, what it was and what the re-walk says
      u32 pos = s.bin[k].start_pos;
      for (u32 i = 0; i < std::min(a.ncmd, b.ncmd); ++i) {
        const BrCmd& x = old_cmds[(size_t)k * s.cmd_stride + i]; const BrCmd& y = m.cmd_blocks[(size_t)k * s.cmd_stride + i];
        if (memcmp(&x, &y, sizeof(BrCmd))) {
          fprintf(stderr, "verify: chunk %u (run of launch %u) command %u at input %u: fixpoint insert %u copy %u dist_prefix %u extra %u | rewalk insert %u copy %u dist_prefix %u extra %u\n", k, a.epoch, i, pos,
                  x.insert_len, x.copy_len & 0x1FFFFFF, x.dist_prefix, x.dist_extra, y.insert_len, y.copy_len & 0x1FFFFFF, y.dist_prefix, y.dist_extra);
          break;
        }
        pos += x.insert_len + (x.copy_len & 0x1FFFFFF);
      }
    }
    if (s.changed_bits[k] || !same_cmds)
      fprintf(stderr, "verify: chunk %u [%u..%u) start %u: %u bits differ, out-state %s (ncmd %u/%u out_pos %u/%u)\n", k, s.bin[k].pos, s.bin[k].end,
              s.bin[k].start_pos, s.changed_bits[k], same ? "same" : "DIFFERENT", a.ncmd, b.ncmd, a.out_pos, b.out_pos);
  }
  s.epoch = epoch0;
  std::copy(old.begin(), old.end(), m.bout.begin()); std::copy(used0.begin(), used0.end(), m.bin_used.begin());
  std::copy(old_cmds.begin(), old_cmds.end(), m.cmd_blocks.begin());
  std::copy(latest0.begin(), latest0.end(), m.bits_latest.begin()); std::copy(srch0.begin(), srch0.end(), m.srch_latest.begin());
  std::copy(counters0.begin(), counters0.end(), m.counters.begin()); std::copy(key_flips0.begin(), key_flips0.end(), m.key_flips.begin());
  std::copy(saw0.begin(), saw0.end(), m.saw.begin()); std::copy(changed_bits0.begin(), changed_bits0.end(), m.changed_bits.begin());
  std::copy(bitdep0.begin(), bitdep0.end(), m.bitdep_epoch.begin()); std::copy(changed_epoch0.begin(), changed_epoch0.end(), m.changed_epoch.begin());
  std::copy(blks0.begin(), blks0.end(), m.plan.blk.begin());
  return ndiff;
}

// Runs the LZ77 stage; returns the commands of every metablock back to back.
extern "C" long sim_lz77(int q, int lgwin, const u8* in, u32 n, BrCmd* cmds_out, u32 cmds_cap,
                         u32* mb_info /* [5*i]: start,end,ncmd,compress,cmd_off */, u32 mb_cap, u32* stats) {
  SimStream* m = sim_setup(q, lgwin, n, in, n);
  if (!m) return -1;
  if (const int e = sim_lz77_fixpoint(*m)) { delete m; return e; }
  u32 nm = m->s.counters[1], total = m->s.counters[2];
  if (total > cmds_cap || nm > mb_cap) { delete m; return -2; }
  memcpy(cmds_out, m->cmds_all.data(), (size_t)total * sizeof(BrCmd));
  for (u32 i = 0; i < nm; ++i) {
    const BrMetaBlock& b = m->s.mbs[i];
    mb_info[5 * i] = b.start; mb_info[5 * i + 1] = b.end; mb_info[5 * i + 2] = b.ncmd;
    mb_info[5 * i + 3] = b.compress; mb_info[5 * i + 4] = b.cmd_off;
  }
  stats[0] = (u32)m->iterations; stats[1] = (u32)m->block_runs; stats[2] = m->s.P.nblocks;
  delete m;
  return nm;
}

// The position index of a one-shot job as the sim builds it (the counterpart of the product's br_debug_sort hook).
extern "C" int sim_debug_sort(int q, int lgwin, const u8* in, u32 n, u32* S_out, u32* seg_out) {
  SimStream* m = sim_setup(q, lgwin, n, in, n);
  if (!m) return 0;
  memcpy(S_out, m->S.data(), (size_t)n * 4);
  memcpy(seg_out, m->seg.data(), (size_t)(m->s.P.nbuckets + 2) * 4);
  delete m;
  return 1;
}

#ifdef BR_SIM_ENTROPY
// ---- the data-parallel entropy stage (br_entropy2.h), run element by element
struct SimEnt {
  BrEnt e;
  std::vector<u32> lit_ord, cmd_pos, dist_ord, lit_pos, lit_cmd, lit_len, cmd_len, lit_bit_base, cmd_mb, outbits;
  std::vector<u16> dist_sym;
  std::vector<BrMbAux> aux;
  std::vector<u8> scratch;
  BrMbLayout L;
};
// k_mb_setup and (qualities 4..9) k_split for one metablock, with a one-thread CTA
static void sim_split_mb(const BrStream& s, const BrEnt& e, const BrMetaBlock& mb, BrMbAux& a, u8* sc, u32* smem) {
  BrMbMem* M = (BrMbMem*)sc;
  br_mb_aux_init(a, mb, e, s.P.disable_ctx ? 1u : br_decide_context_modeling(s, mb.start, mb.end - mb.start, M->sc.rle_syms));
  if (s.P.mb_kind) return;
  for (int cat = 0; cat < 3; ++cat) {
    const BrSplitCat k = br_split_cat(cat, a.which);
    const u32 nblk = br_mb2_nblk(cat, mb.nlit, mb.ncmd);
    br_split_cta(s, e, mb, a, cat, k.A, k.nc, k.min_block, k.thr, a.nsym[cat], br_mb2_types(sc, a, cat, nblk),
                 br_mb2_lengths(sc, a, cat, nblk), BR_SPLIT_HIST(M, cat), smem);
  }
}
// E0 and E1 (the pipeline's launch_e01) over the commands cmds[0 .. C) of the metablocks s.mbs[0 .. nm), with E.e wired
// to E's arrays, those of the later stages sized too.  E.L: the metablocks' layout; the scratch starts filled with sc_fill.
static void sim_e01(const BrStream& s, u32 nm, const BrCmd* cmds, u32 C, SimEnt& E, u8 sc_fill) {
  BrEnt& e = E.e;
  e.cmds = cmds; e.total_cmds = C;
  E.lit_ord.assign(C + 1, 0); E.cmd_pos.assign(C + 1, 0); E.dist_ord.assign(C + 1, 0);
  for (u32 i = 0; i < C; ++i) {
    u32 a, b, d; br_cmd_scan_inputs(cmds[i], &a, &b, &d);
    E.lit_ord[i + 1] = E.lit_ord[i] + a; E.cmd_pos[i + 1] = E.cmd_pos[i] + b; E.dist_ord[i + 1] = E.dist_ord[i] + d;
  }
  e.total_lits = E.lit_ord[C]; e.total_dist = E.dist_ord[C];
  E.lit_pos.assign(e.total_lits + 1, 0); E.lit_cmd.assign(e.total_lits + 1, 0); E.dist_sym.assign(e.total_dist + 1, 0);
  E.lit_len.assign(e.total_lits + 2, 0); E.cmd_len.assign(C + 2, 0); E.lit_bit_base.assign(C + 1, 0); E.cmd_mb.assign(C + 1, 0);
  E.aux.assign(nm, BrMbAux());
  for (u32 i = 0; i < nm; ++i)
    for (u32 c = s.mbs[i].cmd_off; c < s.mbs[i].cmd_off + s.mbs[i].ncmd; ++c) E.cmd_mb[c] = i;
  E.scratch.assign(E.L.scratch_bytes + 256, sc_fill); E.outbits.assign(E.L.out_words + 64, 0);
  e.lit_ord = E.lit_ord.data(); e.cmd_pos = E.cmd_pos.data(); e.dist_ord = E.dist_ord.data();
  e.lit_pos = E.lit_pos.data(); e.lit_cmd = E.lit_cmd.data(); e.dist_sym = E.dist_sym.data();
  e.lit_len = E.lit_len.data(); e.cmd_len = E.cmd_len.data(); e.lit_bit_base = E.lit_bit_base.data();
  e.cmd_mb = E.cmd_mb.data(); e.aux = E.aux.data(); e.scratch = E.scratch.data(); e.scratch_off = E.L.scratch_off.data();
  e.outbits = E.outbits.data(); e.out_off = E.L.out_off.data();
  for (u32 c = 0; c < C; c += BR_WARP) br_expand_cmds(e, c);
}
static void sim_entropy2(SimStream& m, SimEnt& E) {
  BrStream& s = m.s;
  u32 nm = s.counters[1], C = s.counters[2];
  BrEnt& e = E.e;
  br_mb_layout(s.P, s.mbs, nm, E.L);
  sim_e01(s, nm, m.cmds_all.data(), C, E, 0);
  std::vector<u32> smem(64 * 1024);
  for (u32 i = 0; i < nm; ++i) {
    const BrMetaBlock& mb = s.mbs[i];
    if (!mb.compress) continue;
    BrMbAux& a = E.aux[i];
    u8* sc = E.scratch.data() + E.L.scratch_off[i];
    sim_split_mb(s, e, mb, a, sc, smem.data());
    if (s.P.mb_kind) { br_prep_flat(s, e, mb, a, sc, E.outbits.data() + E.L.out_off[i]); continue; }
    br_prep_codes(s, mb, a, sc, E.outbits.data() + E.L.out_off[i]);
  }
  for (u32 o = 0; o < e.total_lits; ++o) br_lit_bits(s, e, o);
  for (u32 i = 0; i < C; ++i) br_cmd_bits(s, e, i);
  { u32 acc = 0; for (u32 o = 0; o <= e.total_lits; ++o) { u32 v = E.lit_len[o]; E.lit_len[o] = acc; acc += v; } }
  { u32 acc = 0; for (u32 i = 0; i <= C; ++i) { u32 v = E.cmd_len[i]; E.cmd_len[i] = acc; acc += v; } }
  for (u32 i = 0; i < C; ++i) br_emit_cmd(s, e, i);
  for (u32 o = 0; o < e.total_lits; ++o) br_emit_lit(s, e, o);
}

// Full pipeline; returns compressed size or negative error.  cuts: see br_pipeline.h BrCuts.
// stats: nstats words (SIM_ST_*).
static long sim_compress_impl(int q, int lgwin, u32 size_hint, const u8* in, u32 n, u8* out, size_t out_cap, u32* stats,
                              const BrCuts* cuts, const SimSched* sched = nullptr, u32 nstats = SIM_ST_MODEL_COST + 1) {
  if (n == 0) { if (out_cap < 1) return -3; out[0] = 6; return 1; }
#ifdef BR_SIM_DEBUG
  memset(br_sim_cnt, 0, sizeof(br_sim_cnt)); memset(br_sim_bnd, 0, sizeof(br_sim_bnd));
#endif
  SimStream* m = sim_setup(q, lgwin, size_hint, in, n, cuts, sched);
  if (!m) return -1;
  BrStream& s = m->s;
  std::vector<u8> res;
  int rounds = 0;
  for (;;) {
    ++rounds;
    if (const int e = sim_lz77_fixpoint(*m)) { delete m; return e; }
    u32 nm = s.counters[1];
    SimEnt E;
    sim_entropy2(*m, E);
    if (getenv("BR_SIM_CHUNKAT")) { const u32 at = (u32)atoi(getenv("BR_SIM_CHUNKAT"));
      for (u32 k = 0; k < s.P.nblocks; ++k) if (s.bin[k].pos <= at + 3000 && s.bin[k].end + 3000 > at)
        fprintf(stderr, "CHUNK %u [%u,%u) blk [%u,%u) start %u dc %d %d %d %d rh %u se %u | out_pos %u ncmd %u dc %d %d %d %d valid %u epoch %u\n", k, s.bin[k].pos, s.bin[k].end, s.bin[k].blk_start, s.bin[k].blk_end,
                s.bin[k].start_pos, s.bin[k].dc[0], s.bin[k].dc[1], s.bin[k].dc[2], s.bin[k].dc[3], s.bin[k].apply_rh, s.bin[k].store_end, s.bout[k].out_pos, s.bout[k].ncmd, s.bout[k].dc[0], s.bout[k].dc[1], s.bout[k].dc[2], s.bout[k].dc[3], s.bout[k].valid, s.bout[k].epoch); }
    if (getenv("BR_SIM_MBS")) {   // the last metablock's commands (debugging against an instrumented reference)
      u32 which = nm - 1;
      if (getenv("BR_DBG_MB")) for (u32 i = 0; i < nm; ++i) if (s.mbs[i].start == (u32)atoi(getenv("BR_DBG_MB"))) which = i;
      const BrMetaBlock& lm = s.mbs[which]; u32 pos = lm.start;
      for (u32 i = 0; i < lm.ncmd; ++i) { const BrCmd& c = m->cmds_all[lm.cmd_off + i];
        fprintf(stderr, "SIMCMD %u ins %u copy %u dprefix %u dextra %u\n", pos, c.insert_len, c.copy_len & 0x1FFFFFF, c.dist_prefix & 0x3FF, c.dist_extra); pos += c.insert_len + (c.copy_len & 0x1FFFFFF); }
    }
    if (getenv("BR_SIM_MBS"))   // metablock table (debugging against an instrumented reference)
      for (u32 i = 0; i < nm; ++i) fprintf(stderr, "SIMMB start %u bytes %u ncmd %u nlit %u last %u compress %u bits %u\n", s.mbs[i].start, s.mbs[i].end - s.mbs[i].start,
                                           s.mbs[i].ncmd, s.mbs[i].nlit, s.mbs[i].is_last, s.mbs[i].compress, s.mbs[i].out_bits);
    // stream assembly (br_assemble.h): the scan, then the copies word by word, as k_assemble_copy does them
    std::vector<u32> outw(E.L.out_cap / 4 + 16, 0);
    std::vector<BrCopyDesc> desc(nm + 1);
    std::vector<u64> cut_end((cuts ? cuts->n : 0) + 2, 0), stream_end(s.P.multi + 2, 0);
    u32 r4[4] = {0, 0, 0, 0};
    br_assemble_scan(s, E.L.out_off.data(), outw.data(), desc.data(), r4, m->plan.with_header, cuts ? cuts->kind : nullptr,
                     cut_end.data(), stream_end.data());
    const bool redo = r4[2] != 0;
    if (!redo) {
      for (u32 i = 0; i < nm; ++i)
        for (u32 w = 0, nw = br_copy_words(desc[i]); w < nw; ++w) br_copy_word(desc[i], w, E.outbits.data(), s.data, outw.data());
      const u64 total = ((u64)r4[1] << 32) | r4[0];
      res.assign((u8*)outw.data(), (u8*)outw.data() + total);
      if (cuts && cuts->end_bit) for (u32 i = 0; i < r4[3]; ++i) cuts->end_bit[i] = cut_end[i];
      if (cuts && cuts->stream_end) for (u32 i = 0; i < s.P.multi; ++i) cuts->stream_end[i] = stream_end[i];
      break;
    }
    if (rounds > (int)m->plan.max_rounds) { delete m; return -4; }
  }
  m->st[SIM_ST_LAUNCHES] = (u32)m->iterations; m->st[SIM_ST_WALKS] = (u32)m->block_runs; m->st[SIM_ST_CHUNKS] = s.P.nblocks;
  m->st[SIM_ST_ROUNDS] = (u32)rounds; m->st[SIM_ST_MODEL_COST] = (u32)m->model_cost; m->st[SIM_ST_RAN_CAP] = m->plan.ran_cap;
#ifdef BR_SIM_DEBUG
  m->st[SIM_ST_PREDICT_OK] = (u32)br_sim_bnd[0]; m->st[SIM_ST_PREDICT_NO] = (u32)br_sim_bnd[1];
#endif
  memcpy(stats, m->st, std::min<u32>(nstats, SIM_ST_WORDS) * sizeof(u32));
  delete m;
  if (res.size() > out_cap) return -3;
  memcpy(out, res.data(), res.size());
  return (long)res.size();
}
extern "C" long sim_compress(int q, int lgwin, const u8* in, u32 n, u8* out, size_t out_cap, u32* stats) {
  return sim_compress_impl(q, lgwin, n, in, n, out, out_cap, stats, nullptr);
}
extern "C" long sim_compress_cuts(int q, int lgwin, u32 size_hint, const u8* in, u32 n, const u32* cut_pos, const u32* cut_kind, u32 ncuts,
                                  int is_final, int with_header, int finish_empty, u64* end_bit, u8* out, size_t out_cap, u32* stats,
                                  int lgblock, int disable_ctx, u32 stream_offset) {
  const BrCuts c = {cut_pos, cut_kind, ncuts, is_final, with_header, finish_empty, end_bit, lgblock, disable_ctx, stream_offset, nullptr};
  return sim_compress_impl(q, lgwin, size_hint, in, n, out, out_cap, stats, &c);
}

// E4 alone on synthetic metablocks: the counterpart of the product's br_debug_codes hook, with its arguments.  A job of at
// most BR_CODE_WARP_MAX codes takes the warp workers' functions with one lane, as br_prep_codes does; a larger one the
// thread workers' functions over a pool of tree areas, each worker taking the codes k_codes gives it, in its order.  The
// scratch, the warps' shared copy and the tree areas start with the device hook's pattern.
extern "C" int sim_debug_codes(u32 n_mbs, const u32* counts, const u32* histos, u32 code_ctas, u32* H, u8* depth, u16* bits,
                               u32* offsets, u32* out, u32 out_words, u32* info) {
  std::vector<BrMetaBlock> mbs; std::vector<BrMbAux> aux; BrMbLayout L; std::vector<u8> sc;
  if (n_mbs == 0 || !br_codes_synth(counts, n_mbs, histos, 0xA5, mbs, aux, L, sc)) return 0;
  BrStream s; memset(&s, 0, sizeof(s));
  s.P.n = n_mbs * BR_SYNTH_MB_BYTES; s.mbs = mbs.data();
  br_bind_tables(s, g_t.blob.data(), g_t.log2tab.data(), (u32)g_t.log2tab.size());
  std::vector<u32> outbits(L.out_words + 64, 0), code_base(n_mbs + 1, 0);
  for (u32 i = 0; i < n_mbs; ++i) code_base[i + 1] = code_base[i] + (mbs[i].compress ? br_mb_code_count(aux[i]) : 0u);   // k_code_count + scan
  const u32 total = code_base[n_mbs];
  const bool warps = total <= BR_CODE_WARP_MAX;
  const u32 nwk = warps ? total : (code_ctas ? code_ctas : (L.code_workers + 63) / 64) * 64;
  std::vector<BrHTree> pool(warps ? 1 : (size_t)nwk * BR_CODE_TREE_NODES);
  memset(pool.data(), 0xA5, pool.size() * sizeof(BrHTree));
  std::vector<u8> smem(sizeof(BrCodeSmem), 0xA5);
  BrCodeSmem* S = (BrCodeSmem*)smem.data();
  auto code = [&](u32 t, u32 wk, bool store) {
    const u32 m = br_upper_index(code_base.data(), n_mbs, t);
    u8* msc = sc.data() + L.scratch_off[m];
    u32* mout = outbits.data() + L.out_off[m];
    if (warps) { if (store) br_code_store_warp(mbs[m], aux[m], msc, t - code_base[m], S, mout); else br_code_build_warp(mbs[m], aux[m], msc, t - code_base[m], S); }
    else { BrHTree* tree = pool.data() + (size_t)wk * BR_CODE_TREE_NODES;
           if (store) br_code_store(mbs[m], aux[m], msc, t - code_base[m], tree, mout); else br_code_build(mbs[m], aux[m], msc, t - code_base[m], tree); }
  };
  for (int store = 0; store < 2; ++store) {
    if (store)
      for (u32 i = 0; i < n_mbs; ++i)
        if (mbs[i].compress) br_mb_header(s, mbs[i], aux[i], sc.data() + L.scratch_off[i], outbits.data() + L.out_off[i]);
    for (u32 wk = 0; wk < nwk; ++wk)
      for (u32 t = wk; t < total; t += nwk) code(t, wk, store != 0);
  }
  br_codes_collect(mbs, aux, L, sc.data(), H, depth, bits, offsets);
  for (u32 i = 0; i < n_mbs; ++i) {
    if (!mbs[i].compress) continue;
    const size_t have = (i + 1 < n_mbs ? L.out_off[i + 1] : L.out_words) - L.out_off[i];
    memcpy(out + (size_t)i * out_words, outbits.data() + L.out_off[i], 4 * std::min<size_t>(have, out_words));
  }
  info[0] = total; info[1] = warps ? 1u : 2u; info[2] = nwk;
  return 1;
}

// E0..E4 on metablocks the caller describes: the counterpart of the product's br_debug_split hook, with its arguments.  E2
// and E3 by sim_split_mb (one-thread CTAs), E4 by br_prep_codes, metablock by metablock, on a scratch that starts with
// the device hook's pattern.
extern "C" long sim_debug_split(const u8* in, u32 n, const BrCmd* cmds, u32 ncmd, const u32* mbw, u32 n_mbs, int quality,
                                u32 size_hint, int disable_ctx, u32* out, size_t out_cap) {
  if (n == 0 || n_mbs == 0 || quality < 4 || quality > 9) return 0;
  BrStream s; memset(&s, 0, sizeof(s));
  s.P.quality = quality; s.P.n = n; s.P.size_hint = size_hint; s.P.disable_ctx = disable_ctx ? 1u : 0u;
  std::vector<BrMetaBlock> mbs; SimEnt E;
  if (!br_split_synth(s.P, mbw, n_mbs, cmds, ncmd, mbs, E.L)) return 0;
  std::vector<u8> data((size_t)n + 64, 0);
  memcpy(data.data(), in, n);
  s.data = data.data(); s.mbs = mbs.data();
  br_bind_tables(s, g_t.blob.data(), g_t.log2tab.data(), (u32)g_t.log2tab.size());
  sim_e01(s, n_mbs, cmds, ncmd, E, 0xA5);
  std::vector<u32> smem(64 * 1024);
  std::vector<std::vector<u32>> recs;
  for (u32 i = 0; i < n_mbs; ++i) {
    if (!mbs[i].compress) continue;
    u8* msc = E.scratch.data() + E.L.scratch_off[i];
    sim_split_mb(s, E.e, mbs[i], E.aux[i], msc, smem.data());
    recs.emplace_back();
    br_split_record(mbs[i], E.aux[i], msc, recs.back());
    u32* mout = E.outbits.data() + E.L.out_off[i];
    br_prep_codes(s, mbs[i], E.aux[i], msc, mout);
    u32 nbits;
    memcpy(&nbits, msc + br_split_code_end_off(mbs[i], E.aux[i]), 4);
    br_split_record_bits(recs.back(), mout, nbits);
  }
  return (long)br_split_put(recs, out, out_cap);
}
#endif

// ------------------------------------------------------------------ quality 1 (br_q1.h)
#ifdef BR_SIM_ENTROPY
#include "../../brotli_b200/csrc/br_q1_plan.h"
// One stream through the q1 device code with a one-lane warp and a one-thread CTA.
extern "C" long sim_q1_compress_seg(int lgwin, const u8* in, u32 n, const size_t* calls, size_t ncalls, u8* out, size_t out_cap,
                                    int with_header, int end_op, u32 start_bits, u32* end_bit) {
  std::vector<BrQ1Stream> streams; std::vector<BrQ1Frag> frags; std::vector<BrQ1Block> blocks;
  br_q1_plan_stream(lgwin, 0, 0, 0, n, calls, ncalls, streams, frags, blocks, with_header, end_op, start_bits);
  const size_t bound = br_q1_stream_bound(frags, streams[0]);
  std::vector<u8> din((size_t)n + 64, 0); memcpy(din.data(), in, n);
  std::vector<u32> dout(bound / 4 + 16, 0), cmds((size_t)n + 16), hdr(blocks.size() * BR_Q1_HDR_WORDS + 1, 0), counters(16, 0);
  std::vector<u8> lits((size_t)n + 16);
  std::vector<BrQ1Codes> codes(blocks.size() + 1);
  std::vector<int> table((size_t)1 << 17);
  BrQ1 q; memset(&q, 0, sizeof(q));
  q.in = din.data(); q.out = dout.data(); q.cmds = cmds.data(); q.lits = lits.data();
  q.streams = streams.data(); q.frags = frags.data(); q.blocks = blocks.data(); q.codes = codes.data(); q.hdr = hdr.data();
  q.tables = table.data(); q.table_slot = 1u << 17; q.nstreams = 1; q.nfrags = (u32)frags.size(); q.nblocks = (u32)blocks.size();
  q.first_width = 8; q.counters = counters.data(); q.log2tab = g_t.log2tab.data(); q.log2tab_n = (u32)std::min<size_t>(g_t.log2tab.size(), 4096);
  for (u32 f = 0; f < q.nfrags; ++f) {
    if (getenv("BR_SIM_Q1_SHM") && frags[f].size <= 65536) {
      // the on-chip variant (u16 table, input copy aligned like the TMA destination of k_q1_parse_shm)
      std::vector<u16> t16((size_t)1 << 16, 0);
      const u32 a0 = frags[f].start & ~15u;
      std::vector<u8> buf((size_t)65536 + 128, 0);
      size_t nb = (size_t)(frags[f].start - a0) + frags[f].size + 16;
      if (a0 + nb > din.size()) nb = din.size() - a0;
      memcpy(buf.data(), din.data() + a0, nb);
      br_q1_parse_fragment_shm(q, f, t16.data(), buf.data());
    } else br_q1_parse_fragment(q, f, table.data());
  }
  BrQ1Smem* sm = new BrQ1Smem();
  for (u32 b = 0; b < q.nblocks; ++b) br_q1_prep_block(q, b, sm);
  delete sm;
  br_q1_chain_stream(q, 0);
  u32 scratch[8];
  for (u32 b = 0; b < q.nblocks; ++b) br_q1_emit_block(q, b, scratch);
  const size_t sz = streams[0].out_bytes;
  if (end_bit) *end_bit = streams[0].end_bit;
  if (sz > out_cap) return -1;
  memcpy(out, dout.data(), sz);
  return (long)sz;
}
extern "C" long sim_q1_compress(int lgwin, const u8* in, u32 n, const size_t* calls, size_t ncalls, u8* out, size_t out_cap) {
  return sim_q1_compress_seg(lgwin, in, n, calls, ncalls, out, out_cap, 1, 2, 0, nullptr);
}
#endif

#ifdef BR_SIM_ENTROPY
#include "../../brotli_b200/csrc/br_driver.h"
// A batch of independent streams laid end to end (cuts of kind 3, br_pipeline.h): bounds[k] = end of stream k (bounds[ns-1] = n).
// stream_end[k] receives the byte offset where stream k ends in `out`.
static long sim_compress_multi_impl(int q, int lgwin, const u8* in, u32 n, const u32* bounds, u32 nstreams, u64* stream_end,
                                    u8* out, size_t out_cap, u32* stats, const SimSched* sched, u32 nstats) {
  std::vector<size_t> sizes(nstreams);
  for (u32 k = 0; k < nstreams; ++k) sizes[k] = bounds[k] - (k ? bounds[k - 1] : 0);
  br_driver::GroupCuts g(sizes.data(), nullptr, nstreams);
  const long r = sim_compress_impl(q, lgwin, g.hint, in, n, out, out_cap, stats, &g.c, sched, nstats);
  if (r >= 0 && stream_end) std::copy(g.ends.begin(), g.ends.begin() + nstreams, stream_end);
  return r;
}
extern "C" long sim_compress_multi(int q, int lgwin, const u8* in, u32 n, const u32* bounds, u32 nstreams, u64* stream_end,
                                   u8* out, size_t out_cap, u32* stats) {
  return sim_compress_multi_impl(q, lgwin, in, n, bounds, nstreams, stream_end, out, out_cap, stats, nullptr, SIM_ST_MODEL_COST + 1);
}

// The fixpoint under an explicit schedule (SimSched; its fields replace the BR_SIM_* switches).  One stream, optionally cut
// (cut_pos / cut_kind / ncuts / size_hint as sim_compress_cuts, the stream finished, with its header), or a batch of streams when
// every cut is of kind 3 (stream_end as sim_compress_multi).  stats: SIM_ST_WORDS words.  Returns the compressed size, or
// a negative error (SIM_ERR_CAPACITY: a launch appended more entries than an array of the product holds).
extern "C" long sim_compress_sched(int q, int lgwin, const u8* in, u32 n, const u32* cut_pos, const u32* cut_kind, u32 ncuts,
                                   u32 size_hint, const SimSched* sched, u64* stream_end, u8* out, size_t out_cap, u32* stats) {
  bool batch = ncuts > 0;
  for (u32 i = 0; i < ncuts; ++i) batch = batch && cut_kind[i] == 3;
  if (batch) {
    std::vector<u32> bounds(cut_pos, cut_pos + ncuts); bounds.push_back(n);
    return sim_compress_multi_impl(q, lgwin, in, n, bounds.data(), ncuts + 1, stream_end, out, out_cap, stats, sched, SIM_ST_WORDS);
  }
  const BrCuts c = {cut_pos, cut_kind, ncuts, 1, 1, 0, nullptr, 0, 0, 0, nullptr};
  return sim_compress_impl(q, lgwin, size_hint, in, n, out, out_cap, stats, ncuts ? &c : nullptr, sched, SIM_ST_WORDS);
}

// ------------------------------------------------------------------ the C API's host driver (br_driver.h) over the sim
// The driver's backend: sim_compress_impl and sim_q1_compress_seg stand in for the device pipelines.
static int sim_backend_compress(const br_driver::Params& p, u32 size_hint, const u8* in, size_t n, const BrCuts* cuts, u8* out,
                                size_t cap, size_t* got, std::vector<u8>* vec) {
  if (!br_driver::supported(p) || n == 0 || n > (1u << 30)) return 0;
  std::vector<u8> res(n + n / 2 + 4096 + 64 * (size_t)(cuts ? cuts->n : 0));
  u32 st[SIM_ST_WORDS];
  const long r = sim_compress_impl(p.quality, br_driver::window_of(p), size_hint, in, (u32)n, res.data(), res.size(), st, cuts);
  if (r < 0) return 0;
  res.resize((size_t)r);
  *got = res.size();
  if (vec) { vec->swap(res); return 1; }
  if (res.size() > cap) return 2;
  memcpy(out, res.data(), res.size());
  return 1;
}
static int sim_backend_q1_segment(int lgwin, const u8* in, size_t n, const std::vector<size_t>& calls, int with_header, int end_op,
                                  u32 start_bits, u32* end_bit, std::vector<u8>& out) {
  out.resize(2 * n + 100000);
  const long r = sim_q1_compress_seg(lgwin, in, (u32)n, calls.data(), calls.size(), out.data(), out.size(), with_header, end_op,
                                     start_bits, end_bit);
  if (r < 0) return 0;
  out.resize((size_t)r);
  return 1;
}
static const br_driver::Backend kSimBackend = {sim_backend_compress, sim_backend_q1_segment};

// A sequence of BrotliEncoderCompressStream calls through the driver, as tests/brotli_libs.py ref_stream_ops sends them to
// the reference: quality, lgwin and nparams further (BrotliEncoderParameter id, value) pairs; call i hands sizes[i] bytes
// of `data` (from where the call before stopped) with operation ops[i], and the output is drained in 64 KiB pieces until
// the input is taken and no output is left.  q1_segment_bytes (0: the product's) is the input of one quality-1 segment.
// Returns the stream's size in `out`, -1 when a call fails, -2 when `cap` is too small.
extern "C" long sim_stream_ops(int q, int lgwin, const u32* param_ids, const u32* param_vals, u32 nparams, const u8* data,
                               const size_t* sizes, const int* ops, size_t n_ops, size_t q1_segment_bytes, u8* out, size_t cap) {
  br_driver::Stream s{br_driver::BrAlloc<u8>()};
  br_driver::set_parameter(s.params, BROTLI_PARAM_QUALITY, (u32)q);
  br_driver::set_parameter(s.params, BROTLI_PARAM_LGWIN, (u32)lgwin);
  for (u32 i = 0; i < nparams; ++i)
    if (!br_driver::set_parameter(s.params, (BrotliEncoderParameter)param_ids[i], param_vals[i])) return -1;
  if (q1_segment_bytes) s.q1_segment_bytes = q1_segment_bytes;
  std::vector<u8> buf(1 << 16);
  size_t got = 0, pos = 0;
  try {
    for (size_t i = 0; i < n_ops; ++i) {
      size_t avail_in = sizes[i];
      const u8* next_in = data + pos;
      pos += sizes[i];
      for (;;) {
        size_t avail_out = buf.size();
        u8* next_out = buf.data();
        if (!br_driver::compress_stream(kSimBackend, s, (BrotliEncoderOperation)ops[i], &avail_in, &next_in, &avail_out, &next_out,
                                        nullptr))
          return -1;
        const size_t k = buf.size() - avail_out;
        if (got + k > cap) return -2;
        memcpy(out + got, buf.data(), k);
        got += k;
        if (avail_in == 0 && !br_driver::has_more_output(s)) break;
      }
    }
  } catch (const std::bad_alloc&) { return -1; }
  return (long)got;
}

// br_driver::plan_groups: group_of[i] receives the group of stream i, or -1 for a stream that goes one by one.  Returns the
// number of groups.
extern "C" size_t sim_plan_groups(const size_t* sizes, size_t count, long* group_of) {
  std::vector<std::vector<size_t>> groups;
  std::vector<size_t> single;
  br_driver::plan_groups(sizes, count, groups, single);
  for (size_t i : single) group_of[i] = -1;
  for (size_t g = 0; g < groups.size(); ++g)
    for (size_t i : groups[g]) group_of[i] = (long)g;
  return groups.size();
}

// BrotliEncoderCompress through the driver: *encoded_size is the capacity of `out` in, the size out.  Returns the BROTLI_BOOL.
extern "C" int sim_compress_oneshot(int q, int lgwin, const u8* in, size_t n, size_t* encoded_size, u8* out) {
  return br_driver::compress_oneshot(kSimBackend, q, lgwin, BROTLI_MODE_GENERIC, n, in, encoded_size, out);
}
#endif
