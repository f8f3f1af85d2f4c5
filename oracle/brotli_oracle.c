/* oracle/brotli_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * A plain-C, single-threaded CPU restatement of the google/brotli encoder hot
 * path for qualities 5..9 (bucket-ring hashers H5/H6 and their SIMD twins
 * H58/H68) and the greedy per-metablock entropy pipeline, plus -- as groundwork
 * for SURVEY.md section 8f rank 1 -- qualities 2..4 (single-slot / sweep hashers
 * H2, H3, H4, H54, fast / trivial / context-free meta-block stores), for one-shot
 * BrotliEncoderCompress(quality, lgwin, GENERIC, n, ...) calls.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may
 * load this library; brotli_b200/ never does.  Parity is PINNED: the
 * restatement is checked bit-for-bit against the compiled reference
 * (oracle/_ref/libbrotli_ref.so) in tests/test_oracle.py, because the
 * reference ships no encoder golden vectors (SURVEY.md section 0, T7).
 *
 * Differences in formulation (results identical):
 *   - no ring buffer: the whole input is addressed by absolute position; the
 *     reference's ring-wrap skip rules are evaluated on (pos & ring_mask);
 *   - the one byte the reference may read just past the current input block
 *     (hash_longest_match64_inc.h:196,245) is modelled by stale_byte();
 *   - SIMD hashers H58/H68 are restated in their scalar H5/H6 form.
 *
 * Every function cites the reference file:line it follows (paths relative to
 * /root/reference/c/enc unless noted).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------ tables */
static uint8_t  g_size_bits[32];
static uint32_t g_offsets[32];
static const uint8_t* g_dict;         /* 122784 bytes, RFC 7932 appendix A */
static const uint16_t* g_hash_words;  /* dictionary_hash_inc.h:2 */
static const uint8_t* g_hash_lengths; /* dictionary_hash_inc.h:987 */
static const uint8_t* g_ctx_lut;      /* common/context.c */
static uint8_t* g_blob;
static double g_log2_small[256];

/* fast_log.c:13 -- literals carry an 'f' suffix, i.e. float-rounded. */
static void init_log2(void) {
  int i;
  g_log2_small[0] = 0.0;
  for (i = 1; i < 256; ++i) g_log2_small[i] = (double)(float)log2((double)i);
}
/* fast_log.h:51 FastLog2 */
static double fast_log2(size_t v) {
  if (v < 256) return g_log2_small[v];
  return log2((double)v);
}
double oracle_fast_log2(size_t v) { return fast_log2(v); }

/* Edge counters: how often the entropy stage took the branches that ordinary data rarely reaches, so that a test
 * can prove its input still reaches the branch it was built for (tests/entropy_cases.py).  They only count; the
 * output never depends on them.  A metablock replaced by a raw one (encode.c:604) leaves them as they were.
 *   retry_*: count_limit doublings in BrotliCreateHuffmanTree for symbol trees (depth 15; told apart by alphabet
 *       size: 256 literals, 704 commands, 64 / 140 distances, other: block switches and context maps) and the
 *       code-length code (retry_cl, depth 5), and in BrotliBuildAndStoreHuffmanTreeFast (retry_fast, depth 14)
 *   simple_nsym1..4, simple_select0/1: codes stored as simple prefix codes by NSYM; for NSYM 4 the tree-select bit
 *   rle_lt16 / rle_lt28 / rle_full: exits of BrotliOptimizeHuffmanCountsForRle (its nonzeros < 5 exit cannot be
 *       taken behind the first one); rle_holes: counts filled
 *   reps7 / reps11: the reps == 7 (non-zero) and reps == 11 (zero) special cases of the code-length run writers
 *   rle_use_nz / rle_use_z: DecideOverRleUse chose runs for a tree of more than 50 symbols
 *   ctx_nc1/2/3/13: compressed metablocks (quality 4+) by literal context count; lit_cap_nc*: those whose literal
 *       split reached the 256 / nc type cap; split_back: blocks merged into the type before last (action 2)
 *   max_lit_types / max_lit_trees / max_cmd_types / max_dist_types: per metablock
 *   max_insert / max_copy / max_block_len / max_distance: the longest emitted (distance: explicit codes only)
 *   codes: the literal, command and distance prefix codes stored by compressed metablocks, summed
 *   rle_good / rle_stride: smoothed histograms with runs marked good_for_rle / with a stride of counts averaged
 *   cl_single: code-length codes of one symbol (stored with zero bits); cl_skip2 / cl_skip3: HSKIP 2 / 3;
 *       cl_trim: code-length codes whose trailing zero lengths are left out
 * The same for the match search (find_longest_match, tests/test_search_probe.py):
 *   srch_dc_len2: searches won by a len-2 distance-cache match; srch_ring_break: the ring-buffer stop
 *       (cur_m + best_len > rmask); srch_ring_skip: a candidate skipped by prev_m + best_len > rmask;
 *   srch_tie_max: a candidate as long as a best length that already equals max_length (the stale byte decides);
 *   srch_wrap_cut: a ring cut short by a wrapped uint16 counter (oracle_search_probe);
 *   srch_dict_hit: a static-dictionary item taken; srch_gate_closed: the dictionary gate (hash.h:186) closed
 * And for the greedy block splitter (splitter_finish_block, tests/split_cases.py), counted at every block decision:
 *   split_tie: a block kept apart from a new type only because a diff equals the threshold exactly (`>` against `>=`);
 *   back_tie: a block merged, not sent back to the type before last, only because diff[1] == diff[0] - 20 exactly;
 *   split_clamp: a histogram of cost below 1 bit per symbol, raised to its symbol count (bit_cost.c:35);
 *   split_pad / split_pad_empty: a final block shorter than the shortest block, padded to it (empty: the symbols
 *       ended exactly at a block's end); split_grow: a second merge in a row that grows the target block size;
 *   cmd_cap / dist_cap: compressed metablocks whose command / distance split reached 256 types */
#define EDGE_FIELDS(X) X(retry_lit) X(retry_cmd) X(retry_dist) X(retry_other) X(retry_cl) X(retry_fast) \
  X(simple_nsym1) X(simple_nsym2) X(simple_nsym3) X(simple_nsym4) X(simple_select0) X(simple_select1) X(rle_lt16) X(rle_lt28) X(rle_full) X(rle_holes) \
  X(reps7) X(reps11) X(rle_use_nz) X(rle_use_z) X(ctx_nc1) X(ctx_nc2) X(ctx_nc3) X(ctx_nc13) X(lit_cap_nc1) \
  X(lit_cap_nc2) X(lit_cap_nc3) X(lit_cap_nc13) X(split_back) X(max_lit_types) X(max_lit_trees) X(max_cmd_types) \
  X(max_dist_types) X(max_insert) X(max_copy) X(max_block_len) X(max_distance) X(codes) \
  X(rle_good) X(rle_stride) X(cl_single) X(cl_skip2) X(cl_skip3) X(cl_trim) \
  X(srch_dc_len2) X(srch_ring_break) X(srch_ring_skip) X(srch_tie_max) X(srch_wrap_cut) X(srch_dict_hit) X(srch_gate_closed) \
  X(split_tie) X(back_tie) X(split_clamp) X(split_pad) X(split_pad_empty) X(split_grow) X(cmd_cap) X(dist_cap)
#define EDGE_MEMBER(f) uint64_t f;
#define EDGE_NAME(f) #f ","
static _Thread_local struct { EDGE_FIELDS(EDGE_MEMBER) } g_edge;   /* per thread: callers may run the oracle in a pool */
#define EDGE_MAX(f, v) do { if ((uint64_t)(v) > g_edge.f) g_edge.f = (uint64_t)(v); } while (0)
void oracle_edge_stats_reset(void) { memset(&g_edge, 0, sizeof(g_edge)); }
/* The counters as uint64 words in the order of oracle_edge_stats_names(); returns how many there are. */
size_t oracle_edge_stats(uint64_t* out, size_t cap) {
  const size_t n = sizeof(g_edge) / sizeof(uint64_t);
  if (out) memcpy(out, &g_edge, (cap < n ? cap : n) * sizeof(uint64_t));
  return n;
}
const char* oracle_edge_stats_names(void) { return EDGE_FIELDS(EDGE_NAME); }

int oracle_init(const uint8_t* blob, size_t len) {
  const uint8_t* p;
  if (len != 8 + 32 + 128 + 122784 + 65536 + 32768 + 2048) return 0;
  free(g_blob);
  g_blob = (uint8_t*)malloc(len);
  memcpy(g_blob, blob, len);
  p = g_blob + 8;
  memcpy(g_size_bits, p, 32); p += 32;
  memcpy(g_offsets, p, 128); p += 128;
  g_dict = p; p += 122784;
  g_hash_words = (const uint16_t*)p; p += 65536;
  g_hash_lengths = p; p += 32768;
  g_ctx_lut = p;
  init_log2();
  return 1;
}

/* command.c:15-24 / RFC 7932 section 5 */
static const uint32_t kInsBase[24] = {0, 1, 2, 3, 4, 5, 6, 8, 10, 14, 18, 26,
    34, 50, 66, 98, 130, 194, 322, 578, 1090, 2114, 6210, 22594};
static const uint32_t kInsExtra[24] = {0, 0, 0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4,
    4, 5, 5, 6, 7, 8, 9, 10, 12, 14, 24};
static const uint32_t kCopyBase[24] = {2, 3, 4, 5, 6, 7, 8, 9, 10, 12, 14, 18,
    22, 30, 38, 54, 70, 102, 134, 198, 326, 582, 1094, 2118};
static const uint32_t kCopyExtra[24] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 2, 2, 3,
    3, 4, 4, 5, 5, 6, 7, 8, 9, 10, 24};
/* common/constants.c:10 / RFC 7932 section 6 block count codes */
static const uint16_t kBlockLenOffset[26] = {1, 5, 9, 13, 17, 25, 33, 41, 49,
    65, 81, 97, 113, 145, 177, 209, 241, 305, 369, 497, 753, 1265, 2289, 4337,
    8433, 16625};
static const uint8_t kBlockLenNbits[26] = {2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4,
    5, 5, 5, 5, 6, 6, 7, 8, 9, 10, 11, 12, 13, 24};

static uint32_t log2floor(size_t n) {
  uint32_t r = 0;
  while (n >>= 1) ++r;
  return r;
}

/* -------------------------------------------------------------- bit writer */
/* write_bits.h:33 BrotliWriteBits (LSB first; storage pre-zeroed ahead) */
typedef struct { uint8_t* buf; size_t ix; } BitW;
static void wbits(BitW* w, size_t n, uint64_t bits) {
  uint8_t* p = &w->buf[w->ix >> 3];
  uint64_t v = (uint64_t)*p;
  size_t i;
  v |= bits << (w->ix & 7);
  for (i = 0; i < 8; ++i) p[i] = (uint8_t)(v >> (8 * i));
  w->ix += n;
}

/* ---------------------------------------------------------------- commands */
typedef struct {
  uint32_t insert_len, copy_len, dist_extra;
  uint16_t cmd_prefix, dist_prefix;
} Cmd;

/* command.h:31 */
static uint16_t ins_code(size_t n) {
  if (n < 6) return (uint16_t)n;
  if (n < 130) { uint32_t nb = log2floor(n - 2) - 1u;
    return (uint16_t)((nb << 1) + ((n - 2) >> nb) + 2); }
  if (n < 2114) return (uint16_t)(log2floor(n - 66) + 10);
  if (n < 6210) return 21;
  if (n < 22594) return 22;
  return 23;
}
/* command.h:49 */
static uint16_t copy_code(size_t n) {
  if (n < 10) return (uint16_t)(n - 2);
  if (n < 134) { uint32_t nb = log2floor(n - 6) - 1u;
    return (uint16_t)((nb << 1) + ((n - 6) >> nb) + 4); }
  if (n < 2118) return (uint16_t)(log2floor(n - 70) + 12);
  return 23;
}
/* command.h:62 CombineLengthCodes */
static uint16_t combine_codes(uint16_t ic, uint16_t cc, int use_last) {
  uint16_t bits64 = (uint16_t)((cc & 7u) | ((ic & 7u) << 3u));
  if (use_last && ic < 8u && cc < 16u) return (cc < 8u) ? bits64 : (bits64 | 64u);
  { uint32_t off = 2u * ((cc >> 3u) + 3u * (ic >> 3u));
    off = (off << 5u) + 0x40u + ((0x520D40u >> off) & 0xC0u);
    return (uint16_t)(off | bits64); }
}
static uint16_t length_code(size_t ins, size_t copy, int use_last) {
  return combine_codes(ins_code(ins), copy_code(copy), use_last);
}
/* prefix.h:23 PrefixEncodeCopyDistance with NPOSTFIX=0, NDIRECT=0 */
static void prefix_encode_distance(size_t dcode, uint16_t* code, uint32_t* extra) {
  if (dcode < 16) { *code = (uint16_t)dcode; *extra = 0; return; }
  { size_t dist = 4 + (dcode - 16);
    size_t bucket = log2floor(dist) - 1;
    size_t prefix = (dist >> bucket) & 1;
    size_t offset = (2 + prefix) << bucket;
    size_t nbits = bucket;
    *code = (uint16_t)((nbits << 10) | (16 + 2 * (nbits - 1) + prefix));
    *extra = (uint32_t)(dist - offset); }
}
/* command.h:120 InitCommand */
static void init_cmd(Cmd* c, size_t ins, size_t copylen, int delta, size_t dcode) {
  uint32_t d = (uint8_t)((int8_t)delta);
  c->insert_len = (uint32_t)ins;
  c->copy_len = (uint32_t)(copylen | (d << 25));
  prefix_encode_distance(dcode, &c->dist_prefix, &c->dist_extra);
  c->cmd_prefix = length_code(ins, (size_t)((int)copylen + delta),
                              (c->dist_prefix & 0x3FF) == 0);
}
/* command.h:138 InitInsertCommand */
static void init_insert_cmd(Cmd* c, size_t ins) {
  c->insert_len = (uint32_t)ins;
  c->copy_len = 4u << 25;
  c->dist_extra = 0;
  c->dist_prefix = 16;
  c->cmd_prefix = length_code(ins, 4, 0);
}
static uint32_t cmd_copy_len(const Cmd* c) { return c->copy_len & 0x1FFFFFF; }
/* command.h:176 CommandCopyLenCode */
static uint32_t cmd_copy_len_code(const Cmd* c) {
  uint32_t m = c->copy_len >> 25;
  int32_t delta = (int8_t)((uint8_t)(m | ((m & 0x40) << 1)));
  return (uint32_t)((int32_t)(c->copy_len & 0x1FFFFFF) + delta);
}
/* command.h:147 CommandRestoreDistanceCode (NPOSTFIX=NDIRECT=0) */
static uint32_t cmd_restore_dcode(const Cmd* c) {
  uint32_t dcode = c->dist_prefix & 0x3FFu;
  if (dcode < 16) return dcode;
  { uint32_t nbits = c->dist_prefix >> 10;
    uint32_t hcode = dcode - 16;
    uint32_t offset = ((2u + (hcode & 1u)) << nbits) - 4u;
    return offset + c->dist_extra + 16; }
}

/* ------------------------------------------------------------ encoder state */
typedef struct {
  int quality, lgwin, lgblock;
  size_t size_hint;
  /* hasher: quality.h:172 ChooseHasher */
  int hash64;       /* 1: H6/H68 (5-byte hash), 0: H5/H58 (4-byte hash) */
  int bucket_bits, block_bits, ndist;
  size_t hash_type_len, store_lookahead;
  uint16_t* num;
  uint32_t* buckets;
  /* qualities 2..4: hash_longest_match_quickly_inc.h (H2, H3, H4, H54): one position per slot */
  int quick, qk_bits, qk_sweep_bits, qk_hash_len, qk_dict;
  uint32_t* qk_table;
  size_t dict_lookups, dict_matches;
  size_t rmask;     /* ring buffer mask: quality.h:99 ComputeRbBits */
  const uint8_t* data;
  size_t n;
  int dist_cache[16];
  int saved_dist_cache[4];
  size_t last_insert_len;
  Cmd* cmds;
  size_t num_cmds, num_literals;
  size_t last_flush_pos;
  uint8_t prev_byte, prev_byte2;
  uint8_t carry; unsigned carry_bits;   /* encode.c last_bytes_/last_bytes_bits_ */
  uint8_t* out; size_t out_pos, out_cap; int overflow;
  /* probe hook (tests only) */
  void (*cmd_hook)(const Cmd*, size_t, size_t, size_t);
} Enc;

static uint64_t load64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }
static uint32_t load32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }

/* hash_longest_match64_inc.h:23 / hash_longest_match_inc.h:23 HashBytes.
   The 8-byte load may run past the end of the input; only 5 bytes matter
   (multiplier is shifted left by 24) and those always lie inside. */
static size_t hash_key(const Enc* e, size_t pos) {
  if (e->hash64) {
    uint8_t tmp[8] = {0};
    size_t avail = e->n - pos; uint64_t v;
    if (avail >= 8) v = load64(e->data + pos);
    else { memcpy(tmp, e->data + pos, avail); v = load64(tmp); }
    return (size_t)((v * (0x1FE35A7BD3579BD3ull << 24)) >> (64 - 15));
  } else {
    uint32_t h = load32(e->data + pos) * 0x1E35A7BDu;
    return (size_t)(h >> (32 - e->bucket_bits));
  }
}
/* hash_longest_match64_inc.h:107 Store */
static size_t quick_key(const Enc* e, size_t pos);
static void hstore(Enc* e, size_t pos) {
  size_t key;
  if (e->quick) {   /* hash_longest_match_quickly_inc.h:96 Store */
    const size_t off = pos & (size_t)(((1u << e->qk_sweep_bits) - 1u) << 3);
    e->qk_table[(quick_key(e, pos) + off) & (((size_t)1 << e->qk_bits) - 1)] = (uint32_t)pos;
    return;
  }
  key = hash_key(e, pos);
  size_t minor = e->num[key] & ((1u << e->block_bits) - 1);
  e->buckets[(key << e->block_bits) + minor] = (uint32_t)pos;
  ++e->num[key];
}

/* find_match_length.h:20 */
static size_t match_len(const uint8_t* a, const uint8_t* b, size_t limit) {
  size_t i = 0;
  while (i < limit && a[i] == b[i]) ++i;
  return i;
}

/* The reference compares data[cur_ix_masked + best_len]; when best_len equals
   max_length that byte lies at the end of the current input block, i.e. not yet
   written.  encode.c:890 zeroes 7 bytes there during the first lap of the ring
   buffer; on later laps the slot still holds the byte from one ring size ago. */
static uint8_t stale_byte(const Enc* e, size_t pos_end) {
  if (pos_end <= e->rmask) return 0;
  return e->data[pos_end - (e->rmask + 1)];
}
static uint8_t cur_byte(const Enc* e, size_t cur, size_t off, size_t max_length) {
  if (off < max_length) return e->data[cur + off];
  return stale_byte(e, cur + max_length);
}

typedef struct { size_t len, distance, score; int len_code_delta; } SR;

#define SCORE_BASE (30 * 8 * sizeof(size_t))
/* hash.h:123-138 */
static size_t score_normal(size_t len, size_t back) {
  return SCORE_BASE + 135 * len - 30 * log2floor(back);
}
static size_t score_last(size_t len) { return 135 * len + SCORE_BASE + 15; }
static size_t penalty_last(size_t i) { return 39 + ((0x1CA10 >> (i & 0xE)) & 0xE); }

/* hash.h:140 TestStaticDictionaryItem */
static int test_dict_item(size_t len, size_t word_idx, const uint8_t* data,
    size_t max_length, size_t max_backward, size_t max_distance, SR* out) {
  size_t offset = g_offsets[len] + len * word_idx;
  size_t matchlen, backward, score;
  if (len > max_length) return 0;
  matchlen = match_len(data, &g_dict[offset], len);
  if (matchlen + 10 <= len || matchlen == 0) return 0;
  { size_t cut = len - matchlen;
    size_t transform_id = (cut << 2) +
        (size_t)((0x071B520ADA2D3200ull >> (cut * 6)) & 0x3F);
    backward = max_backward + 1 + word_idx + (transform_id << g_size_bits[len]); }
  if (backward > max_distance) return 0;
  score = score_normal(matchlen, backward);
  if (score < out->score) return 0;
  out->len = matchlen;
  out->len_code_delta = (int)len - (int)matchlen;
  out->distance = backward;
  out->score = score;
  return 1;
}
/* hash.h:179 SearchInStaticDictionary; shallow (the quickly hashers) probes one slot instead of two */
static void search_static_dict_n(Enc* e, const uint8_t* data, size_t max_length,
    size_t max_backward, size_t max_distance, SR* out, size_t probes) {
  size_t key, i;
  if (e->dict_matches < (e->dict_lookups >> 7)) { ++g_edge.srch_gate_closed; return; }
  key = ((load32(data) * 0x1E35A7BDu) >> (32 - 14)) << 1;
  for (i = 0; i < probes; ++i, ++key) {
    e->dict_lookups++;
    if (g_hash_lengths[key] != 0) {
      if (test_dict_item(g_hash_lengths[key], g_hash_words[key], data,
                         max_length, max_backward, max_distance, out)) {
        e->dict_matches++;
        ++g_edge.srch_dict_hit;
      }
    }
  }
}
static void search_static_dict(Enc* e, const uint8_t* data, size_t max_length,
    size_t max_backward, size_t max_distance, SR* out) {
  search_static_dict_n(e, data, max_length, max_backward, max_distance, out, 2);
}

/* hash_longest_match_quickly_inc.h:27 HashBytes: HASH_LEN bytes, kHashMul64, top BUCKET_BITS bits */
static size_t quick_key(const Enc* e, size_t pos) {
  uint8_t tmp[8] = {0};
  size_t avail = e->n - pos; uint64_t v;
  if (avail >= 8) v = load64(e->data + pos);
  else { memcpy(tmp, e->data + pos, avail); v = load64(tmp); }
  return (size_t)(((v << (64 - 8 * e->qk_hash_len)) * 0x1FE35A7BD3579BD3ull) >> (64 - e->qk_bits));
}
/* hash_longest_match_quickly_inc.h:147 FindLongestMatch: the last distance, then the BUCKET_SWEEP slots
   key, key+8, ... (mod table size); the position is filed in the slot its own low bits select. */
static void quick_find_longest_match(Enc* e, size_t cur, size_t max_length,
    size_t max_backward, size_t dict_distance, size_t max_distance, SR* out) {
  const uint8_t* data = e->data;
  const size_t sweep = (size_t)1 << e->qk_sweep_bits, mask = ((size_t)1 << e->qk_bits) - 1;
  const size_t best_len_in = out->len;
  const size_t key = quick_key(e, cur);
  const size_t min_score = out->score;
  size_t best_score = out->score, best_len = best_len_in;
  const size_t cached = (size_t)e->dist_cache[0];
  size_t prev = cur - cached, i;
  int compare_char = cur_byte(e, cur, best_len_in, max_length);
  out->len_code_delta = 0;
  if (prev < cur && cached <= max_backward) {
    if (compare_char == data[prev + best_len]) {
      const size_t len = match_len(data + prev, data + cur, max_length);
      if (len >= 4) {
        const size_t score = score_last(len);
        if (best_score < score) {
          out->len = len; out->distance = cached; out->score = score;
          if (sweep == 1) { e->qk_table[key] = (uint32_t)cur; return; }
          best_len = len; best_score = score;
          compare_char = cur_byte(e, cur, len, max_length);
        }
      }
    }
  }
  if (sweep == 1) {
    size_t backward, len;
    prev = e->qk_table[key];
    e->qk_table[key] = (uint32_t)cur;
    backward = cur - prev;
    if (compare_char != data[prev + best_len_in]) return;
    if (backward == 0 || backward > max_backward) return;
    len = match_len(data + prev, data + cur, max_length);
    if (len >= 4) {
      const size_t score = score_normal(len, backward);
      if (best_score < score) { out->len = len; out->distance = backward; out->score = score; return; }
    }
  } else {
    for (i = 0; i < sweep; ++i) {
      size_t backward, len;
      prev = e->qk_table[(key + (i << 3)) & mask];
      backward = cur - prev;
      if (compare_char != data[prev + best_len]) continue;
      if (backward == 0 || backward > max_backward) continue;
      len = match_len(data + prev, data + cur, max_length);
      if (len >= 4) {
        const size_t score = score_normal(len, backward);
        if (best_score < score) {
          best_len = len; out->len = len;
          compare_char = cur_byte(e, cur, len, max_length);
          best_score = score; out->score = score; out->distance = backward;
        }
      }
    }
  }
  if (e->qk_dict && min_score == out->score)
    search_static_dict_n(e, data + cur, max_length, dict_distance, max_distance, out, 1);
  if (sweep != 1) e->qk_table[(key + (cur & ((sweep - 1) << 3))) & mask] = (uint32_t)cur;
}

/* hash_longest_match64_inc.h:157 / hash_longest_match_inc.h:156 FindLongestMatch */
static void find_longest_match(Enc* e, size_t cur, size_t max_length,
    size_t max_backward, size_t dict_distance, size_t max_distance, SR* out) {
  const uint8_t* data = e->data;
  if (e->quick) { quick_find_longest_match(e, cur, max_length, max_backward, dict_distance, max_distance, out); return; }
  const size_t rmask = e->rmask;
  const size_t cur_m = cur & rmask;
  size_t min_score = out->score, best_score = out->score, best_len = out->len;
  size_t key = hash_key(e, cur);
  uint32_t* bucket = &e->buckets[key << e->block_bits];
  size_t block_size = (size_t)1 << e->block_bits, block_mask = block_size - 1;
  size_t i;
  out->len = 0; out->len_code_delta = 0;
  for (i = 0; i < (size_t)e->ndist; ++i) {
    size_t backward = (size_t)e->dist_cache[i];
    size_t prev = cur - backward, prev_m, len;
    if (prev >= cur) continue;
    if (backward > max_backward) continue;
    prev_m = prev & rmask;
    if (cur_m + best_len > rmask) { ++g_edge.srch_ring_break; break; }
    if (prev_m + best_len > rmask) { ++g_edge.srch_ring_skip; continue; }
    if (best_len == max_length && match_len(data + prev, data + cur, max_length) == max_length) ++g_edge.srch_tie_max;
    if (cur_byte(e, cur, best_len, max_length) != data[prev + best_len]) continue;
    len = match_len(data + prev, data + cur, max_length);
    if (len >= 3 || (len == 2 && i < 2)) {
      size_t score = score_last(len);
      if (best_score < score) {
        if (i != 0) score -= penalty_last(i);
        if (best_score < score) {
          best_score = score; best_len = len;
          out->len = len; out->distance = backward; out->score = score;
        }
      }
    }
  }
  if (out->len == 2) ++g_edge.srch_dc_len2;
  if (best_len < 3) best_len = 3;
  {
    size_t nk = e->num[key];
    size_t down = nk > block_size ? nk - block_size : 0;
    for (i = nk; i > down;) {
      size_t prev = bucket[--i & block_mask], prev_m, len, k;
      size_t backward = cur - prev;
      int eq = 1;
      if (backward > max_backward) break;
      prev_m = prev & rmask;
      if (cur_m + best_len > rmask) { ++g_edge.srch_ring_break; break; }
      if (prev_m + best_len > rmask) { ++g_edge.srch_ring_skip; continue; }
      if (best_len == max_length && match_len(data + prev, data + cur, max_length) == max_length) ++g_edge.srch_tie_max;
      /* 4 bytes ending at best_len (hash_longest_match64_inc.h:246,
         hash_longest_match_inc.h:243) */
      for (k = 0; k < 4; ++k)
        if (cur_byte(e, cur, best_len - 3 + k, max_length) !=
            data[prev + best_len - 3 + k]) { eq = 0; break; }
      if (!eq) continue;
      if (e->hash64) {
        if (load32(data + cur) != load32(data + prev)) continue;
        len = match_len(data + prev + 4, data + cur + 4, max_length - 4) + 4;
      } else {
        len = match_len(data + prev, data + cur, max_length);
        if (len < 4) continue;
      }
      { size_t score = score_normal(len, backward);
        if (best_score < score) {
          best_score = score; best_len = len;
          out->len = len; out->distance = backward; out->score = score; } }
    }
    bucket[e->num[key] & block_mask] = (uint32_t)cur;
    ++e->num[key];
  }
  if (min_score == out->score)
    search_static_dict(e, data + cur, max_length, dict_distance, max_distance, out);
}

/* hash.h:80 PrepareDistanceCache */
static void prepare_dist_cache(int* dc, int ndist) {
  if (ndist > 4) {
    int l = dc[0];
    dc[4] = l - 1; dc[5] = l + 1; dc[6] = l - 2; dc[7] = l + 2; dc[8] = l - 3; dc[9] = l + 3;
    if (ndist > 10) {
      int n = dc[1];
      dc[10] = n - 1; dc[11] = n + 1; dc[12] = n - 2; dc[13] = n + 2; dc[14] = n - 3; dc[15] = n + 3;
    }
  }
}
/* backward_references.c:87 ComputeDistanceCode */
static size_t compute_distance_code(size_t distance, size_t max_distance, const int* dc) {
  if (distance <= max_distance) {
    size_t d3 = distance + 3;
    size_t o0 = d3 - (size_t)dc[0], o1 = d3 - (size_t)dc[1];
    if (distance == (size_t)dc[0]) return 0;
    if (distance == (size_t)dc[1]) return 1;
    if (o0 < 7) return (0x9750468 >> (4 * o0)) & 0xF;
    if (o1 < 7) return (0xFDB1ACE >> (4 * o1)) & 0xF;
    if (distance == (size_t)dc[2]) return 2;
    if (distance == (size_t)dc[3]) return 3;
  }
  return distance + 15;
}

/* backward_references_inc.h:10 CreateBackwardReferences */
static void create_backward_references(Enc* e, size_t num_bytes, size_t position) {
  const size_t max_backward_limit = ((size_t)1 << e->lgwin) - 16;
  const size_t max_dist_param = 0x3FFFFFC;
  size_t insert_length = e->last_insert_len;
  const size_t pos_end = position + num_bytes;
  const size_t store_end = num_bytes >= e->store_lookahead ?
      position + num_bytes - e->store_lookahead + 1 : position;
  const size_t window = e->quality < 9 ? 64 : 512;
  size_t apply_random_heuristics = position + window;
  const size_t kMinScore = SCORE_BASE + 100;
  Cmd* cmds = e->cmds + e->num_cmds;
  size_t ncmd = 0;
  prepare_dist_cache(e->dist_cache, e->ndist);
  while (position + e->hash_type_len < pos_end) {
    size_t max_length = pos_end - position;
    size_t max_distance = position < max_backward_limit ? position : max_backward_limit;
    size_t dictionary_start = max_distance;
    SR sr;
    sr.len = 0; sr.len_code_delta = 0; sr.distance = 0; sr.score = kMinScore;
    find_longest_match(e, position, max_length, max_distance, dictionary_start,
                       max_dist_param, &sr);
    if (sr.score > kMinScore) {
      int delayed = 0;
      --max_length;
      for (;; --max_length) {
        SR sr2;
        /* backward_references_inc.h:127 MIN_QUALITY_FOR_EXTENSIVE_REFERENCE_SEARCH */
        sr2.len = e->quality < 5 ? (sr.len - 1 < max_length ? sr.len - 1 : max_length) : 0;
        sr2.len_code_delta = 0; sr2.distance = 0; sr2.score = kMinScore;
        max_distance = position + 1 < max_backward_limit ? position + 1 : max_backward_limit;
        dictionary_start = max_distance;
        find_longest_match(e, position + 1, max_length, max_distance,
                           dictionary_start, max_dist_param, &sr2);
        if (sr2.score >= sr.score + 175) {
          ++position; ++insert_length; sr = sr2;
          if (++delayed < 4 && position + e->hash_type_len < pos_end) continue;
        }
        break;
      }
      apply_random_heuristics = position + 2 * sr.len + window;
      dictionary_start = position < max_backward_limit ? position : max_backward_limit;
      {
        size_t dcode = compute_distance_code(sr.distance, dictionary_start, e->dist_cache);
        if (sr.distance <= dictionary_start && dcode > 0) {
          e->dist_cache[3] = e->dist_cache[2];
          e->dist_cache[2] = e->dist_cache[1];
          e->dist_cache[1] = e->dist_cache[0];
          e->dist_cache[0] = (int)sr.distance;
          prepare_dist_cache(e->dist_cache, e->ndist);
        }
        init_cmd(&cmds[ncmd++], insert_length, sr.len, sr.len_code_delta, dcode);
      }
      e->num_literals += insert_length;
      insert_length = 0;
      {
        size_t range_start = position + 2;
        size_t range_end = position + sr.len < store_end ? position + sr.len : store_end;
        size_t i;
        if (sr.distance < (sr.len >> 2)) {
          size_t t = position + sr.len - (sr.distance << 2);
          if (t < range_start) t = range_start;
          range_start = range_end < t ? range_end : t;
        }
        for (i = range_start; i < range_end; ++i) hstore(e, i);
      }
      position += sr.len;
    } else {
      ++insert_length;
      ++position;
      if (position > apply_random_heuristics) {
        if (position > apply_random_heuristics + 4 * window) {
          size_t margin = e->store_lookahead - 1 > 4 ? e->store_lookahead - 1 : 4;
          size_t pos_jump = position + 16 < pos_end - margin ? position + 16 : pos_end - margin;
          for (; position < pos_jump; position += 4) { hstore(e, position); insert_length += 4; }
        } else {
          size_t margin = e->store_lookahead - 1 > 2 ? e->store_lookahead - 1 : 2;
          size_t pos_jump = position + 8 < pos_end - margin ? position + 8 : pos_end - margin;
          for (; position < pos_jump; position += 2) { hstore(e, position); insert_length += 2; }
        }
      }
    }
  }
  insert_length += pos_end - position;
  e->last_insert_len = insert_length;
  e->num_cmds += ncmd;
}

/* --------------------------------------------------------- entropy helpers */
/* bit_cost.c:18 BrotliBitsEntropy -- sequential order, no FMA; clamps (nullable) counts the histograms raised to their
   symbol count */
static double bits_entropy_c(const uint32_t* pop, size_t size, uint64_t* clamps) {
  size_t sum = 0, i;
  double retval = 0;
  for (i = 0; i < size; ++i) {
    size_t p = pop[i];
    sum += p;
    retval -= (double)p * fast_log2(p);
  }
  if (sum) retval += (double)sum * fast_log2(sum);
  if (retval < (double)sum) { retval = (double)sum; if (clamps) ++*clamps; }
  return retval;
}
static double bits_entropy(const uint32_t* pop, size_t size) { return bits_entropy_c(pop, size, NULL); }
/* encode.c:258 EstimateEntropy */
static double estimate_entropy(const uint32_t* pop, size_t size) {
  size_t total = 0, i;
  double result = 0;
  for (i = 0; i < size; ++i) {
    uint32_t p = pop[i];
    total += p;
    result += (double)p * fast_log2(p);
  }
  result = (double)total * fast_log2(total) - result;
  return result;
}

typedef struct { int16_t left, right_or_value; uint32_t count; } HTree;

/* entropy_encode.c:20 BrotliSetDepth */
static int set_depth(int p0, HTree* pool, uint8_t* depth, int max_depth) {
  int stack[16]; int level = 0; int p = p0;
  stack[0] = -1;
  for (;;) {
    if (pool[p].left >= 0) {
      level++;
      if (level > max_depth) return 0;
      stack[level] = pool[p].right_or_value;
      p = pool[p].left;
      continue;
    } else {
      depth[pool[p].right_or_value] = (uint8_t)level;
    }
    while (level >= 0 && stack[level] == -1) level--;
    if (level < 0) return 1;
    p = stack[level];
    stack[level] = -1;
  }
}
static int htree_less(const HTree* a, const HTree* b) {
  if (a->count != b->count) return a->count < b->count;
  return a->right_or_value > b->right_or_value;
}
/* entropy_encode.c:68 BrotliCreateHuffmanTree.  The comparator is a strict
   total order (count, then symbol index descending), so any sort yields the
   order of entropy_encode.h:82 SortHuffmanTreeItems. */
static void create_huffman_tree(const uint32_t* data, size_t length, int tree_limit,
                                HTree* tree, uint8_t* depth) {
  uint32_t count_limit;
  HTree sentinel; sentinel.count = 0xFFFFFFFFu; sentinel.left = -1; sentinel.right_or_value = -1;
  for (count_limit = 1;; count_limit *= 2) {
    size_t n = 0, i, j, k;
    for (i = length; i != 0;) {
      --i;
      if (data[i]) {
        tree[n].count = data[i] > count_limit ? data[i] : count_limit;
        tree[n].left = -1; tree[n].right_or_value = (int16_t)i; ++n;
      }
    }
    if (n == 1) { depth[tree[0].right_or_value] = 1; break; }
    for (i = 1; i < n; ++i) {  /* insertion sort */
      HTree t = tree[i]; size_t q = i;
      while (q > 0 && htree_less(&t, &tree[q - 1])) { tree[q] = tree[q - 1]; --q; }
      tree[q] = t;
    }
    tree[n] = sentinel; tree[n + 1] = sentinel;
    i = 0; j = n + 1;
    for (k = n - 1; k != 0; --k) {
      size_t left, right;
      if (tree[i].count <= tree[j].count) { left = i; ++i; } else { left = j; ++j; }
      if (tree[i].count <= tree[j].count) { right = i; ++i; } else { right = j; ++j; }
      { size_t j_end = 2 * n - k;
        tree[j_end].count = tree[left].count + tree[right].count;
        tree[j_end].left = (int16_t)left;
        tree[j_end].right_or_value = (int16_t)right;
        tree[j_end + 1] = sentinel; }
    }
    if (set_depth((int)(2 * n - 1), tree, depth, tree_limit)) break;
    if (tree_limit == 5) ++g_edge.retry_cl;
    else if (length == 256) ++g_edge.retry_lit;
    else if (length == 704) ++g_edge.retry_cmd;
    else if (length == 64 || length == 140) ++g_edge.retry_dist;
    else ++g_edge.retry_other;
  }
}
/* entropy_encode.c:474 BrotliConvertBitDepthsToSymbols */
static uint16_t reverse_bits(size_t nbits, uint16_t bits) {
  uint16_t r = 0; size_t i;
  for (i = 0; i < nbits; ++i) { r = (uint16_t)((r << 1) | (bits & 1)); bits >>= 1; }
  return r;
}
static void depths_to_symbols(const uint8_t* depth, size_t len, uint16_t* bits) {
  uint16_t bl_count[16] = {0}, next_code[16]; size_t i; int code = 0;
  for (i = 0; i < len; ++i) ++bl_count[depth[i]];
  bl_count[0] = 0; next_code[0] = 0;
  for (i = 1; i < 16; ++i) { code = (code + bl_count[i - 1]) << 1; next_code[i] = (uint16_t)code; }
  for (i = 0; i < len; ++i)
    if (depth[i]) bits[i] = reverse_bits(depth[i], next_code[depth[i]]++);
}

/* entropy_encode.c:241 BrotliOptimizeHuffmanCountsForRle; integer types as in
   the reference (256 * uint32 stays 32-bit). */
static void optimize_counts_for_rle(size_t length, uint32_t* counts, uint8_t* good_for_rle) {
  size_t nonzero_count = 0, stride, limit, sum, i;
  const size_t streak_limit = 1240;
  for (i = 0; i < length; i++) if (counts[i]) ++nonzero_count;
  if (nonzero_count < 16) { ++g_edge.rle_lt16; return; }
  while (length != 0 && counts[length - 1] == 0) --length;
  if (length == 0) return;
  {
    size_t nonzeros = 0; uint32_t smallest_nonzero = 1 << 30;
    for (i = 0; i < length; ++i)
      if (counts[i] != 0) { ++nonzeros; if (smallest_nonzero > counts[i]) smallest_nonzero = counts[i]; }
    if (nonzeros < 5) return;
    if (smallest_nonzero < 4) {
      size_t zeros = length - nonzeros;
      if (zeros < 6)
        for (i = 1; i < length - 1; ++i)
          if (counts[i - 1] != 0 && counts[i] == 0 && counts[i + 1] != 0) { counts[i] = 1; ++g_edge.rle_holes; }
    }
    if (nonzeros < 28) { ++g_edge.rle_lt28; return; }
  }
  ++g_edge.rle_full;
  memset(good_for_rle, 0, length);
  {
    uint32_t symbol = counts[0]; size_t step = 0;
    for (i = 0; i <= length; ++i) {
      if (i == length || counts[i] != symbol) {
        if ((symbol == 0 && step >= 5) || (symbol != 0 && step >= 7)) {
          size_t k; for (k = 0; k < step; ++k) good_for_rle[i - k - 1] = 1;
          ++g_edge.rle_good;
        }
        step = 1;
        if (i != length) symbol = counts[i];
      } else ++step;
    }
  }
  stride = 0;
  limit = (uint32_t)(256u * (counts[0] + counts[1] + counts[2]) / 3u + 420u);
  sum = 0;
  for (i = 0; i <= length; ++i) {
    if (i == length || good_for_rle[i] || (i != 0 && good_for_rle[i - 1]) ||
        ((size_t)(uint32_t)(256u * counts[i]) - limit + streak_limit) >= 2 * streak_limit) {
      if (stride >= 4 || (stride >= 3 && sum == 0)) {
        size_t k, count = (sum + stride / 2) / stride;
        if (count == 0) count = 1;
        if (sum == 0) count = 0;
        for (k = 0; k < stride; ++k) counts[i - k - 1] = (uint32_t)count;
        ++g_edge.rle_stride;
      }
      stride = 0; sum = 0;
      if (i < length - 2) limit = (uint32_t)(256u * (counts[i] + counts[i + 1] + counts[i + 2]) / 3u + 420u);
      else if (i < length) limit = (uint32_t)(256u * counts[i]);
      else limit = 0;
    }
    ++stride;
    if (i != length) {
      sum += counts[i];
      if (stride >= 4) limit = (256 * sum + stride / 2) / stride;
      if (stride == 4) limit += 120;
    }
  }
}

/* entropy_encode.c:160,198 repetition writers; :372 DecideOverRleUse; :402 */
static void rev(uint8_t* v, size_t s, size_t e) {
  --e; while (s < e) { uint8_t t = v[s]; v[s] = v[e]; v[e] = t; ++s; --e; }
}
static void write_reps(uint8_t prev, uint8_t value, size_t reps, size_t* ts,
                       uint8_t* tree, uint8_t* extra) {
  if (prev != value) { tree[*ts] = value; extra[*ts] = 0; ++(*ts); --reps; }
  if (reps == 7) { tree[*ts] = value; extra[*ts] = 0; ++(*ts); --reps; ++g_edge.reps7; }
  if (reps < 3) {
    size_t i; for (i = 0; i < reps; ++i) { tree[*ts] = value; extra[*ts] = 0; ++(*ts); }
  } else {
    size_t start = *ts;
    reps -= 3;
    for (;;) {
      tree[*ts] = 16; extra[*ts] = reps & 0x3; ++(*ts);
      reps >>= 2;
      if (reps == 0) break;
      --reps;
    }
    rev(tree, start, *ts); rev(extra, start, *ts);
  }
}
static void write_reps_zeros(size_t reps, size_t* ts, uint8_t* tree, uint8_t* extra) {
  if (reps == 11) { tree[*ts] = 0; extra[*ts] = 0; ++(*ts); --reps; ++g_edge.reps11; }
  if (reps < 3) {
    size_t i; for (i = 0; i < reps; ++i) { tree[*ts] = 0; extra[*ts] = 0; ++(*ts); }
  } else {
    size_t start = *ts;
    reps -= 3;
    for (;;) {
      tree[*ts] = 17; extra[*ts] = reps & 0x7; ++(*ts);
      reps >>= 3;
      if (reps == 0) break;
      --reps;
    }
    rev(tree, start, *ts); rev(extra, start, *ts);
  }
}
static void write_huffman_tree(const uint8_t* depth, size_t length, size_t* ts,
                               uint8_t* tree, uint8_t* extra) {
  uint8_t prev = 8; size_t i, new_length = length;
  int rle_nz = 0, rle_z = 0;
  for (i = 0; i < length; ++i) { if (depth[length - i - 1] == 0) --new_length; else break; }
  if (length > 50) {
    size_t tz = 0, tnz = 0, cz = 1, cnz = 1;
    for (i = 0; i < new_length;) {
      uint8_t v = depth[i]; size_t reps = 1, k;
      for (k = i + 1; k < new_length && depth[k] == v; ++k) ++reps;
      if (reps >= 3 && v == 0) { tz += reps; ++cz; }
      if (reps >= 4 && v != 0) { tnz += reps; ++cnz; }
      i += reps;
    }
    rle_nz = tnz > cnz * 2; rle_z = tz > cz * 2;
    g_edge.rle_use_nz += rle_nz; g_edge.rle_use_z += rle_z;
  }
  for (i = 0; i < new_length;) {
    uint8_t v = depth[i]; size_t reps = 1;
    if ((v != 0 && rle_nz) || (v == 0 && rle_z)) {
      size_t k; for (k = i + 1; k < new_length && depth[k] == v; ++k) ++reps;
    }
    if (v == 0) write_reps_zeros(reps, ts, tree, extra);
    else { write_reps(prev, v, reps, ts, tree, extra); prev = v; }
    i += reps;
  }
}

/* brotli_bit_stream.c:165 */
static void store_hufftree_of_hufftree(int num_codes, const uint8_t* cl_depth, BitW* w) {
  static const uint8_t kOrder[18] = {1, 2, 3, 4, 0, 5, 17, 6, 16, 7, 8, 9, 10, 11, 12, 13, 14, 15};
  static const uint8_t kSym[6] = {0, 7, 3, 2, 1, 15};
  static const uint8_t kLen[6] = {2, 4, 3, 2, 2, 4};
  size_t skip = 0, to_store = 18, i;
  if (num_codes > 1)
    for (; to_store > 0; --to_store) if (cl_depth[kOrder[to_store - 1]] != 0) break;
  if (cl_depth[kOrder[0]] == 0 && cl_depth[kOrder[1]] == 0) {
    skip = 2;
    if (cl_depth[kOrder[2]] == 0) skip = 3;
  }
  if (skip == 2) ++g_edge.cl_skip2; else if (skip == 3) ++g_edge.cl_skip3;
  if (to_store < 18) ++g_edge.cl_trim;
  wbits(w, 2, skip);
  for (i = skip; i < to_store; ++i) { size_t l = cl_depth[kOrder[i]]; wbits(w, kLen[l], kSym[l]); }
}
/* brotli_bit_stream.c:283 BrotliStoreHuffmanTree */
static void store_huffman_tree(const uint8_t* depths, size_t num, HTree* tree, BitW* w) {
  uint8_t ht[704], hx[704]; size_t hs = 0, i;
  uint8_t cl_depth[18] = {0}; uint16_t cl_bits[18]; uint32_t histo[18] = {0};
  int num_codes = 0; size_t code = 0;
  write_huffman_tree(depths, num, &hs, ht, hx);
  for (i = 0; i < hs; ++i) ++histo[ht[i]];
  for (i = 0; i < 18; ++i) {
    if (histo[i]) {
      if (num_codes == 0) { code = i; num_codes = 1; }
      else if (num_codes == 1) { num_codes = 2; break; }
    }
  }
  create_huffman_tree(histo, 18, 5, tree, cl_depth);
  depths_to_symbols(cl_depth, 18, cl_bits);
  store_hufftree_of_hufftree(num_codes, cl_depth, w);
  if (num_codes == 1) { cl_depth[code] = 0; ++g_edge.cl_single; }
  for (i = 0; i < hs; ++i) {
    size_t ix = ht[i];
    wbits(w, cl_depth[ix], cl_bits[ix]);
    if (ix == 16) wbits(w, 2, hx[i]);
    else if (ix == 17) wbits(w, 3, hx[i]);
  }
}
/* brotli_bit_stream.c:242 StoreSimpleHuffmanTree */
static void store_simple_tree(const uint8_t* depths, size_t* symbols, size_t num,
                              size_t max_bits, BitW* w) {
  size_t i, j;
  wbits(w, 2, 1);
  wbits(w, 2, num - 1);
  for (i = 0; i < num; i++)
    for (j = i + 1; j < num; j++)
      if (depths[symbols[j]] < depths[symbols[i]]) { size_t t = symbols[j]; symbols[j] = symbols[i]; symbols[i] = t; }
  for (i = 0; i < num; ++i) wbits(w, max_bits, symbols[i]);
  if (num == 4) wbits(w, 1, depths[symbols[0]] == 1 ? 1 : 0);
  if (num == 2) ++g_edge.simple_nsym2;
  else if (num == 3) ++g_edge.simple_nsym3;
  else { ++g_edge.simple_nsym4; if (depths[symbols[0]] == 1) ++g_edge.simple_select1; else ++g_edge.simple_select0; }
}
/* brotli_bit_stream.c:349 BuildAndStoreHuffmanTree */
static void build_and_store_tree(const uint32_t* histo, size_t histo_len, size_t alphabet_size,
                                 HTree* tree, uint8_t* depth, uint16_t* bits, BitW* w) {
  size_t count = 0, s4[4] = {0}, i, max_bits = 0;
  for (i = 0; i < histo_len; i++) {
    if (histo[i]) {
      if (count < 4) s4[count] = i; else if (count > 4) break;
      count++;
    }
  }
  { size_t c = alphabet_size - 1; while (c) { c >>= 1; ++max_bits; } }
  if (count <= 1) {
    wbits(w, 4, 1);
    wbits(w, max_bits, s4[0]);
    depth[s4[0]] = 0; bits[s4[0]] = 0;
    ++g_edge.simple_nsym1;
    return;
  }
  memset(depth, 0, histo_len);
  create_huffman_tree(histo, histo_len, 15, tree, depth);
  depths_to_symbols(depth, histo_len, bits);
  if (count <= 4) store_simple_tree(depth, s4, count, max_bits, w);
  else store_huffman_tree(depth, histo_len, tree, w);
}

/* One prefix code of a metablock of quality 4+, with exactly the calls store_compressed_metablock makes for it: the count
   smoothing, then the Huffman construction and the store into a fresh bit writer.  histo: len (256, 704 or 64) counts.
   H_out: the smoothed counts; depth_out / bits_out: zero, then what build_and_store_tree writes (with one symbol or none
   only that symbol's entry); stored: the code's bits, stored_cap bytes; *nbits: its size in bits.  Returns 0 when len is
   not an alphabet size of such a metablock or the code does not fit stored_cap. */
int oracle_build_code(const uint32_t* histo, size_t len, uint32_t* H_out, uint8_t* depth_out, uint16_t* bits_out,
                      uint8_t* stored, size_t stored_cap, size_t* nbits) {
  uint8_t good_for_rle[704];
  HTree* tree; BitW w; size_t nbytes;
  if (len != 256 && len != 704 && len != 64) return 0;
  tree = (HTree*)malloc(sizeof(HTree) * (2 * 704 + 1));
  w.buf = (uint8_t*)calloc(2 * len + 256, 1); w.ix = 0;   /* (at most 8 bits a code length, and the code-length code) */
  memcpy(H_out, histo, len * 4);
  memset(depth_out, 0, len); memset(bits_out, 0, len * 2);
  optimize_counts_for_rle(len, H_out, good_for_rle);
  build_and_store_tree(H_out, len, len, tree, depth_out, bits_out, &w);
  *nbits = w.ix;
  nbytes = (w.ix + 7) / 8;
  if (nbytes <= stored_cap) memcpy(stored, w.buf, nbytes);
  free(w.buf); free(tree);
  return nbytes <= stored_cap;
}

/* brotli_bit_stream.c:106 */
static void store_varlen_uint8(size_t n, BitW* w) {
  if (n == 0) wbits(w, 1, 0);
  else { size_t nb = log2floor(n); wbits(w, 1, 1); wbits(w, 3, nb); wbits(w, nb, n - ((size_t)1 << nb)); }
}
/* brotli_bit_stream.c:33 BlockLengthPrefixCode */
static uint32_t block_len_code(uint32_t len) {
  uint32_t code = (len >= 177) ? (len >= 753 ? 20 : 14) : (len >= 41 ? 7 : 0);
  while (code < 25 && len >= kBlockLenOffset[code + 1]) ++code;
  return code;
}
/* brotli_bit_stream.c:70 BrotliEncodeMlen + :120 header */
static void store_mlen(size_t length, BitW* w) {
  size_t lg = (length == 1) ? 1 : log2floor((uint32_t)(length - 1)) + 1;
  size_t mnibbles = (lg < 16 ? 16 : (lg + 3)) / 4;
  wbits(w, 2, mnibbles - 4);
  wbits(w, mnibbles * 4, length - 1);
}
/* brotli_bit_stream.c:1321 BrotliStoreUncompressedMetaBlock */
static void store_uncompressed(int is_final, const uint8_t* data, size_t pos, size_t len, BitW* w) {
  wbits(w, 1, 0);
  store_mlen(len, w);
  wbits(w, 1, 1);
  w->ix = (w->ix + 7u) & ~(size_t)7u;
  w->buf[w->ix >> 3] = 0;
  memcpy(&w->buf[w->ix >> 3], data + pos, len);
  w->ix += len << 3;
  w->buf[w->ix >> 3] = 0;
  if (is_final) {
    wbits(w, 1, 1); wbits(w, 1, 1);
    w->ix = (w->ix + 7u) & ~(size_t)7u;
    w->buf[w->ix >> 3] = 0;
  }
}

/* ------------------------------------------------------- greedy block split */
typedef struct {
  size_t num_types, num_blocks;
  uint8_t* types; uint32_t* lengths;
} Split;

/* metablock_inc.h:14 BlockSplitter and metablock.c:463 ContextBlockSplitter in
   one restatement: num_contexts histograms per block type. */
typedef struct {
  size_t alphabet, num_contexts, max_block_types, min_block_size;
  double split_threshold;
  size_t num_blocks; Split* split;
  uint32_t* histograms;     /* [(max_types+1)*num_contexts][alphabet] */
  size_t histograms_size;   /* in histograms (types*contexts) */
  size_t target_block_size, block_size, curr_ix, last_ix[2];
  double last_entropy[2 * 13];
  size_t merge_last_count;
  uint32_t* combined;       /* [2*num_contexts][alphabet] */
} Splitter;

static void splitter_init(Splitter* s, size_t alphabet, size_t num_contexts,
    size_t min_block_size, double thr, size_t num_symbols, Split* split) {
  size_t max_num_blocks = num_symbols / min_block_size + 1;
  size_t max_num_types;
  memset(s, 0, sizeof(*s));
  s->alphabet = alphabet; s->num_contexts = num_contexts;
  s->max_block_types = 256 / num_contexts;
  s->min_block_size = min_block_size; s->split_threshold = thr;
  s->split = split; s->target_block_size = min_block_size;
  max_num_types = max_num_blocks < s->max_block_types + 1 ? max_num_blocks : s->max_block_types + 1;
  split->types = (uint8_t*)calloc(max_num_blocks + 1, 1);
  split->lengths = (uint32_t*)calloc(max_num_blocks + 1, 4);
  split->num_blocks = max_num_blocks; split->num_types = 0;
  s->histograms_size = max_num_types * num_contexts;
  s->histograms = (uint32_t*)calloc((max_num_types + 1) * num_contexts * alphabet, 4);
  s->combined = (uint32_t*)calloc(2 * num_contexts * alphabet, 4);
}
static void splitter_finish_block(Splitter* s, int is_final) {
  Split* split = s->split;
  const size_t nc = s->num_contexts, A = s->alphabet;
  double* last_entropy = s->last_entropy;
  uint32_t* H = s->histograms;
  size_t i, k;
  if (s->block_size < s->min_block_size) {
    if (s->block_size) ++g_edge.split_pad; else if (s->num_blocks) ++g_edge.split_pad_empty;
    s->block_size = s->min_block_size;
  }
  if (s->num_blocks == 0) {
    split->lengths[0] = (uint32_t)s->block_size;
    split->types[0] = 0;
    for (i = 0; i < nc; ++i) {
      last_entropy[i] = bits_entropy_c(H + i * A, A, &g_edge.split_clamp);
      last_entropy[nc + i] = last_entropy[i];
    }
    ++s->num_blocks; ++split->num_types;
    s->curr_ix += nc;
    if (s->curr_ix < s->histograms_size) memset(H + s->curr_ix * A, 0, nc * A * 4);
    s->block_size = 0;
  } else if (s->block_size > 0) {
    double entropy[13], combined_entropy[26], diff[2] = {0.0, 0.0};
    for (i = 0; i < nc; ++i) {
      size_t cur = s->curr_ix + i, j;
      entropy[i] = bits_entropy_c(H + cur * A, A, &g_edge.split_clamp);
      for (j = 0; j < 2; ++j) {
        size_t jx = j * nc + i, last = s->last_ix[j] + i;
        for (k = 0; k < A; ++k) s->combined[jx * A + k] = H[cur * A + k] + H[last * A + k];
        combined_entropy[jx] = bits_entropy_c(s->combined + jx * A, A, &g_edge.split_clamp);
        diff[j] += combined_entropy[jx] - entropy[i] - last_entropy[jx];
      }
    }
    if (split->num_types < s->max_block_types && diff[0] >= s->split_threshold && diff[1] >= s->split_threshold &&
        (diff[0] == s->split_threshold || diff[1] == s->split_threshold))
      ++g_edge.split_tie;
    else if (!(split->num_types < s->max_block_types && diff[0] > s->split_threshold && diff[1] > s->split_threshold) &&
             diff[1] == diff[0] - 20.0)
      ++g_edge.back_tie;
    if (split->num_types < s->max_block_types &&
        diff[0] > s->split_threshold && diff[1] > s->split_threshold) {
      split->lengths[s->num_blocks] = (uint32_t)s->block_size;
      split->types[s->num_blocks] = (uint8_t)split->num_types;
      s->last_ix[1] = s->last_ix[0];
      s->last_ix[0] = split->num_types * nc;
      for (i = 0; i < nc; ++i) { last_entropy[nc + i] = last_entropy[i]; last_entropy[i] = entropy[i]; }
      ++s->num_blocks; ++split->num_types;
      s->curr_ix += nc;
      if (s->curr_ix < s->histograms_size) memset(H + s->curr_ix * A, 0, nc * A * 4);
      s->block_size = 0; s->merge_last_count = 0; s->target_block_size = s->min_block_size;
    } else if (diff[1] < diff[0] - 20.0) {
      size_t t;
      split->lengths[s->num_blocks] = (uint32_t)s->block_size;
      split->types[s->num_blocks] = split->types[s->num_blocks - 2];
      t = s->last_ix[0]; s->last_ix[0] = s->last_ix[1]; s->last_ix[1] = t;
      for (i = 0; i < nc; ++i) {
        memcpy(H + (s->last_ix[0] + i) * A, s->combined + (nc + i) * A, A * 4);
        last_entropy[nc + i] = last_entropy[i];
        last_entropy[i] = combined_entropy[nc + i];
        memset(H + (s->curr_ix + i) * A, 0, A * 4);
      }
      ++s->num_blocks;
      s->block_size = 0; s->merge_last_count = 0; s->target_block_size = s->min_block_size;
      ++g_edge.split_back;
    } else {
      split->lengths[s->num_blocks - 1] += (uint32_t)s->block_size;
      for (i = 0; i < nc; ++i) {
        memcpy(H + (s->last_ix[0] + i) * A, s->combined + i * A, A * 4);
        last_entropy[i] = combined_entropy[i];
        if (split->num_types == 1) last_entropy[nc + i] = last_entropy[i];
        memset(H + (s->curr_ix + i) * A, 0, A * 4);
      }
      s->block_size = 0;
      if (++s->merge_last_count > 1) { s->target_block_size += s->min_block_size; ++g_edge.split_grow; }
    }
  }
  if (is_final) {
    s->histograms_size = split->num_types * nc;
    split->num_blocks = s->num_blocks;
  }
}
static void splitter_add(Splitter* s, size_t symbol, size_t context) {
  ++s->histograms[(s->curr_ix + context) * s->alphabet + symbol];
  ++s->block_size;
  if (s->block_size == s->target_block_size) splitter_finish_block(s, 0);
}
static void splitter_free(Splitter* s) {
  free(s->histograms); free(s->combined); free(s->split->types); free(s->split->lengths);
}

/* ---------------------------------------------- literal context modelling */
static const uint32_t kCtxMapContinuation[64] = {1, 1, 2, 2};
static const uint32_t kCtxMapSimpleUTF8[64] = {0, 0, 1, 1};
static const uint32_t kCtxMapComplexUTF8[64] = {
  11, 11, 12, 12, 0, 0, 0, 0, 1, 1, 9, 9, 2, 2, 2, 2, 1, 1, 1, 1, 8, 3, 3, 3,
  1, 1, 1, 1, 2, 2, 2, 2, 8, 4, 4, 4, 8, 7, 4, 4, 8, 0, 0, 0, 3, 3, 3, 3,
  5, 5, 10, 5, 5, 5, 10, 5, 6, 6, 6, 6, 6, 6, 6, 6};
#define CTX_UTF8(p1, p2) (g_ctx_lut[1024 + (p1)] | g_ctx_lut[1024 + 256 + (p2)])

/* encode.c:277 ChooseContextMap */
static void choose_context_map(int quality, uint32_t* bigram, size_t* nctx, const uint32_t** map) {
  uint32_t mono[3] = {0}, two[6] = {0}; size_t total, i; double entropy[4];
  for (i = 0; i < 9; ++i) { mono[i % 3] += bigram[i]; two[i % 6] += bigram[i]; }
  entropy[1] = estimate_entropy(mono, 3);
  entropy[2] = estimate_entropy(two, 3) + estimate_entropy(two + 3, 3);
  entropy[3] = 0;
  for (i = 0; i < 3; ++i) entropy[3] += estimate_entropy(bigram + 3 * i, 3);
  total = mono[0] + mono[1] + mono[2];
  entropy[0] = 1.0 / (double)total;
  entropy[1] *= entropy[0]; entropy[2] *= entropy[0]; entropy[3] *= entropy[0];
  if (quality < 7) entropy[3] = entropy[1] * 10;
  if (entropy[1] - entropy[2] < 0.2 && entropy[1] - entropy[3] < 0.2) *nctx = 1;
  else if (entropy[2] - entropy[3] < 0.02) { *nctx = 2; *map = kCtxMapSimpleUTF8; }
  else { *nctx = 3; *map = kCtxMapContinuation; }
}
/* encode.c:341 ShouldUseComplexStaticContextMap + :424 DecideOver... */
static void decide_context_modeling(const Enc* e, size_t start_pos, size_t length,
                                    size_t* nctx, const uint32_t** map) {
  const uint8_t* in = e->data;
  if (e->quality < 5 || length < 64) return;
  if (e->size_hint >= (1u << 20)) {
    const size_t end_pos = start_pos + length;
    uint32_t combined[32] = {0}, ctxh[13 * 32]; uint32_t total = 0; double entropy[3]; size_t i, sp;
    memset(ctxh, 0, sizeof(ctxh));
    for (sp = start_pos; sp + 64 <= end_pos; sp += 4096) {
      const size_t stride_end = sp + 64;
      uint8_t prev2 = in[sp], prev1 = in[sp + 1]; size_t pos;
      for (pos = sp + 2; pos < stride_end; ++pos) {
        const uint8_t lit = in[pos];
        const uint8_t ctx = (uint8_t)kCtxMapComplexUTF8[CTX_UTF8(prev1, prev2)];
        ++total; ++combined[lit >> 3]; ++ctxh[(ctx << 5) + (lit >> 3)];
        prev2 = prev1; prev1 = lit;
      }
    }
    entropy[1] = estimate_entropy(combined, 32);
    entropy[2] = 0;
    for (i = 0; i < 13; ++i) entropy[2] += estimate_entropy(ctxh + (i << 5), 32);
    entropy[0] = 1.0 / (double)total;
    entropy[1] *= entropy[0]; entropy[2] *= entropy[0];
    if (!(entropy[2] > 3.0 || entropy[1] - entropy[2] < 0.2)) {
      *nctx = 13; *map = kCtxMapComplexUTF8; return;
    }
  }
  {
    static const int lut[4] = {0, 0, 1, 2};
    const size_t end_pos = start_pos + length;
    uint32_t bigram[9] = {0}; size_t sp;
    for (sp = start_pos; sp + 64 <= end_pos; sp += 4096) {
      const size_t stride_end = sp + 64;
      int prev = lut[in[sp] >> 6] * 3; size_t pos;
      for (pos = sp + 1; pos < stride_end; ++pos) {
        const uint8_t lit = in[pos];
        ++bigram[prev + lut[lit >> 6]];
        prev = lut[lit >> 6] * 3;
      }
    }
    choose_context_map(e->quality, bigram, nctx, map);
  }
}

/* encode.c:457 ShouldCompress */
static int should_compress(const Enc* e, size_t bytes) {
  if (bytes <= 2) return 0;
  if (e->num_cmds < (bytes >> 8) + 2) {
    if ((double)e->num_literals > 0.99 * (double)bytes) {
      uint32_t histo[256] = {0};
      const double thr = (double)bytes * 7.92 * (1.0 / 13.0);
      size_t t = (bytes + 12) / 13, i; size_t pos = e->last_flush_pos;
      for (i = 0; i < t; i++) { ++histo[e->data[pos]]; pos += 13; }
      if (bits_entropy(histo, 256) > thr) return 0;
    }
  }
  return 1;
}

/* ------------------------------------------------------- store a metablock */
typedef struct {
  size_t hist_len, num_types, num_blocks;
  const uint8_t* types; const uint32_t* lengths;
  size_t last_type, second_last_type;
  uint8_t type_depths[258]; uint16_t type_bits[258];
  uint8_t len_depths[26]; uint16_t len_bits[26];
  size_t block_ix, block_len, entropy_ix;
  uint8_t* depths; uint16_t* bits;
} BlockEnc;

static size_t next_type_code(size_t* last, size_t* second, uint8_t type) {
  size_t code = (type == *last + 1) ? 1u : (type == *second) ? 0u : type + 2u;
  *second = *last; *last = type;
  return code;
}
static void store_block_switch(BlockEnc* b, uint32_t block_len, uint8_t block_type, int is_first, BitW* w) {
  size_t typecode = next_type_code(&b->last_type, &b->second_last_type, block_type);
  uint32_t lencode;
  if (!is_first) wbits(w, b->type_depths[typecode], b->type_bits[typecode]);
  lencode = block_len_code(block_len);
  wbits(w, b->len_depths[lencode], b->len_bits[lencode]);
  wbits(w, kBlockLenNbits[lencode], block_len - kBlockLenOffset[lencode]);
}
/* brotli_bit_stream.c:760 BuildAndStoreBlockSplitCode */
static void build_and_store_block_split_code(BlockEnc* b, HTree* tree, BitW* w) {
  uint32_t type_histo[258], length_histo[26]; size_t i, last = 1, second = 0;
  memset(type_histo, 0, (b->num_types + 2) * 4);
  memset(length_histo, 0, sizeof(length_histo));
  for (i = 0; i < b->num_blocks; ++i) {
    size_t tc = next_type_code(&last, &second, b->types[i]);
    if (i != 0) ++type_histo[tc];
    ++length_histo[block_len_code(b->lengths[i])];
  }
  store_varlen_uint8(b->num_types - 1, w);
  if (b->num_types > 1) {
    build_and_store_tree(type_histo, b->num_types + 2, b->num_types + 2, tree, b->type_depths, b->type_bits, w);
    build_and_store_tree(length_histo, 26, 26, tree, b->len_depths, b->len_bits, w);
    store_block_switch(b, b->lengths[0], b->types[0], 1, w);
  }
}
static void block_enc_init(BlockEnc* b, size_t hist_len, const Split* s) {
  memset(b, 0, sizeof(*b));
  b->hist_len = hist_len; b->num_types = s->num_types; b->types = s->types;
  b->lengths = s->lengths; b->num_blocks = s->num_blocks;
  b->last_type = 1; b->second_last_type = 0;
  b->block_len = s->num_blocks == 0 ? 0 : s->lengths[0];
}
/* brotli_bit_stream.c:879 StoreSymbol / :898 StoreSymbolWithContext */
static void store_symbol(BlockEnc* b, size_t symbol, BitW* w) {
  if (b->block_len == 0) {
    size_t ix = ++b->block_ix;
    b->block_len = b->lengths[ix];
    b->entropy_ix = b->types[ix] * b->hist_len;
    store_block_switch(b, b->lengths[ix], b->types[ix], 0, w);
  }
  --b->block_len;
  wbits(w, b->depths[b->entropy_ix + symbol], b->bits[b->entropy_ix + symbol]);
}
static void store_symbol_ctx(BlockEnc* b, size_t symbol, size_t context,
                             const uint32_t* cmap, BitW* w) {
  if (b->block_len == 0) {
    size_t ix = ++b->block_ix;
    b->block_len = b->lengths[ix];
    b->entropy_ix = (size_t)b->types[ix] << 6;
    store_block_switch(b, b->lengths[ix], b->types[ix], 0, w);
  }
  --b->block_len;
  { size_t ix = cmap[b->entropy_ix + context] * b->hist_len + symbol;
    wbits(w, b->depths[ix], b->bits[ix]); }
}
/* brotli_bit_stream.c:794 StoreTrivialContextMap */
static void store_trivial_context_map(size_t num_types, size_t context_bits, HTree* tree, BitW* w) {
  store_varlen_uint8(num_types - 1, w);
  if (num_types > 1) {
    size_t repeat_code = context_bits - 1u, repeat_bits = (1u << repeat_code) - 1u;
    size_t alphabet = num_types + repeat_code, i;
    uint32_t histo[272]; uint8_t depths[272]; uint16_t bits[272];
    memset(histo, 0, alphabet * 4);
    wbits(w, 1, 1); wbits(w, 4, repeat_code - 1);
    histo[repeat_code] = (uint32_t)num_types;
    histo[0] = 1;
    for (i = context_bits; i < alphabet; ++i) histo[i] = 1;
    build_and_store_tree(histo, alphabet, alphabet, tree, depths, bits, w);
    for (i = 0; i < num_types; ++i) {
      size_t code = (i == 0 ? 0 : i + context_bits - 1);
      wbits(w, depths[code], bits[code]);
      wbits(w, depths[repeat_code], bits[repeat_code]);
      wbits(w, repeat_code, repeat_bits);
    }
    wbits(w, 1, 1);
  }
}
/* brotli_bit_stream.c:683 EncodeContextMap (+ :592 MTF, :624 RLE of zeros) */
static void encode_context_map(const uint32_t* cmap, size_t cmap_size, size_t num_clusters,
                               HTree* tree, BitW* w) {
  uint32_t* rle; uint32_t max_prefix = 6; size_t n_rle = 0, i;
  uint32_t histo[272]; uint8_t depths[272]; uint16_t bits[272];
  store_varlen_uint8(num_clusters - 1, w);
  if (num_clusters == 1) return;
  rle = (uint32_t*)malloc(cmap_size * 4);
  { uint8_t mtf[256]; uint32_t maxv = cmap[0]; size_t sz;
    for (i = 1; i < cmap_size; ++i) if (cmap[i] > maxv) maxv = cmap[i];
    for (i = 0; i <= maxv; ++i) mtf[i] = (uint8_t)i;
    sz = maxv + 1;
    for (i = 0; i < cmap_size; ++i) {
      size_t idx = 0, k; uint8_t v;
      while (idx < sz && mtf[idx] != (uint8_t)cmap[i]) ++idx;
      rle[i] = (uint32_t)idx;
      v = mtf[idx];
      for (k = idx; k != 0; --k) mtf[k] = mtf[k - 1];
      mtf[0] = v;
    } }
  { uint32_t max_reps = 0;
    for (i = 0; i < cmap_size;) {
      uint32_t reps = 0;
      for (; i < cmap_size && rle[i] != 0; ++i) ;
      for (; i < cmap_size && rle[i] == 0; ++i) ++reps;
      if (reps > max_reps) max_reps = reps;
    }
    { uint32_t mp = max_reps > 0 ? log2floor(max_reps) : 0;
      if (mp < max_prefix) max_prefix = mp; }
    for (i = 0; i < cmap_size;) {
      if (rle[i] != 0) { rle[n_rle++] = rle[i] + max_prefix; ++i; }
      else {
        uint32_t reps = 1; size_t k;
        for (k = i + 1; k < cmap_size && rle[k] == 0; ++k) ++reps;
        i += reps;
        while (reps != 0) {
          if (reps < (2u << max_prefix)) {
            uint32_t p = log2floor(reps);
            rle[n_rle++] = p + ((reps - (1u << p)) << 9);
            break;
          } else {
            rle[n_rle++] = max_prefix + (((1u << max_prefix) - 1u) << 9);
            reps -= (2u << max_prefix) - 1u;
          }
        }
      }
    } }
  memset(histo, 0, sizeof(histo));
  for (i = 0; i < n_rle; ++i) ++histo[rle[i] & 511];
  { int use_rle = max_prefix > 0;
    wbits(w, 1, (uint64_t)use_rle);
    if (use_rle) wbits(w, 4, max_prefix - 1); }
  build_and_store_tree(histo, num_clusters + max_prefix, num_clusters + max_prefix, tree, depths, bits, w);
  for (i = 0; i < n_rle; ++i) {
    uint32_t sym = rle[i] & 511, extra = rle[i] >> 9;
    wbits(w, depths[sym], bits[sym]);
    if (sym > 0 && sym <= max_prefix) wbits(w, sym, extra);
  }
  wbits(w, 1, 1);
  free(rle);
}

static void edge_cmd(const Cmd* c, int lgwin) {
  const uint32_t dcode = cmd_restore_dcode(c);
  EDGE_MAX(max_insert, c->insert_len);
  EDGE_MAX(max_copy, cmd_copy_len(c));
  /* backward references only: a static-dictionary word lies beyond max_backward (encode.c:1240) */
  if (cmd_copy_len(c) && c->cmd_prefix >= 128 && dcode >= 16 && dcode - 15 <= ((1u << lgwin) - 16))
    EDGE_MAX(max_distance, dcode - 15);
}

/* brotli_bit_stream.c:82 StoreCommandExtra */
static void store_cmd_extra(const Cmd* c, BitW* w) {
  uint32_t clc = cmd_copy_len_code(c);
  uint16_t ic = ins_code(c->insert_len), cc = copy_code(clc);
  uint32_t insn = kInsExtra[ic];
  uint64_t insv = c->insert_len - kInsBase[ic], copyv = clc - kCopyBase[cc];
  wbits(w, insn + kCopyExtra[cc], (copyv << insn) | insv);
}

/* A compressed metablock in the making: the literal context choice, the greedy splits with their histograms, then
   the context map and the block encoders of its header. */
typedef struct {
  size_t nctx; const uint32_t* smap;
  Split lit_split, cmd_split, dist_split;
  Splitter ls, cs, ds;
  uint32_t* lit_cmap; size_t lit_cmap_size;
  BlockEnc le, ce, de;
  HTree* tree;
} MbStore;

/* encode.c:561 DecideOverLiteralContextModeling (skipped under disable_ctx) + metablock.c:708
   BrotliBuildMetaBlockGreedyInternal: the splits and their histograms, not yet smoothed. */
static void mb_build_splits(const Enc* e, size_t start_pos, int disable_ctx, size_t length, MbStore* s) {
  const uint8_t* in = e->data;
  const Cmd* cmds = e->cmds; const size_t ncmd = e->num_cmds;
  size_t num_literals = 0, i, pos;
  uint8_t p1 = e->prev_byte, p2 = e->prev_byte2;
  memset(s, 0, sizeof(*s));
  s->nctx = 1;
  if (!disable_ctx) decide_context_modeling(e, start_pos, length, &s->nctx, &s->smap);
  for (i = 0; i < ncmd; ++i) num_literals += cmds[i].insert_len;
  splitter_init(&s->ls, 256, s->nctx, 512, 400.0, num_literals, &s->lit_split);
  splitter_init(&s->cs, 704, 1, 1024, 500.0, ncmd, &s->cmd_split);
  splitter_init(&s->ds, 64, 1, 512, 100.0, ncmd, &s->dist_split);
  pos = start_pos;
  for (i = 0; i < ncmd; ++i) {
    const Cmd c = cmds[i]; size_t j;
    splitter_add(&s->cs, c.cmd_prefix, 0);
    for (j = c.insert_len; j != 0; --j) {
      uint8_t lit = in[pos];
      if (s->nctx == 1) splitter_add(&s->ls, lit, 0);
      else splitter_add(&s->ls, lit, s->smap[CTX_UTF8(p1, p2)]);
      p2 = p1; p1 = lit; ++pos;
    }
    pos += cmd_copy_len(&c);
    if (cmd_copy_len(&c)) {
      p2 = in[pos - 2]; p1 = in[pos - 1];
      if (c.cmd_prefix >= 128) splitter_add(&s->ds, c.dist_prefix & 0x3FF, 0);
    }
  }
  splitter_finish_block(&s->ls, 1);
  splitter_finish_block(&s->cs, 1);
  splitter_finish_block(&s->ds, 1);
}

/* metablock.c:677 MapStaticContexts, :841 OptimizeHistograms and brotli_bit_stream.c:947 BrotliStoreMetaBlock up to
   the last prefix code: the header, the block-split codes, the context maps and every code. */
static void mb_store_header_and_codes(MbStore* s, size_t length, int is_last, BitW* w) {
  const size_t nctx = s->nctx;
  size_t i;
  uint8_t good_for_rle[704];
  s->tree = (HTree*)malloc(sizeof(HTree) * (2 * 704 + 1));
  if (nctx > 1) {  /* metablock.c:677 MapStaticContexts */
    size_t j;
    s->lit_cmap_size = s->lit_split.num_types << 6;
    s->lit_cmap = (uint32_t*)malloc(s->lit_cmap_size * 4);
    for (i = 0; i < s->lit_split.num_types; ++i)
      for (j = 0; j < 64; ++j) s->lit_cmap[(i << 6) + j] = (uint32_t)(i * nctx) + s->smap[j];
  }
  if (nctx == 1) ++g_edge.ctx_nc1; else if (nctx == 2) ++g_edge.ctx_nc2; else if (nctx == 3) ++g_edge.ctx_nc3; else ++g_edge.ctx_nc13;
  if (s->lit_split.num_types == 256 / nctx) {
    if (nctx == 1) ++g_edge.lit_cap_nc1; else if (nctx == 2) ++g_edge.lit_cap_nc2; else if (nctx == 3) ++g_edge.lit_cap_nc3;
    else ++g_edge.lit_cap_nc13;
  }
  if (s->cmd_split.num_types == 256) ++g_edge.cmd_cap;
  if (s->dist_split.num_types == 256) ++g_edge.dist_cap;
  EDGE_MAX(max_lit_types, s->lit_split.num_types); EDGE_MAX(max_lit_trees, s->ls.histograms_size);
  g_edge.codes += s->ls.histograms_size + s->cs.histograms_size + s->ds.histograms_size;
  EDGE_MAX(max_cmd_types, s->cmd_split.num_types); EDGE_MAX(max_dist_types, s->dist_split.num_types);
  { const Split* sp[3] = {&s->lit_split, &s->cmd_split, &s->dist_split}; size_t k;   /* lengths are stored with 2+ types only */
    for (k = 0; k < 3; ++k)
      if (sp[k]->num_types > 1)
        for (i = 0; i < sp[k]->num_blocks; ++i) EDGE_MAX(max_block_len, sp[k]->lengths[i]); }
  for (i = 0; i < s->ls.histograms_size; ++i) optimize_counts_for_rle(256, s->ls.histograms + i * 256, good_for_rle);
  for (i = 0; i < s->cs.histograms_size; ++i) optimize_counts_for_rle(704, s->cs.histograms + i * 704, good_for_rle);
  for (i = 0; i < s->ds.histograms_size; ++i) optimize_counts_for_rle(64, s->ds.histograms + i * 64, good_for_rle);

  /* header: brotli_bit_stream.c:120 */
  wbits(w, 1, (uint64_t)is_last);
  if (is_last) wbits(w, 1, 0);
  store_mlen(length, w);
  if (!is_last) wbits(w, 1, 0);

  block_enc_init(&s->le, 256, &s->lit_split);
  block_enc_init(&s->ce, 704, &s->cmd_split);
  block_enc_init(&s->de, 64, &s->dist_split);
  build_and_store_block_split_code(&s->le, s->tree, w);
  build_and_store_block_split_code(&s->ce, s->tree, w);
  build_and_store_block_split_code(&s->de, s->tree, w);
  wbits(w, 2, 0);  /* NPOSTFIX */
  wbits(w, 4, 0);  /* NDIRECT >> NPOSTFIX */
  for (i = 0; i < s->lit_split.num_types; ++i) wbits(w, 2, 2);  /* CONTEXT_UTF8 */
  if (s->lit_cmap_size == 0) store_trivial_context_map(s->ls.histograms_size, 6, s->tree, w);
  else encode_context_map(s->lit_cmap, s->lit_cmap_size, s->ls.histograms_size, s->tree, w);
  store_trivial_context_map(s->ds.histograms_size, 2, s->tree, w);

  s->le.depths = (uint8_t*)malloc(s->ls.histograms_size * 256 + 1); s->le.bits = (uint16_t*)malloc(s->ls.histograms_size * 512 + 2);
  s->ce.depths = (uint8_t*)malloc(s->cs.histograms_size * 704 + 1); s->ce.bits = (uint16_t*)malloc(s->cs.histograms_size * 1408 + 2);
  s->de.depths = (uint8_t*)malloc(s->ds.histograms_size * 64 + 1); s->de.bits = (uint16_t*)malloc(s->ds.histograms_size * 128 + 2);
  for (i = 0; i < s->ls.histograms_size; ++i)
    build_and_store_tree(s->ls.histograms + i * 256, 256, 256, s->tree, s->le.depths + i * 256, s->le.bits + i * 256, w);
  for (i = 0; i < s->cs.histograms_size; ++i)
    build_and_store_tree(s->cs.histograms + i * 704, 704, 704, s->tree, s->ce.depths + i * 704, s->ce.bits + i * 704, w);
  for (i = 0; i < s->ds.histograms_size; ++i)
    build_and_store_tree(s->ds.histograms + i * 64, 64, 64, s->tree, s->de.depths + i * 64, s->de.bits + i * 64, w);
}
static void mb_free(MbStore* s) {
  free(s->le.depths); free(s->le.bits); free(s->ce.depths); free(s->ce.bits); free(s->de.depths); free(s->de.bits);
  free(s->lit_cmap); free(s->tree);
  splitter_free(&s->ls); splitter_free(&s->cs); splitter_free(&s->ds);
}

static void store_compressed_metablock(Enc* e, size_t start_pos, size_t length,
                                       int is_last, BitW* w) {
  const uint8_t* in = e->data;
  const Cmd* cmds = e->cmds; const size_t ncmd = e->num_cmds;
  size_t i, pos;
  uint8_t p1, p2;
  MbStore s;
  mb_build_splits(e, start_pos, 0, length, &s);
  mb_store_header_and_codes(&s, length, is_last, w);
  pos = start_pos; p1 = e->prev_byte; p2 = e->prev_byte2;
  for (i = 0; i < ncmd; ++i) {
    const Cmd c = cmds[i]; size_t j;
    edge_cmd(&c, e->lgwin);
    store_symbol(&s.ce, c.cmd_prefix, w);
    store_cmd_extra(&c, w);
    if (s.lit_cmap_size == 0) {
      for (j = c.insert_len; j != 0; --j) { store_symbol(&s.le, in[pos], w); ++pos; }
    } else {
      for (j = c.insert_len; j != 0; --j) {
        uint8_t lit = in[pos];
        store_symbol_ctx(&s.le, lit, CTX_UTF8(p1, p2), s.lit_cmap, w);
        p2 = p1; p1 = lit; ++pos;
      }
    }
    pos += cmd_copy_len(&c);
    if (cmd_copy_len(&c)) {
      p2 = in[pos - 2]; p1 = in[pos - 1];
      if (c.cmd_prefix >= 128) {
        store_symbol(&s.de, c.dist_prefix & 0x3FF, w);
        wbits(w, c.dist_prefix >> 10, c.dist_extra);
      }
    }
  }
  if (is_last) { w->ix = (w->ix + 7u) & ~(size_t)7u; w->buf[w->ix >> 3] = 0; }
  mb_free(&s);
}

/* The entropy stage of quality 4..9 up to the last prefix code, on metablocks the caller describes (the counterpart of
   the product's br_debug_split hook, with its arguments): mbw holds 7 words per metablock (start, end, first command,
   command count, is_last, compress, base: the first byte of its stream, where the literal context starts from zeros).
   cmds: 16 bytes each (oracle_make_cmd), covering the input in order.  For every compressed metablock the record of
   br_split_record: which, num_types[3], num_blocks[3], the bit count; per category types and lengths (a word each); the
   histograms before smoothing (literal rows of 256, command rows of 704, distance rows of 64); then the header, the
   block-split codes, the context maps and every prefix code as (bits + 31) / 32 words.  Writes at most cap words to
   out and returns the words the records take, 0 on a description that does not hold together (metablocks that do not
   follow each other, or commands that do not cover their metablock exactly), as br_split_synth rejects it. */
size_t oracle_split(const uint8_t* in, size_t n, const Cmd* cmds, size_t ncmd, const uint32_t* mbw, size_t n_mbs,
                    int quality, size_t size_hint, int disable_ctx, uint32_t* out, size_t cap) {
  size_t k = 0, m, c = 0, i, covered = 0;
#define PUT(v) do { if (k < cap) out[k] = (uint32_t)(v); ++k; } while (0)
  if (quality < 4 || quality > 9) return 0;
  for (m = 0; m < n_mbs; ++m) {
    const uint32_t* w = mbw + 7 * m;
    const size_t start = w[0], end = w[1], base = w[6];
    Enc e; MbStore s; BitW bw; uint8_t* buf; size_t cat;
    if (w[2] != c || w[3] == 0 || c + w[3] > ncmd || end <= start || end > n || base > start || start != covered) return 0;
    { size_t span = 0;
      for (i = c; i < c + w[3]; ++i) span += (size_t)cmds[i].insert_len + cmd_copy_len(&cmds[i]);
      if (span != end - start) return 0; }
    c += w[3]; covered = end;
    if (!w[5]) continue;
    memset(&e, 0, sizeof(e));
    e.quality = quality; e.size_hint = size_hint; e.data = in; e.n = n;
    e.cmds = (Cmd*)(cmds + w[2]); e.num_cmds = w[3];
    e.prev_byte = start >= base + 1 ? in[start - 1] : 0; e.prev_byte2 = start >= base + 2 ? in[start - 2] : 0;
    mb_build_splits(&e, start, disable_ctx, end - start, &s);
    PUT(s.nctx);
    PUT(s.lit_split.num_types); PUT(s.cmd_split.num_types); PUT(s.dist_split.num_types);
    PUT(s.lit_split.num_blocks); PUT(s.cmd_split.num_blocks); PUT(s.dist_split.num_blocks);
    { const size_t at_bits = k; const Split* sp[3] = {&s.lit_split, &s.cmd_split, &s.dist_split};
      const Splitter* sr[3] = {&s.ls, &s.cs, &s.ds};
      PUT(0);
      for (cat = 0; cat < 3; ++cat) {
        for (i = 0; i < sp[cat]->num_blocks; ++i) PUT(sp[cat]->types[i]);
        for (i = 0; i < sp[cat]->num_blocks; ++i) PUT(sp[cat]->lengths[i]);
      }
      for (cat = 0; cat < 3; ++cat)
        for (i = 0; i < sr[cat]->histograms_size * sr[cat]->alphabet; ++i) PUT(sr[cat]->histograms[i]);
      buf = (uint8_t*)calloc(2 * (end - start) + 4096 + 1024 * (s.ls.histograms_size + s.cs.histograms_size + s.ds.histograms_size), 1);
      bw.buf = buf; bw.ix = 0;
      mb_store_header_and_codes(&s, end - start, (int)w[4], &bw);
      if (at_bits < cap) out[at_bits] = (uint32_t)bw.ix;
      for (i = 0; i < (bw.ix + 31) / 32; ++i) { uint32_t v; memcpy(&v, buf + 4 * i, 4); PUT(v); }
      free(buf); }
    mb_free(&s);
  }
#undef PUT
  return c == ncmd && covered == n ? k : 0;
}
/* The static literal context map of nctx contexts (2, 3 or 13; encode.c:277, :341), 64 entries. */
int oracle_static_context_map(size_t nctx, uint32_t* out) {
  const uint32_t* map = nctx == 2 ? kCtxMapSimpleUTF8 : nctx == 3 ? kCtxMapContinuation : nctx == 13 ? kCtxMapComplexUTF8 : NULL;
  if (!map) return 0;
  memcpy(out, map, 64 * 4);
  return 1;
}
/* command.h:120 InitCommand for callers that build command lists (the split tests): insert, copy length, the delta of
   the copy length code and the distance code (0..15: the last-distance codes, else distance + 15). */
void oracle_make_cmd(uint32_t insert, uint32_t copy, int copy_code_delta, uint32_t dcode, Cmd* out) {
  init_cmd(out, insert, copy, copy_code_delta, dcode);
}
/* command.h:138 InitInsertCommand */
void oracle_make_insert_cmd(uint32_t insert, Cmd* out) { init_insert_cmd(out, insert); }

static void emit(Enc* e, const uint8_t* p, size_t n) {
  if (e->out_pos + n > e->out_cap) { e->overflow = 1; return; }
  memcpy(e->out + e->out_pos, p, n);
  e->out_pos += n;
}

static void store_metablock_fast_trivial(Enc* e, size_t start_pos, size_t length, int is_last, BitW* w);

/* encode.c:498 WriteMetaBlockInternal + tail of encode.c:985 EncodeData */
static void write_metablock(Enc* e, size_t end_pos, int is_last) {
  const size_t bytes = end_pos - e->last_flush_pos;
  uint8_t* storage = (uint8_t*)calloc(2 * bytes + 503 + 16, 1);
  BitW w; w.buf = storage; w.ix = e->carry_bits;
  storage[0] = e->carry;
  if (e->cmd_hook) e->cmd_hook(e->cmds, e->num_cmds, e->last_flush_pos, bytes);
  if (bytes == 0) {
    wbits(&w, 2, 3);
    w.ix = (w.ix + 7u) & ~(size_t)7u;
  } else if (!should_compress(e, bytes)) {
    memcpy(e->dist_cache, e->saved_dist_cache, 4 * sizeof(int));
    store_uncompressed(is_last, e->data, e->last_flush_pos, bytes, &w);
  } else {
    const size_t edge_words = sizeof(g_edge) / sizeof(uint64_t);
    uint64_t edge_before[sizeof(g_edge) / sizeof(uint64_t)];
    oracle_edge_stats(edge_before, edge_words);
    if (e->quality < 4) store_metablock_fast_trivial(e, e->last_flush_pos, bytes, is_last, &w);   /* encode.c:543-556 */
    else store_compressed_metablock(e, e->last_flush_pos, bytes, is_last, &w);
    if (bytes + 4 < (w.ix >> 3)) {
      memcpy(&g_edge, edge_before, sizeof(g_edge));
      memcpy(e->dist_cache, e->saved_dist_cache, 4 * sizeof(int));
      memset(storage, 0, 2 * bytes + 503 + 16);
      storage[0] = e->carry; w.ix = e->carry_bits;
      store_uncompressed(is_last, e->data, e->last_flush_pos, bytes, &w);
    }
  }
  emit(e, storage, w.ix >> 3);
  e->carry = storage[w.ix >> 3];
  e->carry_bits = (unsigned)(w.ix & 7u);
  free(storage);
  e->last_flush_pos = end_pos;
  if (end_pos > 0) e->prev_byte = e->data[end_pos - 1];
  if (end_pos > 1) e->prev_byte2 = e->data[end_pos - 2];
  e->num_cmds = 0; e->num_literals = 0;
  memcpy(e->saved_dist_cache, e->dist_cache, sizeof(e->saved_dist_cache));
}

/* encode.c:905 ExtendLastCommand (no compound dictionary) */
static void extend_last_command(Enc* e, size_t* bytes, size_t* pos) {
  Cmd* last = &e->cmds[e->num_cmds - 1];
  uint64_t max_backward = ((uint64_t)1 << e->lgwin) - 16;
  uint64_t last_copy_len = last->copy_len & 0x1FFFFFF;
  uint64_t last_processed = *pos - last_copy_len;
  uint64_t max_distance = last_processed < max_backward ? last_processed : max_backward;
  uint64_t cmd_dist = (uint64_t)e->dist_cache[0];
  uint32_t dcode = cmd_restore_dcode(last);
  if (dcode < 16 || dcode - 15 == cmd_dist) {
    if (cmd_dist <= max_distance) {
      while (*bytes != 0 && e->data[*pos] == e->data[*pos - cmd_dist]) {
        last->copy_len++; (*bytes)--; (*pos)++;
      }
    }
    last->cmd_prefix = length_code(last->insert_len,
        (size_t)((int)(last->copy_len & 0x1FFFFFF) + (int)(last->copy_len >> 25)),
        (last->dist_prefix & 0x3FF) == 0);
  }
}

/* Block size, hasher and ring buffer of an encoder for (quality, lgwin, BROTLI_PARAM_LGBLOCK (0: the encoder's choice),
   BROTLI_PARAM_SIZE_HINT); returns MaxMetablockSize. */
static size_t setup_hasher(Enc* e, int quality, int lgwin, int lgblock_user, size_t size_hint) {
  e->quality = quality; e->lgwin = lgwin; e->size_hint = size_hint;
  /* quality.h:75 ComputeLgBlock */
  e->lgblock = quality < 4 ? 14 : 16;
  if (quality >= 9 && lgwin > 16) e->lgblock = lgwin < 18 ? lgwin : 18;
  if (lgblock_user && quality >= 4) e->lgblock = lgblock_user > 24 ? 24 : lgblock_user < 16 ? 16 : lgblock_user;
  if (quality < 5) {
    /* quality.h:172 ChooseHasher: H2, H3, H4, and H54 for quality 4 on inputs >= 1 MiB (hash.h:251-338) */
    e->quick = 1; e->qk_hash_len = 5;
    if (quality == 2) { e->qk_bits = 16; e->qk_sweep_bits = 0; e->qk_dict = 1; }
    else if (quality == 3) { e->qk_bits = 16; e->qk_sweep_bits = 1; e->qk_dict = 0; }
    else if (size_hint >= (1u << 20)) { e->qk_bits = 20; e->qk_sweep_bits = 2; e->qk_dict = 0; e->qk_hash_len = 7; }
    else { e->qk_bits = 17; e->qk_sweep_bits = 2; e->qk_dict = 1; }
    e->qk_table = (uint32_t*)calloc((size_t)1 << e->qk_bits, 4);
    e->ndist = 1;
    e->hash_type_len = 8; e->store_lookahead = 8;
  } else {
    e->hash64 = (size_hint >= (1u << 20) && lgwin >= 19);
    e->block_bits = quality - 1;
    e->bucket_bits = e->hash64 ? 15 : (quality < 7 ? 14 : 15);
    e->ndist = quality < 7 ? 4 : quality < 9 ? 10 : 16;
    e->hash_type_len = e->hash64 ? 8 : 4;
    e->store_lookahead = e->hash_type_len;
    e->num = (uint16_t*)calloc((size_t)1 << e->bucket_bits, 2);
    e->buckets = (uint32_t*)calloc((size_t)1 << (e->bucket_bits + e->block_bits), 4);
  }
  { int rb = 1 + (lgwin > e->lgblock ? lgwin : e->lgblock);
    e->rmask = ((size_t)1 << rb) - 1;
    return (size_t)1 << (rb < 24 ? rb : 24); }
}

/* One-shot driver: encode.c:1296 BrotliEncoderCompress ->
   :1634 CompressStream(FINISH) -> :985 EncodeData per input block. */
static int oracle_compress_impl(int quality, int lgwin, size_t n, const uint8_t* in,
    size_t* out_n, uint8_t* out, void (*hook)(const Cmd*, size_t, size_t, size_t)) {
  Enc e; size_t pos = 0, block, max_mb;
  if (!g_blob) return 0;
  if (quality < 2 || quality > 9 || lgwin > 24) return 0;
  if (quality >= 5 ? lgwin < 17 : lgwin < 10) return 0;      /* lgwin <= 16 at quality 5+: H40..42, not restated */
  if (n == 0) { if (*out_n < 1) return 0; out[0] = 6; *out_n = 1; return 1; }
  memset(&e, 0, sizeof(e));
  e.data = in; e.n = n;
  e.cmd_hook = hook;
  max_mb = setup_hasher(&e, quality, lgwin, 0, n);
  e.dist_cache[0] = 4; e.dist_cache[1] = 11; e.dist_cache[2] = 15; e.dist_cache[3] = 16;
  memcpy(e.saved_dist_cache, e.dist_cache, 16);
  e.cmds = (Cmd*)malloc(sizeof(Cmd) * (max_mb / 2 + (1u << e.lgblock) + 64));
  e.out = out; e.out_cap = *out_n;
  /* encode.c:203 EncodeWindowBits */
  if (lgwin == 16) { e.carry = 0; e.carry_bits = 1; }
  else if (lgwin == 17) { e.carry = 1; e.carry_bits = 7; }
  else if (lgwin > 17) { e.carry = (uint8_t)(((lgwin - 17) << 1) | 1); e.carry_bits = 4; }
  else { e.carry = (uint8_t)(((lgwin - 8) << 4) | 1); e.carry_bits = 7; }
  block = (size_t)1 << e.lgblock;
  while (pos < n) {
    size_t bytes = n - pos < block ? n - pos : block;
    size_t p = pos, end = pos + bytes;
    int is_last = end == n;
    /* hash_longest_match64_inc.h:127 StitchToPreviousBlock */
    if (bytes >= e.hash_type_len - 1 && p >= 3) { hstore(&e, p - 3); hstore(&e, p - 2); hstore(&e, p - 1); }
    if (e.num_cmds && e.last_insert_len == 0) extend_last_command(&e, &bytes, &p);
    create_backward_references(&e, bytes, p);
    {
      const size_t processed = end - e.last_flush_pos;
      const int next_fits = processed + block <= max_mb;
      /* encode.c:1152: below quality 4 at most MAX_NUM_DELAYED_SYMBOLS literals + commands are buffered */
      const int should_flush = quality < 4 && e.num_literals + e.num_cmds >= 0x2FFF;
      if (!is_last && !should_flush && next_fits && e.num_literals < max_mb / 8 && e.num_cmds < max_mb / 8) {
        pos = end; continue;
      }
    }
    if (e.last_insert_len > 0) {
      init_insert_cmd(&e.cmds[e.num_cmds++], e.last_insert_len);
      e.num_literals += e.last_insert_len;
      e.last_insert_len = 0;
    }
    write_metablock(&e, end, is_last);
    pos = end;
  }
  free(e.num); free(e.buckets); free(e.qk_table); free(e.cmds);
  if (e.overflow) return 0;
  *out_n = e.out_pos;
  return 1;
}

#include "brotli_oracle_q1.h"

/* brotli_bit_stream.c:1196 BrotliStoreMetaBlockTrivial (quality 3) and :1243 BrotliStoreMetaBlockFast
   (quality 2): one code per category, no block splits, no contexts. */
static void store_metablock_fast_trivial(Enc* e, size_t start_pos, size_t length, int is_last, BitW* w) {
  const uint8_t* in = e->data;
  const Cmd* cmds = e->cmds; const size_t ncmd = e->num_cmds;
  uint32_t lit_histo[256], cmd_histo[704], dist_histo[140];
  uint8_t lit_depth[256], cmd_depth[704], dist_depth[140];
  uint16_t lit_bits[256], cmd_bits[704], dist_bits[140];
  HTree* tree = (HTree*)malloc(sizeof(HTree) * (2 * 704 + 1));
  size_t i, pos = start_pos, nlit = 0, ndist = 0;
  g_edge.codes += 3;
  memset(lit_histo, 0, sizeof(lit_histo)); memset(cmd_histo, 0, sizeof(cmd_histo)); memset(dist_histo, 0, sizeof(dist_histo));
  memset(lit_depth, 0, sizeof(lit_depth)); memset(cmd_depth, 0, sizeof(cmd_depth)); memset(dist_depth, 0, sizeof(dist_depth));
  memset(lit_bits, 0, sizeof(lit_bits)); memset(cmd_bits, 0, sizeof(cmd_bits)); memset(dist_bits, 0, sizeof(dist_bits));
  for (i = 0; i < ncmd; ++i) {          /* :1133 BuildHistograms */
    const Cmd c = cmds[i]; size_t j;
    ++cmd_histo[c.cmd_prefix];
    for (j = c.insert_len; j != 0; --j) { ++lit_histo[in[pos]]; ++pos; }
    nlit += c.insert_len;
    pos += cmd_copy_len(&c);
    if (cmd_copy_len(&c) && c.cmd_prefix >= 128) { ++dist_histo[c.dist_prefix & 0x3FF]; ++ndist; }
  }
  /* :120 StoreCompressedMetaBlockHeader, then 13 zero bits: one block type per category, NPOSTFIX / NDIRECT 0,
     context mode, trivial context maps */
  wbits(w, 1, (uint64_t)is_last);
  if (is_last) wbits(w, 1, 0);
  store_mlen(length, w);
  if (!is_last) wbits(w, 1, 0);
  wbits(w, 13, 0);
  if (e->quality == 3) {
    build_and_store_tree(lit_histo, 256, 256, tree, lit_depth, lit_bits, w);
    build_and_store_tree(cmd_histo, 704, 704, tree, cmd_depth, cmd_bits, w);
    build_and_store_tree(dist_histo, 140, 64, tree, dist_depth, dist_bits, w);
  } else if (ncmd <= 128) {
    /* static command / distance codes of entropy_encode_static.h: depths 9 (symbols < 448) and 11, resp. 6;
       their serialised forms (:524, :538) are what brotli_bit_stream.c:283 makes of those depths */
    q1_build_and_store_tree_fast(lit_histo, nlit, 8, lit_depth, lit_bits, w);
    for (i = 0; i < 704; ++i) cmd_depth[i] = i < 448 ? 9 : 11;
    for (i = 0; i < 64; ++i) dist_depth[i] = 6;
    depths_to_symbols(cmd_depth, 704, cmd_bits);
    depths_to_symbols(dist_depth, 64, dist_bits);
    wbits(w, 56, 0x0092624416307003ull); wbits(w, 3, 0);
    wbits(w, 28, 0x0369DC03u);
  } else {
    q1_build_and_store_tree_fast(lit_histo, nlit, 8, lit_depth, lit_bits, w);
    q1_build_and_store_tree_fast(cmd_histo, ncmd, 10, cmd_depth, cmd_bits, w);
    q1_build_and_store_tree_fast(dist_histo, ndist, 6, dist_depth, dist_bits, w);
  }
  pos = start_pos;
  for (i = 0; i < ncmd; ++i) {          /* :1159 StoreDataWithHuffmanCodes */
    const Cmd c = cmds[i]; size_t j;
    edge_cmd(&c, e->lgwin);
    wbits(w, cmd_depth[c.cmd_prefix], cmd_bits[c.cmd_prefix]);
    store_cmd_extra(&c, w);
    for (j = c.insert_len; j != 0; --j) { wbits(w, lit_depth[in[pos]], lit_bits[in[pos]]); ++pos; }
    pos += cmd_copy_len(&c);
    if (cmd_copy_len(&c) && c.cmd_prefix >= 128) {
      const size_t dc = c.dist_prefix & 0x3FF;
      wbits(w, dist_depth[dc], dist_bits[dc]);
      wbits(w, c.dist_prefix >> 10, c.dist_extra);
    }
  }
  if (is_last) { w->ix = (w->ix + 7u) & ~(size_t)7u; w->buf[w->ix >> 3] = 0; }
  free(tree);
}

int oracle_brotli_compress(int quality, int lgwin, size_t n, const uint8_t* in,
                           size_t* out_n, uint8_t* out) {
  if (quality == 1) {
    if (n == 0) { if (*out_n < 1) return 0; out[0] = 6; *out_n = 1; return 1; }   /* encode.c:1310 */
    {
      /* encode.c:1345: a stream longer than BrotliEncoderMaxCompressedSize (:1251) is replaced by
         the raw stream of :1264 MakeUncompressedStream (window 10, empty metadata block, raw
         meta-blocks of at most 2^24 bytes, empty last meta-block) */
      const size_t cap = *out_n, bound = n + 4 * (n >> 14) + 6;
      size_t got = cap + 2 * n + 65536;
      uint8_t* tmp = (uint8_t*)malloc(got);
      int ok = oracle_brotli_compress_q1(lgwin, n, in, 0, NULL, &got, tmp);
      if (ok && got <= bound) {
        ok = got <= cap;
        if (ok) { memcpy(out, tmp, got); *out_n = got; }
      } else if (ok) {
        size_t o = 0, off = 0;
        ok = cap >= bound;
        if (ok) {
          out[o++] = 0x21; out[o++] = 0x03;
          while (off < n) {
            const uint32_t len = n - off > (1u << 24) ? (1u << 24) : (uint32_t)(n - off);
            const uint32_t nib = len > (1u << 20) ? 2 : len > (1u << 16) ? 1 : 0;   /* MNIBBLES - 4 */
            const uint32_t hdr = (nib << 1) | ((len - 1) << 3) | (1u << (19 + 4 * nib));
            uint32_t k;
            for (k = 0; k < 3 + (nib == 2); ++k) out[o++] = (uint8_t)(hdr >> (8 * k));
            memcpy(out + o, in + off, len); o += len; off += len;
          }
          out[o++] = 3;
          *out_n = o;
        }
      }
      free(tmp);
      return ok;
    }
  }
  return oracle_compress_impl(quality, lgwin, n, in, out_n, out, NULL);
}
/* tests: cb(cmds(16B each), ncmds, metablock_start, metablock_bytes) */
int oracle_brotli_compress_hook(int quality, int lgwin, size_t n, const uint8_t* in,
    size_t* out_n, uint8_t* out, void (*hook)(const void*, size_t, size_t, size_t)) {
  return oracle_compress_impl(quality, lgwin, n, in, out_n, out,
      (void (*)(const Cmd*, size_t, size_t, size_t))hook);
}

/* tests/test_search_probe.py: one FindLongestMatch per probe, from a fully specified hash-table state.
 * data: one stream (n bytes, followed by at least 16 readable bytes); snap / own: one byte per position of the stream, the
 * stored bits of the two bitmaps.  Position q counts as inserted in front of a search when q >= p0 ? own[q] : snap[q].
 * probes (16 words each, ascending cur): cur, p0, base, pend, max_backward, dict_distance, dc[0..3], len_in, score_in,
 * dict_l (lo, hi), dict_m (lo, hi).  Positions count from the batch's first byte: the stream starts at `base`.
 * res (16 words each): len, distance, score, delta, dict lookups and matches added, gate checks, gate closed, whether cur
 * was inserted, whether it was searched; the rest zero.
 * Before each search the probe's stream is hashed into a fresh table in position order: every inserted q < cur.  Only
 * the bucket (H5 / H6) or the slots (quick hashers) the search reads can affect it, so only the positions filed there are
 * inserted.  The insertion of cur that the search makes is undone afterwards. */
int oracle_search_probe(int quality, int lgwin, int lgblock, size_t size_hint, const uint8_t* data, size_t n,
                        const uint8_t* snap, const uint8_t* own, const uint32_t* probes, size_t nprobes, uint32_t* res) {
  Enc e; size_t i, nkeys, hashable;
  uint32_t *start, *pos;
  if (!g_blob || quality < 2 || quality > 9) return 0;
  memset(&e, 0, sizeof(e));
  e.data = data; e.n = n;
  setup_hasher(&e, quality, lgwin, lgblock, size_hint);
  /* positions by bucket / slot (counting sort); the last HashTypeLength - 1 are never inserted */
  nkeys = e.quick ? (size_t)1 << e.qk_bits : (size_t)1 << e.bucket_bits;
  hashable = n >= e.hash_type_len ? n - e.hash_type_len + 1 : 0;
  start = (uint32_t*)calloc(nkeys + 2, 4); pos = (uint32_t*)malloc(4 * (hashable + 1));
  {
    uint32_t* key = (uint32_t*)malloc(4 * (hashable + 1));
    const size_t qmask = ((size_t)1 << e.qk_bits) - 1;
    for (i = 0; i < hashable; ++i) {
      key[i] = (uint32_t)(e.quick ? (quick_key(&e, i) + (i & (((1u << e.qk_sweep_bits) - 1u) << 3))) & qmask : hash_key(&e, i));
      ++start[key[i] + 2];
    }
    for (i = 2; i < nkeys + 2; ++i) start[i] += start[i - 1];
    for (i = 0; i < hashable; ++i) pos[start[key[i] + 1]++] = (uint32_t)i;
    free(key);
  }
  for (i = 0; i < nprobes; ++i) {
    const uint32_t* pr = probes + 16 * i;
    uint32_t* r = res + 16 * i;
    const size_t base = pr[2], cur = pr[0] - base, p0 = pr[1] > base ? pr[1] - base : 0, pend = pr[3] - base;
    const size_t block_size = (size_t)1 << e.block_bits;
    const uint64_t dict_l = ((uint64_t)pr[13] << 32) | pr[12], dict_m = ((uint64_t)pr[15] << 32) | pr[14];
    const uint64_t closed0 = g_edge.srch_gate_closed;
    size_t keys[4], nk = 0, k, j, key = 0;
    SR sr;
    if (e.quick) {
      const size_t sweep = (size_t)1 << e.qk_sweep_bits, mask = ((size_t)1 << e.qk_bits) - 1;
      key = quick_key(&e, cur);
      for (k = 0; k < sweep; ++k) { keys[nk++] = (key + (k << 3)) & mask; e.qk_table[keys[k]] = 0; }
    } else {
      key = hash_key(&e, cur);
      keys[nk++] = key; e.num[key] = 0;
    }
    for (k = 0; k < nk; ++k) {
      size_t c = 0;
      for (j = start[keys[k]]; j < start[keys[k] + 1] && pos[j] < cur; ++j) {
        const size_t q = pos[j];
        if (q >= p0 ? own[q] : snap[q]) { hstore(&e, q); ++c; }
      }
      if (!e.quick && c >= 65536 && (c & 0xFFFF) < block_size) ++g_edge.srch_wrap_cut;
    }
    for (k = 0; k < 4; ++k) e.dist_cache[k] = (int)pr[6 + k];
    prepare_dist_cache(e.dist_cache, e.ndist);
    e.dict_lookups = (size_t)dict_l; e.dict_matches = (size_t)dict_m;
    sr.len = pr[10]; sr.score = pr[11]; sr.distance = 0; sr.len_code_delta = 0;
    find_longest_match(&e, cur, pend - cur, pr[4], pr[5], 0x3FFFFFC, &sr);
    if (!e.quick) --e.num[key];   /* (the quick hashers' slots are refilled by the next probe) */
    memset(r, 0, 16 * 4);
    r[0] = (uint32_t)sr.len; r[1] = (uint32_t)sr.distance; r[2] = (uint32_t)sr.score; r[3] = (uint32_t)sr.len_code_delta;
    r[4] = (uint32_t)(e.dict_lookups - dict_l); r[5] = (uint32_t)(e.dict_matches - dict_m);
    r[7] = (uint32_t)(g_edge.srch_gate_closed - closed0);
    r[6] = r[7] + (r[4] != 0);
    r[8] = r[9] = 1;
  }
  free(start); free(pos); free(e.num); free(e.buckets); free(e.qk_table);
  return 1;
}
