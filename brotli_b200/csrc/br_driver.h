// br_driver.h -- the host driver of the BrotliEncoder* C ABI, free of CUDA: what c/enc/encode.c does around its encoder.
// It compresses through a Backend: the GPU in br_api.cc, the CPU simulation in tests/sim/br_sim.cc.
#pragma once
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <new>
#include <vector>
#include <brotli/encode.h>
#include "br_pipeline.h"

namespace br_driver {

struct Params {
  int mode = BROTLI_MODE_GENERIC, quality = 11, lgwin = 22, lgblock = 0;
  uint32_t size_hint = 0, disable_ctx = 0, large_window = 0, npostfix = 0, ndirect = 0, stream_offset = 0,
           base64 = 0;
};
// What the pipeline implements; everything else must fail rather than emit different bytes.
inline bool supported(Params p) {
  if (p.quality > 11) p.quality = 11;          // quality.h:60 SanitizeParams
  if (p.quality < 0) p.quality = 0;
  if (p.quality <= 2) p.large_window = 0;      // quality.h:63: no large window with the static entropy codes; lgwin clamps to 24
  if (p.lgwin < 10) p.lgwin = 10;
  if (p.lgwin > 24 && !p.large_window) p.lgwin = 24;
  if (p.quality < 1 || p.quality > 9) return false;   /* quality 0: one-pass fragment coder; 10, 11: Zopfli path */
  if (p.quality <= 4 ? p.lgwin > 24 : (p.lgwin < 17 || p.lgwin > 24)) return false;   /* quality 1..4: any regular window */
  if (p.large_window || p.npostfix || p.ndirect || p.base64) return false;
  if (p.stream_offset && p.quality < 5) return false;   /* STREAM_OFFSET: quality 5..9 only */
  /* LGBLOCK and DISABLE_LITERAL_CONTEXT_MODELING are honoured at quality 5..9; at quality 1 the reference ignores both
     (quality.h:79: lgblock = lgwin; no context modeling in the fragment coder) */
  if (p.mode == BROTLI_MODE_FONT) return false;
  return true;
}
// The window of supported parameters after quality.h:60 SanitizeParams: what the pipeline compresses with.
inline int window_of(const Params& p) { return p.lgwin < 10 ? 10 : p.lgwin > 24 ? 24 : p.lgwin; }
inline int lgblock_of(const Params& p) {   /* quality.h:76 ComputeLgBlock, quality >= 2 */
  if (p.quality < 4) return 14;
  if (p.lgblock != 0) return p.lgblock > 24 ? 24 : p.lgblock < 16 ? 16 : p.lgblock;
  return (p.quality >= 9 && p.lgwin > 16) ? (p.lgwin < 18 ? p.lgwin : 18) : 16;
}
// The parameters of a one-shot call (encode.c:1329): a window above 24 asks for the large window, which supported()
// refuses unless quality <= 2 drops it again.
inline Params oneshot_params(int quality, int lgwin, int mode = BROTLI_MODE_GENERIC) {
  Params p; p.quality = quality; p.lgwin = lgwin; p.mode = mode;
  if (lgwin > 24) p.large_window = 1;
  return p;
}
inline BROTLI_BOOL set_parameter(Params& p, BrotliEncoderParameter id, uint32_t value) {
  switch (id) {
    case BROTLI_PARAM_MODE: p.mode = (int)value; return BROTLI_TRUE;
    case BROTLI_PARAM_QUALITY: p.quality = (int)value; return BROTLI_TRUE;
    case BROTLI_PARAM_LGWIN: p.lgwin = (int)value; return BROTLI_TRUE;
    case BROTLI_PARAM_LGBLOCK: p.lgblock = (int)value; return BROTLI_TRUE;
    case BROTLI_PARAM_DISABLE_LITERAL_CONTEXT_MODELING:
      if (value != 0 && value != 1) return BROTLI_FALSE;
      p.disable_ctx = value; return BROTLI_TRUE;
    case BROTLI_PARAM_SIZE_HINT: p.size_hint = value; return BROTLI_TRUE;
    case BROTLI_PARAM_LARGE_WINDOW: p.large_window = !!value; return BROTLI_TRUE;
    case BROTLI_PARAM_NPOSTFIX: p.npostfix = value; return BROTLI_TRUE;
    case BROTLI_PARAM_NDIRECT: p.ndirect = value; return BROTLI_TRUE;
    case BROTLI_PARAM_STREAM_OFFSET:
      if (value > (1u << 30)) return BROTLI_FALSE;
      p.stream_offset = value; return BROTLI_TRUE;
    case BROTLI_PARAM_BASE64_MODE: p.base64 = value & 1; return BROTLI_TRUE;
    case BROTLI_PARAM_MAX_BASE64_REGIONS: return BROTLI_TRUE;
    case BROTLI_PARAM_SIMD_HASHER: return value > 2 ? BROTLI_FALSE : BROTLI_TRUE;  /* output-equivalent */
    default: return BROTLI_FALSE;
  }
}

// c/enc/encode.c:1264 MakeUncompressedStream
inline size_t make_uncompressed_stream(const uint8_t* input, size_t input_size, uint8_t* output) {
  size_t size = input_size, result = 0, offset = 0;
  if (input_size == 0) { output[0] = 6; return 1; }
  output[result++] = 0x21;
  output[result++] = 0x03;
  while (size > 0) {
    uint32_t nibbles = 0, chunk, bits;
    chunk = size > (1u << 24) ? (1u << 24) : (uint32_t)size;
    if (chunk > (1u << 16)) nibbles = chunk > (1u << 20) ? 2 : 1;
    bits = (nibbles << 1) | ((chunk - 1) << 3) | (1u << (19 + 4 * nibbles));
    output[result++] = (uint8_t)bits;
    output[result++] = (uint8_t)(bits >> 8);
    output[result++] = (uint8_t)(bits >> 16);
    if (nibbles == 2) output[result++] = (uint8_t)(bits >> 24);
    memcpy(&output[result], &input[offset], chunk);
    result += chunk; offset += chunk; size -= chunk;
  }
  output[result++] = 3;
  return result;
}
inline size_t max_compressed_size(size_t input_size) {  /* encode.c:1251 */
  size_t num_large_blocks = input_size >> 14;
  size_t overhead = 2 + (4 * num_large_blocks) + 3 + 1;
  size_t result = input_size + overhead;
  if (input_size == 0) return 2;
  return (result < input_size) ? 0 : result;
}
// encode.c:1337-1353: a compressed stream of `got` bytes for an input of `n` bytes, in a buffer of `cap` bytes, is kept
// when it fits both the buffer and BrotliEncoderMaxCompressedSize; otherwise the raw stream takes its place when the
// buffer holds that bound; otherwise the call fails.
enum Fit { kKeep, kRaw, kFail };
inline bool within_bound(size_t got, size_t n) { const size_t bound = max_compressed_size(n); return !(bound && got > bound); }
inline Fit fit_stream(size_t got, size_t cap, size_t n) {
  if (got <= cap && within_bound(got, n)) return kKeep;
  return (max_compressed_size(n) && cap >= max_compressed_size(n)) ? kRaw : kFail;
}

// Streams shorter than 1 MiB go through the pipeline in groups, one job per group (the streams laid end to end, cuts of
// kind 3 in br_pipeline.h), so the launches, the fixpoint's host round trips and the copies are paid once per group.  A
// group holds at most kBatchGroupBytes ...
static const size_t kBatchGroupBytes = (size_t)128 << 20;
// ... and at most this many streams: every metablock owns ~1.9 MB of scratch in the entropy stage (histograms for up to 256
// block types per category, br_entropy.h BrMbMem), and a stream is at least one metablock
static const size_t kBatchGroupStreams = 8192;
static const size_t kBatchStreamBytes = (size_t)1 << 20;
// Splits streams 0..count-1 into groups of consecutive small streams, in order; `single` receives the empty and the long
// ones, which go one by one.
inline void plan_groups(const size_t* sizes, size_t count, std::vector<std::vector<size_t>>& groups, std::vector<size_t>& single) {
  size_t group_bytes = 0;
  for (size_t i = 0; i < count; ++i) {
    if (sizes[i] == 0 || sizes[i] >= kBatchStreamBytes) { single.push_back(i); continue; }
    if (groups.empty() || group_bytes + sizes[i] > kBatchGroupBytes || groups.back().size() >= kBatchGroupStreams) {
      groups.emplace_back(); group_bytes = 0;
    }
    groups.back().push_back(i); group_bytes += sizes[i];
  }
}
// The cuts of a group of k >= 1 streams, stream j of size sizes[idx ? idx[j] : j]: the stream boundaries, kind 3, the
// largest stream as the size hint; the pipeline fills `ends` (stream_end) with the byte offset where each stream ends.
struct GroupCuts {
  std::vector<uint32_t> pos, kind;
  std::vector<uint64_t> ends;
  BrCuts c;
  uint32_t hint = 0;
  size_t n = 0;
  GroupCuts(const size_t* sizes, const size_t* idx, size_t k) : pos(k, 0), kind(k, 3), ends(k + 1, 0) {
    for (size_t j = 0; j < k; ++j) {
      const size_t sz = sizes[idx ? idx[j] : j];
      n += sz;
      if (j + 1 < k) pos[j] = (uint32_t)n;
      if (sz > hint) hint = (uint32_t)sz;
    }
    memset(&c, 0, sizeof(c));
    c.pos = pos.data(); c.kind = kind.data(); c.n = (uint32_t)(k - 1); c.is_final = 1; c.with_header = 1; c.stream_end = ends.data();
  }
  GroupCuts(const GroupCuts&) = delete;   // c points into the vectors
};

// Buffers of an encoder instance come from the caller's allocator pair when one was given (encode.h:295-306).
template <class T> struct BrAlloc {
  typedef T value_type;
  brotli_alloc_func af = nullptr; brotli_free_func ff = nullptr; void* opaque = nullptr;
  BrAlloc() {}
  BrAlloc(brotli_alloc_func a, brotli_free_func f, void* o) : af(a), ff(f), opaque(o) {}
  template <class U> BrAlloc(const BrAlloc<U>& o) : af(o.af), ff(o.ff), opaque(o.opaque) {}
  T* allocate(size_t n) {
    void* p = af ? af(opaque, n * sizeof(T)) : malloc(n * sizeof(T));
    if (!p) throw std::bad_alloc();
    return (T*)p;
  }
  void deallocate(T* p, size_t) { if (ff) ff(opaque, p); else free(p); }
  template <class U> bool operator==(const BrAlloc<U>& o) const { return af == o.af && ff == o.ff && opaque == o.opaque; }
  template <class U> bool operator!=(const BrAlloc<U>& o) const { return !(*this == o); }
};
typedef std::vector<uint8_t, BrAlloc<uint8_t>> ByteVec;
// LSB-first bit writer over a byte vector (c/enc/write_bits.h:33)
struct BitOut {
  std::vector<uint8_t>& v; uint32_t pb;   // pb: bits used in the last byte (0 = byte aligned)
  void put(uint32_t n, uint64_t bits) {
    for (uint32_t i = 0; i < n; ++i) {
      if (pb == 0) v.push_back(0);
      if ((bits >> i) & 1) v.back() |= (uint8_t)(1u << pb);
      pb = (pb + 1) & 7;
    }
  }
  void align() { pb = 0; }
};
inline void put_window_bits(BitOut& w, int lgwin) {   // encode.c:185 EncodeWindowBits
  if (lgwin == 16) w.put(1, 0);
  else if (lgwin == 17) w.put(7, 1);
  else if (lgwin > 17) w.put(4, (uint64_t)(((lgwin - 17) << 1) | 1));
  else w.put(7, (uint64_t)(((lgwin - 8) << 4) | 1));
}
// encode.c:1228 WriteMetadataHeader + the body (encode.c:1584)
inline void put_metadata(BitOut& w, const std::vector<uint8_t>& meta) {
  const size_t size = meta.size();
  w.put(1, 0); w.put(2, 3); w.put(1, 0);
  if (size == 0) w.put(2, 0);
  else {
    uint32_t nbits = size == 1 ? 1 : (32u - (uint32_t)__builtin_clz((uint32_t)size - 1));
    uint32_t nbytes = (nbits + 7) / 8;
    w.put(2, nbytes); w.put(8 * nbytes, size - 1);
  }
  w.align();
  w.v.insert(w.v.end(), meta.begin(), meta.end());
}

struct Backend {
  // Quality 2..9: [in, in + n) with these cuts (nullable) into `vec` (resized to the stream) or, when vec is null, into
  // out[0, cap); *got = the stream's size.  0 = failed, 1 = done, 2 = compressed but larger than cap.
  int (*compress)(const Params& p, uint32_t size_hint, const uint8_t* in, size_t n, const BrCuts* cuts, uint8_t* out, size_t cap,
                  size_t* got, std::vector<uint8_t>* vec);
  // Quality 1: one segment of a stream as br_q1_compress_batch compresses it (its with_header, end_op, start_bits, end_bit);
  // calls: the sizes of the CompressStream calls that delivered it.  1 = done.
  int (*q1_segment)(int lgwin, const uint8_t* in, size_t n, const std::vector<size_t>& calls, int with_header, int end_op,
                    uint32_t start_bits, uint32_t* end_bit, std::vector<uint8_t>& out);
};

// What a quality-1 stream carries from one segment to the next (encode.c:1445 last_bytes_ / last_bytes_bits_): the bits of
// its last, incomplete byte, and whether the window bits went out.
struct Q1Tail { uint32_t bits = 0; uint8_t byte = 0; bool header_done = false; };
// The product's segment: at most this much input (bit offsets inside a segment are 32-bit); a stream is any number of them.
static const size_t kQ1SegmentBytes = (size_t)1 << 27;

inline int q1_segment(const Backend& b, const Params& p, const uint8_t* in, size_t n, const std::vector<size_t>& calls, int end_op,
                      Q1Tail& t, ByteVec& out) {
  const int with_header = !t.header_done;
  if (n == 0) {
    /* nothing to parse: window bits (encode.c:1006), ISLAST + ISEMPTY (compress_fragment_two_pass.c:641) or the
       padding block of a FLUSH (encode.c:1356) behind the pending bits */
    std::vector<uint8_t> v;
    BitOut w{v, t.bits};
    if (t.bits) v.push_back((uint8_t)(t.byte & ((1u << t.bits) - 1u)));
    if (with_header) put_window_bits(w, window_of(p) < 18 ? 18 : window_of(p));   /* encode.c:673 */
    if (end_op == 2) { w.put(2, 3); w.align(); }
    else if (end_op == 1 && w.pb) { w.put(6, 6); w.align(); }
    t.bits = w.pb; t.byte = w.pb ? v.back() : 0;   // a partial last byte stays pending
    out.insert(out.end(), v.begin(), v.end() - (w.pb ? 1 : 0));
  } else {
    std::vector<uint8_t> seg; uint32_t end_bit = 0;
    if (!b.q1_segment(window_of(p), in, n, calls, with_header, end_op, t.bits, &end_bit, seg) || seg.empty()) return 0;
    if (t.bits) seg[0] |= (uint8_t)(t.byte & ((1u << t.bits) - 1u));
    t.bits = 0; t.byte = 0;
    if (end_op == 0 && (end_bit & 7)) { t.bits = end_bit & 7; t.byte = seg.back(); seg.pop_back(); }
    out.insert(out.end(), seg.begin(), seg.end());
  }
  t.header_done = true;
  return 1;
}

// [in, in+n) as delivered by `calls` (nullptr: one call), through the backend in segments of at most seg_bytes.  A call
// that straddles a segment is split at a multiple of the fragment size (1 << lgwin), which leaves the reference's fragments
// (encode.c:1425) as they were.  Complete bytes are appended to `out`; end_op as in br_q1_host.h.
inline int q1_run(const Backend& b, const Params& p, size_t seg_bytes, const uint8_t* in, size_t n, const size_t* calls,
                  size_t ncalls, int end_op, Q1Tail& t, ByteVec& out) {
  const size_t limit = (size_t)1 << window_of(p);
  if (seg_bytes < limit) return 0;   // a segment must hold a whole fragment, or a long call never makes progress
  if (!calls) { calls = &n; ncalls = 1; }
  size_t ci = 0, rem = ncalls ? calls[0] : 0, pos = 0;
  for (;;) {
    std::vector<size_t> sc; size_t seg_n = 0;
    while (ci < ncalls) {
      const size_t room = seg_bytes - seg_n;
      if (rem <= room) { sc.push_back(rem); seg_n += rem; ++ci; rem = ci < ncalls ? calls[ci] : 0; continue; }
      const size_t part = room / limit * limit;
      if (part) { sc.push_back(part); seg_n += part; rem -= part; }
      break;
    }
    const bool last = ci >= ncalls;
    if (!q1_segment(b, p, in + pos, seg_n, sc, last ? end_op : 0, t, out)) return 0;
    pos += seg_n;
    if (last) return pos == n;
  }
}

// encode.c:1296 BrotliEncoderCompress; quality 2..9 compresses straight into the caller's buffer.
inline BROTLI_BOOL compress_oneshot(const Backend& b, int quality, int lgwin, int mode, size_t input_size, const uint8_t* input_buffer,
                                    size_t* encoded_size, uint8_t* encoded_buffer) {
  const size_t out_size = *encoded_size;
  if (out_size == 0) return BROTLI_FALSE;
  if (input_size == 0) { *encoded_size = 1; *encoded_buffer = 6; return BROTLI_TRUE; }
  Params p = oneshot_params(quality, lgwin, mode);
  p.size_hint = (uint32_t)input_size;
  if (!supported(p)) { *encoded_size = 0; return BROTLI_FALSE; }
  size_t got = 0;
  ByteVec q1_out; Q1Tail tail;
  const int ok = quality == 1 ? q1_run(b, p, kQ1SegmentBytes, input_buffer, input_size, nullptr, 0, 2, tail, q1_out)
                              : b.compress(p, (uint32_t)input_size, input_buffer, input_size, nullptr, encoded_buffer, out_size, &got, nullptr);
  if (quality == 1) got = q1_out.size();
  *encoded_size = 0;
  if (!ok) return BROTLI_FALSE;   /* the pipeline failed: fail loudly, never substitute other bytes */
  switch (fit_stream(got, out_size, input_size)) {
    case kKeep: if (quality == 1) memcpy(encoded_buffer, q1_out.data(), got); *encoded_size = got; return BROTLI_TRUE;
    case kRaw: *encoded_size = make_uncompressed_stream(input_buffer, input_size, encoded_buffer); return BROTLI_TRUE;
    default: return BROTLI_FALSE;
  }
}

// A FLUSH (kind 1) or EMIT_METADATA (kind 2) operation at input position pos (quality 2..9).
struct StreamEvent { uint32_t pos; int kind; std::vector<uint8_t> meta; };

struct Stream {
  Params params;
  bool initialized = false, compressed = false, hint_fixed = false;
  Q1Tail q1_tail;                // quality 1: pending bits between segments, window bits sent
  size_t q1_segment_bytes = kQ1SegmentBytes;   // quality 1: input of one segment; PROCESS runs one at half of it
  bool flint_done = false;       // STREAM_OFFSET: the cut behind the first two bytes has been recorded
  bool meta_open = false;        // quality 2..9: the last operation was EMIT_METADATA
  ByteVec input, output;
  std::vector<size_t> calls;     // quality 1: bytes brought by each CompressStream call (encode.c:1425 cuts fragments per call)
  std::vector<StreamEvent> events;   // quality 2..9: the FLUSH / EMIT_METADATA operations so far
  size_t wire_sent = 0;          // quality 2..9: bytes of the stream already handed to `output`
  size_t out_pos = 0;
  uint64_t total_out = 0;
  explicit Stream(const BrAlloc<uint8_t>& a) : input(a), output(a) {}
};

// The whole stream for the operations seen so far (quality 2..9): the backend compresses the accumulated input cut at the
// positions of the FLUSH / EMIT_METADATA operations (br_kernels.cu k_assemble_scan pads behind a FLUSH); metadata blocks and
// everything that happens before the first input byte are spliced in here.  Every call reproduces the bytes of the call
// before as a prefix: the parse is causal, and each cut ends on a byte boundary.
inline int build_wire(const Backend& b, const Stream& s, bool is_final, bool finish_empty, std::vector<uint8_t>& W) {
  const size_t n = s.input.size();
  W.clear();
  BitOut w{W, 0};
  size_t e = 0;
  const std::vector<StreamEvent>& ev = s.events;
  const bool lead = !ev.empty() && ev[0].pos == 0;
  const bool continued = s.params.stream_offset != 0;   /* encode.c:675: a stream that continues another one has no window bits */
  if (lead || n == 0) {
    if (!continued) put_window_bits(w, window_of(s.params));
    for (; e < ev.size() && ev[e].pos == 0; ++e) {
      if (ev[e].kind == 1) { if (w.pb) { w.put(6, 6); w.align(); } }   // encode.c:1356 InjectBytePaddingBlock
      else put_metadata(w, ev[e].meta);
    }
  }
  if (n == 0) {
    if (is_final) { w.put(2, 3); w.align(); }   // encode.c:1006: ISLAST + ISEMPTY
    return 1;
  }
  std::vector<uint32_t> cut_pos, cut_kind;
  for (size_t i = e; i < ev.size(); ++i)
    if (cut_pos.empty() || cut_pos.back() != ev[i].pos) { cut_pos.push_back(ev[i].pos); cut_kind.push_back((uint32_t)ev[i].kind); }
  const bool cut_at_end = !cut_pos.empty() && cut_pos.back() == n;
  std::vector<uint64_t> end_bit(cut_pos.size() + 1, 0);
  BrCuts c; c.pos = cut_pos.data(); c.kind = cut_kind.data(); c.n = (uint32_t)cut_pos.size();
  c.is_final = (is_final && !cut_at_end) ? 1 : 0; c.with_header = (lead || continued) ? 0 : 1;
  c.stream_offset = s.params.stream_offset;
  c.finish_empty = (c.is_final && finish_empty) ? 1 : 0; c.end_bit = end_bit.data();
  c.lgblock = s.params.lgblock; c.disable_ctx = (int)s.params.disable_ctx; c.stream_end = nullptr;
  if (!c.is_final && !cut_at_end) return 0;   // (callers only build the wire at a cut or at FINISH)
  std::vector<uint8_t> D;
  size_t got = 0;
  if (!b.compress(s.params, s.params.size_hint, s.input.data(), n, &c, nullptr, 0, &got, &D)) return 0;
  size_t from = 0;
  for (size_t i = 0; i < cut_pos.size(); ++i) {
    const uint64_t eb = end_bit[i];
    size_t upto, next;
    if (cut_kind[i] == 1) { next = (size_t)(((eb & 7) ? eb + 6 : eb) + 7) >> 3; upto = next; }   // the backend wrote the padding block
    else { upto = (size_t)((eb + 7) >> 3); next = upto; }
    W.insert(W.end(), D.begin() + (long)from, D.begin() + (long)upto);
    w.pb = cut_kind[i] == 2 ? (uint32_t)(eb & 7) : 0;
    for (; e < ev.size() && ev[e].pos == cut_pos[i]; ++e)
      if (ev[e].kind == 2) put_metadata(w, ev[e].meta);   // (a FLUSH on a byte boundary emits nothing)
    w.align();
    from = next;
  }
  W.insert(W.end(), D.begin() + (long)from, D.end());
  if (is_final && cut_at_end) W.push_back(3);   // encode.c:520: empty last metablock on a byte boundary
  return 1;
}

inline bool is_finished(const Stream& s) { return s.compressed && s.out_pos == s.output.size(); }
inline bool has_more_output(const Stream& s) { return s.out_pos < s.output.size(); }
inline void push_output(Stream& s, size_t* available_out, uint8_t** next_out, size_t* total_out) {
  size_t avail = s.output.size() - s.out_pos;
  if (avail && *available_out && next_out && *next_out) {
    size_t c = avail < *available_out ? avail : *available_out;
    memcpy(*next_out, s.output.data() + s.out_pos, c);
    *next_out += c; *available_out -= c; s.out_pos += c; s.total_out += c;
  }
  if (total_out) *total_out = (size_t)s.total_out;
}

/* encode.c:1634.  Quality 2..9: the input is accumulated on the host; every FLUSH / EMIT_METADATA / FINISH sends the
   whole stream so far through the backend, cut where those operations happened (build_wire), and hands out the bytes
   that are new.  The bytes equal the reference's for the same call sequence (SURVEY.md section 0, T6: the size hint is frozen
   when the reference would have frozen it, at its first EncodeData call).  Cost: a stream with k flushes is compressed k
   times, and host memory grows with the stream (at most 1 GiB, then PROCESS fails) -- the reference's bounded-memory
   streaming needs the pipeline to resume from a saved window, which it does not do yet.
   Quality 1 (encode.c:1425): every call compresses its own fragments; FLUSH is cheap.
   Throws std::bad_alloc when the caller's allocator fails. */
inline BROTLI_BOOL compress_stream(const Backend& b, Stream& s, BrotliEncoderOperation op, size_t* available_in,
                                   const uint8_t** next_in, size_t* available_out, uint8_t** next_out, size_t* total_out) {
  s.initialized = true;
  const bool q1 = s.params.quality == 1;
  if (!supported(s.params)) return BROTLI_FALSE;
  if (op == BROTLI_OPERATION_EMIT_METADATA && q1) return BROTLI_FALSE;   /* not built for the fragment coder */
  if (s.compressed && (*available_in != 0 || op == BROTLI_OPERATION_EMIT_METADATA)) return BROTLI_FALSE;   /* input after finish */
  if (s.compressed || (op == BROTLI_OPERATION_EMIT_METADATA && *available_in == 0 && s.meta_open && has_more_output(s))) {
    /* encode.c:1549 ProcessMetadata: a metadata block stays open until its bytes have been handed out, so the calls that
       drain it (encode.h:473) add no block of their own */
    push_output(s, available_out, next_out, total_out);
    return BROTLI_TRUE;
  }
  s.meta_open = op == BROTLI_OPERATION_EMIT_METADATA;
  if (op == BROTLI_OPERATION_EMIT_METADATA) {
    if (*available_in > (1u << 24)) return BROTLI_FALSE;   /* encode.c:1552 */
  } else {
    if (!q1 && s.input.size() + *available_in > ((size_t)1 << 30)) return BROTLI_FALSE;   /* positions are 32-bit in the pipeline */
    if (q1 && (*available_in || op == BROTLI_OPERATION_FINISH)) s.calls.push_back(*available_in);
    s.input.insert(s.input.end(), *next_in, *next_in + *available_in);
  }
  const bool finish_without_input = op == BROTLI_OPERATION_FINISH && *available_in == 0;
  if (!q1 && !s.hint_fixed) {
    /* encode.c:1619 UpdateSizeHint runs at the first EncodeData: when the first input block (1 << lgblock) is full
       or the operation is not PROCESS. */
    if (op != BROTLI_OPERATION_PROCESS || s.input.size() >= ((size_t)1 << lgblock_of(s.params)) ||
        (s.params.stream_offset && s.input.size() >= 2)) {
      /* (an estimate of zero -- an operation before any input -- is taken again at the next EncodeData) */
      if (s.params.size_hint == 0) s.params.size_hint = (uint32_t)s.input.size();
      s.hint_fixed = s.params.size_hint != 0;
    }
  }
  if (s.params.stream_offset && !s.flint_done && s.input.size() >= 2 &&
      !(s.input.size() == 2 && op == BROTLI_OPERATION_FINISH)) {
    /* encode.c:1704: with a stream offset the first two bytes are flushed on their own (unless the stream ends there) */
    s.events.push_back(StreamEvent{2, 1, {}});
    s.flint_done = true;
  }
  if (op == BROTLI_OPERATION_EMIT_METADATA)
    s.events.push_back(StreamEvent{(uint32_t)s.input.size(), 2, std::vector<uint8_t>(*next_in, *next_in + *available_in)});
  else if (op == BROTLI_OPERATION_FLUSH && !q1)
    s.events.push_back(StreamEvent{(uint32_t)s.input.size(), 1, {}});
  *next_in += *available_in;
  *available_in = 0;
  if (op != BROTLI_OPERATION_PROCESS || (q1 && s.input.size() >= s.q1_segment_bytes / 2)) {
    s.output.erase(s.output.begin(), s.output.begin() + (long)s.out_pos); s.out_pos = 0;
    if (q1) {   /* encode.c:1425: the calls decide the fragments; running a segment whenever half of one waits keeps
                   memory bounded, and only the pending bits of the last byte carry over (Q1Tail) */
      const int end_op = op == BROTLI_OPERATION_FINISH ? 2 : op == BROTLI_OPERATION_FLUSH ? 1 : 0;
      if (!q1_run(b, s.params, s.q1_segment_bytes, s.input.data(), s.input.size(), s.calls.data(), s.calls.size(), end_op,
                  s.q1_tail, s.output))
        return BROTLI_FALSE;
      s.input.clear(); s.calls.clear();
    } else {
      const size_t last_cut = s.events.empty() ? 0 : s.events.back().pos;
      const size_t bs = (size_t)1 << lgblock_of(s.params);
      /* FINISH without input right behind a full input block: that block was already encoded as a non-last one */
      const bool finish_empty = finish_without_input && s.input.size() > last_cut && (s.input.size() - last_cut) % bs == 0;
      std::vector<uint8_t> W;
      if (!build_wire(b, s, op == BROTLI_OPERATION_FINISH, finish_empty, W) || W.size() < s.wire_sent) return BROTLI_FALSE;
      s.output.insert(s.output.end(), W.begin() + (long)s.wire_sent, W.end());
      s.wire_sent = W.size();
    }
    if (op == BROTLI_OPERATION_FINISH) { s.compressed = true; ByteVec(s.input.get_allocator()).swap(s.input); }
  }
  push_output(s, available_out, next_out, total_out);
  return BROTLI_TRUE;
}

inline const uint8_t* take_output(Stream& s, size_t* size) {   /* encode.c:1742 */
  const size_t avail = s.output.size() - s.out_pos;
  if (*size == 0 || *size > avail) *size = avail;
  if (*size == 0) return nullptr;
  const uint8_t* result = s.output.data() + s.out_pos;
  s.out_pos += *size; s.total_out += *size;
  return result;
}

}  // namespace br_driver
