// br_api.cc -- the BrotliEncoder* C ABI (include/brotli_b200.h) on top of the GPU pipeline: the per-thread device jobs,
// the backend the host driver (br_driver.h) compresses through, and the entry points.  No compression happens on the host.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <new>
#include <thread>
#include <vector>
#include "../../include/brotli_b200.h"
#include "br_driver.h"
#include "br_q1_host.h"

using namespace br_driver;

namespace {

struct TlsJob {
  BrJob* job = nullptr;
  BrQ1Job* q1 = nullptr;
  uint8_t* d_in = nullptr; size_t d_in_cap = 0;
  uint8_t* h_stage = nullptr; size_t h_stage_cap = 0;   // pinned staging area of the stream batches
  double last[16] = {0};
  double last_q1[12] = {0};
  ~TlsJob() { if (d_in) cudaFree(d_in); if (h_stage) cudaFreeHost(h_stage); if (job) br_job_destroy(job); if (q1) br_q1_job_destroy(q1); }
};
thread_local TlsJob tls;

bool have_device() {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    static bool warned = false;
    if (!warned) { warned = true; fprintf(stderr, "brotli_b200: no CUDA device; this library has no CPU path\n"); }
    return false;
  }
  return true;
}
bool ensure_q1() {
  if (tls.q1) return true;
  if (!have_device()) return false;
  tls.q1 = br_q1_job_create();
  return tls.q1 != nullptr;
}
bool ensure_job() {
  if (tls.job) return true;
  if (!have_device()) return false;
  tls.job = br_job_create();
  return tls.job != nullptr;
}
// Grow-only buffers of this thread: room for n bytes of device input, or of pinned staging.
bool reserve_d_in(size_t n) {
  if (tls.d_in_cap >= n) return true;
  if (tls.d_in) cudaFree(tls.d_in);
  tls.d_in = nullptr; tls.d_in_cap = 0;
  if (cudaMalloc(&tls.d_in, n + 64) != cudaSuccess) { cudaGetLastError(); return false; }
  tls.d_in_cap = n;
  return true;
}
bool reserve_h_stage(size_t n) {
  if (tls.h_stage_cap >= n) return true;
  if (tls.h_stage) cudaFreeHost(tls.h_stage);
  tls.h_stage = nullptr; tls.h_stage_cap = 0;
  if (cudaMallocHost(&tls.h_stage, n + 64) != cudaSuccess) { cudaGetLastError(); return false; }
  tls.h_stage_cap = n;
  return true;
}
void record_q1_stats() {
  const BrQ1Stats* s = br_q1_job_stats(tls.q1);
  double* o = tls.last_q1;
  o[0] = s->ms_total; o[1] = s->ms_h2d; o[2] = s->ms_parse; o[3] = s->ms_code; o[4] = s->ms_pack; o[5] = s->ms_d2h;
  o[6] = (double)s->streams; o[7] = (double)s->fragments; o[8] = (double)s->blocks; o[9] = (double)s->in_bytes;
  o[10] = (double)s->out_bytes; o[11] = (double)s->launches;
}
void record_stats() {
  const BrJobStats* s = br_job_stats(tls.job);
  tls.last[0] = s->ms_total; tls.last[1] = s->ms_index; tls.last[2] = s->ms_lz77; tls.last[3] = s->ms_entropy;
  tls.last[4] = s->ms_assemble; tls.last[5] = s->lz77_iterations; tls.last[6] = (double)s->block_runs;
  tls.last[7] = s->nblocks; tls.last[8] = s->n_metablocks; tls.last[9] = s->launches;
  tls.last[10] = s->ms_walk; tls.last[11] = s->ms_encode; tls.last[12] = s->walk_launches;
  tls.last[13] = s->encode_launches; tls.last[14] = (double)s->walk_bytes; tls.last[15] = (double)s->total_cmds;
}

// The driver's backend on the device (Backend::compress): host buffer -> device -> pipeline -> host vector / buffer.
int compress_host(const Params& p, uint32_t size_hint, const uint8_t* in, size_t n, const BrCuts* cuts, uint8_t* out, size_t out_cap,
                  size_t* out_n, std::vector<uint8_t>* out_vec) {
  if (!supported(p) || n == 0 || n > (1u << 30)) return 0;
  if (!ensure_job() || !reserve_d_in(n)) return 0;
  cudaStream_t st = (cudaStream_t)br_job_stream(tls.job);
  if (cudaMemcpyAsync(tls.d_in, in, n, cudaMemcpyHostToDevice, st) != cudaSuccess) return 0;
  const uint8_t* d_out = nullptr; size_t sz = 0;
  if (!br_job_compress_device(tls.job, p.quality, window_of(p), size_hint, tls.d_in, (uint32_t)n, &d_out, &sz, cuts)) return 0;
  record_stats();
  if (out_vec) { out_vec->resize(sz); out = out_vec->data(); out_cap = sz; }
  if (sz > out_cap) { *out_n = sz; return 2; }   /* compressed, but the caller's buffer is too small (encode.c:1336: "not finished") */
  if (cudaMemcpyAsync(out, d_out, sz, cudaMemcpyDeviceToHost, st) != cudaSuccess) return 0;
  if (cudaStreamSynchronize(st) != cudaSuccess) return 0;
  *out_n = sz;
  return 1;
}

// Quality 1 (two-pass fragment coder, br_q1.cu): one segment of one stream = a batch of one.
int device_q1_segment(int lgwin, const uint8_t* in, size_t n, const std::vector<size_t>& calls, int with_header, int end_op,
                      uint32_t start_bits, uint32_t* end_bit, std::vector<uint8_t>& out) {
  if (!ensure_q1() || n > (1u << 28)) return 0;
  const size_t cap = n + 16 + 12 * (n / ((size_t)1 << lgwin) + calls.size() + 2);
  out.resize(cap);
  const uint8_t* ins[1] = {in}; size_t in_n[1] = {n};
  const size_t* cl[1] = {calls.data()}; size_t ncl[1] = {calls.size()};
  uint8_t* outs[1] = {out.data()}; size_t out_n[1] = {cap}; int ok[1] = {0};
  if (!br_q1_compress_batch(tls.q1, lgwin, 1, ins, in_n, cl, ncl, nullptr, outs, out_n, ok, 1, with_header, end_op, &start_bits, end_bit))
    return 0;
  record_q1_stats();
  out.resize(out_n[0]);
  return 1;
}
const Backend kDevice = {compress_host, device_q1_segment};

template <class F> void batch_threads(int threads, size_t count, F f) {
  if (threads <= 1 || count < 64) { f(0, count); return; }
  std::vector<std::thread> th;
  for (int t = 0; t < threads; ++t) {
    const size_t a = count * (size_t)t / (size_t)threads, b = count * (size_t)(t + 1) / (size_t)threads;
    if (a < b) th.emplace_back([=, &f] { f(a, b); });
  }
  for (auto& t : th) t.join();
}
// One group of br_driver::plan_groups as one device job, through the pinned staging area: one upload, one download, and
// BrotliEncoderCompress's raw-stream rule per stream.  idx: the streams of the group; encoded_sizes: capacity in, size
// out (0 = failed).  Returns the number of streams compressed.
size_t compress_stream_group(const Params& p, const std::vector<size_t>& idx, const uint8_t* const* inputs,
                             const size_t* input_sizes, uint8_t* const* outputs, size_t* encoded_sizes, int threads) {
  const size_t k = idx.size();
  auto fail_all = [&]() { for (size_t i : idx) encoded_sizes[i] = 0; return (size_t)0; };
  if (!ensure_job()) return fail_all();
  GroupCuts g(input_sizes, idx.data(), k);
  const size_t n = g.n;
  const size_t out_bound = n + (n >> 3) + 4096 + 64 * k;
  if (!reserve_h_stage(n > out_bound ? n : out_bound) || !reserve_d_in(n)) return fail_all();
  uint8_t* hs = tls.h_stage;
  batch_threads(threads, k, [&](size_t a, size_t b) {
    for (size_t j = a; j < b; ++j) memcpy(hs + (j ? g.pos[j - 1] : 0), inputs[idx[j]], input_sizes[idx[j]]);
  });
  cudaStream_t st = (cudaStream_t)br_job_stream(tls.job);
  if (cudaMemcpyAsync(tls.d_in, hs, n, cudaMemcpyHostToDevice, st) != cudaSuccess) return fail_all();
  const uint8_t* d_out = nullptr; size_t sz = 0;
  if (!br_job_compress_device(tls.job, p.quality, window_of(p), g.hint, tls.d_in, (uint32_t)n, &d_out, &sz, k > 1 ? &g.c : nullptr))
    return fail_all();
  record_stats();
  if (k == 1) g.ends[0] = sz;
  if (sz > tls.h_stage_cap || g.ends[k - 1] != sz) return fail_all();
  if (cudaMemcpyAsync(hs, d_out, sz, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) return fail_all();
  std::vector<uint8_t> good(k, 0);
  batch_threads(threads, k, [&](size_t a, size_t b) {
    for (size_t j = a; j < b; ++j) {
      const size_t i = idx[j], from = j ? (size_t)g.ends[j - 1] : 0, got = (size_t)g.ends[j] - from;
      switch (fit_stream(got, encoded_sizes[i], input_sizes[i])) {
        case kKeep: memcpy(outputs[i], hs + from, got); encoded_sizes[i] = got; good[j] = 1; break;
        case kRaw: encoded_sizes[i] = make_uncompressed_stream(inputs[i], input_sizes[i], outputs[i]); good[j] = 1; break;
        default: encoded_sizes[i] = 0;
      }
    }
  });
  size_t ok = 0;
  for (size_t j = 0; j < k; ++j) ok += good[j];
  return ok;
}

}  // namespace

struct BrotliEncoderStateStruct {
  brotli_alloc_func alloc_func; brotli_free_func free_func; void* opaque;
  Stream s;
  BrotliEncoderStateStruct(brotli_alloc_func a, brotli_free_func f, void* o)
      : alloc_func(a), free_func(f), opaque(o), s(BrAlloc<uint8_t>(a, f, o)) {}
};

extern "C" {

uint32_t BrotliEncoderVersion(void) { return 0x1002000; }  /* c/common/version.h:18: 1.2.0 */

int BrotliB200Available(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n > 0;
}

void BrotliB200LastStats(double out[16]) { memcpy(out, tls.last, sizeof(tls.last)); }
void BrotliB200LastStatsQ1(double out[12]) { memcpy(out, tls.last_q1, sizeof(tls.last_q1)); }

size_t BrotliEncoderMaxCompressedSize(size_t input_size) { return max_compressed_size(input_size); }

BROTLI_BOOL BrotliEncoderCompress(int quality, int lgwin, BrotliEncoderMode mode, size_t input_size,
    const uint8_t* input_buffer, size_t* encoded_size, uint8_t* encoded_buffer) {
  return compress_oneshot(kDevice, quality, lgwin, mode, input_size, input_buffer, encoded_size, encoded_buffer);
}

BROTLI_BOOL BrotliB200CompressDevice(int quality, int lgwin, size_t input_size, const void* d_input,
                                     size_t* encoded_size, void* d_encoded) {
  const Params p = oneshot_params(quality, lgwin);
  if (!supported(p) || input_size == 0 || input_size > (1u << 30) || !ensure_job()) return BROTLI_FALSE;
  const uint8_t* d_out = nullptr; size_t sz = 0;
  if (!br_job_compress_device(tls.job, quality, window_of(p), (uint32_t)input_size, (const uint8_t*)d_input,
                              (uint32_t)input_size, &d_out, &sz, nullptr)) return BROTLI_FALSE;
  record_stats();
  if (sz > *encoded_size) return BROTLI_FALSE;
  cudaStream_t st = (cudaStream_t)br_job_stream(tls.job);
  if (cudaMemcpyAsync(d_encoded, d_out, sz, cudaMemcpyDeviceToDevice, st) != cudaSuccess) return BROTLI_FALSE;
  if (cudaStreamSynchronize(st) != cudaSuccess) return BROTLI_FALSE;
  *encoded_size = sz;
  return BROTLI_TRUE;
}

size_t BrotliB200CompressBatch(int quality, int lgwin, size_t count, const uint8_t* const* inputs,
    const size_t* input_sizes, uint8_t* const* outputs, size_t* encoded_sizes, int threads) {
  if (threads < 1) threads = 1;
  const Params p = oneshot_params(quality, lgwin);
  if (!supported(p) || (quality == 1 && count && !ensure_q1())) { for (size_t i = 0; i < count; ++i) encoded_sizes[i] = 0; return 0; }
  if (quality == 1 && count) {
    /* one device batch: all streams through the same four launches (br_q1.cu) */
    std::vector<int> ok(count, 0);
    std::vector<size_t> caps(encoded_sizes, encoded_sizes + count);
    br_q1_compress_batch(tls.q1, window_of(p), count, inputs, input_sizes, nullptr, nullptr, nullptr, outputs, encoded_sizes, ok.data(), threads, 1, 2, nullptr, nullptr);
    record_q1_stats();
    size_t good = 0;
    for (size_t i = 0; i < count; ++i) {
      /* what the one-shot wrapper adds per stream: encode.c:1310 (empty input) and :1345 (raw-stream rule) */
      if (input_sizes[i] == 0) {
        if (caps[i] >= 1) { outputs[i][0] = 6; encoded_sizes[i] = 1; ++good; } else encoded_sizes[i] = 0;
        continue;
      }
      switch (ok[i] ? fit_stream(encoded_sizes[i], caps[i], input_sizes[i]) : kFail) {
        case kKeep: ++good; break;
        case kRaw: encoded_sizes[i] = make_uncompressed_stream(inputs[i], input_sizes[i], outputs[i]); ++good; break;
        default: encoded_sizes[i] = 0;
      }
    }
    return good;
  }
  /* quality 2..9: streams below 1 MiB go through the device in groups (compress_stream_group); the others one by one,
     `threads` host workers each with its own CUDA stream */
  std::vector<std::vector<size_t>> groups;
  std::vector<size_t> big;
  plan_groups(input_sizes, count, groups, big);
  size_t ok = 0;
  for (const std::vector<size_t>& g : groups) ok += compress_stream_group(p, g, inputs, input_sizes, outputs, encoded_sizes, threads);
  if (big.empty()) return ok;
  if ((size_t)threads > big.size()) threads = (int)big.size();
  std::vector<size_t> okc((size_t)threads, 0);
  int dev = 0; cudaGetDevice(&dev);
  std::vector<std::thread> th;
  for (int t = 0; t < threads; ++t)
    th.emplace_back([&, t] {
      cudaSetDevice(dev);
      for (size_t bi = (size_t)t; bi < big.size(); bi += (size_t)threads) {
        const size_t i = big[bi];
        size_t sz = encoded_sizes[i];
        if (BrotliEncoderCompress(quality, lgwin, BROTLI_MODE_GENERIC, input_sizes[i], inputs[i], &sz, outputs[i])) {
          encoded_sizes[i] = sz; ++okc[(size_t)t];
        } else encoded_sizes[i] = 0;
      }
    });
  for (int t = 0; t < threads; ++t) { th[(size_t)t].join(); ok += okc[(size_t)t]; }
  return ok;
}

size_t BrotliB200CompressBatchDevice(int quality, int lgwin, size_t count, const void* d_inputs, const uint64_t* input_offsets,
    const size_t* input_sizes, void* d_encoded, size_t encoded_capacity, uint64_t* encoded_offsets, size_t* encoded_sizes) {
  const Params p = oneshot_params(quality, lgwin);
  if (!count || !supported(p)) return 0;
  for (size_t i = 0; i < count; ++i) if (input_sizes[i] == 0) return 0;
  /* encode.c:1345: above BrotliEncoderMaxCompressedSize the one-shot wrapper substitutes the raw stream, which needs the
     host copy of the input: such a stream is reported as failed here (size 0) */
  if (quality != 1) {
    /* quality 2..9: streams below 1 MiB (longer ones: BrotliB200CompressDevice) in the groups of compress_stream_group,
       without the host staging: a group whose streams lie back to back in d_inputs is read in place, otherwise it is
       gathered with device copies; the job's output is dense and goes to d_encoded as it is. */
    std::vector<std::vector<size_t>> groups;
    std::vector<size_t> single;
    plan_groups(input_sizes, count, groups, single);
    if (!single.empty() || !ensure_job()) return 0;
    cudaStream_t st = (cudaStream_t)br_job_stream(tls.job);
    const uint8_t* din = (const uint8_t*)d_inputs;
    uint8_t* dout = (uint8_t*)d_encoded;
    size_t used = 0, good = 0, a = 0;   // a: the first stream of the group (groups are consecutive, in order)
    for (size_t i = 0; i < count; ++i) encoded_sizes[i] = 0;
    bool failed = false;
    for (const std::vector<size_t>& idx : groups) {
      const size_t k = idx.size();
      GroupCuts g(input_sizes + a, nullptr, k);
      bool packed = true;
      for (size_t j = a + 1; j < a + k; ++j) if (input_offsets[j] != input_offsets[j - 1] + input_sizes[j - 1]) packed = false;
      const uint8_t* src = din + input_offsets[a];
      if (!packed) {
        if (!reserve_d_in(g.n)) { failed = true; break; }
        for (size_t j = 0; j < k && !failed; ++j)
          if (cudaMemcpyAsync(tls.d_in + (j ? g.pos[j - 1] : 0), din + input_offsets[a + j], input_sizes[a + j], cudaMemcpyDeviceToDevice, st) != cudaSuccess)
            failed = true;
        if (failed) break;
        src = tls.d_in;
      }
      const uint8_t* d_o = nullptr; size_t sz = 0;
      if (!br_job_compress_device(tls.job, quality, window_of(p), g.hint, src, (uint32_t)g.n, &d_o, &sz, k > 1 ? &g.c : nullptr)) { failed = true; break; }
      record_stats();
      if (k == 1) g.ends[0] = sz;
      if (g.ends[k - 1] != sz || used + sz > encoded_capacity) { failed = true; break; }
      if (cudaMemcpyAsync(dout + used, d_o, sz, cudaMemcpyDeviceToDevice, st) != cudaSuccess) { failed = true; break; }
      for (size_t j = 0; j < k; ++j) {
        const size_t from = j ? (size_t)g.ends[j - 1] : 0, got = (size_t)g.ends[j] - from;
        encoded_offsets[a + j] = used + from;
        if (within_bound(got, input_sizes[a + j])) { encoded_sizes[a + j] = got; ++good; }
      }
      used += sz;
      a += k;
    }
    for (size_t i = a; i < count; ++i) encoded_offsets[i] = used;   /* (streams behind a failure) */
    encoded_offsets[count] = used;
    if (cudaStreamSynchronize(st) != cudaSuccess) return 0;
    return failed ? 0 : good;
  }
  if (!ensure_q1()) return 0;
  BrQ1Packed pk; pk.d_in = (const uint8_t*)d_inputs; pk.in_off = input_offsets; pk.d_out = (uint8_t*)d_encoded;
  pk.out_cap = encoded_capacity; pk.out_off = encoded_offsets;
  std::vector<int> ok(count, 0);
  if (!br_q1_compress_batch(tls.q1, window_of(p), count, nullptr, input_sizes, nullptr, nullptr, &pk, nullptr, encoded_sizes, ok.data(), 1, 1, 2, nullptr, nullptr)) return 0;
  record_q1_stats();
  size_t good = 0;
  for (size_t i = 0; i < count; ++i) {
    if (within_bound(encoded_sizes[i], input_sizes[i])) ++good; else encoded_sizes[i] = 0;
  }
  return good;
}

BrotliEncoderState* BrotliEncoderCreateInstance(brotli_alloc_func alloc_func, brotli_free_func free_func, void* opaque) {
  if ((alloc_func == nullptr) != (free_func == nullptr)) return nullptr;   /* encode.h:295 */
  void* mem = alloc_func ? alloc_func(opaque, sizeof(BrotliEncoderState)) : malloc(sizeof(BrotliEncoderState));
  if (!mem) return nullptr;
  return new (mem) BrotliEncoderState(alloc_func, free_func, opaque);
}
void BrotliEncoderDestroyInstance(BrotliEncoderState* state) {
  if (!state) return;
  brotli_free_func ff = state->free_func; void* opaque = state->opaque;
  state->~BrotliEncoderStateStruct();
  if (ff) ff(opaque, state); else free(state);
}

BROTLI_BOOL BrotliEncoderSetParameter(BrotliEncoderState* s, BrotliEncoderParameter p, uint32_t value) {
  if (s->s.initialized) return BROTLI_FALSE;   /* encode.c:63 */
  return set_parameter(s->s.params, p, value);
}

BrotliEncoderPreparedDictionary* BrotliEncoderPrepareDictionary(BrotliSharedDictionaryType, size_t, const uint8_t*, int,
    brotli_alloc_func, brotli_free_func, void*) { return nullptr; }
void BrotliEncoderDestroyPreparedDictionary(BrotliEncoderPreparedDictionary*) {}
BROTLI_BOOL BrotliEncoderAttachPreparedDictionary(BrotliEncoderState*, const BrotliEncoderPreparedDictionary*) {
  return BROTLI_FALSE;
}

BROTLI_BOOL BrotliEncoderCompressStream(BrotliEncoderState* s, BrotliEncoderOperation op, size_t* available_in,
    const uint8_t** next_in, size_t* available_out, uint8_t** next_out, size_t* total_out) {
  try { return compress_stream(kDevice, s->s, op, available_in, next_in, available_out, next_out, total_out); }
  catch (const std::bad_alloc&) { return BROTLI_FALSE; }   /* the reference reports allocation failure the same way */
}

BROTLI_BOOL BrotliEncoderIsFinished(BrotliEncoderState* s) { return is_finished(s->s) ? BROTLI_TRUE : BROTLI_FALSE; }
BROTLI_BOOL BrotliEncoderHasMoreOutput(BrotliEncoderState* s) { return has_more_output(s->s) ? BROTLI_TRUE : BROTLI_FALSE; }
const uint8_t* BrotliEncoderTakeOutput(BrotliEncoderState* s, size_t* size) { return take_output(s->s, size); }

}  // extern "C"
