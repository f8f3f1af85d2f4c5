// br_pipeline.h -- host-visible interface of the per-stream GPU pipeline (br_kernels.cu).
#pragma once
#include <stddef.h>
#include <stdint.h>
struct BrJob;
struct BrJobStats {
  float ms_total, ms_index, ms_lz77, ms_entropy, ms_assemble;
  float ms_walk, ms_encode;          // summed durations of the k_walk / k_encode_mb launches
  uint32_t walk_launches, encode_launches;
  uint64_t walk_bytes, total_cmds;   // input bytes walked (all launches), commands emitted
  uint32_t lz77_iterations, nblocks, n_metablocks, rounds, launches;
  uint64_t block_runs, in_bytes, out_bytes;
};
// A stream cut by FLUSH / EMIT_METADATA operations (c/enc/encode.c:1634): pos[i] (sorted, in (0, n]) = input position where
// the i-th such operation ended the input, kind[i] = 1 FLUSH, 2 EMIT_METADATA.  is_final = 0: FINISH has not been seen, the
// stream ends behind the cut at n.  with_header = 0: the window bits were already sent.  end_bit (host, nullable) receives
// the bit position in the output where the metablock in front of each cut ended.
// finish_empty: FINISH came without input right behind a full input block (BrParams::finish_empty).
// lgblock (0 = default) / disable_ctx / stream_offset: BROTLI_PARAM_LGBLOCK / DISABLE_LITERAL_CONTEXT_MODELING / STREAM_OFFSET
// (the caller passes with_header = 0 and the cut behind the first two bytes that a stream offset implies, encode.c:1704).
// kind[i] = 3: the input is a BATCH of independent streams laid end to end and pos[i] is where one ends and the next begins
// (all cuts are of this kind then; every stream is shorter than 1 MiB and size_hint is the largest of them): each stream is
// compressed as BrotliEncoderCompress would compress it alone, its bytes start on a byte boundary of the output and
// stream_end[k] (host, n + 1 entries) receives the byte offset where stream k ends.
struct BrCuts { const uint32_t* pos; const uint32_t* kind; uint32_t n; int is_final; int with_header; int finish_empty; uint64_t* end_bit;
                int lgblock; int disable_ctx; uint32_t stream_offset; uint64_t* stream_end; };
extern "C" {
BrJob* br_job_create(void);
void br_job_destroy(BrJob*);
const BrJobStats* br_job_stats(const BrJob*);
void* br_job_stream(BrJob*);
int br_job_compress_device(BrJob* job, int quality, int lgwin, uint32_t size_hint,
                           const uint8_t* d_in, uint32_t n, const uint8_t** d_out, size_t* out_size, const BrCuts* cuts);
int br_debug_sort(int quality, int lgwin, const uint8_t* h_in, uint32_t n, uint32_t* h_S, uint32_t* h_seg);
int br_debug_index(int quality, int lgwin, const uint8_t* h_in, uint32_t n, uint32_t* h_S, uint32_t* h_seg, uint32_t* h_rank,
                   uint32_t* h_keys);
}
