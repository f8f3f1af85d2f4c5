/* brotli_b200.h -- C ABI of libbrotlienc_b200.so.
 *
 * Drop-in boundary: the encoder half of google/brotli's public API,
 * /root/reference/c/include/brotli/encode.h (function by function below), with identical
 * names, argument meaning, enum values and error behaviour, so that the `brotli` CLI
 * (c/tools/brotli.c:1357), the Python extension (python/_brotli.c:403,529), the Go wrapper
 * (go/cbrotli/writer.go:30) and the JNI wrapper (java/org/brotli/wrapper/enc/encoder_jni.cc:78)
 * can link against this library instead of libbrotlienc.  See INTEGRATION.md.
 *
 * The hot path runs on an NVIDIA H100 (sm_90a).  There is NO CPU implementation inside
 * the library: without a CUDA device, or for parameters outside the implemented path
 * (quality 1..9, no custom dictionary, modes GENERIC/TEXT: limits below), the entry points
 * return BROTLI_FALSE / NULL instead of producing different bytes.
 *
 * Plain C: pointers and sizes only, no torch / CUDA types.
 */
#ifndef BROTLI_B200_H_
#define BROTLI_B200_H_
/* The reference API itself -- the 13 BROTLI_ENC_API functions of c/include/brotli/encode.h (SetParameter :289,
 * CreateInstance :306, DestroyInstance :314, PrepareDictionary :343, DestroyPreparedDictionary :348,
 * AttachPreparedDictionary :361, MaxCompressedSize :375, Compress :405, CompressStream :473, IsFinished :486,
 * HasMoreOutput :495, TakeOutput :526, Version :542) -- is declared in include/brotli/encode.h of this repository with the
 * reference's own types (no re-definition here, so this header mixes with <brotli/encode.h> and <brotli/decode.h>).
 *
 * Limits of the implemented path (everything else returns BROTLI_FALSE / NULL, never other bytes):
 *   quality 1..4 (lgwin 10..24) and quality 5..9 (lgwin 17..24), modes GENERIC / TEXT, default NPOSTFIX / NDIRECT, no
 *   dictionaries, no LARGE_WINDOW.  (Qualities 2..4 -- hash_longest_match_quickly_inc.h, brotli_bit_stream.c:1196-1317 --
 *   are the newest path: see DESIGN.md section 3d for what has and has not been run on a GPU.)  BROTLI_PARAM_LGBLOCK, DISABLE_LITERAL_CONTEXT_MODELING, SIZE_HINT and (quality 5..9)
 *   STREAM_OFFSET are honoured.  Quality 1: streams of any size, compressed in device segments of <= 128 MiB as the calls
 *   arrive (bounded memory).  Quality 2..9: one stream <= 1 GiB -- BrotliEncoderCompressStream fails on the PROCESS call
 *   that crosses it; the stream so far is kept in host memory and recompressed at every FLUSH (see csrc/br_driver.h).
 *   FLUSH, FINISH and (quality 2..9) EMIT_METADATA follow encode.h:93-157. */
#include <brotli/encode.h>
#ifdef __cplusplus
extern "C" {
#endif

#define BROTLI_B200_API BROTLI_ENC_API

/* ---- device-resident extensions (not in the reference API) ------------------------ */
/* Same as BrotliEncoderCompress but input and output live in DEVICE memory of the current
 * CUDA device (plain device pointers).  *encoded_size: in = capacity, out = bytes written. */
BROTLI_B200_API BROTLI_BOOL BrotliB200CompressDevice(int quality, int lgwin, size_t input_size, const void* d_input, size_t* encoded_size, void* d_encoded);
/* Many independent streams (SURVEY.md 8e: one stream per shard / per object).  Inputs and
 * outputs are host pointers; every stream comes out exactly as BrotliEncoderCompress(quality, lgwin, GENERIC) gives it.
 * Quality 2..4: one device job per stream, on `threads` host workers.
 * Quality 5..9: streams shorter than 1 MiB are laid end to end and run as ONE device job per group of <= 128 MiB / 8192 streams (one
 * set of launches, one copy each way; `threads` parallelises the host-side packing); longer streams are spread over
 * `threads` host workers, each with its own CUDA stream.  Quality 1 (compress_fragment_two_pass.c:612, one independent
 * fragment coder per stream): the whole batch is ONE device batch -- four kernel launches, one copy each way.  encoded_sizes[i]: in = capacity of outputs[i], out = bytes written.
 * Returns the number of streams compressed successfully. */
BROTLI_B200_API size_t BrotliB200CompressBatch(int quality, int lgwin, size_t count, const uint8_t* const* inputs, const size_t* input_sizes, uint8_t* const* outputs, size_t* encoded_sizes, int threads);
/* Device resident batches.  Quality 2..9: `count` non-empty streams of less than 1 MiB each sit in one device buffer, stream i
 * at d_inputs + input_offsets[i]; consecutive streams are grouped into device jobs of <= 128 MiB / 8192 streams (a group whose
 * streams lie back to back is read in place).  The compressed streams are packed DENSELY into d_encoded in input order:
 * stream i at d_encoded + encoded_offsets[i] (count + 1 entries, last = bytes used), encoded_sizes[i] bytes (0 = above
 * BrotliEncoderMaxCompressedSize: that stream must go through the host call).  The inputs must be complete before the call (it
 * runs on the calling thread's own CUDA stream and returns when the outputs are complete).  Returns the number of streams
 * compressed, 0 if a job failed or d_encoded is too small.
 * Quality 1, device resident: `count` non-empty streams sit in ONE device buffer, stream i at d_inputs + input_offsets[i]
 * (host array), input_sizes[i] bytes (host array).  The compressed streams are packed into d_encoded (device), stream i at
 * d_encoded + encoded_offsets[i] (host array of count + 1 entries, 16-byte aligned starts, last = bytes used),
 * encoded_sizes[i] bytes (host array; 0 = that stream must go through the host call: it compressed to more than
 * BrotliEncoderMaxCompressedSize).  Bytes equal BrotliEncoderCompress(1, lgwin, GENERIC, ...) per stream.
 * Returns the number of streams compressed. */
BROTLI_B200_API size_t BrotliB200CompressBatchDevice(int quality, int lgwin, size_t count, const void* d_inputs, const uint64_t* input_offsets, const size_t* input_sizes, void* d_encoded, size_t encoded_capacity, uint64_t* encoded_offsets, size_t* encoded_sizes);
/* Timings (milliseconds, CUDA events) and counters of the calling thread's last compress call.
 * out[0..15]: total, index (hash+sort), lz77, entropy, assemble, lz77 iterations, block runs,
 * blocks, metablocks, kernel launches, summed k_walk ms, k_encode_mb ms, k_walk launches,
 * k_encode_mb launches, input bytes walked over all k_walk launches, commands emitted. */
BROTLI_B200_API void BrotliB200LastStats(double out[16]);
/* quality-1 batch pipeline of the calling thread's last call: ms total / h2d / parse / code / pack / d2h, then
   streams, fragments, blocks, input bytes, compressed bytes, launches */
BROTLI_B200_API void BrotliB200LastStatsQ1(double out[12]);
/* 1 if a usable CUDA device is present. */
BROTLI_B200_API int BrotliB200Available(void);

#ifdef __cplusplus
}
#endif
#endif  /* BROTLI_B200_H_ */
