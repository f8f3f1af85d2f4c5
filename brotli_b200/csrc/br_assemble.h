// br_assemble.h -- stream assembly: where every metablock's bits go in the output (serial scan over the metablock
// records; the copies themselves are data parallel, k_assemble_copy).  Shared by the CUDA pipeline and the CPU sim.
#pragma once
#include "br_entropy2.h"

struct BrCopyDesc { u64 dst_bit; u64 src_off; u32 nbits; u32 kind; };  // kind 0: bit copy from outbits, 1: raw bytes from input
// encode.c:185 EncodeWindowBits (lgwin 10..24; no large window)
BR_DEV u32 br_put_window_bits(u32* out, u64 bit, int lgwin) {
  if (lgwin == 16) { br_put_bits_at(out + (bit >> 5), (u32)(bit & 31), 1, 0); return 1; }
  if (lgwin == 17) { br_put_bits_at(out + (bit >> 5), (u32)(bit & 31), 7, 1); return 7; }
  if (lgwin < 17) { br_put_bits_at(out + (bit >> 5), (u32)(bit & 31), 7, (u64)(((lgwin - 8) << 4) | 1)); return 7; }
  br_put_bits_at(out + (bit >> 5), (u32)(bit & 31), 4, (u64)(((lgwin - 17) << 1) | 1));
  return 4;
}
// res[0..1]: total bytes (u64), res[2]: number of metablocks that need the late fallback (marked in force_unc under the
// number of their first chunk, which is what the chain looks up when it forms the metablock again: the FIRST
// such metablock of every stream -- storing it raw restores the distance cache behind it, so the rest of that stream is
// parsed again), res[3]: cuts seen.
// with_header: the stream starts here (window bits); 0 when the caller already sent them (a FLUSH / EMIT_METADATA before any
// input).  cut_kind[i] says what ended the i-th flushed metablock: 1 = FLUSH (encode.c:1356 InjectBytePaddingBlock: an empty
// metadata block pads to a byte boundary unless the stream stands on one), 2 = EMIT_METADATA (encode.c:1549: no padding
// block -- the caller merges its metadata header into the pending bits -- and the next metablock starts on the next byte
// boundary).  cut_end_bit[i] receives the bit position where that metablock ended (before any padding).
// Batch of streams (BrParams::multi): every stream starts on a byte boundary with its own window bits; stream_end[k]
// receives the byte offset where the k-th stream ends.
BR_DEV void br_assemble_scan(const BrStream& s, const u64* out_off, u32* out, BrCopyDesc* desc, u32* res,
                             int with_header, const u32* cut_kind, u64* cut_end_bit, u64* stream_end) {
  u64 bit = 0;
  u32 ncut = 0, nstream = 0;
  const int lgwin = s.P.lgwin;
  const u32 nm = s.counters[1];
  u32 fallbacks = 0;
  bool skip = false;   // behind a fallback: the rest of the stream will be parsed again, its sizes mean nothing
  for (u32 i = 0; i < nm; ++i) {
    BrMetaBlock mb = s.mbs[i];
    const u32 bytes = mb.end - mb.start;
    if (mb.start == mb.base) {
      skip = false;
      if (i == 0 ? with_header != 0 : true) bit += br_put_window_bits(out, bit, lgwin);
    }
    BrCopyDesc d;
    if (mb.compress) {
      u64 storage_ix = (bit & 7) + mb.out_bits;
      if (mb.is_last) storage_ix = (storage_ix + 7) & ~7ull;
      if ((u64)bytes + 4 < (storage_ix >> 3) && !skip) { s.force_unc[mb.first_block] = 1; ++fallbacks; skip = true; }   // encode.c:604
      d.dst_bit = bit; d.src_off = out_off[i]; d.nbits = mb.out_bits; d.kind = 0;
      bit += mb.out_bits;
      if (mb.is_last) bit = (bit + 7) & ~7ull;
    } else {
      // brotli_bit_stream.c:1321 BrotliStoreUncompressedMetaBlock
      u32* w32 = out + (bit >> 5); u32 sh = (u32)(bit & 31);   // write relative to a word base to keep ix in 32 bits
      u32 ix = sh;
      br_put_bits_at(w32, ix, 1, 0); ix += 1;
      { u32 lg = bytes == 1 ? 1 : br_log2floor(bytes - 1) + 1; u32 mn = (lg < 16 ? 16 : (lg + 3)) / 4;
        br_put_bits_at(w32, ix, 2, mn - 4); ix += 2; br_put_bits_at(w32, ix, mn * 4, bytes - 1); ix += mn * 4; }
      br_put_bits_at(w32, ix, 1, 1); ix += 1;
      bit += ix - sh;
      bit = (bit + 7) & ~7ull;
      d.dst_bit = bit; d.src_off = mb.start; d.nbits = bytes; d.kind = 1;
      bit += (u64)bytes * 8;
      if (mb.is_last) { br_put_bits_at(out + (bit >> 5), (u32)(bit & 31), 2, 3); bit += 2; bit = (bit + 7) & ~7ull; }
    }
    desc[i] = d;
    if (mb.empty_last) { br_put_bits_at(out + (bit >> 5), (u32)(bit & 31), 2, 3); bit += 2; bit = (bit + 7) & ~7ull; }   // encode.c:520
    if (mb.flushed && !mb.is_last) {
      cut_end_bit[ncut] = bit;
      if (cut_kind[ncut] == 1 && (bit & 7)) { br_put_bits_at(out + (bit >> 5), (u32)(bit & 31), 6, 6); bit += 6; }
      bit = (bit + 7) & ~7ull;
      ++ncut;
    }
    if (mb.is_last && stream_end) stream_end[nstream++] = bit >> 3;
  }
  u64 total = (bit + 7) >> 3;
  res[0] = (u32)total; res[1] = (u32)(total >> 32); res[2] = fallbacks; res[3] = ncut;
}
// The copy of a descriptor goes word by word, in any order: br_copy_words words, word i by br_copy_word.  Bits: 32 from
// outbits put at dst_bit + 32 i.  Raw bytes (byte aligned): the input bytes that fall into the i-th destination word.
BR_DEV u32 br_copy_words(const BrCopyDesc& d) {
  if (d.kind == 0) return (d.nbits + 31) / 32;
  const u64 dst_byte = d.dst_bit >> 3;
  return (u32)(((dst_byte + d.nbits - 1) >> 2) - (dst_byte >> 2) + 1);
}
BR_DEV void br_copy_word(const BrCopyDesc& d, u32 i, const u32* outbits, const u8* data, u32* out) {
  if (d.kind == 0) {
    u32 nb = (i + 1) * 32 <= d.nbits ? 32 : d.nbits - i * 32;
    u32 v = outbits[d.src_off + i];
    if (nb < 32) v &= (1u << nb) - 1;
    u64 db = d.dst_bit + (u64)i * 32;
    br_put_bits_at(out + (db >> 5), (u32)(db & 31), nb, v);
  } else {
    u64 dst_byte = d.dst_bit >> 3, first_word = dst_byte >> 2, wbyte = (first_word + i) << 2;
    u32 v = 0;
    for (u32 b = 0; b < 4; ++b) {
      u64 ob = wbyte + b;
      if (ob >= dst_byte && ob < dst_byte + d.nbits) v |= (u32)data[d.src_off + (ob - dst_byte)] << (8 * b);
    }
    if (v) br_atomic_or(out + first_word + i, v);
  }
}
