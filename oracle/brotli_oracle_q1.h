/* oracle/brotli_oracle_q1.h -- TEST INFRASTRUCTURE, NOT PRODUCT (included by brotli_oracle.c).
 *
 * CPU restatement of the quality-1 path (SURVEY.md section 8, row F1): the two-pass fragment
 * coder of compress_fragment_two_pass.c driven by encode.c:1425 BrotliEncoderCompressStreamFast.
 * Positions are indices into the fragment, not pointers.  Word layout of the intermediate
 * command stream (one u32 = code | extra << 8) follows compress_fragment_two_pass.c:112-226:
 *   [0,24)   insert-length code c            (command.h:31 code, base/extra of RFC 7932 s.5)
 *   [24,40)  copy of (len-2) with the last distance, copy code c' = code-24 (c' < 16)
 *   [40,64)  copy-length code c = code-40
 *   [64,128) distance code = code-64 (64 = "last distance"; 80.. = ordinary codes 16..)
 */

/* compress_fragment_two_pass.c:32 Hash / :39 HashBytesAtOffset (v = 8 bytes at the position) */
static uint32_t q1_hash(uint64_t v, size_t shift, size_t min_match) {
  return (uint32_t)(((v << ((8 - min_match) * 8)) * 0x1E35A7BDull) >> shift);
}
/* :47 IsMatch */
static int q1_is_match(const uint8_t* a, const uint8_t* b, size_t min_match) {
  if (load32(a) != load32(b)) return 0;
  return min_match == 4 || (a[4] == b[4] && a[5] == b[5]);
}
/* RFC 7932 section 5 tables in closed form (the reference spells them out at :464-479) */
static uint32_t q1_ins_extra(uint32_t c) { return c < 6 ? 0 : c < 16 ? (c - 4) >> 1 : c < 21 ? c - 10 : c == 21 ? 12 : c == 22 ? 14 : 24; }
static uint32_t q1_ins_base(uint32_t c) {
  if (c < 6) return c;
  if (c < 16) { uint32_t nb = (c - 4) >> 1; return ((2 + (c & 1)) << nb) + 2; }
  if (c < 22) return (1u << (c - 10)) + 66;
  return c == 22 ? 6210 : 22594;
}
static uint32_t q1_copy_extra(uint32_t c) { return c < 8 ? 0 : c < 18 ? (c - 6) >> 1 : c < 23 ? c - 12 : 24; }
static uint32_t q1_copy_base(uint32_t c) {
  if (c < 8) return c + 2;
  if (c < 18) { uint32_t nb = (c - 6) >> 1; return ((2 + (c & 1)) << nb) + 6; }
  if (c < 23) return (1u << (c - 12)) + 70;
  return 2118;
}
static uint32_t q1_word_extra_bits(uint32_t code) {   /* :460 kNumExtraBits */
  if (code < 24) return q1_ins_extra(code);
  if (code < 40) return q1_copy_extra(code - 24);
  if (code < 64) return q1_copy_extra(code - 40);
  if (code < 80) return 0;
  return ((code - 80) >> 1) + 1;
}
/* :112 EmitInsertLen, :145 EmitCopyLen, :170 EmitCopyLenLastDistance, :213 EmitDistance */
static uint32_t* q1_emit_insert(uint32_t n, uint32_t* w) {
  uint32_t c = ins_code(n);
  *w++ = c | ((n - q1_ins_base(c)) << 8);
  return w;
}
static uint32_t* q1_emit_copy(uint32_t n, uint32_t* w) {
  uint32_t c = copy_code(n);
  *w++ = (c + 40) | ((n - q1_copy_base(c)) << 8);
  return w;
}
static uint32_t* q1_emit_copy_last(uint32_t n, uint32_t* w) {
  uint32_t m = n - 2, c = copy_code(m), x = (m - q1_copy_base(c)) << 8;
  if (c < 16) { *w++ = (c + 24) | x; }
  else { *w++ = (c + 40) | x; *w++ = 64; }
  return w;
}
static uint32_t* q1_emit_distance(uint32_t distance, uint32_t* w) {
  uint32_t d = distance + 3, nb = log2floor(d) - 1, prefix = (d >> nb) & 1;
  *w++ = (2 * (nb - 1) + prefix + 80) | ((d - ((2 + prefix) << nb)) << 8);
  return w;
}

/* :283-?,:341-?  the table refresh after a copy that ends at `ip`; returns the candidate for ip.
   `first` selects the variant used after the first copy of a run, whose min_match == 4 form
   stores ip-1 under the hash of ip-3 (offset 0 used twice, :339). */
static uint32_t q1_refresh_table(const uint8_t* base, size_t ip, int* table, size_t shift,
                                 size_t min_match, int first) {
  uint32_t cur;
  if (min_match == 4) {
    uint64_t v = load64(base + ip - 3);
    cur = q1_hash(v >> 24, shift, 4);
    table[q1_hash(v, shift, 4)] = (int)(ip - 3);
    table[q1_hash(v >> 8, shift, 4)] = (int)(ip - 2);
    table[q1_hash(first ? v : v >> 16, shift, 4)] = (int)(ip - 1);
  } else {
    uint64_t v = load64(base + ip - 5);
    table[q1_hash(v, shift, 6)] = (int)(ip - 5);
    table[q1_hash(v >> 8, shift, 6)] = (int)(ip - 4);
    table[q1_hash(v >> 16, shift, 6)] = (int)(ip - 3);
    v = load64(base + ip - 2);
    cur = q1_hash(v >> 16, shift, 6);
    table[q1_hash(v, shift, 6)] = (int)(ip - 2);
    table[q1_hash(v >> 8, shift, 6)] = (int)(ip - 1);
  }
  { uint32_t cand = (uint32_t)table[cur]; table[cur] = (int)ip; return cand; }
}

/* :228 CreateCommands.  base = start of the fragment, [start, start+block_size) the block,
   remaining = bytes from `start` to the end of the fragment. */
static void q1_create_commands(const uint8_t* base, size_t start, size_t block_size, size_t remaining,
                               int* table, size_t table_bits, size_t min_match,
                               uint8_t** literals, uint32_t** commands) {
  const size_t shift = 64 - table_bits;
  const size_t ip_end = start + block_size;
  const long kMaxDistance = (1L << 18) - 16;
  size_t ip = start, next_emit = start;
  int last_distance = -1;
  uint32_t* w = *commands; uint8_t* lit = *literals;
  if (block_size >= 16) {
    size_t len_limit = block_size - min_match < remaining - 16 ? block_size - min_match : remaining - 16;
    const size_t ip_limit = start + len_limit;
    uint32_t next_hash;
    ++ip;
    next_hash = q1_hash(load64(base + ip), shift, min_match);
    for (;;) {
      uint32_t skip = 32;
      size_t next_ip = ip, cand = 0;
      int found = 0;
      while (!found) {                         /* :277 trawl */
        uint32_t h = next_hash, step = skip++ >> 5;
        ip = next_ip;
        next_ip = ip + step;
        if (next_ip > ip_limit) goto remainder;
        next_hash = q1_hash(load64(base + next_ip), shift, min_match);
        if (last_distance > 0 && q1_is_match(base + ip, base + ip - last_distance, min_match)) {
          /* :291 with last_distance == -1 the candidate is ip + 1, which :292 rejects */
          table[h] = (int)ip; cand = ip - (size_t)last_distance; found = 1; break;
        }
        cand = (size_t)table[h];
        table[h] = (int)ip;
        if (q1_is_match(base + ip, base + cand, min_match) && (long)(ip - cand) <= kMaxDistance) found = 1;
      }
      {                                        /* :309 first copy of the run, with its literals */
        size_t matched = min_match + match_len(base + cand + min_match, base + ip + min_match, ip_end - ip - min_match);
        int distance = (int)(ip - cand);
        size_t insert = ip - next_emit;
        w = q1_emit_insert((uint32_t)insert, w);
        memcpy(lit, base + next_emit, insert); lit += insert;
        if (distance == last_distance) *w++ = 64;
        else { w = q1_emit_distance((uint32_t)distance, w); last_distance = distance; }
        w = q1_emit_copy_last((uint32_t)matched, w);
        ip += matched; next_emit = ip;
        if (ip >= ip_limit) goto remainder;
        cand = q1_refresh_table(base, ip, table, shift, min_match, 1);
      }
      while ((long)(ip - cand) <= kMaxDistance && q1_is_match(base + ip, base + cand, min_match)) {   /* :377 */
        size_t matched = min_match + match_len(base + cand + min_match, base + ip + min_match, ip_end - ip - min_match);
        last_distance = (int)(ip - cand);
        w = q1_emit_copy((uint32_t)matched, w);
        w = q1_emit_distance((uint32_t)last_distance, w);
        ip += matched; next_emit = ip;
        if (ip >= ip_limit) goto remainder;
        cand = q1_refresh_table(base, ip, table, shift, min_match, 0);
      }
      ++ip;
      next_hash = q1_hash(load64(base + ip), shift, min_match);
    }
  }
remainder:
  if (next_emit < ip_end) {
    size_t insert = ip_end - next_emit;
    w = q1_emit_insert((uint32_t)insert, w);
    memcpy(lit, base + next_emit, insert); lit += insert;
  }
  *commands = w; *literals = lit;
}

/* entropy_encode.h:82 SortHuffmanTreeItems with brotli_bit_stream.c:398's count-only comparator:
   not a total order, so the insertion / shell sort sequence itself is part of the format. */
static void q1_sort_by_count(HTree* it, size_t n) {
  static const size_t gaps[6] = {132, 57, 23, 10, 4, 1};
  size_t i;
  if (n < 13) {
    for (i = 1; i < n; ++i) {
      HTree t = it[i]; size_t k = i;
      while (k > 0 && t.count < it[k - 1].count) { it[k] = it[k - 1]; --k; }
      it[k] = t;
    }
  } else {
    int g;
    for (g = n < 57 ? 2 : 0; g < 6; ++g) {
      size_t gap = gaps[g];
      for (i = gap; i < n; ++i) {
        HTree t = it[i]; size_t j = i;
        for (; j >= gap && t.count < it[j - gap].count; j -= gap) it[j] = it[j - gap];
        it[j] = t;
      }
    }
  }
}
/* the static code-length code of entropy_encode_static.h:20,82: depths {4 x13, 5, 5, 0, 4, 4};
   its canonical bit-reversed codes and the zero / non-zero run encodings (:93-,:263-) are derived. */
static const uint8_t q1_cl_depth[18] = {4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 5, 5, 0, 4, 4};
static void q1_store_static_cl_code(BitW* w) {
  /* brotli_bit_stream.c:165 applied to q1_cl_depth: HSKIP 0, then 15 x "length 4" (2 bits, value 1)
     for symbols 1,2,3,4,0,5,17,6,16,7..12 and 2 x "length 5" (4 bits, value 15) for 13, 14 */
  store_hufftree_of_hufftree(2, q1_cl_depth, w);
}
static void q1_write_run(uint32_t sym, size_t reps, const uint16_t* cl_bits, BitW* w) {
  /* entropy_encode.c:160/198 run coding without their "7"/"11" special cases folded in here;
     sym 16: 2 extra bits, sym 17: 3 extra bits; digits most-significant first */
  uint8_t digits[16]; int nd = 0;
  const uint32_t xb = sym == 16 ? 2 : 3;
  for (;;) {
    digits[nd++] = (uint8_t)(reps & ((1u << xb) - 1));
    reps >>= xb;
    if (reps == 0) break;
    --reps;
  }
  while (nd--) { wbits(w, q1_cl_depth[sym], cl_bits[sym]); wbits(w, xb, digits[nd]); }
}
/* brotli_bit_stream.c:404 BrotliBuildAndStoreHuffmanTreeFast */
static void q1_build_and_store_tree_fast(const uint32_t* histo, size_t total, size_t max_bits,
                                         uint8_t* depth, uint16_t* bits, BitW* w) {
  HTree tree[2 * 704 + 2];
  size_t count = 0, symbols[4] = {0, 0, 0, 0}, length = 0, left = total, i;
  uint16_t cl_bits[18];
  while (left != 0) {
    if (histo[length]) { if (count < 4) symbols[count] = length; ++count; left -= histo[length]; }
    ++length;
  }
  if (count <= 1) {
    wbits(w, 4, 1); wbits(w, max_bits, symbols[0]);
    depth[symbols[0]] = 0; bits[symbols[0]] = 0;
    ++g_edge.simple_nsym1;
    return;
  }
  memset(depth, 0, length);
  {
    uint32_t limit;
    HTree sentinel; sentinel.count = 0xFFFFFFFFu; sentinel.left = -1; sentinel.right_or_value = -1;
    for (limit = 1;; limit *= 2) {
      size_t n = 0, a, b, k;
      for (i = length; i != 0;) {
        --i;
        if (histo[i]) { tree[n].count = histo[i] >= limit ? histo[i] : limit; tree[n].left = -1; tree[n].right_or_value = (int16_t)i; ++n; }
      }
      q1_sort_by_count(tree, n);
      tree[n] = sentinel; tree[n + 1] = sentinel;
      a = 0; b = n + 1;
      for (k = n - 1; k > 0; --k) {
        size_t l, r, parent = 2 * n - k;
        if (tree[a].count <= tree[b].count) l = a++; else l = b++;
        if (tree[a].count <= tree[b].count) r = a++; else r = b++;
        tree[parent].count = tree[l].count + tree[r].count;
        tree[parent].left = (int16_t)l; tree[parent].right_or_value = (int16_t)r;
        tree[parent + 1] = sentinel;
      }
      if (set_depth((int)(2 * n - 1), tree, depth, 14)) break;
      ++g_edge.retry_fast;
    }
  }
  depths_to_symbols(depth, length, bits);
  if (count <= 4) {
    size_t j;
    wbits(w, 2, 1); wbits(w, 2, count - 1);
    for (i = 0; i < count; i++)
      for (j = i + 1; j < count; j++)
        if (depth[symbols[j]] < depth[symbols[i]]) { size_t t = symbols[j]; symbols[j] = symbols[i]; symbols[i] = t; }
    for (i = 0; i < count; ++i) wbits(w, max_bits, symbols[i]);
    if (count == 4) wbits(w, 1, depth[symbols[0]] == 1 ? 1 : 0);
    if (count == 2) ++g_edge.simple_nsym2;
    else if (count == 3) ++g_edge.simple_nsym3;
    else { ++g_edge.simple_nsym4; if (depth[symbols[0]] == 1) ++g_edge.simple_select1; else ++g_edge.simple_select0; }
    return;
  }
  depths_to_symbols(q1_cl_depth, 18, cl_bits);
  q1_store_static_cl_code(w);
  {
    uint8_t prev = 8;
    for (i = 0; i < length;) {
      const uint8_t v = depth[i]; size_t reps = 1, k;
      for (k = i + 1; k < length && depth[k] == v; ++k) ++reps;
      i += reps;
      if (v == 0) {
        /* kZeroReps[reps]: the generic zero-run writer (entropy_encode.c:198) under the static code */
        if (reps == 11) { wbits(w, q1_cl_depth[0], cl_bits[0]); --reps; }
        if (reps < 3) { while (reps--) wbits(w, q1_cl_depth[0], cl_bits[0]); }
        else q1_write_run(17, reps - 3, cl_bits, w);
      } else {
        if (prev != v) { wbits(w, q1_cl_depth[v], cl_bits[v]); --reps; }
        if (reps < 3) { while (reps--) wbits(w, q1_cl_depth[v], cl_bits[v]); }
        else q1_write_run(16, reps - 3, cl_bits, w);
        prev = v;
      }
    }
  }
}

/* :58 BuildAndStoreCommandPrefixCode.  order[] lists the 64 insert/copy words in the order of
   their symbols in the full 704-symbol alphabet, sym704() is that symbol. */
static uint32_t q1_sym704(uint32_t code) {
  if (code < 8) return 128 + 8 * code;
  if (code < 16) return 256 + 8 * (code - 8);
  if (code < 24) return 448 + 8 * (code - 16);
  if (code < 32) return code - 24;
  if (code < 40) return 64 + (code - 32);
  if (code < 48) return 128 + (code - 40);
  if (code < 56) return 192 + (code - 48);
  return 384 + (code - 56);
}
static void q1_store_command_code(const uint32_t* histo, uint8_t* depth, uint16_t* bits, BitW* w) {
  HTree tree[2 * 704 + 1];
  uint8_t perm_depth[64], full[704];
  uint16_t perm_bits[64];
  uint32_t k;
  memset(depth, 0, 128);
  create_huffman_tree(histo, 64, 15, tree, depth);
  create_huffman_tree(histo + 64, 64, 14, tree, depth + 64);
  for (k = 0; k < 64; ++k) {
    uint32_t code = k < 24 ? k + 24 : k < 32 ? k - 24 : k < 40 ? k + 16 : k < 48 ? k - 32 : k < 56 ? k + 8 : k - 40;
    perm_depth[k] = depth[code];
  }
  memset(perm_bits, 0, sizeof(perm_bits));
  depths_to_symbols(perm_depth, 64, perm_bits);
  for (k = 0; k < 64; ++k) {
    uint32_t code = k < 24 ? k + 24 : k < 32 ? k - 24 : k < 40 ? k + 16 : k < 48 ? k - 32 : k < 56 ? k + 8 : k - 40;
    bits[code] = perm_bits[k];
  }
  depths_to_symbols(depth + 64, 64, bits + 64);
  memset(full, 0, sizeof(full));
  for (k = 24; k < 64; ++k) full[q1_sym704(k)] = depth[k];
  for (k = 0; k < 24; ++k) full[q1_sym704(k)] = depth[k];
  store_huffman_tree(full, 704, tree, w);
  store_huffman_tree(depth + 64, 64, tree, w);
}

/* :197 BrotliStoreMetaBlockHeader */
static void q1_store_mb_header(size_t len, int uncompressed, BitW* w) {
  size_t nibbles = len <= (1u << 16) ? 4 : len <= (1u << 20) ? 5 : 6;
  wbits(w, 1, 0); wbits(w, 2, nibbles - 4); wbits(w, nibbles * 4, len - 1); wbits(w, 1, (uint64_t)uncompressed);
}
/* :548 EmitUncompressedMetaBlock */
static void q1_emit_uncompressed(const uint8_t* in, size_t n, BitW* w) {
  q1_store_mb_header(n, 1, w);
  w->ix = (w->ix + 7) & ~(size_t)7;
  memcpy(w->buf + (w->ix >> 3), in, n);
  w->ix += n << 3;
  w->buf[w->ix >> 3] = 0;
}
/* :526 ShouldCompress */
static int q1_should_compress(const uint8_t* in, size_t n, size_t num_literals) {
  double corpus = (double)n;
  if ((double)num_literals < 0.98 * corpus) return 1;
  {
    uint32_t histo[256]; size_t i;
    const double max_cost = corpus * 8 * 0.98 / 43;
    memset(histo, 0, sizeof(histo));
    for (i = 0; i < n; i += 43) ++histo[in[i]];
    return bits_entropy(histo, 256) < max_cost;
  }
}
/* :458 StoreCommands */
static void q1_store_commands(const uint8_t* lits, size_t nlit, const uint32_t* cmds, size_t ncmd, BitW* w) {
  uint32_t lit_histo[256], cmd_histo[128];
  uint8_t lit_depth[256], cmd_depth[128];
  uint16_t lit_bits[256], cmd_bits[128];
  size_t i;
  memset(lit_histo, 0, sizeof(lit_histo)); memset(cmd_histo, 0, sizeof(cmd_histo));
  memset(lit_depth, 0, sizeof(lit_depth)); memset(lit_bits, 0, sizeof(lit_bits));
  memset(cmd_bits, 0, sizeof(cmd_bits));
  for (i = 0; i < nlit; ++i) ++lit_histo[lits[i]];
  q1_build_and_store_tree_fast(lit_histo, nlit, 8, lit_depth, lit_bits, w);
  for (i = 0; i < ncmd; ++i) ++cmd_histo[cmds[i] & 0xFF];
  cmd_histo[1] += 1; cmd_histo[2] += 1; cmd_histo[64] += 1; cmd_histo[84] += 1;
  q1_store_command_code(cmd_histo, cmd_depth, cmd_bits, w);
  for (i = 0; i < ncmd; ++i) {
    const uint32_t code = cmds[i] & 0xFF, extra = cmds[i] >> 8;
    wbits(w, cmd_depth[code], cmd_bits[code]);
    wbits(w, q1_word_extra_bits(code), extra);
    if (code < 24) {
      uint32_t j, ins = q1_ins_base(code) + extra;
      for (j = 0; j < ins; ++j) { wbits(w, lit_depth[*lits], lit_bits[*lits]); ++lits; }
    }
  }
}

/* :612 BrotliCompressFragmentTwoPass (+ :563 Impl) for one fragment. */
static void q1_compress_fragment(const uint8_t* in, size_t n, int is_last, uint32_t* cmd_buf, uint8_t* lit_buf,
                                 int* table, size_t table_size, BitW* w) {
  const size_t start_ix = w->ix;
  const size_t table_bits = log2floor(table_size);
  const size_t min_match = table_bits <= 15 ? 4 : 6;
  size_t off = 0;
  while (off < n) {
    size_t block = n - off < ((size_t)1 << 17) ? n - off : ((size_t)1 << 17);
    uint32_t* c = cmd_buf; uint8_t* l = lit_buf;
    q1_create_commands(in, off, block, n - off, table, table_bits, min_match, &l, &c);
    if (q1_should_compress(in + off, block, (size_t)(l - lit_buf))) {
      q1_store_mb_header(block, 0, w);
      wbits(w, 13, 0);
      q1_store_commands(lit_buf, (size_t)(l - lit_buf), cmd_buf, (size_t)(c - cmd_buf), w);
    } else {
      q1_emit_uncompressed(in + off, block, w);
    }
    off += block;
  }
  if (w->ix - start_ix > 31 + (n << 3)) {    /* :635 larger than one raw meta-block: redo it raw */
    size_t b = start_ix >> 3, e = (w->ix >> 3) + 9;
    w->buf[b] &= (uint8_t)((1u << (start_ix & 7)) - 1);
    memset(w->buf + b + 1, 0, e - b - 1);
    w->ix = start_ix;
    q1_emit_uncompressed(in, n, w);
  }
  if (is_last) { wbits(w, 1, 1); wbits(w, 1, 1); w->ix = (w->ix + 7) & ~(size_t)7; }
}

/* encode.c:1425 BrotliEncoderCompressStreamFast seen from the caller: every CompressStream call
   that brings `a` bytes is cut into fragments of at most 1 << lgwin bytes, each compressed with
   a freshly zeroed table (encode.c:156 GetHashTable); FINISH closes the stream after the last
   fragment of its call (an empty one if it brought no bytes).  call_sizes == NULL: one call. */
/* ops (nullable): per call 0 = PROCESS, 1 = FLUSH, 2 = FINISH; NULL = PROCESS ... PROCESS, FINISH.  A FLUSH
   call compresses what it brought and then, if the stream is not byte aligned, appends the 6-bit empty
   metadata block of encode.c:1356 InjectBytePaddingBlock. */
int oracle_brotli_compress_q1_ops(int lgwin, size_t n, const uint8_t* in, size_t ncalls, const size_t* call_sizes,
                                  const int* ops, size_t* out_n, uint8_t* out) {
  const size_t limit = (size_t)1 << lgwin;
  const size_t cap = *out_n;
  uint32_t* cmd_buf; uint8_t* lit_buf; int* table; uint8_t* buf;
  BitW w; size_t pos = 0, ci, one = n;
  int hdr_lgwin = lgwin < 18 ? 18 : lgwin;
  if (lgwin < 10 || lgwin > 24) return 0;
  if (!call_sizes) { call_sizes = &one; ncalls = 1; ops = NULL; }
  buf = (uint8_t*)calloc(2 * n + 1024 + 16 * (n / 1024 + ncalls + 4), 1);
  cmd_buf = (uint32_t*)malloc(4u << 17); lit_buf = (uint8_t*)malloc(1u << 17);
  table = (int*)malloc(sizeof(int) << 17);
  w.buf = buf; w.ix = 0;
  wbits(&w, 4, (uint64_t)(((hdr_lgwin - 17) << 1) | 1));      /* encode.c:203 EncodeWindowBits, lgwin > 17 */
  for (ci = 0; ci < ncalls; ++ci) {
    size_t a = call_sizes[ci];
    const int op = ops ? ops[ci] : (ci + 1 == ncalls ? 2 : 0);
    if (a != 0 || op == 2) {
      do {
        size_t frag = a < limit ? a : limit, ts = 256;
        while (ts < ((size_t)1 << 17) && ts < frag) ts <<= 1;       /* encode.c:148 HashTableSize */
        memset(table, 0, ts * sizeof(int));
        q1_compress_fragment(in + pos, frag, op == 2 && frag == a, cmd_buf, lit_buf, table, ts, &w);
        pos += frag; a -= frag;
      } while (a != 0);
    }
    if (op == 1 && (w.ix & 7) != 0) { wbits(&w, 6, 6); w.ix = (w.ix + 7) & ~(size_t)7; }
  }
  free(cmd_buf); free(lit_buf); free(table);
  { size_t bytes = (w.ix + 7) >> 3; int ok = bytes <= cap;
    if (ok) { memcpy(out, buf, bytes); *out_n = bytes; }
    free(buf); return ok; }
}
int oracle_brotli_compress_q1(int lgwin, size_t n, const uint8_t* in, size_t ncalls, const size_t* call_sizes,
                              size_t* out_n, uint8_t* out) {
  return oracle_brotli_compress_q1_ops(lgwin, n, in, ncalls, call_sizes, NULL, out_n, out);
}
