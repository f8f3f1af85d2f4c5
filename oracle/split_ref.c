/* oracle/split_ref.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * Runs the reference encoder's greedy block splitter (c/enc/metablock.c BrotliBuildMetaBlockGreedy, linked from the
 * unmodified reference sources by oracle/Makefile into oracle/_ref/split_ref) on metablocks read from stdin, so that
 * tests/test_entropy_split.py can pin the oracle's splitter to it.  Input, little-endian u32 words unless noted, per
 * metablock: nctx (1, 2, 3 or 13), prev_byte, prev_byte2, length, ncmd, the 64-entry static context map, then length
 * data bytes and ncmd commands of 16 bytes (the reference's Command layout).  A zero word ends the input.  Output, one
 * line per metablock: for literals, commands and distances the number of types and of blocks, the types, the lengths
 * and the histograms (literal rows of 256, command rows of 704, the first 64 symbols of distance rows), all as decimal
 * numbers separated by spaces. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "enc/command.h"
#include "enc/memory.h"
#include "enc/metablock.h"
#include "common/context.h"

static int rd(void* p, size_t n) { return fread(p, 1, n, stdin) == n; }

static void put_split(const BlockSplit* s) {
  size_t i;
  printf(" %zu %zu", s->num_types, s->num_blocks);
  for (i = 0; i < s->num_blocks; ++i) printf(" %u", s->types[i]);
  for (i = 0; i < s->num_blocks; ++i) printf(" %u", s->lengths[i]);
}

int main(void) {
  for (;;) {
    uint32_t h[5], map[64];
    uint8_t* data; Command* cmds;
    MemoryManager m; MetaBlockSplit mb; size_t i, k;
    if (!rd(h, 4) || h[0] == 0) return 0;
    if (!rd(h + 1, 16) || !rd(map, sizeof(map))) return 1;
    data = (uint8_t*)malloc(h[3] + 8); cmds = (Command*)malloc(h[4] * sizeof(Command) + 1);
    if (!rd(data, h[3]) || !rd(cmds, h[4] * sizeof(Command))) return 1;
    BrotliInitMemoryManager(&m, 0, 0, 0);
    InitMetaBlockSplit(&mb);
    BrotliBuildMetaBlockGreedy(&m, data, 0, (size_t)-1 >> 2, NULL, 0, (uint8_t)h[1], (uint8_t)h[2],
                               BROTLI_CONTEXT_LUT(CONTEXT_UTF8), h[0], h[0] > 1 ? map : NULL, cmds, h[4], &mb);
    put_split(&mb.literal_split); put_split(&mb.command_split); put_split(&mb.distance_split);
    for (i = 0; i < mb.literal_histograms_size; ++i) for (k = 0; k < 256; ++k) printf(" %u", mb.literal_histograms[i].data_[k]);
    for (i = 0; i < mb.command_histograms_size; ++i) for (k = 0; k < 704; ++k) printf(" %u", mb.command_histograms[i].data_[k]);
    for (i = 0; i < mb.distance_histograms_size; ++i) for (k = 0; k < 64; ++k) printf(" %u", mb.distance_histograms[i].data_[k]);
    printf("\n");
    DestroyMetaBlockSplit(&m, &mb);
    free(data); free(cmds);
  }
}
