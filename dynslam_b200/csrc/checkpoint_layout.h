// checkpoint_layout.h — section offsets of a checkpoint (the layout include/b200fusion.h documents). The checkpoint oracle
// restates them on its own (oracle/checkpoint_oracle.c), so the engine-vs-oracle comparison checks this code too.
#pragma once
#include "../../include/b200fusion.h"

/* Fills h->section[] and h->totalBytes from the geometry, flags and counts of h (all non-negative); returns totalBytes. */
static inline uint64_t checkpoint_layout(b200_checkpoint_header *h) {
  const uint64_t px = (uint64_t)h->img_w * (uint64_t)h->img_h, noTotal = (uint64_t)h->numBuckets + (uint64_t)h->excessSize;
  const uint64_t vis = (uint64_t)(h->noVisibleBlocks < h->numBlocks ? h->noVisibleBlocks : h->numBlocks);
  const int fwd = (h->flags & B200_CK_HAS_FORWARD) != 0;
  const uint64_t len[B200_CK_SECTIONS] = {
    4 * (uint64_t)h->noEntries, 20 * (uint64_t)h->noEntries, 4 * (uint64_t)h->numBlocks, 4 * (uint64_t)h->excessSize,
    (h->flags & B200_CK_HAS_SWAP_STATES) ? noTotal : 0, 4 * (uint64_t)h->noVisBytes, (uint64_t)h->noVisBytes, 12 * vis,
    8 * px, 16 * px, 4 * px, fwd ? 16 * px : 0, fwd ? 4 * px : 0, 4 * (uint64_t)h->noSnapshots, 12 * (uint64_t)h->noQueueItems,
    4 * (uint64_t)h->noBlocks, 4096 * (uint64_t)h->noBlocks};
  uint64_t off = B200_CHECKPOINT_HEADER_BYTES;
  for (int i = 0; i < B200_CK_SECTIONS; ++i) {
    const uint64_t a = (i == B200_CK_BLOCK_DATA) ? 4096 : 16;
    off = (off + a - 1) & ~(a - 1);
    h->section[i][0] = off; h->section[i][1] = len[i];
    off += len[i];
  }
  h->totalBytes = off;
  return off;
}
