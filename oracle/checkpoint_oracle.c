/*
 * checkpoint_oracle.c — TEST INFRASTRUCTURE ONLY. Serial restatement of b200_checkpoint_save / b200_checkpoint_load
 * (dynslam_b200/csrc/checkpoint.cu, format in include/b200fusion.h) over the CPU oracle's state (tsdf_oracle.c): the
 * engine's checkpoint of a state equals oracle_checkpoint_save's bytes of the same state whenever the engine has dropped
 * no snapshot (the oracle's queue is unbounded; it stores an overwritten snapshot, loaded from an engine's checkpoint, as
 * one of count -1, which its Decay sweeps as nothing).
 *
 * The oracle engine's fields are private to tsdf_oracle.c; the struct below restates its layout (that file is frozen).
 * The section offsets are restated here from the format's description in include/b200fusion.h (place_sections), not taken
 * from the engine's code, so that the engine-vs-oracle byte comparison also checks the engine's layout.
 */
#include "../include/b200fusion.h"

#include <stdlib.h>
#include <string.h>

typedef struct snap { int count; int frameIdx; b200_vec3i *items; struct snap *next; } snap;
typedef struct oracle_engine {
  int noTotalEntries;
  uint8_t *allocType;
  int16_t *blockCoords;
  int frameIdx;
  long totalDecayed;
  snap *q_head, *q_tail; int q_size;
  int16_t *allocatedBlockPositions; int allocatedCap;
  int noIntegratedBlocks;
} oracle_engine;

static int entry_is_reset(const b200_hash_entry *h) {
  return h->pos[0] == 0 && h->pos[1] == 0 && h->pos[2] == 0 && h->_pad == 0 && h->offset == 0 && h->ptr == -2 && h->allocatedTime == 0;
}

static int block_is_reset(const b200_voxel *v) {
  for (int i = 0; i < 512; ++i)
    if (v[i].sdf != 32767 || v[i].w_depth || v[i].clr[0] || v[i].clr[1] || v[i].clr[2] || v[i].w_color || v[i]._pad) return 0;
  return 1;
}

static int has_forward(const b200_render_state *rs) { return rs->d_forwardProjection && rs->d_fwdProjMissingPoints; }

/* The layout include/b200fusion.h describes: the 512-byte header, then each section in order at the next 16-byte boundary,
   the voxel payload at the next 4096-byte boundary; totalBytes = the end of the payload. */
static uint64_t place_sections(b200_checkpoint_header *h) {
  const uint64_t px = (uint64_t)h->img_w * (uint64_t)h->img_h;
  const uint64_t entries = (uint64_t)h->numBuckets + (uint64_t)h->excessSize;
  const uint64_t listed = (uint64_t)(h->noVisibleBlocks < h->numBlocks ? h->noVisibleBlocks : h->numBlocks);
  const int swap = (h->flags & B200_CK_HAS_SWAP_STATES) != 0, fwd = (h->flags & B200_CK_HAS_FORWARD) != 0;
  uint64_t bytes[B200_CK_SECTIONS];
  bytes[B200_CK_HASH_INDEX] = sizeof(uint32_t) * (uint64_t)h->noEntries;
  bytes[B200_CK_HASH_ENTRIES] = sizeof(b200_hash_entry) * (uint64_t)h->noEntries;
  bytes[B200_CK_ALLOCATION_LIST] = sizeof(int32_t) * (uint64_t)h->numBlocks;
  bytes[B200_CK_EXCESS_LIST] = sizeof(int32_t) * (uint64_t)h->excessSize;
  bytes[B200_CK_SWAP_STATES] = swap ? entries : 0;
  bytes[B200_CK_VIS_INDEX] = sizeof(uint32_t) * (uint64_t)h->noVisBytes;
  bytes[B200_CK_VIS_VALUE] = (uint64_t)h->noVisBytes;
  bytes[B200_CK_VISIBLE_LIST] = sizeof(b200_vec3i) * listed;
  bytes[B200_CK_MINMAX] = sizeof(b200_vec2f) * px;
  bytes[B200_CK_RAYCAST_RESULT] = sizeof(b200_vec4f) * px;
  bytes[B200_CK_RAYCAST_IMAGE] = sizeof(b200_vec4u) * px;
  bytes[B200_CK_FWD_PROJECTION] = fwd ? sizeof(b200_vec4f) * px : 0;
  bytes[B200_CK_FWD_MISSING] = fwd ? sizeof(int32_t) * px : 0;
  bytes[B200_CK_QUEUE_COUNTS] = sizeof(int32_t) * (uint64_t)h->noSnapshots;
  bytes[B200_CK_QUEUE_ITEMS] = sizeof(b200_vec3i) * (uint64_t)h->noQueueItems;
  bytes[B200_CK_BLOCK_IDS] = sizeof(uint32_t) * (uint64_t)h->noBlocks;
  bytes[B200_CK_BLOCK_DATA] = sizeof(b200_voxel) * 512 * (uint64_t)h->noBlocks;
  uint64_t at = B200_CHECKPOINT_HEADER_BYTES;
  for (int i = 0; i < B200_CK_SECTIONS; ++i) {
    const uint64_t align = i == B200_CK_BLOCK_DATA ? 4096 : 16;
    if (at % align) at += align - at % align;
    h->section[i][0] = at;
    h->section[i][1] = bytes[i];
    at += bytes[i];
  }
  h->totalBytes = at;
  return at;
}

/* *size = the checkpoint's size; with out != NULL and capacity >= *size the checkpoint is written. Returns a b200_status. */
int oracle_checkpoint_save(const oracle_engine *e, const b200_scene *s, const b200_render_state *rs, void *out, size_t capacity,
                           size_t *size) {
  const int noTotal = s->numBuckets + s->excessSize;
  const size_t px = (size_t)rs->img_w * rs->img_h;
  b200_checkpoint_header h;
  memset(&h, 0, sizeof(h));
  memcpy(h.magic, B200_CHECKPOINT_MAGIC, 8);
  h.version = B200_CHECKPOINT_VERSION;
  h.flags = (s->d_swapStates ? B200_CK_HAS_SWAP_STATES : 0u) | (has_forward(rs) ? B200_CK_HAS_FORWARD : 0u);
  h.numBlocks = s->numBlocks; h.numBuckets = s->numBuckets; h.excessSize = s->excessSize; h.img_w = rs->img_w; h.img_h = rs->img_h;
  h.voxelSize = s->voxelSize; h.mu = s->mu; h.maxW = s->maxW; h.viewFrustum_min = s->viewFrustum_min; h.viewFrustum_max = s->viewFrustum_max;
  h.stopIntegratingAtMaxW = s->stopIntegratingAtMaxW; h.useSwapping = s->useSwapping;
  h.lastFreeBlockId = s->lastFreeBlockId; h.lastFreeExcessListId = s->lastFreeExcessListId;
  h.noVisibleBlocks = rs->noVisibleBlocks; h.noFwdProjMissingPoints = has_forward(rs) ? rs->noFwdProjMissingPoints : 0;
  h.frameIdx = e->frameIdx; h.noSnapshots = e->q_size; h.totalDecayed = e->totalDecayed; h.droppedSnapshots = 0;
  for (int i = 0; i < noTotal; ++i) { h.noEntries += !entry_is_reset(&s->d_hash[i]); h.noVisBytes += rs->d_entriesVisibleType[i] != 0; }
  for (int b = 0; b < s->numBlocks; ++b) h.noBlocks += !block_is_reset(s->d_voxels + (size_t)b * 512);
  for (const snap *q = e->q_head; q; q = q->next) h.noQueueItems += q->count > 0 ? q->count : 0;
  const uint64_t total = place_sections(&h);
  *size = (size_t)total;
  if (!out) return B200_OK;
  if (capacity < total) return B200_ERR_INVALID;
  uint8_t *o = (uint8_t *)out;
  memset(o, 0, (size_t)total);
  memcpy(o, &h, sizeof(h));
#define SEC(i) (o + h.section[i][0])
  {
    uint32_t *idx = (uint32_t *)SEC(B200_CK_HASH_INDEX); uint8_t *ent = SEC(B200_CK_HASH_ENTRIES); size_t k = 0;
    for (int i = 0; i < noTotal; ++i)
      if (!entry_is_reset(&s->d_hash[i])) { uint32_t v = (uint32_t)i; memcpy(idx + k, &v, 4); memcpy(ent + 20 * k, &s->d_hash[i], 20); ++k; }
  }
  memcpy(SEC(B200_CK_ALLOCATION_LIST), s->d_allocationList, 4 * (size_t)s->numBlocks);
  memcpy(SEC(B200_CK_EXCESS_LIST), s->d_excessList, 4 * (size_t)s->excessSize);
  if (s->d_swapStates) memcpy(SEC(B200_CK_SWAP_STATES), s->d_swapStates, (size_t)noTotal);
  {
    uint8_t *idx = SEC(B200_CK_VIS_INDEX), *val = SEC(B200_CK_VIS_VALUE); size_t k = 0;
    for (int i = 0; i < noTotal; ++i)
      if (rs->d_entriesVisibleType[i]) { uint32_t v = (uint32_t)i; memcpy(idx + 4 * k, &v, 4); val[k] = rs->d_entriesVisibleType[i]; ++k; }
  }
  memcpy(SEC(B200_CK_VISIBLE_LIST), rs->d_visibleBlockPositions, (size_t)h.section[B200_CK_VISIBLE_LIST][1]);
  memcpy(SEC(B200_CK_MINMAX), rs->d_minmax, 8 * px);
  memcpy(SEC(B200_CK_RAYCAST_RESULT), rs->d_raycastResult, 16 * px);
  memcpy(SEC(B200_CK_RAYCAST_IMAGE), rs->d_raycastImage, 4 * px);
  if (has_forward(rs)) { memcpy(SEC(B200_CK_FWD_PROJECTION), rs->d_forwardProjection, 16 * px); memcpy(SEC(B200_CK_FWD_MISSING), rs->d_fwdProjMissingPoints, 4 * px); }
  {
    uint8_t *cnt = SEC(B200_CK_QUEUE_COUNTS), *items = SEC(B200_CK_QUEUE_ITEMS); size_t j = 0, k = 0;
    for (const snap *q = e->q_head; q; q = q->next, ++j) {
      int32_t c = q->count; memcpy(cnt + 4 * j, &c, 4);
      if (c > 0) { memcpy(items + 12 * k, q->items, 12 * (size_t)c); k += (size_t)c; }
    }
  }
  {
    uint8_t *ids = SEC(B200_CK_BLOCK_IDS), *data = SEC(B200_CK_BLOCK_DATA); size_t k = 0;
    for (int b = 0; b < s->numBlocks; ++b) {
      const b200_voxel *v = s->d_voxels + (size_t)b * 512;
      if (block_is_reset(v)) continue;
      uint32_t id = (uint32_t)b; memcpy(ids + 4 * k, &id, 4); memcpy(data + 4096 * k, v, 4096); ++k;
    }
  }
#undef SEC
  return B200_OK;
}

/* the load's rejections, all decided before anything is written (same rules as checkpoint.cu's ck_validate) */
static int check(const b200_scene *s, const b200_render_state *rs, const uint8_t *p, size_t size, b200_checkpoint_header *h) {
  if (!p || size < sizeof(*h)) return 1;
  memcpy(h, p, sizeof(*h));
  if (memcmp(h->magic, B200_CHECKPOINT_MAGIC, 8) != 0) return 2;
  if (h->version != B200_CHECKPOINT_VERSION) return 3;
  if (h->numBlocks != s->numBlocks || h->numBuckets != s->numBuckets || h->excessSize != s->excessSize || h->img_w != rs->img_w ||
      h->img_h != rs->img_h) return 4;
  if (memcmp(&h->voxelSize, &s->voxelSize, 4) != 0 || memcmp(&h->mu, &s->mu, 4) != 0) return 5;
  if (h->flags & ~(B200_CK_HAS_SWAP_STATES | B200_CK_HAS_FORWARD)) return 6;
  if (((h->flags & B200_CK_HAS_SWAP_STATES) != 0) != (s->d_swapStates != NULL)) return 7;
  if (((h->flags & B200_CK_HAS_FORWARD) != 0) != (has_forward(rs) != 0)) return 8;
  const long long noTotal = (long long)s->numBuckets + s->excessSize, px = (long long)rs->img_w * rs->img_h;
  if (h->noEntries < 0 || h->noEntries > noTotal || h->noVisBytes < 0 || h->noVisBytes > noTotal || h->noBlocks < 0 ||
      h->noBlocks > s->numBlocks || h->noSnapshots < 0 || h->noQueueItems < 0 || h->noQueueItems > (long long)h->noSnapshots * s->numBlocks ||
      h->noVisibleBlocks < 0 || h->noVisibleBlocks > s->numBlocks || h->noFwdProjMissingPoints < 0 || h->noFwdProjMissingPoints > px || h->lastFreeBlockId < -1 ||
      h->lastFreeBlockId >= s->numBlocks || h->lastFreeExcessListId < -1 || h->lastFreeExcessListId >= s->excessSize ||
      h->totalDecayed < 0 || h->droppedSnapshots < 0) return 9;
  b200_checkpoint_header t = *h;
  place_sections(&t);
  if (memcmp(t.section, h->section, sizeof(t.section)) != 0 || t.totalBytes != h->totalBytes) return 10;
  if (size != h->totalBytes) return 11;
  const int secs[3] = {B200_CK_HASH_INDEX, B200_CK_VIS_INDEX, B200_CK_BLOCK_IDS};
  const long long ns[3] = {h->noEntries, h->noVisBytes, h->noBlocks}, bounds[3] = {noTotal, noTotal, s->numBlocks};
  for (int l = 0; l < 3; ++l) {
    long long prev = -1;
    for (long long i = 0; i < ns[l]; ++i) {
      uint32_t v; memcpy(&v, p + h->section[secs[l]][0] + 4 * i, 4);
      if ((long long)v <= prev || (long long)v >= bounds[l]) return 12;
      prev = v;
    }
  }
  long long items = 0;
  for (int j = 0; j < h->noSnapshots; ++j) {
    int32_t n; memcpy(&n, p + h->section[B200_CK_QUEUE_COUNTS][0] + 4 * (size_t)j, 4);
    if (n < -1 || n > s->numBlocks) return 13;
    items += n > 0 ? n : 0;
  }
  if (items != h->noQueueItems) return 14;
  return 0;
}

/* Returns B200_OK, or B200_ERR_INVALID with nothing written (*why, when not NULL, receives which check refused it). */
int oracle_checkpoint_load(oracle_engine *e, b200_scene *s, b200_render_state *rs, const void *in, size_t size, int *why) {
  b200_checkpoint_header h;
  const uint8_t *p = (const uint8_t *)in;
  const int r = check(s, rs, p, size, &h);
  if (why) *why = r;
  if (r) return B200_ERR_INVALID;
  const int noTotal = s->numBuckets + s->excessSize;
  const size_t px = (size_t)rs->img_w * rs->img_h;
#define SEC(i) (p + h.section[i][0])
  /* ResetScene's values first (tsdf_oracle.c oracle_reset_scene), then every listed block, entry and byte */
  b200_voxel rv; memset(&rv, 0, sizeof(rv)); rv.sdf = 32767;
  for (size_t i = 0; i < (size_t)s->numBlocks * 512; ++i) s->d_voxels[i] = rv;
  b200_hash_entry rh; memset(&rh, 0, sizeof(rh)); rh.ptr = -2;
  for (int i = 0; i < noTotal; ++i) s->d_hash[i] = rh;
  memset(rs->d_entriesVisibleType, 0, (size_t)noTotal);
  for (long long k = 0; k < h.noEntries; ++k) {
    uint32_t i; memcpy(&i, SEC(B200_CK_HASH_INDEX) + 4 * k, 4);
    memcpy(&s->d_hash[i], SEC(B200_CK_HASH_ENTRIES) + 20 * k, 20);
  }
  memcpy(s->d_allocationList, SEC(B200_CK_ALLOCATION_LIST), 4 * (size_t)s->numBlocks);
  memcpy(s->d_excessList, SEC(B200_CK_EXCESS_LIST), 4 * (size_t)s->excessSize);
  if (s->d_swapStates) memcpy(s->d_swapStates, SEC(B200_CK_SWAP_STATES), (size_t)noTotal);
  for (long long k = 0; k < h.noVisBytes; ++k) {
    uint32_t i; memcpy(&i, SEC(B200_CK_VIS_INDEX) + 4 * k, 4);
    rs->d_entriesVisibleType[i] = SEC(B200_CK_VIS_VALUE)[k];
  }
  memcpy(rs->d_visibleBlockPositions, SEC(B200_CK_VISIBLE_LIST), (size_t)h.section[B200_CK_VISIBLE_LIST][1]);
  memcpy(rs->d_minmax, SEC(B200_CK_MINMAX), 8 * px);
  memcpy(rs->d_raycastResult, SEC(B200_CK_RAYCAST_RESULT), 16 * px);
  memcpy(rs->d_raycastImage, SEC(B200_CK_RAYCAST_IMAGE), 4 * px);
  if (has_forward(rs)) { memcpy(rs->d_forwardProjection, SEC(B200_CK_FWD_PROJECTION), 16 * px); memcpy(rs->d_fwdProjMissingPoints, SEC(B200_CK_FWD_MISSING), 4 * px); }
  for (long long k = 0; k < h.noBlocks; ++k) {
    uint32_t id; memcpy(&id, SEC(B200_CK_BLOCK_IDS) + 4 * k, 4);
    memcpy(s->d_voxels + (size_t)id * 512, SEC(B200_CK_BLOCK_DATA) + 4096 * k, 4096);
  }
  /* the queue, oldest first */
  while (e->q_head) { snap *q = e->q_head; e->q_head = q->next; free(q->items); free(q); }
  e->q_tail = NULL; e->q_size = 0;
  const uint8_t *items = SEC(B200_CK_QUEUE_ITEMS);
  for (int j = 0; j < h.noSnapshots; ++j) {
    snap *q = (snap *)calloc(1, sizeof(snap));
    memcpy(&q->count, SEC(B200_CK_QUEUE_COUNTS) + 4 * (size_t)j, 4);
    q->frameIdx = h.frameIdx;
    if (q->count > 0) {
      q->items = (b200_vec3i *)malloc(12 * (size_t)q->count);
      memcpy(q->items, items, 12 * (size_t)q->count);
      items += 12 * (size_t)q->count;
    }
    if (e->q_tail) e->q_tail->next = q; else e->q_head = q;
    e->q_tail = q; e->q_size++;
  }
#undef SEC
  e->frameIdx = h.frameIdx;
  e->totalDecayed = (long)h.totalDecayed;
  s->lastFreeBlockId = h.lastFreeBlockId; s->lastFreeExcessListId = h.lastFreeExcessListId;
  rs->noVisibleBlocks = h.noVisibleBlocks; rs->noFwdProjMissingPoints = h.noFwdProjMissingPoints;
  return B200_OK;
}
