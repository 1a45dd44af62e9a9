/*
 * tsdf_oracle.c — TEST INFRASTRUCTURE ONLY. Serial CPU restatement of the reference's
 * voxel-hash allocate -> integrate -> visible-list -> decay -> expected-depth -> raycast ->
 * shading path (AndreiBarsan/DynSLAM, InfiniTAM fork). Nothing under dynslam_b200/ may
 * import, link or call this file; only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs use it, and only as the checker / CPU baseline.
 *
 * Pinning: the reference ships no golden vectors for this path (SURVEY.md 4, 8c). This
 * restatement is pinned against the reference's own DeviceAgnostic per-element functions
 * compiled from /root/reference into oracle/_ref (see oracle/build_ref.sh,
 * tests/test_oracle_vs_ref.py) and against golden vectors generated from that build
 * (tests/golden/).
 *
 * Reference paths below are relative to src/InfiniTAM/InfiniTAM/ITMLib/:
 *   DA/  = Engine/DeviceAgnostic/            CUDA/ = Engine/DeviceSpecific/CUDA/
 *   CPU/ = Engine/DeviceSpecific/CPU/        OR/   = ../ORUtils/
 *
 * Canonical ordering (what makes "bit-exact" well defined; the reference CUDA build is
 * nondeterministic, SURVEY.md finding 4): pixels in raster order, later writer wins a bucket
 * request; requests served in ascending entry index; VBA slot = allocationList[lastFree--];
 * visible list in ascending entry index; decay processes list items in order and pushes freed
 * slots in that order. Floating point: IEEE-754 binary32, no contraction (build with
 * -ffp-contract=off), expression order exactly as written in the reference sources.
 */
#include "../include/b200fusion.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define BS 8
#define BS3 512

/* OR/MathUtils.h:5-23 (macros restated as functions with identical comparison direction) */
static inline float minf_(float a, float b) { return (a < b) ? a : b; }
static inline float maxf_(float a, float b) { return (a < b) ? b : a; }
static inline int mini_(int a, int b) { return (a < b) ? a : b; }
static inline float round_(float x) { return (x < 0) ? (x - 0.5f) : (x + 0.5f); }
static inline int clampi_(int x, int a, int b) { /* CLAMP(x,a,b) = MAX(a, MIN(b, x)) */
  int t = (b < x) ? b : x;
  return (a < t) ? t : a;
}

/* OR/Matrix.h:115-122  Matrix4 * Vector4, m[col*4+row] */
static inline void m4v4(const float *m, const float v[4], float r[4]) {
  r[0] = m[0] * v[0] + m[4] * v[1] + m[8] * v[2] + m[12] * v[3];
  r[1] = m[1] * v[0] + m[5] * v[1] + m[9] * v[2] + m[13] * v[3];
  r[2] = m[2] * v[0] + m[6] * v[1] + m[10] * v[2] + m[14] * v[3];
  r[3] = m[3] * v[0] + m[7] * v[1] + m[11] * v[2] + m[15] * v[3];
}

/* OR/Matrix.h:162-224 */
int oracle_mat4_inv(const float *m, float *dst) {
  float tmp[12], src[16], det;
  for (int i = 0; i < 4; i++) {
    src[i] = m[i * 4]; src[i + 4] = m[i * 4 + 1]; src[i + 8] = m[i * 4 + 2]; src[i + 12] = m[i * 4 + 3];
  }
  tmp[0] = src[10] * src[15]; tmp[1] = src[11] * src[14]; tmp[2] = src[9] * src[15];
  tmp[3] = src[11] * src[13]; tmp[4] = src[9] * src[14]; tmp[5] = src[10] * src[13];
  tmp[6] = src[8] * src[15]; tmp[7] = src[11] * src[12]; tmp[8] = src[8] * src[14];
  tmp[9] = src[10] * src[12]; tmp[10] = src[8] * src[13]; tmp[11] = src[9] * src[12];
  dst[0] = (tmp[0] * src[5] + tmp[3] * src[6] + tmp[4] * src[7]) - (tmp[1] * src[5] + tmp[2] * src[6] + tmp[5] * src[7]);
  dst[1] = (tmp[1] * src[4] + tmp[6] * src[6] + tmp[9] * src[7]) - (tmp[0] * src[4] + tmp[7] * src[6] + tmp[8] * src[7]);
  dst[2] = (tmp[2] * src[4] + tmp[7] * src[5] + tmp[10] * src[7]) - (tmp[3] * src[4] + tmp[6] * src[5] + tmp[11] * src[7]);
  dst[3] = (tmp[5] * src[4] + tmp[8] * src[5] + tmp[11] * src[6]) - (tmp[4] * src[4] + tmp[9] * src[5] + tmp[10] * src[6]);
  det = src[0] * dst[0] + src[1] * dst[1] + src[2] * dst[2] + src[3] * dst[3];
  if (det == 0.0f) return 0;
  dst[4] = (tmp[1] * src[1] + tmp[2] * src[2] + tmp[5] * src[3]) - (tmp[0] * src[1] + tmp[3] * src[2] + tmp[4] * src[3]);
  dst[5] = (tmp[0] * src[0] + tmp[7] * src[2] + tmp[8] * src[3]) - (tmp[1] * src[0] + tmp[6] * src[2] + tmp[9] * src[3]);
  dst[6] = (tmp[3] * src[0] + tmp[6] * src[1] + tmp[11] * src[3]) - (tmp[2] * src[0] + tmp[7] * src[1] + tmp[10] * src[3]);
  dst[7] = (tmp[4] * src[0] + tmp[9] * src[1] + tmp[10] * src[2]) - (tmp[5] * src[0] + tmp[8] * src[1] + tmp[11] * src[2]);
  tmp[0] = src[2] * src[7]; tmp[1] = src[3] * src[6]; tmp[2] = src[1] * src[7];
  tmp[3] = src[3] * src[5]; tmp[4] = src[1] * src[6]; tmp[5] = src[2] * src[5];
  tmp[6] = src[0] * src[7]; tmp[7] = src[3] * src[4]; tmp[8] = src[0] * src[6];
  tmp[9] = src[2] * src[4]; tmp[10] = src[0] * src[5]; tmp[11] = src[1] * src[4];
  dst[8] = (tmp[0] * src[13] + tmp[3] * src[14] + tmp[4] * src[15]) - (tmp[1] * src[13] + tmp[2] * src[14] + tmp[5] * src[15]);
  dst[9] = (tmp[1] * src[12] + tmp[6] * src[14] + tmp[9] * src[15]) - (tmp[0] * src[12] + tmp[7] * src[14] + tmp[8] * src[15]);
  dst[10] = (tmp[2] * src[12] + tmp[7] * src[13] + tmp[10] * src[15]) - (tmp[3] * src[12] + tmp[6] * src[13] + tmp[11] * src[15]);
  dst[11] = (tmp[5] * src[12] + tmp[8] * src[13] + tmp[11] * src[14]) - (tmp[4] * src[12] + tmp[9] * src[13] + tmp[10] * src[14]);
  dst[12] = (tmp[2] * src[10] + tmp[5] * src[11] + tmp[1] * src[9]) - (tmp[4] * src[11] + tmp[0] * src[9] + tmp[3] * src[10]);
  dst[13] = (tmp[8] * src[11] + tmp[0] * src[8] + tmp[7] * src[10]) - (tmp[6] * src[10] + tmp[9] * src[11] + tmp[1] * src[8]);
  dst[14] = (tmp[6] * src[9] + tmp[11] * src[11] + tmp[3] * src[8]) - (tmp[10] * src[11] + tmp[2] * src[8] + tmp[7] * src[9]);
  dst[15] = (tmp[10] * src[10] + tmp[4] * src[8] + tmp[9] * src[9]) - (tmp[8] * src[9] + tmp[11] * src[10] + tmp[5] * src[8]);
  float s = 1 / det;
  for (int i = 0; i < 16; ++i) dst[i] *= s;
  return 1;
}

/* OR/Matrix.h:102-108  r(x,y) += lhs(k,y) * rhs(x,k); (x = column, y = row) */
void oracle_mat4_mul(const float *lhs, const float *rhs, float *out) {
  float r[16];
  for (int i = 0; i < 16; ++i) r[i] = 0.0f;
  for (int x = 0; x < 4; x++) for (int y = 0; y < 4; y++) for (int k = 0; k < 4; k++)
    r[x * 4 + y] += lhs[k * 4 + y] * rhs[x * 4 + k];
  memcpy(out, r, sizeof(r));
}

/* DA/ITMRepresentationAccess.h:10-12 */
static inline int hash_index(int x, int y, int z, int mask) {
  return (int)((((unsigned)x * 73856093u) ^ ((unsigned)y * 19349669u) ^ ((unsigned)z * 83492791u)) & (unsigned)mask);
}

static inline int pos_eq(const b200_hash_entry *e, int x, int y, int z) {
  return e->pos[0] == x && e->pos[1] == y && e->pos[2] == z;
}

/* DA/ITMRepresentationAccess.h:62-85 findBlock; returns -1 when absent */
static int find_block(const b200_hash_entry *table, int numBuckets, int x, int y, int z) {
  int idx = hash_index(x, y, z, numBuckets - 1);
  for (;;) {
    const b200_hash_entry *e = &table[idx];
    if (pos_eq(e, x, y, z) && e->ptr >= 0) return idx;
    if (e->offset < 1) break;
    idx = numBuckets + e->offset - 1;
  }
  return -1;
}

/* DA/ITMRepresentationAccess.h:94-150 findVoxel(blockGridCoords,...): entry + predecessor */
static int find_block_prev(const b200_hash_entry *table, int numBuckets, int x, int y, int z, int *prev) {
  int idx = hash_index(x, y, z, numBuckets - 1);
  *prev = -1;
  for (;;) {
    const b200_hash_entry *e = &table[idx];
    if (pos_eq(e, x, y, z) && e->ptr >= 0) return idx;
    if (e->offset < 1) break;
    *prev = idx;
    idx = numBuckets + e->offset - 1;
  }
  return -1;
}

/* ------------------------------------------------------------------------------------------- */
/* engine state (CUDA/ITMSceneReconstructionEngine_CUDA.h:31-45)                                 */
/* ------------------------------------------------------------------------------------------- */

typedef struct snap { int count; int frameIdx; b200_vec3i *items; struct snap *next; } snap;

typedef struct oracle_engine {
  int noTotalEntries;
  uint8_t *allocType;
  int16_t *blockCoords; /* Vector4s per entry */
  int frameIdx;
  long totalDecayed;
  snap *q_head, *q_tail; int q_size;
  int16_t *allocatedBlockPositions; int allocatedCap;
  int noIntegratedBlocks;
} oracle_engine;

oracle_engine *oracle_engine_create(int numBlocks, int numBuckets, int excessSize) {
  oracle_engine *e = (oracle_engine *)calloc(1, sizeof(*e));
  e->noTotalEntries = numBuckets + excessSize;
  e->allocType = (uint8_t *)calloc(e->noTotalEntries, 1);
  e->blockCoords = (int16_t *)calloc((size_t)e->noTotalEntries * 4, sizeof(int16_t));
  e->allocatedBlockPositions = (int16_t *)calloc((size_t)numBlocks * 4, sizeof(int16_t));
  e->allocatedCap = numBlocks;
  return e;
}

static void queue_clear(oracle_engine *e) {
  while (e->q_head) { snap *s = e->q_head; e->q_head = s->next; free(s->items); free(s); }
  e->q_tail = NULL; e->q_size = 0;
}

void oracle_engine_destroy(oracle_engine *e) {
  if (!e) return;
  queue_clear(e);
  free(e->allocType); free(e->blockCoords); free(e->allocatedBlockPositions); free(e);
}

/* frameVisibleBlocks.push({count, frameIdx, copy of the positions}) — CUDA/..._CUDA.cu:302-316. Allocation pushes its
   visible list here; tests push a snapshot of their own to seed the decay queue. */
void oracle_push_snapshot(oracle_engine *e, const b200_vec3i *positions, int n) {
  snap *sn = (snap *)calloc(1, sizeof(snap));
  sn->count = n; sn->frameIdx = e->frameIdx;
  if (n > 0) {
    sn->items = (b200_vec3i *)malloc(sizeof(b200_vec3i) * (size_t)n);
    memcpy(sn->items, positions, sizeof(b200_vec3i) * (size_t)n);
  }
  if (e->q_tail) e->q_tail->next = sn; else e->q_head = sn;
  e->q_tail = sn; e->q_size++;
}

/* the front (oldest) snapshot: copies up to cap positions to out, returns its count, or -1 when the queue is empty */
int oracle_peek_snapshot(const oracle_engine *e, b200_vec3i *out, int cap) {
  if (!e->q_head) return -1;
  const int n = e->q_head->count;
  if (out && n > 0) memcpy(out, e->q_head->items, sizeof(b200_vec3i) * (size_t)(n < cap ? n : cap));
  return n;
}

void oracle_set_frame_index(oracle_engine *e, int f) { e->frameIdx = f; }
int oracle_frame_index(const oracle_engine *e) { return e->frameIdx; }
long oracle_decayed_block_count(const oracle_engine *e) { return e->totalDecayed; }
int oracle_queue_size(const oracle_engine *e) { return e->q_size; }
int oracle_integrated_blocks(const oracle_engine *e) { return e->noIntegratedBlocks; }

/* ------------------------------------------------------------------------------------------- */
/* ResetScene — CUDA/ITMSceneReconstructionEngine_CUDA.cu:145-172 (CPU twin CPU/..._CPU.cpp:25-45) */
/* ------------------------------------------------------------------------------------------- */
void oracle_reset_scene(oracle_engine *e, b200_scene *s) {
  e->totalDecayed = 0;
  queue_clear(e);
  size_t nvox = (size_t)s->numBlocks * BS3;
  b200_voxel v; memset(&v, 0, sizeof(v)); v.sdf = 32767;
  for (size_t i = 0; i < nvox; ++i) s->d_voxels[i] = v;
  for (int i = 0; i < s->numBlocks; ++i) s->d_allocationList[i] = i;
  s->lastFreeBlockId = s->numBlocks - 1;
  b200_hash_entry h; memset(&h, 0, sizeof(h)); h.ptr = -2;
  int n = s->numBuckets + s->excessSize;
  for (int i = 0; i < n; ++i) s->d_hash[i] = h;
  for (int i = 0; i < s->excessSize; ++i) s->d_excessList[i] = i;
  s->lastFreeExcessListId = s->excessSize - 1;
}

/* ------------------------------------------------------------------------------------------- */
/* buildHashAllocAndVisibleTypePP — DA/ITMSceneReconstructionEngine.h:176-313 (lock branches are */
/* __CUDA_ARCH__-only and drop out of the serial restatement)                                    */
/* ------------------------------------------------------------------------------------------- */
static void mark_pixel(uint8_t *allocType, uint8_t *visType, int x, int y, int16_t *blockCoords,
                       const float *depth, const float *invM, const float invProj[4], float mu,
                       int w, float oneOverVoxelSize, const b200_hash_entry *table, int numBuckets,
                       float vfmin, float vfmax) {
  float d = depth[x + y * w];
  if (d <= 0 || (d - mu) < 0 || (d - mu) < vfmin || (d + mu) > vfmax) return;

  float pz = d;
  float px = pz * (((float)x - invProj[2]) * invProj[0]);
  float py = pz * (((float)y - invProj[3]) * invProj[1]);
  float norm = sqrtf(px * px + py * py + pz * pz);

  float t[4], r[4], point[3], point_e[3], dir[3];
  t[0] = px * (1.0f - mu / norm); t[1] = py * (1.0f - mu / norm); t[2] = pz * (1.0f - mu / norm); t[3] = 1.0f;
  m4v4(invM, t, r);
  point[0] = r[0] * oneOverVoxelSize; point[1] = r[1] * oneOverVoxelSize; point[2] = r[2] * oneOverVoxelSize;
  t[0] = px * (1.0f + mu / norm); t[1] = py * (1.0f + mu / norm); t[2] = pz * (1.0f + mu / norm);
  m4v4(invM, t, r);
  point_e[0] = r[0] * oneOverVoxelSize; point_e[1] = r[1] * oneOverVoxelSize; point_e[2] = r[2] * oneOverVoxelSize;

  dir[0] = point_e[0] - point[0]; dir[1] = point_e[1] - point[1]; dir[2] = point_e[2] - point[2];
  norm = sqrtf(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]);
  int noSteps = (int)ceilf(2.0f * norm);
  float den = (float)(noSteps - 1);
  dir[0] /= den; dir[1] /= den; dir[2] /= den;

  for (int i = 0; i < noSteps; i++) {
    int bx = (short)(int)floorf(point[0]), by = (short)(int)floorf(point[1]), bz = (short)(int)floorf(point[2]);
    int hashIdx = hash_index(bx, by, bz, numBuckets - 1);
    int isFound = 0;
    b200_hash_entry he = table[hashIdx];
    if (pos_eq(&he, bx, by, bz) && he.ptr >= -1) {
      visType[hashIdx] = (he.ptr == -1) ? 2 : 1;
      isFound = 1;
    }
    if (!isFound) {
      int isExcess = 0;
      if (he.ptr >= -1) {
        while (he.offset >= 1) {
          hashIdx = numBuckets + he.offset - 1;
          he = table[hashIdx];
          if (pos_eq(&he, bx, by, bz) && he.ptr >= -1) {
            visType[hashIdx] = (he.ptr == -1) ? 2 : 1;
            isFound = 1;
            break;
          }
        }
        isExcess = 1;
      }
      if (!isFound) {
        allocType[hashIdx] = isExcess ? 2 : 1;
        if (!isExcess) visType[hashIdx] = 1;
        blockCoords[hashIdx * 4 + 0] = (int16_t)bx; blockCoords[hashIdx * 4 + 1] = (int16_t)by;
        blockCoords[hashIdx * 4 + 2] = (int16_t)bz; blockCoords[hashIdx * 4 + 3] = 1;
      }
    }
    point[0] += dir[0]; point[1] += dir[1]; point[2] += dir[2];
  }
}

/* checkPointVisibility<false> / checkBlockVisibility<false> — DA/ITMSceneReconstructionEngine.h:315-397 */
static int point_visible(const float p[4], const float *M, const float proj[4], int w, int h) {
  float b[4];
  m4v4(M, p, b);
  if (b[2] < 1e-10f) return 0;
  b[0] = proj[0] * b[0] / b[2] + proj[2];
  b[1] = proj[1] * b[1] / b[2] + proj[3];
  return (b[0] >= 0 && b[0] < w && b[1] >= 0 && b[1] < h);
}

static int block_visible(const int16_t pos[3], const float *M, const float proj[4], float voxelSize, int w, int h) {
  float p[4];
  float factor = (float)BS * voxelSize;
  p[0] = (float)pos[0] * factor; p[1] = (float)pos[1] * factor; p[2] = (float)pos[2] * factor; p[3] = 1.0f;
  if (point_visible(p, M, proj, w, h)) return 1;           /* 0 0 0 */
  p[2] += factor; if (point_visible(p, M, proj, w, h)) return 1; /* 0 0 1 */
  p[1] += factor; if (point_visible(p, M, proj, w, h)) return 1; /* 0 1 1 */
  p[0] += factor; if (point_visible(p, M, proj, w, h)) return 1; /* 1 1 1 */
  p[2] -= factor; if (point_visible(p, M, proj, w, h)) return 1; /* 1 1 0 */
  p[1] -= factor; if (point_visible(p, M, proj, w, h)) return 1; /* 1 0 0 */
  p[0] -= factor; p[1] += factor; if (point_visible(p, M, proj, w, h)) return 1; /* 0 1 0 */
  p[0] += factor; p[1] -= factor; p[2] += factor; if (point_visible(p, M, proj, w, h)) return 1; /* 1 0 1 */
  return 0;
}

/* ------------------------------------------------------------------------------------------- */
/* AllocateSceneFromDepth — CUDA/..._CUDA.cu:175-358 sequencing, serial bodies from the          */
/* commented CPU engine CPU/..._CPU.cpp:143-298 brought up to the CUDA semantics                  */
/* (allocatedTime :843/:868, position list :984, setToType3 by lookup :776-810, queue :302-317). */
/* Swapping is not restated in the allocate path (ITMLibSettings.cpp:50-55 forbids it).          */
/* Returns 0, 2 (VBA exhausted) or 3 (excess list exhausted) — after mutating state, as the      */
/* reference does (:348-357).                                                                    */
/* ------------------------------------------------------------------------------------------- */
int oracle_allocate_from_depth(oracle_engine *e, b200_scene *s, b200_render_state *rs,
                               const b200_view *v, int onlyUpdateVisibleList, int ompMark) {
  const int w = v->depth_w, h = v->depth_h;
  const int nb = s->numBuckets, noTotal = nb + s->excessSize;
  b200_hash_entry *table = s->d_hash;
  uint8_t *visType = rs->d_entriesVisibleType;
  float invProj[4] = {1.0f / v->proj_d[0], 1.0f / v->proj_d[1], v->proj_d[2], v->proj_d[3]};
  float oneOverVoxelSize = 1.0f / (s->voxelSize * BS);

  int lastFreeVoxelBlockId = s->lastFreeBlockId;
  int lastFreeExcessListId = s->lastFreeExcessListId;
  int noVisible = 0;

  memset(e->allocType, 0, noTotal);

  /* setToType3 — :776-810 */
  for (int i = 0; i < rs->noVisibleBlocks; i++) {
    b200_vec3i p = rs->d_visibleBlockPositions[i];
    int idx = find_block(table, nb, p.x, p.y, p.z);
    if (idx >= 0) visType[idx] = 3;
  }

  /* per-pixel marking; raster order is the canonical order (ompMark is for timing runs only:
     it enables the reference's own pragma site CPU/..._CPU.cpp:166-168 and makes the winner racy) */
  (void)ompMark;
#ifdef _OPENMP
  if (ompMark) {
#pragma omp parallel for schedule(static)
    for (int locId = 0; locId < w * h; locId++) {
      int y = locId / w, x = locId - y * w;
      mark_pixel(e->allocType, visType, x, y, e->blockCoords, v->d_depth, v->invM_d, invProj, s->mu, w,
                 oneOverVoxelSize, table, nb, s->viewFrustum_min, s->viewFrustum_max);
    }
  } else
#endif
  for (int locId = 0; locId < w * h; locId++) {
    int y = locId / w, x = locId - y * w;
    mark_pixel(e->allocType, visType, x, y, e->blockCoords, v->d_depth, v->invM_d, invProj, s->mu, w,
               oneOverVoxelSize, table, nb, s->viewFrustum_min, s->viewFrustum_max);
  }

  if (!onlyUpdateVisibleList) {
    /* allocateVoxelBlocksList — :812-905 in ascending targetIdx (CPU/..._CPU.cpp:186-233) */
    for (int targetIdx = 0; targetIdx < noTotal; targetIdx++) {
      int vbaIdx, exlIdx;
      switch (e->allocType[targetIdx]) {
      case 1:
        vbaIdx = lastFreeVoxelBlockId; lastFreeVoxelBlockId--;
        if (vbaIdx >= 0) {
          b200_hash_entry he; memset(&he, 0, sizeof(he));
          he.pos[0] = e->blockCoords[targetIdx * 4]; he.pos[1] = e->blockCoords[targetIdx * 4 + 1];
          he.pos[2] = e->blockCoords[targetIdx * 4 + 2];
          he.ptr = s->d_allocationList[vbaIdx]; he.offset = 0; he.allocatedTime = e->frameIdx;
          table[targetIdx] = he;
        }
        break;
      case 2:
        vbaIdx = lastFreeVoxelBlockId; lastFreeVoxelBlockId--;
        exlIdx = lastFreeExcessListId; lastFreeExcessListId--;
        if (vbaIdx >= 0 && exlIdx >= 0) {
          b200_hash_entry he; memset(&he, 0, sizeof(he));
          he.pos[0] = e->blockCoords[targetIdx * 4]; he.pos[1] = e->blockCoords[targetIdx * 4 + 1];
          he.pos[2] = e->blockCoords[targetIdx * 4 + 2];
          he.ptr = s->d_allocationList[vbaIdx]; he.offset = 0; he.allocatedTime = e->frameIdx;
          int exlOffset = s->d_excessList[exlIdx];
          table[targetIdx].offset = exlOffset + 1;
          table[nb + exlOffset] = he;
          visType[nb + exlOffset] = 1;
        }
        break;
      default: break;
      }
    }
  }

  /* buildVisibleList<false> — :924-999, ascending entry index (CPU/..._CPU.cpp:236-276) */
  for (int targetIdx = 0; targetIdx < noTotal; targetIdx++) {
    uint8_t t = visType[targetIdx];
    const b200_hash_entry *he = &table[targetIdx];
    if (t == 3) {
      if (!block_visible(he->pos, v->M_d, v->proj_d, s->voxelSize, w, h)) t = 0;
      visType[targetIdx] = t;
    }
    if (t > 0) {
      b200_vec3i p = {he->pos[0], he->pos[1], he->pos[2]};
      if (noVisible < s->numBlocks) rs->d_visibleBlockPositions[noVisible] = p;
      noVisible++;
    }
  }

  rs->noVisibleBlocks = noVisible;
  s->lastFreeBlockId = lastFreeVoxelBlockId;
  s->lastFreeExcessListId = lastFreeExcessListId;

  /* decay queue snapshot + frameIdx++ — :302-317 */
  oracle_push_snapshot(e, rs->d_visibleBlockPositions, noVisible);
  e->frameIdx++;

  if (s->lastFreeBlockId < 0) return B200_ERR_VBA_FULL;
  if (s->lastFreeExcessListId < 0) return B200_ERR_EXCESS_FULL;
  return B200_OK;
}

/* ------------------------------------------------------------------------------------------- */
/* computeUpdatedVoxelDepthInfo — DA/ITMSceneReconstructionEngine.h:14-88                          */
/* ------------------------------------------------------------------------------------------- */
static inline float sdf_to_float(int16_t x) { return (float)(x) / 32767.0f; }   /* ITMLibDefines.h:141 */
static inline int16_t float_to_sdf(float x) { return (int16_t)((x) * 32767.0f); } /* :142 */

static float update_depth(b200_voxel *vox, const float pt_model[4], const float *M_d, const float *proj,
                          float mu, int maxW, const float *depth, int w, int h, int depthWeighting) {
  float pc[4];
  m4v4(M_d, pt_model, pc);
  if (pc[2] <= 0) return -1;
  float ix = proj[0] * pc[0] / pc[2] + proj[2];
  float iy = proj[1] * pc[1] / pc[2] + proj[3];
  if ((ix < 1) || (ix > w - 2) || (iy < 1) || (iy > h - 2)) return -1;
  float dm = depth[(int)(ix + 0.5f) + (int)(iy + 0.5f) * w];
  if (dm <= 0.0) return -1;
  float eta = dm - pc[2];
  if (eta < -mu) return eta;
  float oldF = sdf_to_float(vox->sdf);
  int oldW = vox->w_depth;
  float newF = minf_(1.0f, eta / mu);
  int newW;
  if (depthWeighting) {
    int maxNewW = 10;
    newW = (int)(100.0 / dm);
    if (newW < 1) newW = 1;
    if (newW > maxNewW) newW = maxNewW;
  } else newW = 1;
  newF = oldW * oldF + newW * newF;
  newW = oldW + newW;
  newF /= newW;
  newW = mini_(newW, maxW);
  vox->sdf = float_to_sdf(newF);
  vox->w_depth = (uint8_t)newW;
  return eta;
}

/* interpolateBilinear<Vector4u> — DA/ITMPixelUtils.h:11-39 (xyz only are consumed) */
static void bilinear_rgb(const b200_vec4u *src, float px, float py, int w, float out[3]) {
  int ix = (int)floorf(px), iy = (int)floorf(py);
  float dx = px - (float)ix, dy = py - (float)iy;
  b200_vec4u a, b = {0, 0, 0, 0}, c = {0, 0, 0, 0}, d = {0, 0, 0, 0};
  a = src[ix + iy * w];
  if (dx != 0) b = src[(ix + 1) + iy * w];
  if (dy != 0) c = src[ix + (iy + 1) * w];
  if (dx != 0 && dy != 0) d = src[(ix + 1) + (iy + 1) * w];
  out[0] = ((float)a.x * (1.0f - dx) * (1.0f - dy) + (float)b.x * dx * (1.0f - dy) + (float)c.x * (1.0f - dx) * dy + (float)d.x * dx * dy);
  out[1] = ((float)a.y * (1.0f - dx) * (1.0f - dy) + (float)b.y * dx * (1.0f - dy) + (float)c.y * (1.0f - dx) * dy + (float)d.y * dx * dy);
  out[2] = ((float)a.z * (1.0f - dx) * (1.0f - dy) + (float)b.z * dx * (1.0f - dy) + (float)c.z * (1.0f - dx) * dy + (float)d.z * dx * dy);
}

static inline uint8_t to_uchar_round(float x) { /* Vector3::toUChar, OR/Vector.h:246-248 */
  return (uint8_t)clampi_((int)round_(x), 0, 255);
}

/* computeUpdatedVoxelColorInfo — DA/ITMSceneReconstructionEngine.h:91-128 */
static void update_color(b200_voxel *vox, const float pt_model[4], const float *M_rgb, const float *proj,
                         uint8_t maxW, const b200_vec4u *rgb, int w, int h) {
  float pc[4];
  float oldW = (float)vox->w_color;
  float oldC[3] = {(float)vox->clr[0] / 255.0f, (float)vox->clr[1] / 255.0f, (float)vox->clr[2] / 255.0f};
  m4v4(M_rgb, pt_model, pc);
  float ix = proj[0] * pc[0] / pc[2] + proj[2];
  float iy = proj[1] * pc[1] / pc[2] + proj[3];
  if ((ix < 1) || (ix > w - 2) || (iy < 1) || (iy > h - 2)) return;
  float m[3];
  bilinear_rgb(rgb, ix, iy, w, m);
  m[0] = m[0] / 255.0f; m[1] = m[1] / 255.0f; m[2] = m[2] / 255.0f;
  float newW = 5;
  float newC[3];
  newC[0] = oldC[0] * oldW + m[0] * newW; newC[1] = oldC[1] * oldW + m[1] * newW; newC[2] = oldC[2] * oldW + m[2] * newW;
  newW = oldW + newW;
  newC[0] /= newW; newC[1] /= newW; newC[2] /= newW;
  newW = (newW < maxW) ? newW : maxW;
  vox->clr[0] = to_uchar_round(newC[0] * 255.0f);
  vox->clr[1] = to_uchar_round(newC[1] * 255.0f);
  vox->clr[2] = to_uchar_round(newC[2] * 255.0f);
  vox->w_color = (uint8_t)newW;
}

/* ------------------------------------------------------------------------------------------- */
/* IntegrateIntoScene — CUDA/..._CUDA.cu:361-427, kernel :692-750 (serial body CPU/..._CPU.cpp:73-115 */
/* updated to look blocks up by position and to pass WeightParams)                              */
/* ------------------------------------------------------------------------------------------- */
void oracle_integrate(oracle_engine *e, b200_scene *s, const b200_render_state *rs, const b200_view *v, int omp) {
  e->noIntegratedBlocks = 0;
  if (rs->noVisibleBlocks == 0) return;
  const int stopMaxW = s->stopIntegratingAtMaxW;
  const int approx = !v->requiresFullRendering;
  const float voxelSize = s->voxelSize, mu = s->mu; const int maxW = s->maxW;
  int integrated = 0;
  (void)omp;
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 64) reduction(+ : integrated) if (omp)
#endif
  for (int i = 0; i < rs->noVisibleBlocks; i++) {
    b200_vec3i p = rs->d_visibleBlockPositions[i];
    int entryId = find_block(s->d_hash, s->numBuckets, p.x, p.y, p.z);
    if (entryId < 0) continue;
    const b200_hash_entry *he = &s->d_hash[entryId];
    int gx = he->pos[0] * BS, gy = he->pos[1] * BS, gz = he->pos[2] * BS;
    b200_voxel *blk = &s->d_voxels[(size_t)he->ptr * BS3];
    integrated++;
    for (int z = 0; z < BS; z++) for (int y = 0; y < BS; y++) for (int x = 0; x < BS; x++) {
      int locId = x + y * BS + z * BS * BS;
      if (stopMaxW) if (blk[locId].w_depth == maxW) continue;
      if (approx) if (blk[locId].w_depth != 0) continue;
      float pt[4];
      pt[0] = (float)(gx + x) * voxelSize; pt[1] = (float)(gy + y) * voxelSize; pt[2] = (float)(gz + z) * voxelSize; pt[3] = 1.0f;
      /* ComputeUpdatedVoxelInfo<true,...> — DA/...:147-171 */
      float eta = update_depth(&blk[locId], pt, v->M_d, v->proj_d, mu, maxW, v->d_depth, v->depth_w, v->depth_h, v->depthWeighting);
      if ((eta > mu) || (fabsf(eta / mu) > 0.25f)) continue;
      update_color(&blk[locId], pt, v->M_rgb, v->proj_rgb, (uint8_t)maxW, v->d_rgb, v->rgb_w, v->rgb_h);
    }
  }
  e->noIntegratedBlocks = integrated;
}

/* ------------------------------------------------------------------------------------------- */
/* Decay — CUDA/..._CUDA.cu:509-560; decayVoxel :1120-1197; deleteBlock :1012-1115 (serial: the     */
/* bucket lock never contends). Blocks in list order (partial) / ascending VBA id (full).        */
/* ------------------------------------------------------------------------------------------- */
/* How often each decay branch ran since the last oracle_decay_branches() call: tests use it to check that the branch they
   target really ran. */
enum { DB_AGE_SKIP, DB_VOXEL_RESET, DB_HEAD_WITH_SUCCESSOR, DB_HEAD_ALONE, DB_EXCESS_ENTRY, DB_COUNT };
static long g_decay_branch[DB_COUNT];

/* copies the counters {blocks left alone because age < minAge, voxels reset, deleted bucket heads with a successor, deleted
   bucket heads without one, deleted excess-list entries} to out and clears them */
void oracle_decay_branches(long *out) {
  memcpy(out, g_decay_branch, sizeof(g_decay_branch));
  memset(g_decay_branch, 0, sizeof(g_decay_branch));
}

static void delete_block(b200_scene *s, uint8_t *visType, int x, int y, int z, int *lastFree) {
  b200_hash_entry *table = s->d_hash; const int nb = s->numBuckets;
  int prev;
  int idx = find_block_prev(table, nb, x, y, z, &prev);
  if (idx < 0) return; /* cannot happen in the serial order; the reference would index -1 here */
  int freeListIdx = (*lastFree)++;
  s->d_allocationList[freeListIdx + 1] = table[idx].ptr;
  g_decay_branch[prev != -1 ? DB_EXCESS_ENTRY : (table[idx].offset >= 1 ? DB_HEAD_WITH_SUCCESSOR : DB_HEAD_ALONE)]++;
  if (prev == -1) {
    if (table[idx].offset >= 1) {
      int nextIdx = nb + table[idx].offset - 1;
      table[idx] = table[nextIdx];
      visType[idx] = visType[nextIdx];
      visType[nextIdx] = 0;
      table[nextIdx].offset = 0;
      table[nextIdx].ptr = -2;
    } else {
      table[idx].ptr = -2;
      visType[idx] = 0;
    }
  } else {
    table[prev].offset = table[idx].offset;
    table[idx].offset = 0;
    table[idx].ptr = -2;
    visType[prev] = visType[idx];
    visType[idx] = 0;
  }
}

static void decay_block(b200_scene *s, uint8_t *visType, int x, int y, int z, int minAge, int maxWeight,
                        int currentFrame, int *lastFree) {
  int prev;
  int idx = find_block_prev(s->d_hash, s->numBuckets, x, y, z, &prev);
  if (idx < 0) return;
  int age = currentFrame - s->d_hash[idx].allocatedTime;
  if (age < minAge) { g_decay_branch[DB_AGE_SKIP]++; return; } /* safeToClear == false: nothing touched, never deleted (:1151-1157, :1189) */
  b200_voxel *blk = &s->d_voxels[(size_t)s->d_hash[idx].ptr * BS3];
  int empty = 0;
  for (int i = 0; i < BS3; ++i) {
    int isNoisy = (blk[i].w_depth <= maxWeight);
    if (isNoisy && blk[i].w_depth > 0) {
      blk[i].sdf = 32767; blk[i].w_depth = 0; blk[i].clr[0] = blk[i].clr[1] = blk[i].clr[2] = 0; blk[i].w_color = 0;
      g_decay_branch[DB_VOXEL_RESET]++;
    }
    if (blk[i].w_depth == 0) empty++;
  }
  if (empty == BS3) delete_block(s, visType, x, y, z, lastFree);
}

int oracle_decay(oracle_engine *e, b200_scene *s, b200_render_state *rs, int maxWeight, int minAge, int forceAll) {
  int oldLastFree = s->lastFreeBlockId;
  int lastFree = s->lastFreeBlockId;
  uint8_t *visType = rs->d_entriesVisibleType;
  if (forceAll) {
    /* FullDecay :430-475 + findAllocatedBlocks CUDA/ITMMeshingEngine_CUDA.cu:96-114 */
    int noTotal = s->numBuckets + s->excessSize;
    memset(e->allocatedBlockPositions, 0, sizeof(int16_t) * 4 * (size_t)s->numBlocks);
    for (int i = 0; i < noTotal; ++i) {
      const b200_hash_entry *he = &s->d_hash[i];
      if (he->ptr >= 0) {
        int16_t *p = &e->allocatedBlockPositions[(size_t)he->ptr * 4];
        p[0] = he->pos[0]; p[1] = he->pos[1]; p[2] = he->pos[2]; p[3] = 1;
      }
    }
    for (int b = 0; b < s->numBlocks; ++b) {
      const int16_t *p = &e->allocatedBlockPositions[(size_t)b * 4];
      if (p[3] == 0) continue;
      decay_block(s, visType, p[0], p[1], p[2], minAge, maxWeight, e->frameIdx, &lastFree);
    }
  } else if ((long)e->q_size > minAge) {
    snap *sn = e->q_head;
    e->q_head = sn->next; if (!e->q_head) e->q_tail = NULL; e->q_size--;
    for (int i = 0; i < sn->count; ++i) {
      b200_vec3i p = sn->items[i];
      int idx = find_block(s->d_hash, s->numBuckets, p.x, p.y, p.z); /* decay_device :1214-1221 */
      if (idx < 0) continue;
      const b200_hash_entry *he = &s->d_hash[idx];
      decay_block(s, visType, he->pos[0], he->pos[1], he->pos[2], minAge, maxWeight, e->frameIdx, &lastFree);
    }
    free(sn->items); free(sn);
  }
  s->lastFreeBlockId = lastFree;
  int freed = lastFree - oldLastFree;
  e->totalDecayed += freed;
  return freed;
}

/* ------------------------------------------------------------------------------------------- */
/* FindVisibleBlocks — CUDA/ITMVisualisationEngine_CUDA.cu:151-180, kernel :536-569               */
/* (serial: CPU/ITMVisualisationEngine_CPU.cpp:43-78 updated to positions)                       */
/* ------------------------------------------------------------------------------------------- */
void oracle_find_visible_blocks(const b200_scene *s, b200_render_state *rs, const b200_camera *cam) {
  int noTotal = s->numBuckets + s->excessSize, n = 0;
  for (int i = 0; i < noTotal; ++i) {
    const b200_hash_entry *he = &s->d_hash[i];
    if (he->ptr < 0) continue;
    if (block_visible(he->pos, cam->M, cam->proj, s->voxelSize, rs->img_w, rs->img_h)) {
      b200_vec3i p = {he->pos[0], he->pos[1], he->pos[2]};
      if (n < s->numBlocks) rs->d_visibleBlockPositions[n] = p;
      n++;
    }
  }
  rs->noVisibleBlocks = n;
}

/* ProjectSingleBlock — DA/ITMVisualisationEngine.h:29-71 */
static int project_single_block(const int16_t pos[3], const float *pose, const float *intr, int w, int h,
                                float voxelSize, int ul[2], int lr[2], float zr[2]) {
  ul[0] = w / B200_MINMAX_SUBSAMPLE; ul[1] = h / B200_MINMAX_SUBSAMPLE;
  lr[0] = -1; lr[1] = -1;
  zr[0] = B200_FAR_AWAY; zr[1] = B200_VERY_CLOSE;
  for (int corner = 0; corner < 8; ++corner) {
    int16_t t[3] = {pos[0], pos[1], pos[2]};
    t[0] += (corner & 1) ? 1 : 0; t[1] += (corner & 2) ? 1 : 0; t[2] += (corner & 4) ? 1 : 0;
    float p[4] = {(float)t[0] * (float)BS * voxelSize, (float)t[1] * (float)BS * voxelSize, (float)t[2] * (float)BS * voxelSize, 1.0f};
    float q[4];
    m4v4(pose, p, q);
    if (q[2] < 1e-6) continue;
    float px = (intr[0] * q[0] / q[2] + intr[2]) / B200_MINMAX_SUBSAMPLE;
    float py = (intr[1] * q[1] / q[2] + intr[3]) / B200_MINMAX_SUBSAMPLE;
    if (ul[0] > floorf(px)) ul[0] = (int)floorf(px);
    if (lr[0] < ceilf(px)) lr[0] = (int)ceilf(px);
    if (ul[1] > floorf(py)) ul[1] = (int)floorf(py);
    if (lr[1] < ceilf(py)) lr[1] = (int)ceilf(py);
    if (zr[0] > q[2]) zr[0] = q[2];
    if (zr[1] < q[2]) zr[1] = q[2];
  }
  if (ul[0] < 0) ul[0] = 0;
  if (ul[1] < 0) ul[1] = 0;
  if (lr[0] >= w) lr[0] = w - 1;
  if (lr[1] >= h) lr[1] = h - 1;
  if (ul[0] > lr[0]) return 0;
  if (ul[1] > lr[1]) return 0;
  if (zr[0] < B200_VERY_CLOSE) zr[0] = B200_VERY_CLOSE;
  if (zr[1] < B200_VERY_CLOSE) return 0;
  return 1;
}

/* ------------------------------------------------------------------------------------------- */
/* CreateExpectedDepths — CUDA/ITMVisualisationEngine_CUDA.cu:194-240; projectAndSplitBlocks :572-612; */
/* fillBlocks :614-637. Tile offsets are the list-order prefix; a block whose tiles would cross  */
/* MAX_RENDERING_BLOCKS is dropped (:609). The reference then rasterises whatever stale tiles    */
/* sit in the dropped range; the canonical result treats them as absent (documented deviation,   */
/* only reachable with > 262144 tiles).                                                          */
/* ------------------------------------------------------------------------------------------- */
/* MAX_RENDERING_BLOCKS (DA/ITMVisualisationEngine.h:25); a test hook lowers it so that the overflow rule (Vis_CUDA.cu:609)
 * can be exercised with a few hundred blocks */
static int g_max_rendering_blocks = B200_MAX_RENDERING_BLOCKS;
void oracle_set_max_rendering_blocks(int n) { g_max_rendering_blocks = n > 0 ? n : B200_MAX_RENDERING_BLOCKS; }

void oracle_expected_depths(const b200_scene *s, b200_render_state *rs, const b200_camera *cam) {
  const int w = rs->img_w, h = rs->img_h;
  for (int i = 0; i < w * h; ++i) { rs->d_minmax[i].x = B200_FAR_AWAY; rs->d_minmax[i].y = B200_VERY_CLOSE; }
  unsigned offset = 0;
  for (int i = 0; i < rs->noVisibleBlocks; ++i) {
    b200_vec3i p = rs->d_visibleBlockPositions[i];
    int idx = find_block(s->d_hash, s->numBuckets, p.x, p.y, p.z);
    if (idx < 0) continue;
    int ul[2], lr[2]; float zr[2];
    if (!project_single_block(s->d_hash[idx].pos, cam->M, cam->proj, w, h, s->voxelSize, ul, lr, zr)) continue;
    int rx = (int)ceilf((float)(lr[0] - ul[0] + 1) / 16), ry = (int)ceilf((float)(lr[1] - ul[1] + 1) / 16);
    unsigned required = (unsigned)(rx * ry);
    unsigned out_offset = offset;
    offset += required;
    if (required == 0) continue;
    if (out_offset + required > (unsigned)g_max_rendering_blocks) continue;
    for (int y = ul[1]; y <= lr[1]; ++y) for (int x = ul[0]; x <= lr[0]; ++x) {
      b200_vec2f *px = &rs->d_minmax[x + y * w];
      if (zr[0] < px->x) px->x = zr[0];
      if (zr[1] > px->y) px->y = zr[1];
    }
  }
}

/* ------------------------------------------------------------------------------------------- */
/* readVoxel with IndexCache — DA/ITMRepresentationAccess.h:176-220; cache ITMVoxelBlockHash.h:27-31 */
/* ------------------------------------------------------------------------------------------- */
typedef struct { int bx, by, bz, blockPtr; } idx_cache;
static inline void cache_init(idx_cache *c) { c->bx = c->by = c->bz = 0x7fffffff; c->blockPtr = -1; }

static inline int floordiv8(int p) { return ((p < 0) ? p - BS + 1 : p) / BS; } /* pointToVoxelBlockPos :14-22 */

static const b200_voxel *read_voxel(const b200_scene *s, int px, int py, int pz, int *isFound, idx_cache *c) {
  int bx = floordiv8(px), by = floordiv8(py), bz = floordiv8(pz);
  int linearIdx = px + (py - bx) * BS + (pz - by) * BS * BS - bz * BS3;
  if (bx == c->bx && by == c->by && bz == c->bz) { *isFound = 1; return &s->d_voxels[c->blockPtr + linearIdx]; }
  int hashIdx = hash_index(bx, by, bz, s->numBuckets - 1);
  for (;;) {
    const b200_hash_entry *he = &s->d_hash[hashIdx];
    if (pos_eq(he, bx, by, bz) && he->ptr >= 0) {
      *isFound = 1;
      c->bx = bx; c->by = by; c->bz = bz; c->blockPtr = he->ptr * BS3;
      return &s->d_voxels[c->blockPtr + linearIdx];
    }
    if (he->offset < 1) break;
    hashIdx = s->numBuckets + he->offset - 1;
  }
  *isFound = 0;
  return NULL; /* TVoxel(): sdf 32767, all else 0 */
}

static inline float rv_sdf(const b200_scene *s, int x, int y, int z, int *f, idx_cache *c) {
  const b200_voxel *v = read_voxel(s, x, y, z, f, c);
  return v ? (float)v->sdf : 32767.0f;
}

/* readFromSDF_float_uninterpolated — DA/ITMRepresentationAccess.h:245-250 */
static float sdf_uninterp(const b200_scene *s, const float p[3], int *found, idx_cache *c) {
  const b200_voxel *v = read_voxel(s, (int)round_(p[0]), (int)round_(p[1]), (int)round_(p[2]), found, c);
  return sdf_to_float(v ? v->sdf : 32767);
}

/* readFromSDF_float_interpolated — :252-278 */
static float sdf_interp(const b200_scene *s, const float p[3], int *found, idx_cache *c) {
  float res1, res2, v1, v2;
  float fx = floorf(p[0]), fy = floorf(p[1]), fz = floorf(p[2]);
  float cx = p[0] - fx, cy = p[1] - fy, cz = p[2] - fz;
  int x = (int)fx, y = (int)fy, z = (int)fz;
  v1 = rv_sdf(s, x, y, z, found, c); v2 = rv_sdf(s, x + 1, y, z, found, c);
  res1 = (1.0f - cx) * v1 + cx * v2;
  v1 = rv_sdf(s, x, y + 1, z, found, c); v2 = rv_sdf(s, x + 1, y + 1, z, found, c);
  res1 = (1.0f - cy) * res1 + cy * ((1.0f - cx) * v1 + cx * v2);
  v1 = rv_sdf(s, x, y, z + 1, found, c); v2 = rv_sdf(s, x + 1, y, z + 1, found, c);
  res2 = (1.0f - cx) * v1 + cx * v2;
  v1 = rv_sdf(s, x, y + 1, z + 1, found, c); v2 = rv_sdf(s, x + 1, y + 1, z + 1, found, c);
  res2 = (1.0f - cy) * res2 + cy * ((1.0f - cx) * v1 + cx * v2);
  *found = 1;
  return ((1.0f - cz) * res1 + cz * res2) / 32767.0f; /* SDF_valueToFloat(float) */
}

/* castRay — DA/ITMVisualisationEngine.h:93-179 */
static int cast_ray(b200_vec4f *out, int x, int y, const b200_scene *s, const float *invM, const float invProj[4],
                    float oneOverVoxelSize, float mu, b200_vec2f minmax) {
  float pc[4], r[4], ps[3], pe[3], dir[3], pt[3];
  int hash_found; float sdfValue = 1.0f;
  float totalLength, stepLength, totalLengthMax, stepScale;
  stepScale = mu * oneOverVoxelSize * 1.0f;

  pc[2] = minmax.x;
  pc[0] = pc[2] * (((float)x - invProj[2]) * invProj[0]);
  pc[1] = pc[2] * (((float)y - invProj[3]) * invProj[1]);
  pc[3] = 1.0f;
  totalLength = sqrtf(pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2]) * oneOverVoxelSize;
  m4v4(invM, pc, r);
  ps[0] = r[0] * oneOverVoxelSize; ps[1] = r[1] * oneOverVoxelSize; ps[2] = r[2] * oneOverVoxelSize;

  pc[2] = minmax.y;
  pc[0] = pc[2] * (((float)x - invProj[2]) * invProj[0]);
  pc[1] = pc[2] * (((float)y - invProj[3]) * invProj[1]);
  pc[3] = 1.0f;
  totalLengthMax = sqrtf(pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2]) * oneOverVoxelSize;
  m4v4(invM, pc, r);
  pe[0] = r[0] * oneOverVoxelSize; pe[1] = r[1] * oneOverVoxelSize; pe[2] = r[2] * oneOverVoxelSize;

  dir[0] = pe[0] - ps[0]; dir[1] = pe[1] - ps[1]; dir[2] = pe[2] - ps[2];
  float direction_norm = 1.0f / sqrtf(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]);
  dir[0] *= direction_norm; dir[1] *= direction_norm; dir[2] *= direction_norm;

  pt[0] = ps[0]; pt[1] = ps[1]; pt[2] = ps[2];
  idx_cache cache; cache_init(&cache);

  while (totalLength < totalLengthMax) {
    sdfValue = sdf_uninterp(s, pt, &hash_found, &cache);
    if (!hash_found) {
      stepLength = BS;
    } else {
      float maxSdf = 20.0; float minSdf = -100.0f;
      if ((sdfValue <= maxSdf) && (sdfValue >= minSdf)) sdfValue = sdf_interp(s, pt, &hash_found, &cache);
      if (sdfValue <= 0.0f) break;
      stepLength = maxf_(sdfValue * stepScale, 1.0f);
    }
    pt[0] += stepLength * dir[0]; pt[1] += stepLength * dir[1]; pt[2] += stepLength * dir[2];
    totalLength += stepLength;
  }

  int pt_found;
  if (sdfValue <= 0.0f) {
    stepLength = sdfValue * stepScale;
    pt[0] += stepLength * dir[0]; pt[1] += stepLength * dir[1]; pt[2] += stepLength * dir[2];
    sdfValue = sdf_interp(s, pt, &hash_found, &cache);
    stepLength = sdfValue * stepScale;
    pt[0] += stepLength * dir[0]; pt[1] += stepLength * dir[1]; pt[2] += stepLength * dir[2];
    pt_found = 1;
  } else pt_found = 0;

  out->x = pt[0]; out->y = pt[1]; out->z = pt[2];
  out->w = pt_found ? 1.0f : 0.0f;
  return pt_found;
}

/* GenericRaycast — CUDA/ITMVisualisationEngine_CUDA.cu:242-265, kernel :672-684 */
void oracle_raycast(const b200_scene *s, b200_render_state *rs, const float *invM, const float *proj, int omp) {
  const int w = rs->img_w, h = rs->img_h;
  float oneOverVoxelSize = 1.0f / s->voxelSize;
  float invProj[4] = {1.0f / proj[0], 1.0f / proj[1], proj[2], proj[3]};
  (void)omp;
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 4) if (omp)
#endif
  for (int y = 0; y < h; ++y) for (int x = 0; x < w; ++x) {
    int locId = x + y * w;
    int locId2 = (int)floorf((float)x / B200_MINMAX_SUBSAMPLE) + (int)floorf((float)y / B200_MINMAX_SUBSAMPLE) * w;
    cast_ray(&rs->d_raycastResult[locId], x, y, s, invM, invProj, oneOverVoxelSize, s->mu, rs->d_minmax[locId2]);
  }
}

/* computeSingleNormalFromSDF — DA/ITMRepresentationAccess.h:336-449 (fresh cache per read: the
   4-argument readVoxel overload, :222-228) */
static inline float rvs(const b200_scene *s, int x, int y, int z) {
  idx_cache c; cache_init(&c); int f;
  return rv_sdf(s, x, y, z, &f, &c);
}

static void normal_from_sdf(const b200_scene *s, const float p[3], float ret[3]) {
  float fx = floorf(p[0]), fy = floorf(p[1]), fz = floorf(p[2]);
  float cx = p[0] - fx, cy = p[1] - fy, cz = p[2] - fz;
  int X = (int)fx, Y = (int)fy, Z = (int)fz;
  float nx = 1.0f - cx, ny = 1.0f - cy, nz = 1.0f - cz;
  float fr[4], bk[4], t[4], p1, p2, v1;
  fr[0] = rvs(s, X, Y, Z); fr[1] = rvs(s, X + 1, Y, Z); fr[2] = rvs(s, X, Y + 1, Z); fr[3] = rvs(s, X + 1, Y + 1, Z);
  bk[0] = rvs(s, X, Y, Z + 1); bk[1] = rvs(s, X + 1, Y, Z + 1); bk[2] = rvs(s, X, Y + 1, Z + 1); bk[3] = rvs(s, X + 1, Y + 1, Z + 1);
  /* gradient x */
  p1 = fr[0] * ny * nz + fr[2] * cy * nz + bk[0] * ny * cz + bk[2] * cy * cz;
  t[0] = rvs(s, X - 1, Y, Z); t[1] = rvs(s, X - 1, Y + 1, Z); t[2] = rvs(s, X - 1, Y, Z + 1); t[3] = rvs(s, X - 1, Y + 1, Z + 1);
  p2 = t[0] * ny * nz + t[1] * cy * nz + t[2] * ny * cz + t[3] * cy * cz;
  v1 = p1 * cx + p2 * nx;
  p1 = fr[1] * ny * nz + fr[3] * cy * nz + bk[1] * ny * cz + bk[3] * cy * cz;
  t[0] = rvs(s, X + 2, Y, Z); t[1] = rvs(s, X + 2, Y + 1, Z); t[2] = rvs(s, X + 2, Y, Z + 1); t[3] = rvs(s, X + 2, Y + 1, Z + 1);
  p2 = t[0] * ny * nz + t[1] * cy * nz + t[2] * ny * cz + t[3] * cy * cz;
  ret[0] = (p1 * nx + p2 * cx - v1) / 32767.0f;
  /* gradient y */
  p1 = fr[0] * nx * nz + fr[1] * cx * nz + bk[0] * nx * cz + bk[1] * cx * cz;
  t[0] = rvs(s, X, Y - 1, Z); t[1] = rvs(s, X + 1, Y - 1, Z); t[2] = rvs(s, X, Y - 1, Z + 1); t[3] = rvs(s, X + 1, Y - 1, Z + 1);
  p2 = t[0] * nx * nz + t[1] * cx * nz + t[2] * nx * cz + t[3] * cx * cz;
  v1 = p1 * cy + p2 * ny;
  p1 = fr[2] * nx * nz + fr[3] * cx * nz + bk[2] * nx * cz + bk[3] * cx * cz;
  t[0] = rvs(s, X, Y + 2, Z); t[1] = rvs(s, X + 1, Y + 2, Z); t[2] = rvs(s, X, Y + 2, Z + 1); t[3] = rvs(s, X + 1, Y + 2, Z + 1);
  p2 = t[0] * nx * nz + t[1] * cx * nz + t[2] * nx * cz + t[3] * cx * cz;
  ret[1] = (p1 * ny + p2 * cy - v1) / 32767.0f;
  /* gradient z */
  p1 = fr[0] * nx * ny + fr[1] * cx * ny + fr[2] * nx * cy + fr[3] * cx * cy;
  t[0] = rvs(s, X, Y, Z - 1); t[1] = rvs(s, X + 1, Y, Z - 1); t[2] = rvs(s, X, Y + 1, Z - 1); t[3] = rvs(s, X + 1, Y + 1, Z - 1);
  p2 = t[0] * nx * ny + t[1] * cx * ny + t[2] * nx * cy + t[3] * cx * cy;
  v1 = p1 * cz + p2 * nz;
  p1 = bk[0] * nx * ny + bk[1] * cx * ny + bk[2] * nx * cy + bk[3] * cx * cy;
  t[0] = rvs(s, X, Y, Z + 2); t[1] = rvs(s, X + 1, Y, Z + 2); t[2] = rvs(s, X, Y + 1, Z + 2); t[3] = rvs(s, X + 1, Y + 1, Z + 2);
  p2 = t[0] * nx * ny + t[1] * cx * ny + t[2] * nx * cy + t[3] * cx * cy;
  ret[2] = (p1 * nz + p2 * cz - v1) / 32767.0f;
}

/* computeNormalAndAngle<TVoxel,TIndex> — DA/ITMVisualisationEngine.h:196-210 */
static void normal_and_angle_sdf(int *found, const float p[3], const b200_scene *s, const float light[3], float n[3], float *angle) {
  if (!*found) return;
  normal_from_sdf(s, p, n);
  float normScale = 1.0f / sqrtf(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
  n[0] *= normScale; n[1] *= normScale; n[2] *= normScale;
  *angle = n[0] * light[0] + n[1] * light[1] + n[2] * light[2];
  if (!(*angle > 0.0)) *found = 0;
}

/* readFromSDF_color4u_interpolated_noalpha — DA/ITMRepresentationAccess.h:280-318 */
static void color_interp(const b200_scene *s, const float p[3], float ret[3]) {
  idx_cache c; cache_init(&c); int f;
  float fx = floorf(p[0]), fy = floorf(p[1]), fz = floorf(p[2]);
  float cx = p[0] - fx, cy = p[1] - fy, cz = p[2] - fz;
  int X = (int)fx, Y = (int)fy, Z = (int)fz;
  ret[0] = ret[1] = ret[2] = 0.0f;
  static const int off[8][3] = {{0, 0, 0}, {1, 0, 0}, {0, 1, 0}, {1, 1, 0}, {0, 0, 1}, {1, 0, 1}, {0, 1, 1}, {1, 1, 1}};
  for (int k = 0; k < 8; ++k) {
    const b200_voxel *v = read_voxel(s, X + off[k][0], Y + off[k][1], Z + off[k][2], &f, &c);
    float wx = off[k][0] ? cx : (1.0f - cx), wy = off[k][1] ? cy : (1.0f - cy), wz = off[k][2] ? cz : (1.0f - cz);
    float wgt = wx * wy * wz;
    float r = v ? (float)v->clr[0] : 0.0f, g = v ? (float)v->clr[1] : 0.0f, b = v ? (float)v->clr[2] : 0.0f;
    ret[0] += wgt * r; ret[1] += wgt * g; ret[2] += wgt * b;
  }
  ret[0] = ret[0] / 255.0f; ret[1] = ret[1] / 255.0f; ret[2] = ret[2] / 255.0f;
}

static inline b200_vec4u grey_px(float angle) { /* drawPixelGrey :277-281 */
  float outRes = (0.8f * angle + 0.2f) * 255.0f;
  uint8_t g = (uint8_t)outRes;
  b200_vec4u r = {g, g, g, g};
  return r;
}

static void draw_colour(b200_vec4u *dest, const float p[3], const b200_scene *s) { /* drawPixelColour :290-300 */
  float c[3]; color_interp(s, p, c);
  dest->x = (uint8_t)(c[0] * 255.0f); dest->y = (uint8_t)(c[1] * 255.0f); dest->z = (uint8_t)(c[2] * 255.0f); dest->w = 255;
}

/* drawPixelWeight — DA/ITMVisualisationEngine.h:322-383 with WeightRenderingParams(1.0,false,maxW,2) Vis_CUDA.cu:303-311 */
static void draw_weight(b200_vec4u *dest, const float p[3], const b200_scene *s, float overlayWeight, int differentiate,
                        int maxWeight, int maxNoiseWeight) {
  draw_colour(dest, p, s);
  idx_cache c; cache_init(&c); int f = 0;
  int ix = (int)p[0], iy = (int)p[1], iz = (int)p[2];
  const b200_voxel *v = read_voxel(s, ix, iy, iz, &f, &c);
  int wd = v ? v->w_depth : 0;
  uint8_t intensity = (uint8_t)(255.0f * (((float)wd) / maxWeight));
  int bx = floordiv8(ix), by = floordiv8(iy), bz = floordiv8(iz);
  int blockIdx = find_block(s->d_hash, s->numBuckets, bx, by, bz);
  int isExcess = (blockIdx >= s->numBuckets) && differentiate;
  b200_vec4u saturated = isExcess ? (b200_vec4u){0, 0, 128, 255} : (b200_vec4u){0, 0, 255, 255};
  b200_vec4u noisy = isExcess ? (b200_vec4u){255, 255, 0, 255} : (b200_vec4u){255, 0, 0, 255};
  b200_vec4u gradual = isExcess ? (b200_vec4u){50, intensity, 255, 255} : (b200_vec4u){intensity, intensity, intensity, 255};
  b200_vec4u invalid = {255, 255, 255, 255};
  b200_vec4u ov;
  if (blockIdx < 0) ov = invalid;
  else if (wd <= maxNoiseWeight) ov = noisy;
  else if (wd == maxWeight) ov = saturated;
  else ov = gradual;
  float a = (float)(1.0 - overlayWeight);
  float fr = ((float)dest->x * a) + ((float)ov.x * overlayWeight);
  float fg = ((float)dest->y * a) + ((float)ov.y * overlayWeight);
  float fb = ((float)dest->z * a) + ((float)ov.z * overlayWeight);
  float fa = ((float)dest->w * a) + ((float)ov.w * overlayWeight);
  dest->x = (uint8_t)fr; dest->y = (uint8_t)fg; dest->z = (uint8_t)fb; dest->w = (uint8_t)fa;
}

/* RenderImage_common — CUDA/ITMVisualisationEngine_CUDA.cu:267-343 (+ kernels :735-886) */
void oracle_render_image(const b200_scene *s, b200_render_state *rs, const b200_camera *cam, b200_vec4u *outChar,
                         float *outFloat, int type, int omp) {
  const int w = rs->img_w, h = rs->img_h;
  oracle_raycast(s, rs, cam->invM, cam->proj, omp);
  float light[3] = {-cam->invM[8], -cam->invM[9], -cam->invM[10]};
  (void)omp;
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 4) if (omp)
#endif
  for (int locId = 0; locId < w * h; ++locId) {
    b200_vec4f pr = rs->d_raycastResult[locId];
    float p[3] = {pr.x, pr.y, pr.z};
    int found = pr.w > 0;
    float n[3] = {0, 0, 0}, angle = 0;
    switch (type) {
    case B200_RENDER_COLOUR_FROM_VOLUME:
      normal_and_angle_sdf(&found, p, s, light, n, &angle);
      if (found) draw_colour(&outChar[locId], p, s);
      else outChar[locId] = (b200_vec4u){0, 0, 0, 255};
      break;
    case B200_RENDER_COLOUR_FROM_NORMAL:
      normal_and_angle_sdf(&found, p, s, light, n, &angle);
      if (found) { /* drawPixelNormal :283-288 (alpha untouched) */
        outChar[locId].x = (uint8_t)((0.3f + (-n[0] + 1.0f) * 0.35f) * 255.0f);
        outChar[locId].y = (uint8_t)((0.3f + (-n[1] + 1.0f) * 0.35f) * 255.0f);
        outChar[locId].z = (uint8_t)((0.3f + (-n[2] + 1.0f) * 0.35f) * 255.0f);
      } else outChar[locId] = (b200_vec4u){0, 0, 0, 0};
      break;
    case B200_RENDER_COLOUR_FROM_DEPTH_WEIGHT:
      normal_and_angle_sdf(&found, p, s, light, n, &angle);
      if (found) draw_weight(&outChar[locId], p, s, 1.0f, 0, s->maxW, 2);
      else outChar[locId] = (b200_vec4u){0, 0, 0, 0};
      break;
    case B200_RENDER_DEPTH_MAP:
      if (found) { /* drawPixelDepth :304-320 */
        float ph[4] = {p[0] * s->voxelSize, p[1] * s->voxelSize, p[2] * s->voxelSize, 1.0f}, pc[4];
        m4v4(cam->M, ph, pc);
        outFloat[locId] = pc[2] / pc[3];
      } else outFloat[locId] = 0.0f;
      break;
    case B200_RENDER_SHADED_GREYSCALE:
    default:
      normal_and_angle_sdf(&found, p, s, light, n, &angle);
      if (found) outChar[locId] = grey_px(angle);
      else outChar[locId] = (b200_vec4u){0, 0, 0, 0};
      break;
    }
  }
}

/* computeNormalAndAngle<useSmoothing> — DA/ITMVisualisationEngine.h:212-275 */
static void normal_and_angle_img(int smoothing, int *found, int x, int y, const b200_vec4f *pr, const float light[3],
                                 float voxelSize, int w, int h, float n[3], float *angle) {
  if (!*found) return;
  b200_vec4f xp1, xm1, yp1, ym1;
  if (smoothing) {
    if (y <= 2 || y >= h - 3 || x <= 2 || x >= w - 3) { *found = 0; return; }
    xp1 = pr[(x + 2) + y * w]; yp1 = pr[x + (y + 2) * w]; xm1 = pr[(x - 2) + y * w]; ym1 = pr[x + (y - 2) * w];
  } else {
    if (y <= 1 || y >= h - 2 || x <= 1 || x >= w - 2) { *found = 0; return; }
    xp1 = pr[(x + 1) + y * w]; yp1 = pr[x + (y + 1) * w]; xm1 = pr[(x - 1) + y * w]; ym1 = pr[x + (y - 1) * w];
  }
  float dxx = 0, dxy = 0, dxz = 0, dyx = 0, dyy = 0, dyz = 0;
  int doPlus1 = 0;
  if (xp1.w <= 0 || yp1.w <= 0 || xm1.w <= 0 || ym1.w <= 0) doPlus1 = 1;
  else {
    dxx = xp1.x - xm1.x; dxy = xp1.y - xm1.y; dxz = xp1.z - xm1.z;
    dyx = yp1.x - ym1.x; dyy = yp1.y - ym1.y; dyz = yp1.z - ym1.z;
    float length_diff = maxf_(dxx * dxx + dxy * dxy + dxz * dxz, dyx * dyx + dyy * dyy + dyz * dyz);
    if (length_diff * voxelSize * voxelSize > (0.15f * 0.15f)) doPlus1 = 1;
  }
  if (doPlus1) {
    if (smoothing) {
      xp1 = pr[(x + 1) + y * w]; yp1 = pr[x + (y + 1) * w]; xm1 = pr[(x - 1) + y * w]; ym1 = pr[x + (y - 1) * w];
      dxx = xp1.x - xm1.x; dxy = xp1.y - xm1.y; dxz = xp1.z - xm1.z;
      dyx = yp1.x - ym1.x; dyy = yp1.y - ym1.y; dyz = yp1.z - ym1.z;
    }
    if (xp1.w <= 0 || yp1.w <= 0 || xm1.w <= 0 || ym1.w <= 0) { *found = 0; return; }
  }
  n[0] = -(dxy * dyz - dxz * dyy);
  n[1] = -(dxz * dyx - dxx * dyz);
  n[2] = -(dxx * dyy - dxy * dyx);
  float normScale = 1.0f / sqrtf(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
  n[0] *= normScale; n[1] *= normScale; n[2] *= normScale;
  *angle = n[0] * light[0] + n[1] * light[1] + n[2] * light[2];
  if (!(*angle > 0.0)) *found = 0;
}

/* CreateICPMaps_common — CUDA/ITMVisualisationEngine_CUDA.cu:372-390; processPixelICP<true> DA/...:418-453 */
void oracle_icp_maps(const b200_scene *s, b200_render_state *rs, const b200_view *v, b200_vec4f *points,
                     b200_vec4f *normals, int omp) {
  const int w = rs->img_w, h = rs->img_h;
  oracle_raycast(s, rs, v->invM_d, v->proj_d, omp);
  float light[3] = {-v->invM_d[8], -v->invM_d[9], -v->invM_d[10]};
  const b200_vec4f *pr = rs->d_raycastResult;
  for (int y = 0; y < h; ++y) for (int x = 0; x < w; ++x) {
    int locId = x + y * w;
    b200_vec4f point = pr[locId];
    int found = point.w > 0.0f;
    float n[3] = {0, 0, 0}, angle = 0;
    normal_and_angle_img(1, &found, x, y, pr, light, s->voxelSize, w, h, n, &angle);
    if (found) {
      rs->d_raycastImage[locId] = grey_px(angle);
      points[locId] = (b200_vec4f){point.x * s->voxelSize, point.y * s->voxelSize, point.z * s->voxelSize, 1.0f};
      normals[locId] = (b200_vec4f){n[0], n[1], n[2], 0.0f};
    } else {
      b200_vec4f o = {0.0f, 0.0f, 0.0f, -1.0f};
      points[locId] = o; normals[locId] = o;
      rs->d_raycastImage[locId] = (b200_vec4u){0, 0, 0, 0};
    }
  }
}

/* forwardProjectPixel — DA/ITMVisualisationEngine.h:181-194 */
static int forward_project_pixel(b200_vec4f px, const float *M, const float *proj, int w, int h) {
  float p[4] = {px.x, px.y, px.z, 1}, q[4];
  m4v4(M, p, q);
  float ix = proj[0] * q[0] / q[2] + proj[2];
  float iy = proj[1] * q[1] / q[2] + proj[3];
  if ((ix < 0) || (ix > w - 1) || (iy < 0) || (iy > h - 1)) return -1;
  return (int)(ix + 0.5f) + (int)(iy + 0.5f) * w;
}

/* ForwardRender_common — CUDA/ITMVisualisationEngine_CUDA.cu:393-453 (serial: CPU/ITMVisualisationEngine_CPU.cpp:298-363).
   Canonical order: raster order for the forward splat (later pixel wins) and for the missing list. */
void oracle_forward_render(const b200_scene *s, b200_render_state *rs, const b200_view *v) {
  const int w = rs->img_w, h = rs->img_h;
  float invProj[4] = {1.0f / v->proj_d[0], 1.0f / v->proj_d[1], v->proj_d[2], v->proj_d[3]};
  float light[3] = {-v->invM_d[8], -v->invM_d[9], -v->invM_d[10]};
  float oneOverVoxelSize = 1.0f / s->voxelSize;
  b200_vec4f *fwd = rs->d_forwardProjection;
  memset(fwd, 0, sizeof(b200_vec4f) * (size_t)w * h);
  for (int y = 0; y < h; ++y) for (int x = 0; x < w; ++x) {
    int locId = x + y * w;
    b200_vec4f pixel = rs->d_raycastResult[locId];
    b200_vec4f sc = {pixel.x * s->voxelSize, pixel.y * s->voxelSize, pixel.z * s->voxelSize, pixel.w * s->voxelSize};
    int locId_new = forward_project_pixel(sc, v->M_d, v->proj_d, w, h);
    if (locId_new >= 0) fwd[locId_new] = pixel;
  }
  int n = 0;
  for (int y = 0; y < h; ++y) for (int x = 0; x < w; ++x) {
    int locId = x + y * w;
    int locId2 = (int)floorf((float)x / B200_MINMAX_SUBSAMPLE) + (int)floorf((float)y / B200_MINMAX_SUBSAMPLE) * w;
    b200_vec4f fp = fwd[locId]; b200_vec2f mm = rs->d_minmax[locId2]; float depth = v->d_depth[locId];
    if ((fp.w <= 0) && ((fp.x == 0 && fp.y == 0 && fp.z == 0) || (depth > 0)) && (mm.x < mm.y))
      rs->d_fwdProjMissingPoints[n++] = locId;
  }
  rs->noFwdProjMissingPoints = n;
  for (int i = 0; i < n; ++i) {
    int locId = rs->d_fwdProjMissingPoints[i];
    int y = locId / w, x = locId - y * w;
    int locId2 = (int)floorf((float)x / B200_MINMAX_SUBSAMPLE) + (int)floorf((float)y / B200_MINMAX_SUBSAMPLE) * w;
    cast_ray(&fwd[locId], x, y, s, v->invM_d, invProj, oneOverVoxelSize, s->mu, rs->d_minmax[locId2]);
  }
  for (int y = 0; y < h; ++y) for (int x = 0; x < w; ++x) { /* processPixelForwardRender<true> :455-470 */
    int locId = x + y * w;
    int found = fwd[locId].w > 0.0f; float n3[3] = {0, 0, 0}, angle = 0;
    normal_and_angle_img(1, &found, x, y, fwd, light, s->voxelSize, w, h, n3, &angle);
    rs->d_raycastImage[locId] = found ? grey_px(angle) : (b200_vec4u){0, 0, 0, 0};
  }
}

/* CreatePointCloud_common — CUDA/ITMVisualisationEngine_CUDA.cu:346-369, kernel :820-871.
   Canonical order of the compacted cloud: raster order. invM = pose_d^-1 * calib_rgb_to_depth. */
unsigned oracle_point_cloud(const b200_scene *s, b200_render_state *rs, const b200_view *v, const float *calib,
                            int skipPoints, b200_vec4f *locations, b200_vec4f *colours) {
  const int w = rs->img_w, h = rs->img_h;
  float invM[16];
  oracle_mat4_mul(v->invM_d, calib, invM);
  oracle_raycast(s, rs, invM, v->proj_rgb, 0);
  float light[3] = {-invM[8], -invM[9], -invM[10]};
  unsigned n = 0;
  for (int y = 0; y < h; ++y) for (int x = 0; x < w; ++x) {
    int locId = x + y * w;
    b200_vec4f pr = rs->d_raycastResult[locId];
    float p[3] = {pr.x, pr.y, pr.z};
    int found = pr.w > 0; float nn[3] = {0, 0, 0}, angle = 0;
    normal_and_angle_sdf(&found, p, s, light, nn, &angle);
    rs->d_raycastImage[locId] = found ? grey_px(angle) : (b200_vec4u){0, 0, 0, 0};
    if (skipPoints && ((x % 2 == 0) || (y % 2 == 0))) found = 0;
    if (found) {
      float c[3]; color_interp(s, p, c);
      b200_vec4f tmp = {c[0], c[1], c[2], 1.0f};
      if (tmp.w > 0.0f) { tmp.x /= tmp.w; tmp.y /= tmp.w; tmp.z /= tmp.w; tmp.w = 1.0f; }
      colours[n] = tmp;
      locations[n] = (b200_vec4f){p[0] * s->voxelSize, p[1] * s->voxelSize, p[2] * s->voxelSize, 1.0f};
      n++;
    }
  }
  return n;
}

/* ------------------------------------------------------------------------------------------- */
/* Swapping — DA/ITMSwappingEngine.h:7-63; CUDA/ITMSwappingEngine_CUDA.cu:218-330                   */
/* (serial order: ascending entry index, CPU/ITMSwappingEngine_CPU.cpp)                          */
/* ------------------------------------------------------------------------------------------- */
static void combine_voxel(const b200_voxel *src, b200_voxel *dst, int maxW) {
  { /* combineVoxelDepthInformation */
    int newW = dst->w_depth, oldW = src->w_depth;
    float newF = sdf_to_float(dst->sdf), oldF = sdf_to_float(src->sdf);
    if (oldW != 0) {
      newF = oldW * oldF + newW * newF; newW = oldW + newW; newF /= newW; newW = mini_(newW, maxW);
      dst->w_depth = (uint8_t)newW; dst->sdf = float_to_sdf(newF);
    }
  }
  { /* combineVoxelColorInformation */
    int newW = dst->w_color, oldW = src->w_color;
    if (oldW != 0) {
      float nc[3], oc[3];
      for (int k = 0; k < 3; ++k) { nc[k] = (float)dst->clr[k] / 255.0f; oc[k] = (float)src->clr[k] / 255.0f; }
      for (int k = 0; k < 3; ++k) nc[k] = oc[k] * (float)oldW + nc[k] * (float)newW;
      newW = oldW + newW;
      for (int k = 0; k < 3; ++k) nc[k] /= (float)newW;
      newW = mini_(newW, maxW);
      for (int k = 0; k < 3; ++k) dst->clr[k] = to_uchar_round(nc[k] * 255.0f);
      dst->w_color = (uint8_t)newW;
    }
  }
}

/* buildListToSwapIn :218-232 */
int oracle_swap_list_in(const b200_scene *s, int32_t *neededEntryIDs) {
  int n = 0, noTotal = s->numBuckets + s->excessSize;
  for (int i = 0; i < noTotal; ++i)
    if (s->d_swapStates[i] == 1) { if (n < B200_TRANSFER_BLOCK_NUM) neededEntryIDs[n] = i; n++; }
  return n < B200_TRANSFER_BLOCK_NUM ? n : B200_TRANSFER_BLOCK_NUM;
}

/* integrateOldIntoActiveData :262-281 */
void oracle_swap_integrate_in(b200_scene *s, const b200_voxel *synced, const int32_t *neededEntryIDs, int noNeeded) {
  for (int i = 0; i < noNeeded; ++i) {
    int entryDestId = neededEntryIDs[i];
    const b200_voxel *src = synced + (size_t)i * BS3;
    b200_voxel *dst = s->d_voxels + (size_t)s->d_hash[entryDestId].ptr * BS3;
    for (int v = 0; v < BS3; ++v) combine_voxel(&src[v], &dst[v], s->maxW);
    s->d_swapStates[entryDestId] = 2;
  }
}

/* buildListToSwapOut :234-260, moveActiveDataToTransferBuffer :298-330, cleanMemory :283-296 */
int oracle_swap_out(b200_scene *s, const b200_render_state *rs, b200_voxel *synced, uint8_t *hasSynced, int32_t *neededEntryIDs) {
  int n = 0, noTotal = s->numBuckets + s->excessSize;
  for (int i = 0; i < noTotal; ++i) {
    if (s->d_swapStates[i] == 2 && s->d_hash[i].ptr >= 0 && rs->d_entriesVisibleType[i] == 0) {
      if (n < B200_TRANSFER_BLOCK_NUM) neededEntryIDs[n] = i;
      n++;
    }
  }
  if (n > B200_TRANSFER_BLOCK_NUM) n = B200_TRANSFER_BLOCK_NUM;
  int counter = s->lastFreeBlockId;
  for (int i = 0; i < n; ++i) { /* moveActiveDataToTransferBuffer */
    int id = neededEntryIDs[i];
    b200_voxel *blk = s->d_voxels + (size_t)s->d_hash[id].ptr * BS3;
    memcpy(synced + (size_t)i * BS3, blk, sizeof(b200_voxel) * BS3);
    hasSynced[i] = 1;
    b200_voxel v0; memset(&v0, 0, sizeof(v0)); v0.sdf = 32767;
    for (int v = 0; v < BS3; ++v) blk[v] = v0;
  }
  for (int i = 0; i < n; ++i) { /* cleanMemory */
    int id = neededEntryIDs[i];
    s->d_swapStates[id] = 0;
    int vbaIdx = counter++;
    if (vbaIdx < s->numBlocks - 1) {
      s->d_allocationList[vbaIdx + 1] = s->d_hash[id].ptr;
      s->d_hash[id].ptr = -1;
    }
  }
  if (n > 0) { /* host clamp, Swap_CUDA.cu:199-203 */
    if (counter < 0) counter = 0;
    if (counter > s->numBlocks) counter = s->numBlocks;
    s->lastFreeBlockId = counter;
  }
  return n;
}

void oracle_set_threads(int n) {
#ifdef _OPENMP
  if (n > 0) omp_set_num_threads(n);
#else
  (void)n;
#endif
}

int oracle_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

/* ---- test hooks (used only by tests/test_oracle_vs_ref.py to pin single stages) ------------- */
void oracle_mark_only(oracle_engine *e, const b200_scene *s, uint8_t *visType, const b200_view *v) {
  float invProj[4] = {1.0f / v->proj_d[0], 1.0f / v->proj_d[1], v->proj_d[2], v->proj_d[3]};
  float oneOverVoxelSize = 1.0f / (s->voxelSize * BS);
  memset(e->allocType, 0, e->noTotalEntries);
  for (int locId = 0; locId < v->depth_w * v->depth_h; locId++) {
    int y = locId / v->depth_w, x = locId - y * v->depth_w;
    mark_pixel(e->allocType, visType, x, y, e->blockCoords, v->d_depth, v->invM_d, invProj, s->mu, v->depth_w,
               oneOverVoxelSize, s->d_hash, s->numBuckets, s->viewFrustum_min, s->viewFrustum_max);
  }
}
uint8_t *oracle_alloc_type(oracle_engine *e) { return e->allocType; }
int16_t *oracle_block_coords(oracle_engine *e) { return e->blockCoords; }
int oracle_block_visible(const int16_t *pos, const float *M, const float *proj, float voxelSize, int w, int h) {
  return block_visible(pos, M, proj, voxelSize, w, h);
}
int oracle_project_single_block(const int16_t *pos, const float *pose, const float *intr, int w, int h, float voxelSize,
                                int *ul, int *lr, float *zr) {
  return project_single_block(pos, pose, intr, w, h, voxelSize, ul, lr, zr);
}
void oracle_combine_block(const b200_voxel *src, b200_voxel *dst, int maxW) {
  for (int i = 0; i < BS3; ++i) combine_voxel(&src[i], &dst[i], maxW);
}
int oracle_find_block(const b200_hash_entry *table, int numBuckets, int x, int y, int z) {
  return find_block(table, numBuckets, x, y, z);
}
