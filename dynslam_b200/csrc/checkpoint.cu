// checkpoint.cu — b200_checkpoint_save / b200_checkpoint_load (include/b200fusion.h): one volume's state to a host buffer and
// back, bit for bit.
//
// Save: one persistent launch classifies every voxel block (128-bit loads, warp vote against the reset block), hash entry
// (against the reset entry) and visibility byte (against 0) and compacts the survivors in ascending order with the decoupled
// look-back of common.cuh. One launch gathers everything but the voxel payload (the "small part") into a device staging
// buffer. The buffer then goes down in chunks through two pinned bounce buffers on the copy stream; the blocks of chunk i+1
// are gathered while chunk i is copied down and chunk i-1 is copied out of its bounce buffer on the host.
// Load mirrors it: reset, the chunks up through the bounce buffers, one scatter of the small part, one per block chunk, then
// the decay queue is pushed again snapshot by snapshot through the same path as allocation's pushes.
#include "engine.h"
#include "checkpoint_layout.h"

#include <climits>
#include <cstdio>
#include <cstring>
#include <vector>

#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t _e = (call);                                                                       \
    if (_e != cudaSuccess) {                                                                       \
      snprintf(e->err, sizeof(e->err), "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
      return B200_ERR_CUDA;                                                                        \
    }                                                                                              \
  } while (0)

static_assert(sizeof(b200_checkpoint_header) == B200_CHECKPOINT_HEADER_BYTES, "checkpoint header layout");

#define CK_CHUNK (32ull << 20)        // bytes per pipelined copy, a multiple of the 4 KiB block
#define CK_TILE_BLOCKS 256            // classification: voxel blocks per tile (8 warps x 32)
#define CK_TILE_ENTRIES 1024          // classification: hash entries and visibility bytes per tile (256 threads x 4)
#define CK_SMALL B200_CK_BLOCK_DATA   // sections 0 .. CK_SMALL-1 form the small part

struct CheckpointScratch {
  unsigned *d_blkIds, *d_entIdx, *d_visIdx;   // classification: ascending indices of the blocks / entries / bytes kept
  unsigned long long *d_desc;                 // chained-scan descriptors: block tiles, entry tiles, visibility tiles
  int tilesB, tilesE, classifyGrid, classifyPerSm;   // classifyPerSm: resident classification CTAs per SM (occupancy)
  long long *d_counts, *h_counts;             // noBlocks, noEntries, noVisBytes (device, pinned mirror)
  int *d_qCount; long long *d_qCum, *d_qStart;   // save: the queue table (SNAP_SLOTS entries, cumulative counts + 1)
  int *h_snapCount; long long *h_snapStart;   // pinned copies of the engine's snapshot slots
  struct { int ctr3[3]; int noFwd; long long totalDecayed; } *h_set;   // load: counters uploaded from pinned memory
  uint8_t *d_small; size_t smallCap;
  uint8_t *d_stage[2], *h_bounce[2];
  cudaStream_t copyStream;
  cudaEvent_t evKernel[2], evCopy[2], evSmall;
  // the classification kept for the save that follows a size query
  bool valid; long long launches; const void *voxels, *hash, *visType;
};

// ---- kernels ---------------------------------------------------------------------------------------------------------

// Tiles [0, tilesB) test voxel blocks, [tilesB, tilesB + tilesE) hash entries and visibility bytes; each kind is compacted
// through its own descriptor chain. Tiles come from draw_tile, so every tile's predecessors are owned by running CTAs (common.cuh).
__global__ void __launch_bounds__(256)
k_ck_classify(const uint4 *voxels, int numBlocks, const int *hash, const uint8_t *visType, int noTotal, int tilesB, int tilesE,
              unsigned long long *desc, unsigned gen, unsigned *blkIds, unsigned *entIdx, unsigned *visIdx, long long *counts,
              unsigned *ticket) {
  __shared__ unsigned sm[33];
  __shared__ unsigned base[2];
  __shared__ int sTile;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int t = draw_tile(ticket, tilesB + tilesE, &sTile); t < tilesB + tilesE; t = draw_tile(ticket, tilesB + tilesE, &sTile)) {
    if (t < tilesB) {
      const int first = t * CK_TILE_BLOCKS + warp * 32;
      unsigned mask = 0;                      // bit i: block first + i differs from a reset block
      for (int i = 0; i < 32 && first + i < numBlocks; ++i) {
        const uint4 *p = voxels + (size_t)(first + i) * (BS3 / 2) + lane;
        uint4 v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = ld_stream(p + 32 * k);
        bool pristine = true;                 // two reset voxels {sdf 32767, 0, 0, 0, pad 0} per 16 bytes
#pragma unroll
        for (int k = 0; k < 8; ++k) pristine &= (v[k].x == 0x7fffu) & (v[k].y == 0u) & (v[k].z == 0x7fffu) & (v[k].w == 0u);
        if (!__all_sync(0xffffffffu, pristine)) mask |= 1u << i;
      }
      unsigned total;
      const unsigned local = block_exclusive_scan(lane == 0 ? (unsigned)__popc(mask) : 0u, sm, &total);
      const unsigned warpOff = __shfl_sync(0xffffffffu, local, 0);
      if (warp == 0) {
        const unsigned ex = scan_lookback(desc, gen, t, total);
        if (lane == 0) { base[0] = ex; if (t == tilesB - 1) counts[0] = (long long)ex + total; }
      }
      __syncthreads();
      if ((mask >> lane) & 1u) blkIds[base[0] + warpOff + __popc(mask & ((1u << lane) - 1u))] = (unsigned)(first + lane);
      __syncthreads();
    } else {
      const int te = t - tilesB;
      const int first = te * CK_TILE_ENTRIES + threadIdx.x * 4;
      unsigned hm = 0, vm = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int i = first + k;
        if (i >= noTotal) break;
        const int *w = hash + (size_t)i * 5;   // reset entry: {pos 0, pad 0, offset 0, ptr -2, allocatedTime 0}
        if ((w[0] | w[1] | w[2] | w[4]) != 0 || w[3] != -2) hm |= 1u << k;
        if (visType[i] != 0) vm |= 1u << k;
      }
      unsigned totH, totV;
      const unsigned lh = block_exclusive_scan((unsigned)__popc(hm), sm, &totH);
      const unsigned lv = block_exclusive_scan((unsigned)__popc(vm), sm, &totV);
      if (warp == 0) {
        const unsigned exH = scan_lookback(desc + tilesB, gen, te, totH);
        const unsigned exV = scan_lookback(desc + tilesB + tilesE, gen, te, totV);
        if (lane == 0) {
          base[0] = exH; base[1] = exV;
          if (te == tilesE - 1) { counts[1] = (long long)exH + totH; counts[2] = (long long)exV + totV; }
        }
      }
      __syncthreads();
      unsigned r = base[0] + lh;
      for (int k = 0; k < 4; ++k) if ((hm >> k) & 1u) entIdx[r++] = (unsigned)(first + k);
      r = base[1] + lv;
      for (int k = 0; k < 4; ++k) if ((vm >> k) & 1u) visIdx[r++] = (unsigned)(first + k);
      __syncthreads();
    }
  }
}

// The state buffers a checkpoint covers and where each section of the small part lies.
struct CkBufs {
  int *hash, *allocList, *excessList, *visible, *minmax, *rays, *image, *fwd, *fwdMissing;
  uint8_t *swap, *visType;
  unsigned long long off[CK_SMALL], len[CK_SMALL];
};
// Save only: the classification and the decay queue (snapshot s: qCount[s] items from ring position qStart[s], preceded by
// qCum[s] items of the snapshots before it).
struct CkQueue {
  const unsigned *entIdx, *visIdx, *blkIds;
  const int *qCount; const long long *qCum, *qStart; int nSnap;
  const int *ring; long long ringCap;
};

DEV unsigned ck_word(const CkBufs &b, const CkQueue &q, int sec, long long w) {
  switch (sec) {
  case B200_CK_HASH_INDEX: return q.entIdx[w];
  case B200_CK_HASH_ENTRIES: return (unsigned)b.hash[(size_t)q.entIdx[w / 5] * 5 + w % 5];
  case B200_CK_ALLOCATION_LIST: return (unsigned)b.allocList[w];
  case B200_CK_EXCESS_LIST: return (unsigned)b.excessList[w];
  case B200_CK_VIS_INDEX: return q.visIdx[w];
  case B200_CK_VISIBLE_LIST: return (unsigned)b.visible[w];
  case B200_CK_MINMAX: return (unsigned)b.minmax[w];
  case B200_CK_RAYCAST_RESULT: return (unsigned)b.rays[w];
  case B200_CK_RAYCAST_IMAGE: return (unsigned)b.image[w];
  case B200_CK_FWD_PROJECTION: return (unsigned)b.fwd[w];
  case B200_CK_FWD_MISSING: return (unsigned)b.fwdMissing[w];
  case B200_CK_QUEUE_COUNTS: return (unsigned)q.qCount[w];
  case B200_CK_QUEUE_ITEMS: {
    const long long j = w / 3;
    int lo = 0, hi = q.nSnap;                 // qCum[lo] <= j < qCum[hi]
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (q.qCum[mid] <= j) lo = mid; else hi = mid; }
    return (unsigned)q.ring[((q.qStart[lo] + (j - q.qCum[lo])) % q.ringCap) * 3 + w % 3];
  }
  case B200_CK_BLOCK_IDS: return q.blkIds[w];
  default: return 0u;
  }
}

// blockIdx.y = section; one 32-bit word per thread, the padding up to the next 16-byte boundary written as zeros
__global__ void __launch_bounds__(256) k_ck_gather_small(CkBufs b, CkQueue q, uint8_t *out) {
  const int sec = blockIdx.y;
  const long long len = (long long)b.len[sec], words = ((len + 15) & ~15ll) >> 2;
  unsigned *o = reinterpret_cast<unsigned *>(out + b.off[sec]);
  const bool bytes = sec == B200_CK_SWAP_STATES || sec == B200_CK_VIS_VALUE;
  for (long long w = blockIdx.x * (long long)blockDim.x + threadIdx.x; w < words; w += (long long)gridDim.x * blockDim.x) {
    unsigned v = 0;
    if (bytes) {
      for (int k = 0; k < 4; ++k) {
        const long long i = w * 4 + k;
        if (i < len) v |= (unsigned)(sec == B200_CK_SWAP_STATES ? b.swap[i] : b.visType[q.visIdx[i]]) << (8 * k);
      }
    } else if (w * 4 < len) {
      v = ck_word(b, q, sec, w);
    }
    o[w] = v;
  }
}

// the mirror: writes every section that is state (the index lists and the queue are read from the small part where needed)
__global__ void __launch_bounds__(256) k_ck_scatter_small(CkBufs b, const uint8_t *in) {
  const int sec = blockIdx.y;
  const long long len = (long long)b.len[sec];
  const unsigned *src = reinterpret_cast<const unsigned *>(in + b.off[sec]);
  const unsigned *entIdx = reinterpret_cast<const unsigned *>(in + b.off[B200_CK_HASH_INDEX]);
  const unsigned *visIdx = reinterpret_cast<const unsigned *>(in + b.off[B200_CK_VIS_INDEX]);
  const long long stride = (long long)gridDim.x * blockDim.x, t0 = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (sec == B200_CK_SWAP_STATES || sec == B200_CK_VIS_VALUE) {
    const uint8_t *s8 = in + b.off[sec];
    for (long long i = t0; i < len; i += stride) {
      if (sec == B200_CK_SWAP_STATES) b.swap[i] = s8[i];
      else b.visType[visIdx[i]] = s8[i];
    }
    return;
  }
  int *dst;
  switch (sec) {
  case B200_CK_ALLOCATION_LIST: dst = b.allocList; break;
  case B200_CK_EXCESS_LIST: dst = b.excessList; break;
  case B200_CK_VISIBLE_LIST: dst = b.visible; break;
  case B200_CK_MINMAX: dst = b.minmax; break;
  case B200_CK_RAYCAST_RESULT: dst = b.rays; break;
  case B200_CK_RAYCAST_IMAGE: dst = b.image; break;
  case B200_CK_FWD_PROJECTION: dst = b.fwd; break;
  case B200_CK_FWD_MISSING: dst = b.fwdMissing; break;
  case B200_CK_HASH_ENTRIES: dst = nullptr; break;
  default: return;                            // index lists, queue: not state of their own
  }
  for (long long w = t0; w < (len >> 2); w += stride) {
    if (sec == B200_CK_HASH_ENTRIES) b.hash[(size_t)entIdx[w / 5] * 5 + w % 5] = (int)src[w];
    else dst[w] = (int)src[w];
  }
}

__global__ void __launch_bounds__(256) k_ck_gather_blocks(const uint4 *voxels, const unsigned *ids, long long n16, uint4 *out) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n16; t += (long long)gridDim.x * blockDim.x)
    out[t] = ld_stream(voxels + (size_t)ids[t >> 8] * (BS3 / 2) + (t & 255));
}

__global__ void __launch_bounds__(256) k_ck_scatter_blocks(uint4 *voxels, const unsigned *ids, long long n16, const uint4 *in) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n16; t += (long long)gridDim.x * blockDim.x)
    st_stream(voxels + (size_t)ids[t >> 8] * (BS3 / 2) + (t & 255), ld_stream(in + t));
}

// ---- host --------------------------------------------------------------------------------------------------------------

void checkpoint_release(b200_engine *e) {
  CheckpointScratch *c = e->ck;
  if (!c) return;
  if (c->copyStream) { cudaStreamSynchronize(c->copyStream); cudaStreamDestroy(c->copyStream); }
  cudaFree(c->d_blkIds); cudaFree(c->d_entIdx); cudaFree(c->d_visIdx); cudaFree(c->d_desc); cudaFree(c->d_counts); cudaFreeHost(c->h_counts);
  cudaFree(c->d_qCount); cudaFree(c->d_qCum); cudaFree(c->d_qStart); cudaFreeHost(c->h_snapCount); cudaFreeHost(c->h_snapStart);
  cudaFreeHost(c->h_set); cudaFree(c->d_small);
  for (int i = 0; i < 2; ++i) {
    cudaFree(c->d_stage[i]); cudaFreeHost(c->h_bounce[i]);
    if (c->evKernel[i]) cudaEventDestroy(c->evKernel[i]);
    if (c->evCopy[i]) cudaEventDestroy(c->evCopy[i]);
  }
  if (c->evSmall) cudaEventDestroy(c->evSmall);
  delete c;
  e->ck = nullptr;
}

// Scratch on first use (like the meshing descriptors); the small-part staging grows to smallBytes.
static b200_status ck_ensure(b200_engine *e, size_t smallBytes) {
  if (!e->ck) {
    CheckpointScratch *c = new CheckpointScratch();
    memset(c, 0, sizeof(*c));
    e->ck = c;
    c->tilesB = (e->numBlocks + CK_TILE_BLOCKS - 1) / CK_TILE_BLOCKS;
    c->tilesE = (e->noTotal + CK_TILE_ENTRIES - 1) / CK_TILE_ENTRIES;
    CK(cudaMalloc(&c->d_blkIds, sizeof(unsigned) * (size_t)e->numBlocks));
    CK(cudaMalloc(&c->d_entIdx, sizeof(unsigned) * (size_t)e->noTotal));
    CK(cudaMalloc(&c->d_visIdx, sizeof(unsigned) * (size_t)e->noTotal));
    CK(cudaMalloc(&c->d_desc, sizeof(unsigned long long) * (size_t)(c->tilesB + 2 * c->tilesE)));
    CK(cudaMemset(c->d_desc, 0, sizeof(unsigned long long) * (size_t)(c->tilesB + 2 * c->tilesE)));
    CK(cudaMalloc(&c->d_counts, 4 * sizeof(long long)));
    CK(cudaMallocHost(&c->h_counts, 4 * sizeof(long long)));
    CK(cudaMalloc(&c->d_qCount, sizeof(int) * SNAP_SLOTS));
    CK(cudaMalloc(&c->d_qCum, sizeof(long long) * (SNAP_SLOTS + 1)));
    CK(cudaMalloc(&c->d_qStart, sizeof(long long) * SNAP_SLOTS));
    CK(cudaMallocHost(&c->h_snapCount, sizeof(int) * SNAP_SLOTS));
    CK(cudaMallocHost(&c->h_snapStart, sizeof(long long) * SNAP_SLOTS));
    CK(cudaMallocHost(&c->h_set, sizeof(*c->h_set)));
    for (int i = 0; i < 2; ++i) {
      CK(cudaMalloc(&c->d_stage[i], CK_CHUNK));
      CK(cudaMallocHost(&c->h_bounce[i], CK_CHUNK));
      CK(cudaEventCreateWithFlags(&c->evKernel[i], cudaEventDisableTiming));
      CK(cudaEventCreateWithFlags(&c->evCopy[i], cudaEventDisableTiming));
    }
    CK(cudaEventCreateWithFlags(&c->evSmall, cudaEventDisableTiming));
    CK(cudaStreamCreateWithFlags(&c->copyStream, cudaStreamNonBlocking));
    int perSm = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, k_ck_classify, 256, 0));
    c->classifyPerSm = perSm > 0 ? perSm : 1;
    c->classifyGrid = persistent_grid(e, c->classifyPerSm, (long long)c->tilesB + c->tilesE);
  }
  CheckpointScratch *c = e->ck;
  if (smallBytes > c->smallCap) {
    CK(cudaStreamSynchronize(e->stream));
    cudaFree(c->d_small); c->d_small = nullptr; c->smallCap = 0;
    CK(cudaMalloc(&c->d_small, smallBytes));
    c->smallCap = smallBytes;
  }
  return B200_OK;
}

static bool has_forward(const b200_render_state *rs) { return rs->d_forwardProjection && rs->d_fwdProjMissingPoints; }

static CkBufs ck_bufs(const b200_scene *s, const b200_render_state *rs, const b200_checkpoint_header &h) {
  CkBufs b;
  b.hash = (int *)s->d_hash; b.allocList = s->d_allocationList; b.excessList = s->d_excessList; b.swap = s->d_swapStates;
  b.visType = rs->d_entriesVisibleType; b.visible = (int *)rs->d_visibleBlockPositions; b.minmax = (int *)rs->d_minmax;
  b.rays = (int *)rs->d_raycastResult; b.image = (int *)rs->d_raycastImage; b.fwd = (int *)rs->d_forwardProjection;
  b.fwdMissing = rs->d_fwdProjMissingPoints;
  for (int i = 0; i < CK_SMALL; ++i) { b.off[i] = h.section[i][0]; b.len[i] = h.section[i][1]; }
  return b;
}

static b200_status check_state_args(b200_engine *e, const b200_scene *s, const b200_render_state *rs, const char *what) {
  if (!s || !rs || !rs->d_visibleBlockPositions || !rs->d_entriesVisibleType || !rs->d_minmax || !rs->d_raycastResult ||
      !rs->d_raycastImage || rs->img_w <= 0 || rs->img_h <= 0) {
    snprintf(e->err, sizeof(e->err), "%s: scene and a complete render state are required", what);
    return B200_ERR_INVALID;
  }
  return check_scene(e, s);
}

// One pipelined chunk of the buffer: bytes [off, off + bytes); a chunk of the small part or nBlocks voxel blocks from firstBlock.
struct CkChunk { size_t off, bytes; bool small; long long firstBlock, nBlocks; };

static std::vector<CkChunk> ck_chunks(const b200_checkpoint_header &h) {
  std::vector<CkChunk> v;
  const size_t dataOff = (size_t)h.section[B200_CK_BLOCK_DATA][0];
  for (size_t a = 0; a < dataOff; a += CK_CHUNK) v.push_back({a, dataOff - a < CK_CHUNK ? dataOff - a : (size_t)CK_CHUNK, true, 0, 0});
  const long long per = (long long)(CK_CHUNK / 4096);
  for (long long b0 = 0; b0 < h.noBlocks; b0 += per) {
    const long long n = h.noBlocks - b0 < per ? h.noBlocks - b0 : per;
    v.push_back({dataOff + (size_t)b0 * 4096, (size_t)n * 4096, false, b0, n});
  }
  return v;
}

static int ck_grid(const b200_engine *e, long long work) { return persistent_grid(e, 8, (work + 255) / 256); }

extern "C" {

b200_status b200_checkpoint_save(b200_engine *e, b200_scene *s, b200_render_state *rs, void *h_out, size_t capacity, size_t *size) {
  if (!e) return B200_ERR_INVALID;
  if (!size) { snprintf(e->err, sizeof(e->err), "checkpoint_save: size pointer missing"); return B200_ERR_INVALID; }
  *size = 0;
  b200_status st = check_state_args(e, s, rs, "checkpoint_save"); if (st) return st;
  CK(cudaSetDevice(e->device));
  st = b200_sync(e, s, rs); if (st) return st;     // outstanding frames finished, the expected-depth image complete
  st = ck_ensure(e, 0); if (st) return st;
  CheckpointScratch *c = e->ck;
  // A size query always classifies; the data save right after it reuses that classification if nothing was launched since.
  if (!h_out || !(c->valid && c->launches == e->launches && c->voxels == s->d_voxels && c->hash == s->d_hash &&
                  c->visType == rs->d_entriesVisibleType)) {
    TRACED(e, e->stream, "k_ck_classify",
           k_ck_classify<<<ticket_grid(e, c->classifyPerSm, (long long)c->tilesB + c->tilesE), 256, 0, e->stream>>>((const uint4 *)s->d_voxels, s->numBlocks, (const int *)s->d_hash,
                                                                 rs->d_entriesVisibleType, e->noTotal, c->tilesB, c->tilesE, c->d_desc,
                                                                 ++e->scanGen, c->d_blkIds, c->d_entIdx, c->d_visIdx, c->d_counts,
                                                                 &e->d_ctr->ticket[TK_CK_CLASSIFY]));
    e->launches++;
    CK(cudaMemcpyAsync(c->h_counts, c->d_counts, 3 * sizeof(long long), cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    CK(cudaGetLastError());
    c->valid = true; c->launches = e->launches; c->voxels = s->d_voxels; c->hash = s->d_hash; c->visType = rs->d_entriesVisibleType;
  }
  // the decay queue, oldest first; a snapshot the ring has wrapped over is stored as overwritten (decay.cu's test)
  CK(cudaMemcpyAsync(c->h_snapCount, e->d_snapCount, sizeof(int) * SNAP_SLOTS, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemcpyAsync(c->h_snapStart, e->d_snapStart, sizeof(long long) * SNAP_SLOTS, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  const long long ringHead = e->h_ctr->ringHead;
  std::vector<int> qCount(e->qSize);
  std::vector<long long> qCum(e->qSize + 1, 0), qStart(e->qSize);
  for (int j = 0; j < e->qSize; ++j) {
    const int slot = (e->qHead + j) % SNAP_SLOTS;
    qStart[j] = c->h_snapStart[slot];
    qCount[j] = (ringHead - qStart[j] > e->ringCap) ? -1 : c->h_snapCount[slot];
    qCum[j + 1] = qCum[j] + (qCount[j] > 0 ? qCount[j] : 0);
  }
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
  h.frameIdx = e->frameIdx; h.noSnapshots = e->qSize;
  h.totalDecayed = e->totalDecayed; h.droppedSnapshots = e->droppedSnapshots + e->h_ctr->droppedSnapshots;
  h.noBlocks = c->h_counts[0]; h.noEntries = c->h_counts[1]; h.noVisBytes = c->h_counts[2]; h.noQueueItems = qCum[e->qSize];
  const uint64_t total = checkpoint_layout(&h);
  *size = (size_t)total;
  if (!h_out) return B200_OK;
  if (capacity < total) {
    snprintf(e->err, sizeof(e->err), "checkpoint_save: capacity %zu is below the checkpoint's %llu bytes", capacity, (unsigned long long)total);
    return B200_ERR_INVALID;
  }
  const size_t dataOff = (size_t)h.section[B200_CK_BLOCK_DATA][0];
  st = ck_ensure(e, dataOff); if (st) return st;
  if (e->qSize > 0) {
    CK(cudaMemcpyAsync(c->d_qCount, qCount.data(), sizeof(int) * e->qSize, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(c->d_qCum, qCum.data(), sizeof(long long) * (e->qSize + 1), cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(c->d_qStart, qStart.data(), sizeof(long long) * e->qSize, cudaMemcpyHostToDevice, e->stream));
  }
  const CkBufs b = ck_bufs(s, rs, h);
  const CkQueue q{c->d_entIdx, c->d_visIdx, c->d_blkIds, c->d_qCount, c->d_qCum, c->d_qStart, e->qSize, (const int *)e->d_ring, e->ringCap};
  TRACED(e, e->stream, "k_ck_gather_small",
         k_ck_gather_small<<<dim3(e->smCount * 4, CK_SMALL), 256, 0, e->stream>>>(b, q, c->d_small));
  e->launches++;
  const size_t idsEnd = (size_t)((h.section[B200_CK_BLOCK_IDS][0] + h.section[B200_CK_BLOCK_IDS][1] + 15) & ~15ull);
  if (dataOff > idsEnd) CK(cudaMemsetAsync(c->d_small + idsEnd, 0, dataOff - idsEnd, e->stream));   // padding before the payload
  CK(cudaEventRecord(c->evSmall, e->stream));
  CK(cudaStreamWaitEvent(c->copyStream, c->evSmall, 0));
  // the pipeline: at step i the host copies chunk i-2 out of its bounce buffer while chunk i-1 goes down and chunk i is gathered
  const std::vector<CkChunk> ch = ck_chunks(h);
  const int n = (int)ch.size();
  for (int i = 0; i < n + 2; ++i) {
    if (i >= 2) {
      const CkChunk &d = ch[i - 2];
      CK(cudaEventSynchronize(c->evCopy[i & 1]));
      memcpy((uint8_t *)h_out + d.off, c->h_bounce[i & 1], d.bytes);
    }
    if (i >= n) continue;
    const CkChunk &d = ch[i];
    const int slot = i & 1;
    const uint8_t *src = c->d_small + d.off;
    if (!d.small) {   // the stage's previous chunk (i-2) has been copied down: its event was waited for just above
      TRACED(e, e->stream, "k_ck_gather_blocks",
             k_ck_gather_blocks<<<ck_grid(e, d.nBlocks * 256), 256, 0, e->stream>>>((const uint4 *)s->d_voxels, c->d_blkIds + d.firstBlock,
                                                                                   d.nBlocks * 256, (uint4 *)c->d_stage[slot]));
      e->launches++;
      CK(cudaEventRecord(c->evKernel[slot], e->stream));
      CK(cudaStreamWaitEvent(c->copyStream, c->evKernel[slot], 0));
      src = c->d_stage[slot];
    }
    CK(cudaMemcpyAsync(c->h_bounce[slot], src, d.bytes, cudaMemcpyDeviceToHost, c->copyStream));
    CK(cudaEventRecord(c->evCopy[slot], c->copyStream));
  }
  CK(cudaGetLastError());
  memcpy(h_out, &h, sizeof(h));
  c->valid = false;            // kept for one save only: the next save classifies again
  return B200_OK;
}

// Every rejection is decided here, from the buffer alone, before the load writes anything.
static b200_status ck_validate(b200_engine *e, const b200_scene *s, const b200_render_state *rs, const uint8_t *p, size_t size,
                               b200_checkpoint_header *h) {
#define REJECT(...) do { snprintf(e->err, sizeof(e->err), "checkpoint_load: " __VA_ARGS__); return B200_ERR_INVALID; } while (0)
  if (!p) REJECT("no buffer");
  if (size < sizeof(*h)) REJECT("truncated: %zu bytes, the header alone is %d", size, B200_CHECKPOINT_HEADER_BYTES);
  memcpy(h, p, sizeof(*h));
  if (memcmp(h->magic, B200_CHECKPOINT_MAGIC, 8) != 0) REJECT("not a checkpoint (bad magic)");
  if (h->version != B200_CHECKPOINT_VERSION) REJECT("format version %u, this library reads %d", h->version, B200_CHECKPOINT_VERSION);
  if (h->numBlocks != s->numBlocks || h->numBuckets != s->numBuckets || h->excessSize != s->excessSize || h->img_w != rs->img_w ||
      h->img_h != rs->img_h)
    REJECT("geometry %d blocks, %d buckets, %d excess, %dx%d differs from the target's %d, %d, %d, %dx%d", h->numBlocks, h->numBuckets,
           h->excessSize, h->img_w, h->img_h, s->numBlocks, s->numBuckets, s->excessSize, rs->img_w, rs->img_h);
  if (memcmp(&h->voxelSize, &s->voxelSize, sizeof(float)) != 0 || memcmp(&h->mu, &s->mu, sizeof(float)) != 0)
    REJECT("voxelSize %g / mu %g differ from the target scene's %g / %g", h->voxelSize, h->mu, s->voxelSize, s->mu);
  if (h->flags & ~(B200_CK_HAS_SWAP_STATES | B200_CK_HAS_FORWARD)) REJECT("unknown flags 0x%x", h->flags);
  if (((h->flags & B200_CK_HAS_SWAP_STATES) != 0) != (s->d_swapStates != nullptr))
    REJECT("swap states are present in only one of the checkpoint and the target scene");
  if (((h->flags & B200_CK_HAS_FORWARD) != 0) != has_forward(rs))
    REJECT("forward-projection buffers are present in only one of the checkpoint and the target render state");
  const long long noTotal = (long long)s->numBuckets + s->excessSize, px = (long long)rs->img_w * rs->img_h;
  if (h->noEntries < 0 || h->noEntries > noTotal || h->noVisBytes < 0 || h->noVisBytes > noTotal || h->noBlocks < 0 ||
      h->noBlocks > s->numBlocks || h->noSnapshots < 0 || h->noQueueItems < 0 || h->noQueueItems > (long long)h->noSnapshots * s->numBlocks ||
      h->noVisibleBlocks < 0 || h->noVisibleBlocks > s->numBlocks || h->noFwdProjMissingPoints < 0 || h->noFwdProjMissingPoints > px || h->lastFreeBlockId < -1 ||
      h->lastFreeBlockId >= s->numBlocks || h->lastFreeExcessListId < -1 || h->lastFreeExcessListId >= s->excessSize ||
      h->totalDecayed < 0 || h->droppedSnapshots < 0)
    REJECT("counts out of range");
  b200_checkpoint_header t = *h;
  checkpoint_layout(&t);
  if (memcmp(t.section, h->section, sizeof(t.section)) != 0 || t.totalBytes != h->totalBytes)
    REJECT("the section table disagrees with the header's counts");
  if (size < h->totalBytes) REJECT("truncated: %zu bytes of %llu", size, (unsigned long long)h->totalBytes);
  if (size != h->totalBytes) REJECT("%zu bytes, the header says %llu", size, (unsigned long long)h->totalBytes);
  struct { int sec; long long n, bound; const char *what; } lists[3] = {
    {B200_CK_HASH_INDEX, h->noEntries, noTotal, "hash entry"}, {B200_CK_VIS_INDEX, h->noVisBytes, noTotal, "visibility byte"},
    {B200_CK_BLOCK_IDS, h->noBlocks, s->numBlocks, "voxel block"}};
  for (const auto &l : lists) {
    const uint8_t *a = p + h->section[l.sec][0];
    long long prev = -1;
    for (long long i = 0; i < l.n; ++i) {
      uint32_t v; memcpy(&v, a + 4 * i, 4);
      if ((long long)v <= prev || (long long)v >= l.bound) REJECT("%s index %u out of range or out of order", l.what, v);
      prev = v;
    }
  }
  long long items = 0;
  for (int j = 0; j < h->noSnapshots; ++j) {
    int32_t n; memcpy(&n, p + h->section[B200_CK_QUEUE_COUNTS][0] + 4 * (size_t)j, 4);
    if (n < -1 || n > s->numBlocks) REJECT("decay snapshot %d holds %d items", j, n);
    items += n > 0 ? n : 0;
  }
  if (items != h->noQueueItems) REJECT("the decay queue holds %lld items, the header says %lld", items, (long long)h->noQueueItems);
  return B200_OK;
#undef REJECT
}

b200_status b200_checkpoint_load(b200_engine *e, b200_scene *s, b200_render_state *rs, const void *h_in, size_t size) {
  if (!e) return B200_ERR_INVALID;
  b200_status st = check_state_args(e, s, rs, "checkpoint_load"); if (st) return st;
  if (e->copyStream && (e->slotBusy[0] || e->slotBusy[1])) {
    snprintf(e->err, sizeof(e->err), "checkpoint_load: a host-frame slot is still outstanding (b200_host_frame_wait it first)");
    return B200_ERR_INVALID;
  }
  b200_checkpoint_header h;
  st = ck_validate(e, s, rs, (const uint8_t *)h_in, size, &h); if (st) return st;
  const uint8_t *in = (const uint8_t *)h_in;
  CK(cudaSetDevice(e->device));
  const size_t dataOff = (size_t)h.section[B200_CK_BLOCK_DATA][0];
  st = ck_ensure(e, dataOff); if (st) return st;
  CheckpointScratch *c = e->ck;
  CK(cudaStreamSynchronize(e->stream));            // frames still in flight finish on the state they started on
  c->valid = false;
  e->deadPending = false;
  launch_reset(e, scene_ref(s, nullptr));           // blocks, entries and bytes the checkpoint does not list have their reset values
  // Allocation's request keys carry (frame index + 1) and the largest key wins. The loaded frame index can be lower than
  // this engine's, so keys left by its later frames would outrank every new request: they go with the old state.
  CK(cudaMemsetAsync(e->d_reqKey, 0, sizeof(unsigned long long) * (size_t)e->noTotal, e->stream));
  CK(cudaMemsetAsync(rs->d_entriesVisibleType, 0, (size_t)e->noTotal, e->stream));
  const CkBufs b = ck_bufs(s, rs, h);
  const std::vector<CkChunk> ch = ck_chunks(h);
  bool stageUsed[2] = {false, false};
  for (int i = 0; i < (int)ch.size(); ++i) {
    const CkChunk &d = ch[i];
    const int slot = i & 1;
    if (i >= 2) CK(cudaEventSynchronize(c->evCopy[slot]));   // the bounce buffer's previous chunk is up
    memcpy(c->h_bounce[slot], in + d.off, d.bytes);
    if (d.small) {
      CK(cudaMemcpyAsync(c->d_small + d.off, c->h_bounce[slot], d.bytes, cudaMemcpyHostToDevice, c->copyStream));
      CK(cudaEventRecord(c->evCopy[slot], c->copyStream));
      if (i + 1 == (int)ch.size() || !ch[i + 1].small) {   // the whole small part is up: scatter it
        CK(cudaEventRecord(c->evSmall, c->copyStream));
        CK(cudaStreamWaitEvent(e->stream, c->evSmall, 0));
        TRACED(e, e->stream, "k_ck_scatter_small",
               k_ck_scatter_small<<<dim3(e->smCount * 4, CK_SMALL), 256, 0, e->stream>>>(b, c->d_small));
        e->launches++;
      }
      continue;
    }
    if (stageUsed[slot]) CK(cudaStreamWaitEvent(c->copyStream, c->evKernel[slot], 0));   // the stage's last scatter has read it
    CK(cudaMemcpyAsync(c->d_stage[slot], c->h_bounce[slot], d.bytes, cudaMemcpyHostToDevice, c->copyStream));
    CK(cudaEventRecord(c->evCopy[slot], c->copyStream));
    CK(cudaStreamWaitEvent(e->stream, c->evCopy[slot], 0));
    const unsigned *ids = (const unsigned *)(c->d_small + h.section[B200_CK_BLOCK_IDS][0]) + d.firstBlock;
    TRACED(e, e->stream, "k_ck_scatter_blocks",
           k_ck_scatter_blocks<<<ck_grid(e, d.nBlocks * 256), 256, 0, e->stream>>>((uint4 *)s->d_voxels, ids, d.nBlocks * 256,
                                                                                  (const uint4 *)c->d_stage[slot]));
    e->launches++;
    CK(cudaEventRecord(c->evKernel[slot], e->stream));
    stageUsed[slot] = true;
  }
  // the decay queue: pushed again oldest first through the path allocation uses (a longer queue than this engine holds
  // drops its oldest snapshots there, as a running engine does)
  e->qHead += e->qSize; e->qSize = 0;
  e->droppedSnapshots = h.droppedSnapshots;
  CK(cudaMemsetAsync(&e->d_ctr->droppedSnapshots, 0, sizeof(int), e->stream));
  const b200_vec3i *items = (const b200_vec3i *)(c->d_small + h.section[B200_CK_QUEUE_ITEMS][0]);
  for (int j = 0; j < h.noSnapshots; ++j) {
    int32_t n; memcpy(&n, in + h.section[B200_CK_QUEUE_COUNTS][0] + 4 * (size_t)j, 4);
    launch_push_snapshot(e, items, n, push_snapshot_slot(e));
    if (n > 0) items += n;
  }
  e->frameIdx = h.frameIdx;
  c->h_set->ctr3[0] = h.lastFreeBlockId; c->h_set->ctr3[1] = h.lastFreeExcessListId; c->h_set->ctr3[2] = h.noVisibleBlocks;
  c->h_set->noFwd = h.noFwdProjMissingPoints; c->h_set->totalDecayed = h.totalDecayed;
  CK(cudaMemcpyAsync(&e->d_ctr->lastFreeBlockId, c->h_set->ctr3, 3 * sizeof(int), cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(&e->d_ctr->noFwdMissing, &c->h_set->noFwd, sizeof(int), cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(&e->d_ctr->totalDecayed, &c->h_set->totalDecayed, sizeof(long long), cudaMemcpyHostToDevice, e->stream));
  e->ptrListFor = nullptr;                          // integration takes its no-pointer-list branch
  e->tableVersion++;
  st = download_sync(e, s, rs); if (st) return st;
  rs->noFwdProjMissingPoints = h.noFwdProjMissingPoints;
  return B200_OK;
}

}  // extern "C"
