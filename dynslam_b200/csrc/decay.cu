// decay.cu — voxel Decay() garbage collection for sm_90a (partial: blocks visible minAge frames
// ago; full: every allocated block).
//
// Replaces decay_device / decayFull_device -> decayVoxel -> deleteBlock (reference
// ITMSceneReconstructionEngine_CUDA.cu:1201-1262, :1120-1197, :1012-1115), findAllocatedBlocks
// (ITMMeshingEngine_CUDA.cu:96-114) and the host logic of Decay/PartialDecay/FullDecay (:430-560).
//
// The reference takes a per-bucket lock (4 MiB array memset per call), DROPS a deletion when the
// lock is contended, and pushes freed slots with atomicAdd — nondeterministic. Here the pass is
// split so that it equals the serial oracle (blocks in list order):
//   phase 1  per list item, one CTA iteration: resolve the block once, sweep its 4 KiB with 128-bit
//            loads, reset noisy voxels, decide "block is empty" with a block-wide vote; the first
//            item (list order) that empties a block claims it with a 64-bit atomicMax tag;
//   phase 2  ordered compaction of the claiming items => free-list position = rank in list order;
//   phase 3  chain leaders: for every bucket chain that loses blocks, ONE thread applies that
//            chain's deletions in list order with the reference's unlink rules (incl. the
//            visibility-byte moves and the never-reclaimed excess slots, :1075-1111).
#include "engine.h"

DEV unsigned long long del_tag(unsigned gen, unsigned item) { return ((unsigned long long)gen << 32) | (0xffffffffu - item); }

DEV void item_pos(int mode, const b200_vec3i *ring, long long ringCap, long long s0, const short4 *allocatedPos, int item, int &x, int &y, int &z);
DEV bool chain_leader(const b200_hash_entry *table, int numBuckets, int x, int y, int z, int item, const unsigned long long *delTag, unsigned gen);
DEV void unlink_chain(b200_hash_entry *table, int numBuckets, uint8_t *visType, int head, const unsigned long long *delTag, unsigned gen);
__device__ void decay_commit_body(b200_hash_entry *table, int numBuckets, uint8_t *visType, const b200_vec3i *ring, long long ringCap, long long s0,
                                  const int *itemPtr, const unsigned long long *delTag, unsigned gen, int *allocList, int *delList,
                                  uint8_t *isLeader, DevCounters *ctr, const int *candList, unsigned *sm, int *cand);

// phase 1. MODE 0: items = ring snapshot; MODE 1: items = VBA slots with allocatedPos.w != 0
template <int MODE>
__global__ void __launch_bounds__(256)
k_decay_blocks(b200_voxel *voxels, const b200_hash_entry *table, int numBuckets, const b200_vec3i *ring,
               long long ringCap, const long long *snapStart, const int *snapCount, int slot, const short4 *allocatedPos,
               int numBlocks, int minAge, int maxWeight, int currentFrame, unsigned gen, unsigned long long *delTag,
               int *itemPtr, DevCounters *ctr, int *candList, uint8_t *visType, int *allocList, int *delList, uint8_t *isLeader,
               unsigned long long *span) {
  pdl_wait();            // in the fused frame: the raycast reads the voxels and entries this sweep resets and unlinks
  SpanStamp stamp(span);
  // One WARP per list item (a block = 256 uint4 = 8 per lane, all 8 loads in flight), 8 items per CTA: the per-item chain of
  // dependent loads (ring position -> hash chain -> voxels) overlaps across warps, so the few thousand items of a frame are
  // one wave of warps instead of ~5 sequential items per CTA.
  const int lane = threadIdx.x & 31;
  const int warpsTotal = gridDim.x * (blockDim.x >> 5), warpId = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int n = (MODE == 0) ? snapCount[slot] : numBlocks;
  const long long s0 = (MODE == 0) ? snapStart[slot] : 0;
  // a snapshot the ring has wrapped over since it was taken is gone (b200_engine_config.decayRingItems): sweep nothing
  const bool overwritten = (MODE == 0) && (ctr->ringHead - s0 > ringCap);
  if (overwritten) n = 0;
  if (blockIdx.x == 0 && threadIdx.x == 0) { ctr->decayItems = n; if (overwritten) ctr->droppedSnapshots++; }
  for (int item = warpId; item < n; item += warpsTotal) {
    int x, y, z;
    if (MODE == 0) { b200_vec3i p = ring[(s0 + item) % ringCap]; x = p.x; y = p.y; z = p.z; }
    else {
      short4 p = allocatedPos[item];
      if (p.w == 0) { if (lane == 0) itemPtr[item] = -1; continue; }
      x = p.x; y = p.y; z = p.z;
    }
    // findBlock / findVoxel (:1214, :1138): uniform across the warp
    int idx = hash_index(x, y, z, numBuckets - 1), ptr = -1, allocatedTime = 0;
    for (;;) {
      const int *w = reinterpret_cast<const int *>(table) + (size_t)idx * 5;
      int w0 = w[0], w1 = w[1], off = w[2], p = w[3];     // plain loads: the last CTA of a partial sweep rewrites the table (commit)
      if ((short)(w0 & 0xffff) == x && (short)(w0 >> 16) == y && (short)(w1 & 0xffff) == z && p >= 0) {
        ptr = p; allocatedTime = w[4]; break;
      }
      if (off < 1) break;
      idx = numBuckets + off - 1;
    }
    bool claim = false;
    if (ptr >= 0 && (currentFrame - allocatedTime) >= minAge) {   // safeToClear (:1151-1157)
      uint4 *blk = reinterpret_cast<uint4 *>(voxels + (size_t)ptr * BS3) + lane;
      uint4 raw[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) raw[k] = ld_stream(blk + 32 * k);
      int empty = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        bool ch = false;
        int wd = (raw[k].x >> 16) & 0xff;
        if (wd <= maxWeight && wd > 0) { raw[k].x = 0x00007fffu; raw[k].y &= 0xff000000u; ch = true; wd = 0; }
        empty += (wd == 0);
        wd = (raw[k].z >> 16) & 0xff;
        if (wd <= maxWeight && wd > 0) { raw[k].z = 0x00007fffu; raw[k].w &= 0xff000000u; ch = true; wd = 0; }
        empty += (wd == 0);
        if (ch) st_stream(blk + 32 * k, raw[k]);
      }
      // block-wide count of empty voxels (replaces the 512-int shared-memory tree, ITMCUDAUtils.h:145-160)
      for (int o = 16; o > 0; o >>= 1) empty += __shfl_xor_sync(0xffffffffu, empty, o);
      claim = (empty == BS3);
    }
    if (lane == 0) {
      itemPtr[item] = claim ? ptr : -1;
      if (claim) {
        atomicMax(&delTag[ptr], del_tag(gen, (unsigned)item));
        if (MODE == 0) {   // remember the candidate: the commit ranks the few of them instead of scanning the whole list
          const int c = atomicAdd(&ctr->decayCand, 1);
          if (c < DECAY_CAND_CAP) candList[c] = item;
        }
      }
    }
  }
  if (MODE == 0) {
    // partial decay: the CTA that finishes last commits the pass (rank, elect, unlink, counters) — no second launch
    __shared__ bool lastCta;
    __shared__ unsigned smScan[33];
    __shared__ int smCand[DECAY_CAND_CAP];
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) lastCta = (atomicAdd(&ctr->decayCtasDone, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!lastCta) return;
    __threadfence();
    decay_commit_body(const_cast<b200_hash_entry *>(table), numBuckets, visType, ring, ringCap, s0, itemPtr, delTag, gen, allocList, delList,
                      isLeader, ctr, candList, smScan, smCand);
  }
}

// phase 2: ordered compaction of the claiming items, free-list push by rank (:1072-1073)
#define DEC_TILE 1024
__global__ void __launch_bounds__(256)
k_decay_rank(const int *itemPtr, const unsigned long long *delTag, unsigned gen, int *allocList, int *delList, DevCounters *ctr,
             unsigned long long *scanDesc, unsigned scanGen) {
  __shared__ unsigned sm[33];
  __shared__ unsigned tileBase;
  const int n = ctr->decayItems;
  const int lastFree = ctr->lastFreeBlockId;
  const int noTiles = (n + DEC_TILE - 1) / DEC_TILE;
  for (int tile = blockIdx.x; tile < noTiles; tile += gridDim.x) {
    const int first = tile * DEC_TILE + threadIdx.x * 4;
    unsigned mask = 0;
    int ptrs[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      ptrs[k] = -1;
      const int item = first + k;
      if (item < n) {
        const int p = itemPtr[item];
        if (p >= 0 && delTag[p] == del_tag(gen, (unsigned)item)) { mask |= 1u << k; ptrs[k] = p; }
      }
    }
    unsigned total;
    unsigned local = block_exclusive_scan(__popc(mask), sm, &total);
    if (threadIdx.x < 32) {
      unsigned ex = scan_lookback(scanDesc, scanGen, tile, total);
      if (threadIdx.x == 0) { tileBase = ex; if (tile == noTiles - 1) ctr->decayDeleted = (int)(ex + total); }
    }
    __syncthreads();
    unsigned r = tileBase + local;
#pragma unroll
    for (int k = 0; k < 4; ++k) if (mask & (1u << k)) {
      allocList[lastFree + 1 + (int)r] = ptrs[k];
      delList[r] = first + k;
      r++;
    }
    __syncthreads();
  }
  if (noTiles == 0 && blockIdx.x == 0 && threadIdx.x == 0) ctr->decayDeleted = 0;
}

// item position: MODE 0 = ring snapshot, MODE 1 = allocatedPos[VBA slot]
DEV void item_pos(int mode, const b200_vec3i *ring, long long ringCap, long long s0, const short4 *allocatedPos, int item, int &x, int &y,
                  int &z) {
  if (mode == 0) { const b200_vec3i p = ring[(s0 + item) % ringCap]; x = p.x; y = p.y; z = p.z; }
  else { const short4 p = allocatedPos[item]; x = p.x; y = p.y; z = p.z; }
}

// phase 3a: is deletion r the first (list order) deletion of its bucket chain? (read-only on the table)
DEV bool chain_leader(const b200_hash_entry *table, int numBuckets, int x, int y, int z, int item, const unsigned long long *delTag,
                      unsigned gen) {
  int idx = hash_index(x, y, z, numBuckets - 1);
  unsigned minItem = 0xffffffffu;
  for (;;) {
    const Entry en = load_entry_rw(table, idx);
    if (en.ptr >= 0) {
      const unsigned long long t = delTag[en.ptr];
      if ((unsigned)(t >> 32) == gen) { const unsigned it = 0xffffffffu - (unsigned)(t & 0xffffffffu); if (it < minItem) minItem = it; }
    }
    if (en.offset < 1) break;
    idx = numBuckets + en.offset - 1;
  }
  return minItem == (unsigned)item;
}

// phase 3b: the leader unlinks its chain's claimed blocks in list order — deleteBlock, Reco_CUDA.cu:1032-1111.
// Serial order = ascending list position: repeatedly take the chain entry whose block was claimed by the
// smallest item and unlink it on the evolving chain (findVoxel's idx / prev, :1032-1037).
DEV void unlink_chain(b200_hash_entry *table, int numBuckets, uint8_t *visType, int head, const unsigned long long *delTag, unsigned gen) {
  int *tw = reinterpret_cast<int *>(table);
  for (;;) {
    int found = -1, foundPrev = -1; unsigned best = 0xffffffffu;
    for (int idx = head, prev = -1;;) {
      const Entry en = load_entry_rw(table, idx);
      if (en.ptr >= 0) {
        const unsigned long long t = delTag[en.ptr];
        if ((unsigned)(t >> 32) == gen) {
          const unsigned it = 0xffffffffu - (unsigned)(t & 0xffffffffu);
          if (it < best) { best = it; found = idx; foundPrev = prev; }
        }
      }
      if (en.offset < 1) break;
      prev = idx;
      idx = numBuckets + en.offset - 1;
    }
    if (found < 0) break;
    const int prev = foundPrev;
    int *e = tw + (size_t)found * 5;
    if (prev == -1) {
      if (e[2] >= 1) {                       // ordered entry with a successor: pull the successor in
        const int nextIdx = numBuckets + e[2] - 1;
        int *nx = tw + (size_t)nextIdx * 5;
        e[0] = nx[0]; e[1] = nx[1]; e[2] = nx[2]; e[3] = nx[3]; e[4] = nx[4];
        visType[found] = visType[nextIdx];
        visType[nextIdx] = 0;
        nx[2] = 0; nx[3] = -2;
      } else {                               // ordered entry, no successor
        e[3] = -2;
        visType[found] = 0;
      }
    } else {                                 // excess entry: predecessor inherits the link
      int *pv = tw + (size_t)prev * 5;
      pv[2] = e[2];
      e[2] = 0; e[3] = -2;
      visType[prev] = visType[found];        // (sic) reference quirk, :1109-1110
      visType[found] = 0;
    }
  }
}

template <int MODE>
__global__ void k_decay_elect(const b200_hash_entry *table, int numBuckets, const b200_vec3i *ring, long long ringCap,
                              const long long *snapStart, int slot, const short4 *allocatedPos, const int *delList,
                              const unsigned long long *delTag, unsigned gen, uint8_t *isLeader, const DevCounters *ctr) {
  const int nDel = ctr->decayDeleted;
  const long long s0 = (MODE == 0) ? snapStart[slot] : 0;
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nDel; r += gridDim.x * blockDim.x) {
    const int item = delList[r];
    int x, y, z;
    item_pos(MODE, ring, ringCap, s0, allocatedPos, item, x, y, z);
    isLeader[r] = chain_leader(table, numBuckets, x, y, z, item, delTag, gen) ? 1 : 0;
  }
}

__global__ void k_decay_unlink(b200_hash_entry *table, int numBuckets, uint8_t *visType, const b200_vec3i *ring, long long ringCap,
                               const long long *snapStart, int slot, const short4 *allocatedPos, int mode, const int *delList,
                               const unsigned long long *delTag, unsigned gen, const uint8_t *isLeader, DevCounters *ctr) {
  const int nDel = ctr->decayDeleted;
  const long long s0 = (mode == 0) ? snapStart[slot] : 0;
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nDel; r += gridDim.x * blockDim.x) {
    if (!isLeader[r]) continue;
    int x, y, z;
    item_pos(mode, ring, ringCap, s0, allocatedPos, delList[r], x, y, z);
    unlink_chain(table, numBuckets, visType, hash_index(x, y, z, numBuckets - 1), delTag, gen);
  }
}

// phases 2 + 3 + counters of a PARTIAL decay, run by the LAST CTA of the sweep (k_decay_blocks<0>) — a frame's list is a few
// thousand items and the few dozen blocks it empties are known as unordered candidates by then; a second launch for this cost
// 13 us of the frame. Ordered compaction of the claims, leader election, chain unlinking, counter update. All threads of the
// calling CTA take part; reads of what other CTAs produced go to L2 (__ldcg).
__device__ void decay_commit_body(b200_hash_entry *table, int numBuckets, uint8_t *visType, const b200_vec3i *ring, long long ringCap, long long s0,
                                  const int *itemPtr, const unsigned long long *delTag, unsigned gen, int *allocList, int *delList,
                                  uint8_t *isLeader, DevCounters *ctr, const int *candList, unsigned *sm, int *cand) {
  const int n = *(volatile int *)&ctr->decayItems;
  const int lastFree = *(volatile int *)&ctr->lastFreeBlockId;
  const int nc = *(volatile int *)&ctr->decayCand;
  unsigned running = 0;
  if (nc <= DECAY_CAND_CAP) {
    // Few candidates (a few dozen per frame): keep the winners of the block claims and rank them by list position by
    // counting — the same order the scan over the whole list produces, without walking the list.
    for (int c = threadIdx.x; c < DECAY_CAND_CAP; c += blockDim.x) {
      int v = 0x7fffffff;
      if (c < nc) {
        const int item = __ldcg(candList + c);
        const int ptr = __ldcg(itemPtr + item);
        if (ptr >= 0 && __ldcg(delTag + ptr) == del_tag(gen, (unsigned)item)) v = item;
      }
      cand[c] = v;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < nc; c += blockDim.x) {
      const int v = cand[c];
      if (v == 0x7fffffff) continue;
      int r = 0;
      for (int j = 0; j < nc; ++j) r += (cand[j] < v);
      allocList[lastFree + 1 + r] = __ldcg(itemPtr + v);      // free-list push by list position (:1072-1073)
      delList[r] = v;
    }
    int mine = 0;
    for (int c = threadIdx.x; c < nc; c += blockDim.x) mine += (cand[c] != 0x7fffffff);
    unsigned tot;
    block_exclusive_scan((unsigned)mine, sm, &tot);   // (its barriers also order the writes above before the election below)
    running = tot;
  } else
  for (int base = 0; base < n; base += blockDim.x) {
    const int item = base + threadIdx.x;
    int ptr = -1;
    if (item < n) { ptr = __ldcg(itemPtr + item); if (ptr >= 0 && __ldcg(delTag + ptr) != del_tag(gen, (unsigned)item)) ptr = -1; }
    unsigned total;
    const unsigned r = running + block_exclusive_scan(ptr >= 0 ? 1u : 0u, sm, &total);
    if (ptr >= 0) { allocList[lastFree + 1 + (int)r] = ptr; delList[r] = item; }   // free-list push by list position (:1072-1073)
    running += total;
  }
  const int nDel = (int)running;
  __syncthreads();
  for (int r = threadIdx.x; r < nDel; r += blockDim.x) {
    int x, y, z;
    const int item = delList[r];
    item_pos(0, ring, ringCap, s0, nullptr, item, x, y, z);
    isLeader[r] = chain_leader(table, numBuckets, x, y, z, item, delTag, gen) ? 1 : 0;
  }
  __syncthreads();
  for (int r = threadIdx.x; r < nDel; r += blockDim.x) {
    if (!isLeader[r]) continue;
    int x, y, z;
    item_pos(0, ring, ringCap, s0, nullptr, delList[r], x, y, z);
    unlink_chain(table, numBuckets, visType, hash_index(x, y, z, numBuckets - 1), delTag, gen);
  }
  if (threadIdx.x == 0) {
    ctr->lastFreeBlockId = lastFree + nDel;
    ctr->freedLastDecay = nDel;
    ctr->totalDecayed += nDel;
    ctr->decayDeleted = 0;
    ctr->decayItems = 0;
    ctr->decayCand = 0;
    ctr->decayCtasDone = 0;
  }
}

// finalise: lastFreeBlockId += deleted; freedLastDecay
__global__ void k_decay_finish(DevCounters *ctr) {
  ctr->lastFreeBlockId += ctr->decayDeleted;
  ctr->freedLastDecay = ctr->decayDeleted;
  ctr->totalDecayed += ctr->decayDeleted;
  ctr->decayDeleted = 0;
  ctr->decayItems = 0;
}

// findAllocatedBlocks — ITMMeshingEngine_CUDA.cu:96-114 (after a zero fill)
__global__ void k_find_allocated(const b200_hash_entry *__restrict__ table, int noTotal, short4 *allocatedPos) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < noTotal; i += gridDim.x * blockDim.x) {
    Entry en = load_entry(table, i);
    if (en.ptr >= 0) allocatedPos[en.ptr] = make_short4((short)en.x, (short)en.y, (short)en.z, 1);
  }
}

// b200_diag_push_decay_snapshot / b200_checkpoint_load: n caller positions appended to the ring as snapshot `slot` (one CTA:
// the cursor is read before and moved after every item is written). n == -1: a snapshot that is already overwritten — it
// starts more than ringCap items behind the cursor and takes no room, so k_decay_blocks sweeps nothing for it.
__global__ void k_push_snapshot(const b200_vec3i *positions, int n, b200_vec3i *ring, long long ringCap, long long *snapStart,
                                int *snapCount, int slot, DevCounters *ctr) {
  const long long ringStart = ctr->ringHead;
  if (n < 0) {
    if (threadIdx.x == 0) { snapStart[slot] = ringStart - ringCap - 1; snapCount[slot] = 0; }
    return;
  }
  for (int i = threadIdx.x; i < n; i += blockDim.x) ring[(ringStart + i) % ringCap] = positions[i];
  __syncthreads();
  if (threadIdx.x == 0) publish_snapshot(ctr, snapStart, snapCount, slot, ringStart, n);
}

void launch_push_snapshot(b200_engine *e, const b200_vec3i *positions, int n, int snapSlot) {
  k_push_snapshot<<<1, 256, 0, e->stream>>>(positions, n, e->d_ring, e->ringCap, e->d_snapStart, e->d_snapCount, snapSlot, e->d_ctr);
  e->launches++;
}

static void decay_common(b200_engine *e, const SceneRef &s, int mode, int slot, int minAge, int maxWeight, int frameIdx,
                         long long items, bool fused = false) {
  cudaStream_t st = e->stream;
  const unsigned gen = ++e->decayGen;
  const int grid1 = persistent_grid(e, 6, (items + 7) / 8);   // 8 items (warps) per CTA
  if (mode == 0) {
    trace_begin(e, st, "k_decay_blocks<0>");
    launch_chained(fused, k_decay_blocks<0>, grid1, 256, 0, st, s.voxels, s.hash, s.numBuckets, e->d_ring, e->ringCap, e->d_snapStart,
                   e->d_snapCount, slot, e->d_allocatedPos, s.numBlocks, minAge, maxWeight, frameIdx, gen, e->d_delTag, e->d_itemPtr,
                   e->d_ctr, e->d_candList, s.visType, s.allocationList, e->d_delList, e->d_isLeader,
                   fused ? span_slot(e, SPAN_DECAY) : nullptr);
    trace_end(e, st);
  } else {
    trace_begin(e, st, "k_decay_blocks<1>");
    k_decay_blocks<1><<<grid1, 256, 0, st>>>(s.voxels, s.hash, s.numBuckets, e->d_ring, e->ringCap, e->d_snapStart, e->d_snapCount,
                                            slot, e->d_allocatedPos, s.numBlocks, minAge, maxWeight, frameIdx, gen, e->d_delTag,
                                            e->d_itemPtr, e->d_ctr, e->d_candList, s.visType, s.allocationList, e->d_delList, e->d_isLeader,
                                            nullptr);
    trace_end(e, st);
  }
  if (mode == 0) { e->launches += 1; return; }   // the sweep's last CTA has committed the pass
  const int noTiles = (int)((items + DEC_TILE - 1) / DEC_TILE);
  k_decay_rank<<<persistent_grid(e, 4, noTiles), 256, 0, st>>>(e->d_itemPtr, e->d_delTag, gen, s.allocationList, e->d_delList,
                                                               e->d_ctr, e->d_scanDesc, ++e->scanGen);
  k_decay_elect<1><<<e->smCount, 128, 0, st>>>(s.hash, s.numBuckets, e->d_ring, e->ringCap, e->d_snapStart, slot, e->d_allocatedPos,
                                              e->d_delList, e->d_delTag, gen, e->d_isLeader, e->d_ctr);
  k_decay_unlink<<<e->smCount, 128, 0, st>>>(s.hash, s.numBuckets, s.visType, e->d_ring, e->ringCap, e->d_snapStart, slot,
                                            e->d_allocatedPos, mode, e->d_delList, e->d_delTag, gen, e->d_isLeader, e->d_ctr);
  k_decay_finish<<<1, 1, 0, st>>>(e->d_ctr);
  e->launches += 5;
}

void launch_decay_partial(b200_engine *e, const SceneRef &s, int snapSlot, int minAge, int maxWeight, int frameIdx, bool fused) {
  // item count lives on the device (snapCount[slot]); size the grid for the capacity
  decay_common(e, s, 0, snapSlot, minAge, maxWeight, frameIdx, s.numBlocks, fused);
}

void launch_decay_full(b200_engine *e, const SceneRef &s, int minAge, int maxWeight, int frameIdx) {
  cudaMemsetAsync(e->d_allocatedPos, 0, sizeof(short4) * (size_t)s.numBlocks, e->stream);
  k_find_allocated<<<e->smCount * 8, 256, 0, e->stream>>>(s.hash, s.noTotal, e->d_allocatedPos);
  e->launches++;
  decay_common(e, s, 1, 0, minAge, maxWeight, frameIdx, s.numBlocks);
}
