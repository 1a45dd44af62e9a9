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
//   phase 1  the sweep (decay_sweep.cuh), one warp per list item: resolve the block once, read its 4 KiB with 128-bit loads,
//            apply the reset rule, decide "block is empty" with a warp-wide vote; the first item (list order) that empties a
//            block claims it with a 64-bit atomicMax tag. A full decay stores the resets as it goes; a partial one only
//            records which blocks have voxels to reset, and k_decay_commit stores them;
//   phase 2  ordered compaction of the claiming items => free-list position = rank in list order;
//   phase 3  chain leaders: for every bucket chain that loses blocks, ONE thread applies that
//            chain's deletions in list order with the reference's unlink rules (incl. the
//            visibility-byte moves and the never-reclaimed excess slots, :1075-1111).
#include "decay_sweep.cuh"

DEV void item_pos(int mode, const b200_vec3i *ring, long long ringCap, long long s0, const short4 *allocatedPos, int item, int &x, int &y, int &z);
DEV bool chain_leader(const b200_hash_entry *table, int numBuckets, int x, int y, int z, int item, const unsigned long long *delTag, unsigned gen);
DEV void unlink_chain(b200_hash_entry *table, int numBuckets, uint8_t *visType, int head, const unsigned long long *delTag, unsigned gen);
__device__ void decay_commit_body(b200_hash_entry *table, int numBuckets, uint8_t *visType, const b200_vec3i *ring, long long ringCap, long long s0,
                                  const int *itemPtr, const unsigned long long *delTag, unsigned gen, int *allocList, int *delList,
                                  uint8_t *isLeader, DevCounters *ctr, const int *candList, unsigned *sm, int *cand);

// phase 1 as a grid of its own: full decay (MODE 1), and a partial one (MODE 0) when no raycast carries its sweep
template <int MODE>
__global__ void __launch_bounds__(256) k_decay_sweep(DecaySweep d) {
  pdl_wait();            // in a fused frame without a raycast: the integrate kernel writes the voxels this sweep reads
  pdl_trigger();
  SpanStamp stamp(d.span);
  decay_sweep<MODE>(d, (blockIdx.x * blockDim.x + threadIdx.x) >> 5, gridDim.x * (blockDim.x >> 5));
}

// Partial decay, after everything that reads the voxels: the reset stores of the sweep and phases 2 + 3 + counters, side by side.
// The two touch disjoint memory — the replay writes only the voxels of flagged blocks, the commit reads the claims and writes
// the table, the visibility bytes, the free list and the decay scratch — so neither waits for the other. CTA 0 commits the pass
// as soon as it is past the dependency wait (a chain of dependent L2 round trips in one CTA, the longer of the two); the other
// CTAs replay: a warp per item the sweep flagged reloads its block and applies the reset rule again. Nothing has written those
// voxels since the sweep read them, so the rule changes the same voxels to the same bits. decayItems, which every CTA reads, is
// cleared by the CTA that finishes last (an arrival count: no CTA waits on another).
__global__ void __launch_bounds__(256)
k_decay_commit(b200_voxel *voxels, int maxWeight, const int *resetPtr, b200_hash_entry *table, int numBuckets, const b200_vec3i *ring,
               long long ringCap, const long long *snapStart, int slot, unsigned gen, const unsigned long long *delTag, const int *itemPtr,
               DevCounters *ctr, const int *candList, uint8_t *visType, int *allocList, int *delList, uint8_t *isLeader,
               unsigned long long *span, unsigned long long *commitSpan) {
  pdl_wait();            // in the fused frame: the raycast reads the voxels and entries this kernel resets and unlinks
  SpanStamp stamp(span);
  __shared__ bool lastCta;
  __shared__ unsigned smScan[33];
  __shared__ int smCand[DECAY_CAND_CAP];
  if (blockIdx.x == 0) {
    SpanStamp commitStamp(commitSpan);
    decay_commit_body(table, numBuckets, visType, ring, ringCap, snapStart[slot], itemPtr, delTag, gen, allocList, delList, isLeader, ctr,
                      candList, smScan, smCand);
  }
  const int first = gridDim.x > 1 ? 1 : 0;   // the replaying CTAs: all but CTA 0, or CTA 0 alone on a grid of one
  if ((int)blockIdx.x >= first) {
    const int lane = threadIdx.x & 31;
    const int warps = (gridDim.x - first) * (blockDim.x >> 5), warp = ((blockIdx.x - first) * blockDim.x + threadIdx.x) >> 5;
    const int n = *(volatile int *)&ctr->decayItems;
    for (int item = warp; item < n; item += warps) {
      const int ptr = resetPtr[item];
      if (ptr < 0) continue;
      uint4 *blk = reinterpret_cast<uint4 *>(voxels + (size_t)ptr * BS3) + lane;
      uint4 raw[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) raw[k] = ld_stream(blk + 32 * k);
      int empty = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) if (decay_reset_pair(raw[k], maxWeight, empty)) st_stream(blk + 32 * k, raw[k]);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) lastCta = (atomicAdd(&ctr->decayCtasDone, 1u) == gridDim.x - 1);
  __syncthreads();
  if (lastCta && threadIdx.x == 0) { ctr->decayItems = 0; ctr->decayCtasDone = 0; }
}

// phase 2: ordered compaction of the claiming items, free-list push by rank (:1072-1073)
#define DEC_TILE 1024
__global__ void __launch_bounds__(256)
k_decay_rank(const int *itemPtr, const unsigned long long *delTag, unsigned gen, int *allocList, int *delList, DevCounters *ctr,
             unsigned long long *scanDesc, unsigned scanGen) {
  __shared__ unsigned sm[33];
  __shared__ unsigned tileBase;
  __shared__ int sTile;
  const int n = ctr->decayItems;
  const int lastFree = ctr->lastFreeBlockId;
  const int noTiles = (n + DEC_TILE - 1) / DEC_TILE;
  unsigned *ticket = &ctr->ticket[TK_DECAY_RANK];
  for (int tile = draw_tile(ticket, noTiles, &sTile); tile < noTiles; tile = draw_tile(ticket, noTiles, &sTile)) {
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

// phases 2 + 3 + counters of a PARTIAL decay, run by CTA 0 of k_decay_commit — a frame's list is a few thousand items
// and the few dozen blocks it empties are known as unordered candidates by then; a launch of its own for this cost 13 us of
// the frame. Ordered compaction of the claims, leader election, chain unlinking, counter update. All threads of the
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
    ctr->decayCand = 0;   // (decayItems and decayCtasDone: k_decay_commit's last CTA)
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

DecaySweep decay_sweep_args(b200_engine *e, const SceneRef &s, int snapSlot, int minAge, int maxWeight, int frameIdx, bool fused) {
  DecaySweep d;
  d.voxels = s.voxels; d.table = s.hash; d.numBuckets = s.numBuckets; d.numBlocks = s.numBlocks;
  d.ring = e->d_ring; d.ringCap = e->ringCap; d.snapStart = e->d_snapStart; d.snapCount = e->d_snapCount; d.slot = snapSlot;
  d.allocatedPos = e->d_allocatedPos;
  d.minAge = minAge; d.maxWeight = maxWeight; d.currentFrame = frameIdx; d.gen = ++e->decayGen;
  d.delTag = e->d_delTag; d.itemPtr = e->d_itemPtr; d.resetPtr = e->d_resetPtr; d.candList = e->d_candList; d.ctr = e->d_ctr;
  d.span = fused ? span_slot(e, SPAN_SWEEP) : nullptr;
  return d;
}

// 8 items (warps) per CTA; the item count lives on the device (snapCount[slot]), so the grid is sized for the capacity
static int sweep_grid(const b200_engine *e, const SceneRef &s) { return persistent_grid(e, 6, ((long long)s.numBlocks + 7) / 8); }

void launch_decay_partial(b200_engine *e, const SceneRef &s, const DecaySweep &d, bool swept, bool fused) {
  cudaStream_t st = e->stream;
  if (!swept) {
    trace_begin(e, st, "k_decay_sweep<0>");
    launch_chained(fused, k_decay_sweep<0>, sweep_grid(e, s), 256, 0, st, d);
    trace_end(e, st);
    e->launches++;
  }
  trace_begin(e, st, "k_decay_commit");
  launch_chained(fused, k_decay_commit, persistent_grid(e, 2, ((long long)s.numBlocks + 7) / 8), 256, 0, st, s.voxels, d.maxWeight,
                 (const int *)e->d_resetPtr, s.hash, s.numBuckets, (const b200_vec3i *)e->d_ring, e->ringCap, (const long long *)e->d_snapStart,
                 d.slot, d.gen, (const unsigned long long *)e->d_delTag, (const int *)e->d_itemPtr, e->d_ctr, (const int *)e->d_candList,
                 s.visType, s.allocationList, e->d_delList, e->d_isLeader, fused ? span_slot(e, SPAN_DECAY) : nullptr,
                 fused ? span_slot(e, SPAN_COMMIT) : nullptr);
  trace_end(e, st);
  e->launches++;
}

void launch_decay_full(b200_engine *e, const SceneRef &s, int minAge, int maxWeight, int frameIdx) {
  cudaStream_t st = e->stream;
  cudaMemsetAsync(e->d_allocatedPos, 0, sizeof(short4) * (size_t)s.numBlocks, st);
  k_find_allocated<<<e->smCount * 8, 256, 0, st>>>(s.hash, s.noTotal, e->d_allocatedPos);
  const DecaySweep d = decay_sweep_args(e, s, 0, minAge, maxWeight, frameIdx);
  const unsigned gen = d.gen;
  trace_begin(e, st, "k_decay_sweep<1>");
  k_decay_sweep<1><<<sweep_grid(e, s), 256, 0, st>>>(d);
  trace_end(e, st);
  const int noTiles = (s.numBlocks + DEC_TILE - 1) / DEC_TILE;
  k_decay_rank<<<ticket_grid(e, 4, noTiles), 256, 0, st>>>(e->d_itemPtr, e->d_delTag, gen, s.allocationList, e->d_delList,
                                                               e->d_ctr, e->d_scanDesc, ++e->scanGen);
  k_decay_elect<1><<<e->smCount, 128, 0, st>>>(s.hash, s.numBuckets, e->d_ring, e->ringCap, e->d_snapStart, 0, e->d_allocatedPos,
                                              e->d_delList, e->d_delTag, gen, e->d_isLeader, e->d_ctr);
  k_decay_unlink<<<e->smCount, 128, 0, st>>>(s.hash, s.numBuckets, s.visType, e->d_ring, e->ringCap, e->d_snapStart, 0,
                                            e->d_allocatedPos, 1, e->d_delList, e->d_delTag, gen, e->d_isLeader, e->d_ctr);
  k_decay_finish<<<1, 1, 0, st>>>(e->d_ctr);
  e->launches += 6;
}
