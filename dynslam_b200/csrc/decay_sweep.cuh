// decay_sweep.cuh — the per-item sweep of voxel Decay (decayVoxel, reference ITMSceneReconstructionEngine_CUDA.cu:1120-1197),
// shared by the decay kernels (decay.cu) and by the sweep CTAs that a partial Decay adds to the fused frame's raycast grid
// (vis.cu).
#pragma once
#include "engine.h"

DEV unsigned long long del_tag(unsigned gen, unsigned item) { return ((unsigned long long)gen << 32) | (0xffffffffu - item); }

// The reset rule of decayVoxel (:1151-1162) on the two voxels of one uint4: a voxel of weight 1..maxWeight gets sdf 32767 and
// weight 0, and keeps only its colour bytes' top byte. A function of the old voxel only. Returns whether v changed; `empty`
// counts the voxels whose weight is 0 afterwards.
DEV bool decay_reset_pair(uint4 &v, int maxWeight, int &empty) {
  bool ch = false;
  int wd = (v.x >> 16) & 0xff;
  if (wd <= maxWeight && wd > 0) { v.x = 0x00007fffu; v.y &= 0xff000000u; ch = true; wd = 0; }
  empty += (wd == 0);
  wd = (v.z >> 16) & 0xff;
  if (wd <= maxWeight && wd > 0) { v.z = 0x00007fffu; v.w &= 0xff000000u; ch = true; wd = 0; }
  empty += (wd == 0);
  return ch;
}

// Sweep over the items of a decay pass, one WARP per item (a block = 256 uint4 = 8 per lane, all 8 loads in flight): items
// warp, warp + warps, ... The per-item chain of dependent loads (item position -> hash chain -> voxels) overlaps across warps.
// Per item: resolve the block (findBlock / findVoxel, :1214, :1138), apply the reset rule to its voxels if the block is old
// enough (safeToClear, :1151-1157) and vote whether the block is then empty; the first item (list order) that empties a block
// claims it with a 64-bit atomicMax tag.
//   MODE 1 (full decay, items = VBA slots with allocatedPos.w != 0): the reset voxels are stored in place.
//   MODE 0 (partial decay, items = ring snapshot d.slot): nothing is stored to the voxels or the table, so the sweep may run
//     beside kernels that read them (the fused frame's raycast). Per item it records in resetPtr the block's VBA pointer when
//     the rule changes any of its voxels (else -1); k_decay_commit replays the rule from there, and commits the pass.
template <int MODE>
DEV void decay_sweep(const DecaySweep &d, int warp, int warps) {
  const int lane = threadIdx.x & 31;
  int n = (MODE == 0) ? d.snapCount[d.slot] : d.numBlocks;
  const long long s0 = (MODE == 0) ? d.snapStart[d.slot] : 0;
  // a snapshot the ring has wrapped over since it was taken is gone (b200_engine_config.decayRingItems): sweep nothing
  const bool overwritten = (MODE == 0) && (d.ctr->ringHead - s0 > d.ringCap);
  if (overwritten) n = 0;
  if (warp == 0 && lane == 0) { d.ctr->decayItems = n; if (overwritten) d.ctr->droppedSnapshots++; }
  for (int item = warp; item < n; item += warps) {
    int x, y, z;
    if (MODE == 0) { b200_vec3i p = d.ring[(s0 + item) % d.ringCap]; x = p.x; y = p.y; z = p.z; }
    else {
      short4 p = d.allocatedPos[item];
      if (p.w == 0) { if (lane == 0) d.itemPtr[item] = -1; continue; }
      x = p.x; y = p.y; z = p.z;
    }
    int idx = hash_index(x, y, z, d.numBuckets - 1), ptr = -1, allocatedTime = 0;
    for (;;) {
      const int *w = reinterpret_cast<const int *>(d.table) + (size_t)idx * 5;
      int w0 = w[0], w1 = w[1], off = w[2], p = w[3];
      if ((short)(w0 & 0xffff) == x && (short)(w0 >> 16) == y && (short)(w1 & 0xffff) == z && p >= 0) {
        ptr = p; allocatedTime = w[4]; break;
      }
      if (off < 1) break;
      idx = d.numBuckets + off - 1;
    }
    bool claim = false, reset = false;
    if (ptr >= 0 && (d.currentFrame - allocatedTime) >= d.minAge) {
      uint4 *blk = reinterpret_cast<uint4 *>(d.voxels + (size_t)ptr * BS3) + lane;
      uint4 raw[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) raw[k] = ld_stream(blk + 32 * k);
      int empty = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const bool ch = decay_reset_pair(raw[k], d.maxWeight, empty);
        if (MODE == 1 && ch) st_stream(blk + 32 * k, raw[k]);
        reset |= ch;
      }
      // block-wide count of empty voxels (replaces the 512-int shared-memory tree, ITMCUDAUtils.h:145-160)
      for (int o = 16; o > 0; o >>= 1) empty += __shfl_xor_sync(0xffffffffu, empty, o);
      claim = (empty == BS3);
      if (MODE == 0) reset = __any_sync(0xffffffffu, reset);
    }
    if (lane == 0) {
      d.itemPtr[item] = claim ? ptr : -1;
      if (MODE == 0) {
        d.resetPtr[item] = reset ? ptr : -1;
        // diagnostic counter (a hundred or so flagged blocks per pass: an atomic each, no register held across the loop)
        if (reset) atomicAdd((unsigned long long *)&d.ctr->decayReplays, 1ull);
      }
      if (claim) {
        atomicMax(&d.delTag[ptr], del_tag(d.gen, (unsigned)item));
        if (MODE == 0) {   // remember the candidate: the commit ranks the few of them instead of scanning the whole list
          const int c = atomicAdd(&d.ctr->decayCand, 1);
          if (c < DECAY_CAND_CAP) d.candList[c] = item;
        }
      }
    }
  }
}
