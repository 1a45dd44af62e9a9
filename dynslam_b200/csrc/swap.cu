// swap.cu — device half of ITMSwappingEngine for sm_90a (host<->device streaming of voxel blocks).
//
// Replaces buildListToSwapIn/Out_device, integrateOldIntoActiveData_device,
// moveActiveDataToTransferBuffer_device and cleanMemory_device (reference
// ITMSwappingEngine_CUDA.cu:218-330) and combineVoxel{Depth,Color}Information
// (DeviceAgnostic/ITMSwappingEngine.h:7-63). DynSLAM runs with swapping disabled
// (Utils/ITMLibSettings.cpp:50-55 throws when it is enabled); the interface is kept complete.
// Lists are ordered compactions (ascending entry index, the serial CPU engine's order,
// CPU/ITMSwappingEngine_CPU.cpp), free-list pushes are by list position.
#include "engine.h"

#define SWAP_TILE (256 * 16)
// MODE 0: swap-in list (state == 1); MODE 1: swap-out list (state == 2 && ptr >= 0 && invisible)
template <int MODE>
__global__ void __launch_bounds__(256)
k_swap_list(const uint8_t *__restrict__ swapStates, const b200_hash_entry *__restrict__ table, const uint8_t *__restrict__ visType,
            int noTotal, int *needed, DevCounters *ctr, unsigned long long *scanDesc, unsigned gen) {
  __shared__ unsigned sm[33];
  __shared__ unsigned tileBase;
  __shared__ int sTile;
  const int noTiles = (noTotal + SWAP_TILE - 1) / SWAP_TILE;
  unsigned *ticket = &ctr->ticket[TK_SWAP_LIST];
  for (int tile = draw_tile(ticket, noTiles, &sTile); tile < noTiles; tile = draw_tile(ticket, noTiles, &sTile)) {
    const int first = tile * SWAP_TILE + threadIdx.x * 16;
    unsigned mask = 0;
    for (int k = 0; k < 16; ++k) {
      const int idx = first + k;
      if (idx >= noTotal) break;
      const uint8_t st = swapStates[idx];
      if (MODE == 0) { if (st == 1) mask |= 1u << k; }
      else if (st == 2) {
        Entry en = load_entry(table, idx);
        if (en.ptr >= 0 && visType[idx] == 0) mask |= 1u << k;
      }
    }
    unsigned total;
    unsigned local = block_exclusive_scan(__popc(mask), sm, &total);
    if (threadIdx.x < 32) {
      unsigned ex = scan_lookback(scanDesc, gen, tile, total);
      if (threadIdx.x == 0) {
        tileBase = ex;
        if (tile == noTiles - 1) { int n = (int)(ex + total); ctr->noNeededEntries = n < B200_TRANSFER_BLOCK_NUM ? n : B200_TRANSFER_BLOCK_NUM; }
      }
    }
    __syncthreads();
    unsigned o = tileBase + local;
    while (mask) {
      const int k = __ffs(mask) - 1;
      mask &= mask - 1;
      if (o < B200_TRANSFER_BLOCK_NUM) needed[o] = first + k;
      o++;
    }
  }
}

void launch_swap_list_in(b200_engine *e, const SceneRef &s, int *needed) {
  const int noTiles = (s.noTotal + SWAP_TILE - 1) / SWAP_TILE;
  k_swap_list<0><<<ticket_grid(e, 4, noTiles), 256, 0, e->stream>>>(s.swapStates, s.hash, s.visType, s.noTotal, needed, e->d_ctr,
                                                                       e->d_scanDesc, ++e->scanGen);
  e->launches++;
}
void launch_swap_list_out(b200_engine *e, const SceneRef &s, int *needed) {
  const int noTiles = (s.noTotal + SWAP_TILE - 1) / SWAP_TILE;
  k_swap_list<1><<<ticket_grid(e, 4, noTiles), 256, 0, e->stream>>>(s.swapStates, s.hash, s.visType, s.noTotal, needed, e->d_ctr,
                                                                       e->d_scanDesc, ++e->scanGen);
  e->launches++;
}

DEV int to_uchar_round_s(float x) { return clampi_((int)round_(x), 0, 255); }

// CombineVoxelInformation<true,TVoxel>::compute on packed words (src -> dst)
DEV void combine(unsigned slo, unsigned shi, unsigned &dlo, unsigned &dhi, int maxW) {
  {
    int newW = (dlo >> 16) & 0xff, oldW = (slo >> 16) & 0xff;
    float newF = (float)((short)(dlo & 0xffff)) / 32767.0f, oldF = (float)((short)(slo & 0xffff)) / 32767.0f;
    if (oldW != 0) {
      newF = oldW * oldF + newW * newF; newW = oldW + newW; newF /= newW; newW = mini_(newW, maxW);
      const int sdf = (short)((newF) * 32767.0f);
      dlo = (dlo & 0xff000000u) | ((unsigned)(newW & 0xff) << 16) | ((unsigned)sdf & 0xffffu);
    }
  }
  {
    int newW = (dhi >> 16) & 0xff, oldW = (shi >> 16) & 0xff;
    if (oldW != 0) {
      float n0 = (float)((dlo >> 24) & 0xff) / 255.0f, n1 = (float)(dhi & 0xff) / 255.0f, n2 = (float)((dhi >> 8) & 0xff) / 255.0f;
      const float o0 = (float)((slo >> 24) & 0xff) / 255.0f, o1 = (float)(shi & 0xff) / 255.0f, o2 = (float)((shi >> 8) & 0xff) / 255.0f;
      n0 = o0 * (float)oldW + n0 * (float)newW; n1 = o1 * (float)oldW + n1 * (float)newW; n2 = o2 * (float)oldW + n2 * (float)newW;
      newW = oldW + newW;
      n0 /= (float)newW; n1 /= (float)newW; n2 /= (float)newW;
      newW = mini_(newW, maxW);
      const int c0 = to_uchar_round_s(n0 * 255.0f), c1 = to_uchar_round_s(n1 * 255.0f), c2 = to_uchar_round_s(n2 * 255.0f);
      dlo = (dlo & 0x00ffffffu) | ((unsigned)c0 << 24);
      dhi = (dhi & 0xff000000u) | (unsigned)c1 | ((unsigned)c2 << 8) | ((unsigned)(newW & 0xff) << 16);
    }
  }
}

__global__ void __launch_bounds__(256)
k_swap_integrate_in(b200_voxel *voxels, const b200_hash_entry *table, uint8_t *swapStates, const b200_voxel *synced, const int *needed,
                    int n, int maxW) {
  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    const int entryDestId = needed[i];
    const int ptr = reinterpret_cast<const int *>(table)[(size_t)entryDestId * 5 + 3];
    const uint4 src = reinterpret_cast<const uint4 *>(synced + (size_t)i * BS3)[threadIdx.x];
    uint4 *dp = reinterpret_cast<uint4 *>(voxels + (size_t)ptr * BS3) + threadIdx.x;
    uint4 dst = *dp;
    combine(src.x, src.y, dst.x, dst.y, maxW);
    combine(src.z, src.w, dst.z, dst.w, maxW);
    *dp = dst;
    if (threadIdx.x == 0) swapStates[entryDestId] = 2;
  }
}

void launch_swap_integrate_in(b200_engine *e, const SceneRef &s, const b200_voxel *synced, const int *needed, int n, int maxW) {
  if (n <= 0) return;
  k_swap_integrate_in<<<persistent_grid(e, 4, n), 256, 0, e->stream>>>(s.voxels, s.hash, s.swapStates, synced, needed, n, maxW);
  e->launches++;
}

// moveActiveDataToTransferBuffer + cleanMemory; free-list position = list position (serial order)
__global__ void __launch_bounds__(256)
k_swap_move_out(b200_voxel *voxels, b200_hash_entry *table, uint8_t *swapStates, b200_voxel *synced, uint8_t *hasSynced, const int *needed,
                int n, int *allocList, int numBlocks, DevCounters *ctr) {
  const int lastFree = ctr->lastFreeBlockId;
  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    const int id = needed[i];
    int *ew = reinterpret_cast<int *>(table) + (size_t)id * 5;
    const int ptr = ew[3];
    uint4 *sp = reinterpret_cast<uint4 *>(voxels + (size_t)ptr * BS3) + threadIdx.x;
    reinterpret_cast<uint4 *>(synced + (size_t)i * BS3)[threadIdx.x] = *sp;
    *sp = make_uint4(0x00007fffu, 0u, 0x00007fffu, 0u);
    __syncthreads();
    if (threadIdx.x == 0) {
      hasSynced[i] = 1;
      swapStates[id] = 0;
      const int vbaIdx = lastFree + i;
      if (vbaIdx < numBlocks - 1) { allocList[vbaIdx + 1] = ptr; ew[3] = -1; }
    }
    __syncthreads();
  }
}

__global__ void k_swap_finish(DevCounters *ctr, int n, int numBlocks) {
  int c = ctr->lastFreeBlockId + n;
  if (c < 0) c = 0;
  if (c > numBlocks) c = numBlocks;
  ctr->lastFreeBlockId = c;
}

void launch_swap_move_out(b200_engine *e, const SceneRef &s, b200_voxel *synced, uint8_t *hasSynced, const int *needed, int n) {
  if (n <= 0) return;
  k_swap_move_out<<<persistent_grid(e, 4, n), 256, 0, e->stream>>>(s.voxels, s.hash, s.swapStates, synced, hasSynced, needed, n,
                                                                  s.allocationList, s.numBlocks, e->d_ctr);
  k_swap_finish<<<1, 1, 0, e->stream>>>(e->d_ctr, n, s.numBlocks);
  e->launches += 2;
}
