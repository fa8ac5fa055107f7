// ksg_log.cuh — `merged`: the update log (ksg_set_update_log), written by a pass over the frame's sorted update records.
//
// The `fast` tile kernel writes its log entries itself (ksg_fast.cuh).  The `merged` frame has several apply routes (the per-voxel
// kernels of ksg_voxel.cuh, k_tile_apply, the hot-voxel pre-pass) and the long kernel finishes a voxel's TSDF and its semantic row in
// different warps, so no apply kernel holds a voxel's final state in one place.  The log is therefore written after every apply
// kernel has finished, from the pool:
//
//   k_merged_log_heads   one thread per sorted record: flags the first record of every voxel segment, except the anti-grazing
//                        sentinel (records dropped by anti-grazing sort last) and, under spatial sharding, the tiles this rank does
//                        not own (the test of k_voxel_heads)
//   cub::DeviceSelect    compacts the flagged record indices in record order and stores their count in Counters::pad0
//   k_merged_log_keys    the packed block index of every head; a stable cub::DeviceRadixSort on it puts the blocks in index order
//   k_merged_log_write   one warp per entry: block index, voxblox linear index, distance, weight, colours, label and the C-float
//                        prior row, gathered from the voxel's tile
//
// Record order alone is not reproducible: the tile key holds the block's hash-table position, and which position a new block gets
// depends on which thread wins a concurrent insert.  Entries are therefore ordered by (block index, tile, voxel in the tile): the
// same map history gives the same log bytes on every run and whichever apply route ran, and the entries of one block are contiguous.
// A frame with more entries than the capacity writes none; the count stays the full total.
#pragma once
#include "ksg_voxel.cuh"

namespace ksg {

__global__ void k_merged_log_heads(DevCfg cfg, MapRef map, const uint64_t* __restrict__ rec, long long n, uint8_t* __restrict__ flags) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t kSkipped = ~0ull >> kRecOrdBits;
  const uint64_t vk = rec[i] >> kRecOrdBits;
  bool head = vk != kSkipped && (i == 0 || (rec[i - 1] >> kRecOrdBits) != vk);
  if (head) {
    const uint32_t tk = (uint32_t)(vk >> kRecVoxBits);
    const int pos = (int)(tk / (uint32_t)cfg.tiles_per_block);
    const int slot = map.ht_slot[pos];
    head = slot >= 0 && slot < map.max_blocks;
    if (head && cfg.shard_count > 1)
      head = tile_owner(map.ht_keys[pos], (int)(tk % (uint32_t)cfg.tiles_per_block), cfg.shard_count) == cfg.shard_rank;
  }
  flags[i] = head ? 1 : 0;
}

__global__ void k_merged_log_keys(DevCfg cfg, MapRef map, const uint64_t* __restrict__ rec, const int* __restrict__ heads, int n,
                                  uint64_t* __restrict__ keys) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint32_t tk = (uint32_t)(rec[heads[j]] >> 32);
  keys[j] = map.ht_keys[tk / (uint32_t)cfg.tiles_per_block];
}

__global__ void __launch_bounds__(256) k_merged_log_write(DevCfg cfg, MapRef map, const uint64_t* __restrict__ rec, const int* __restrict__ heads,
                                                          int n, VoxelUpdate* __restrict__ log_head, float* __restrict__ log_prior) {
  const int lane = threadIdx.x & 31;
  const int C = cfg.C;
  const int warps = (gridDim.x * blockDim.x) >> 5;
  for (int e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < n; e += warps) {
    const uint64_t key = rec[heads[e]];
    int pos, tile;
    const uint8_t* chunk = voxel_chunk(cfg, map, (uint32_t)(key >> 32), pos, tile);   // valid: k_merged_log_heads checked the slot
    const int v = (int)((key >> kRecOrdBits) & ((1u << kRecVoxBits) - 1u));
    const float* prow = (const float*)(chunk + cfg.head_bytes) + (size_t)v * C;
    float* dst = log_prior + (size_t)e * C;
    for (int c = lane; c < C; c += 32) dst[c] = prow[c];
    if (lane == 0) {
      const I3 bi = unpack_key(map.ht_keys[pos]);
      const int tps = cfg.tiles_per_side, ts = cfg.tile_side_log2, tm = cfg.tile_side - 1;
      const int lx = (tile % tps) * cfg.tile_side + (v & tm);
      const int ly = ((tile / tps) % tps) * cfg.tile_side + ((v >> ts) & tm);
      const int lz = (tile / (tps * tps)) * cfg.tile_side + (v >> (2 * ts));
      VoxelUpdate u;
      u.bx = bi.x; u.by = bi.y; u.bz = bi.z;
      u.lin_label = (uint32_t)(lx + cfg.vps * (ly + cfg.vps * lz)) | ((uint32_t)(chunk + 4 * cfg.plane_f32)[v] << 24);
      u.dist = ((const float*)chunk)[v];
      u.wgt = ((const float*)(chunk + cfg.plane_f32))[v];
      u.rgba = ((const uint32_t*)(chunk + 2 * cfg.plane_f32))[v];
      u.srgba = ((const uint32_t*)(chunk + 3 * cfg.plane_f32))[v];
      log_head[e] = u;
    }
  }
}

}  // namespace ksg
