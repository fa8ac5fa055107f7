// ksg_voxel.cuh — `merged`: per-VOXEL update kernels (round 2).
//
// Round 1 applied a frame's sorted update records with one CTA per touched 8^3 tile (k_tile_apply).  On the 2 cm workload
// (31 M records, 4 690 tiles) the tiles around the camera hold up to 1.1 M records each, and one CTA (8 warps) worked through such
// a tile alone while most SMs idled.  DRAM traffic was never the limit, so staging tiles in shared memory bought nothing here.  This file drops the tile as the unit of work:
//
//   k_voxel_heads        one thread per sorted record: detects voxel-segment heads, measures the segment (galloping search), and
//                        files it by length: `long` (>= kLongLen records, one item per role) or `short`; tile heads do the updated()
//                        bookkeeping of the block (base.cpp:248)
//   k_voxel_apply_long   warps take long segments from a queue (longest class first): the TSDF recurrence and the semantic
//                        recurrence of a voxel are independent, so they are separate items; software-pipelined row gathers
//   k_voxel_apply_short_t  C <= 32: one thread takes a short segment (the bulk of the voxels: ~17 records each); the hot segments run
//                        beside it on a second stream (the DEEP instance of k_voxel_apply_long), the other long segments behind it
//   k_voxel_apply_short  C > 32: warps take short segments - lean code, high occupancy; it runs CONCURRENTLY with the long kernel on
//                        a second stream, filling the SMs the long tail leaves idle
//
// Per-voxel arithmetic and order are those of k_tile_apply (same device functions): results stay bit-identical.
#pragma once
#include "ksg_kernels.cuh"

namespace ksg {

static constexpr int kLongLen = 96;        // segments of at least this many records are split into a TSDF item and a semantic item
static constexpr int kLongLenThread = 256; // the same split when the short segments go to the thread-per-voxel kernel (C <= 32)
static constexpr int kHotLen = 4096;       // ... and these are queued first
static constexpr int kGrab = 8;            // short items fetched per queue access

struct VoxelQueues {
  unsigned long long* long_items;    // [begin:40][len:23][role:1], hot ones from the front, the others from the back
  unsigned long long* short_items;   // [begin:40][len:24]
  long long long_cap, short_cap;
  int long_len;                      // segments of at least this many records are `long` (>= kLongLen, which sizes long_items)
  int* counters;                     // [0] hot count (front), [1] other long count (back), [2] short count, [3] long cursor, [4] short cursor, [5] hot cursor
};

__device__ __forceinline__ uint8_t* voxel_chunk(const DevCfg& cfg, const MapRef& map, uint32_t tk, int& pos, int& tile) {
  pos = (int)(tk / (uint32_t)cfg.tiles_per_block);
  tile = (int)(tk % (uint32_t)cfg.tiles_per_block);
  const int slot = map.ht_slot[pos];
  if (slot < 0 || slot >= map.max_blocks) return nullptr;
  return map.pool + (uint64_t)slot * cfg.block_stride + (uint64_t)tile * cfg.tile_stride;
}

static constexpr int kHeadsBlock = 1024;      // records per CTA of k_voxel_heads (256 threads x 4)
__global__ void __launch_bounds__(256) k_voxel_heads(DevCfg cfg, Counters* cnt, MapRef map, const uint64_t* __restrict__ rec, long long n, int stamp, VoxelQueues q) {
  // the CTA's 1024 voxel keys (+ the predecessor's) in shared memory: a head finds the end of its segment by scanning shared memory
  // (segments average ~17 records); only a segment that runs past the CTA's range continues with a galloping search in global memory
  __shared__ uint64_t s_vk[kHeadsBlock + 1];
  const long long base = (long long)blockIdx.x * kHeadsBlock;
  const uint64_t kNone = ~0ull;                     // no record here (beyond n)
  for (int t = threadIdx.x; t < kHeadsBlock; t += blockDim.x) {
    const long long i = base + t;
    s_vk[1 + t] = (i < n) ? (rec[i] >> kRecOrdBits) : kNone;
  }
  if (threadIdx.x == 0) s_vk[0] = (base > 0) ? (rec[base - 1] >> kRecOrdBits) : kNone;
  __syncthreads();
  const uint64_t kSkipped = ~0ull >> kRecOrdBits;   // records dropped by anti-grazing sort last (key ~0)
  // short segments are the bulk of the heads (~1.8 M per 640x480 / 2 cm frame): their queue slots are handed out with ONE atomic per
  // CTA (block scan of the per-thread counts) - one atomic per warp and round was ~10^6 same-address atomics = the kernel's whole 0.5 ms
  constexpr int kPerThread = kHeadsBlock / 256;
  unsigned long long mine[kPerThread];
  int n_mine = 0;
#pragma unroll
  for (int k = 0; k < kPerThread; ++k) {
    mine[k] = 0ull;
    const int t = (int)threadIdx.x + k * 256;
    const long long i = base + t;
    if (i >= n) continue;
    const uint64_t vk = s_vk[1 + t];
    if (vk == kSkipped) continue;
    if (s_vk[t] == vk && !(base == 0 && t == 0)) continue;                    // not the first record of its voxel
    const uint32_t tk = (uint32_t)(vk >> kRecVoxBits);
    const int pos = (int)(tk / (uint32_t)cfg.tiles_per_block);
    if ((base == 0 && t == 0) || (uint32_t)(s_vk[t] >> kRecVoxBits) != tk) {   // tile head: updated() bookkeeping is replicated on every shard
      const int old = atomicExch(&map.touched_stamp[pos], stamp);
      if (old != stamp) map.touched_list[atomicAdd(&cnt->n_blocks_touched, 1)] = pos;
      atomicAdd(&cnt->n_tiles, 1);
    }
    if (cfg.shard_count > 1 && tile_owner(map.ht_keys[pos], (int)(tk % (uint32_t)cfg.tiles_per_block), cfg.shard_count) != cfg.shard_rank) continue;
    int j = t + 1;
    while (j < kHeadsBlock && s_vk[1 + j] == vk) ++j;
    long long len = j - t;
    if (j == kHeadsBlock && base + kHeadsBlock < n) {   // the segment reaches the end of the CTA's range: gallop on in global memory
      long long lo = base + kHeadsBlock - 1, hi;       // invariant: rec[lo] belongs to the segment
      long long step = 1;
      for (;;) {
        const long long p = base + kHeadsBlock - 1 + step;
        if (p >= n) { hi = n; break; }
        if ((rec[p] >> kRecOrdBits) != vk) { hi = p; break; }
        lo = p;
        step <<= 1;
      }
      while (hi - lo > 1) { const long long mid = (lo + hi) >> 1; if ((rec[mid] >> kRecOrdBits) == vk) lo = mid; else hi = mid; }
      len = hi - i;
    }
    if (len >= q.long_len) {
      const bool hot = len >= kHotLen;
      const int at = atomicAdd(&q.counters[hot ? 0 : 1], 2);
      if (at + 2 > q.long_cap / 2) { set_err(cnt, 4); continue; }   // cannot happen: long_cap >= 2 * (2 * records / kLongLen)
      const unsigned long long item = ((unsigned long long)i << 24) | ((unsigned long long)len << 1);
      if (hot) { q.long_items[at] = item; q.long_items[at + 1] = item | 1ull; }
      else { q.long_items[q.long_cap - 1 - at] = item; q.long_items[q.long_cap - 2 - at] = item | 1ull; }
    } else {
      mine[k] = ((unsigned long long)i << 24) | (unsigned long long)len;   // never 0: len >= 1
      ++n_mine;
    }
  }
  __shared__ int s_wsum[8];
  __shared__ int s_cta_base;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int incl = n_mine;
  for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
  if (lane == 31) s_wsum[wid] = incl;
  __syncthreads();
  if (threadIdx.x == 0) {
    int tot = 0;
    for (int w = 0; w < 8; ++w) { const int v = s_wsum[w]; s_wsum[w] = tot; tot += v; }
    s_cta_base = tot > 0 ? atomicAdd(&q.counters[2], tot) : 0;
  }
  __syncthreads();
  int at = s_cta_base + s_wsum[wid] + incl - n_mine;
#pragma unroll
  for (int k = 0; k < kPerThread; ++k) {
    if (mine[k] != 0ull) {
      if (at >= q.short_cap) { set_err(cnt, 4); break; }
      q.short_items[at++] = mine[k];
    }
  }
}

struct VoxelCtx {
  uint8_t* chunk;
  int v;          // voxel inside the tile
  F3 center;
};
__device__ __forceinline__ bool voxel_ctx(const DevCfg& cfg, const MapRef& map, uint64_t key, VoxelCtx& c) {
  const uint32_t tk = (uint32_t)(key >> 32);
  int pos, tile;
  c.chunk = voxel_chunk(cfg, map, tk, pos, tile);
  c.v = (int)((key >> kRecOrdBits) & ((1u << kRecVoxBits) - 1u));
  if (!c.chunk) return false;
  const I3 bi = unpack_key(map.ht_keys[pos]);
  const int tps = cfg.tiles_per_side;
  const int tx = tile % tps, ty = (tile / tps) % tps, tz = tile / (tps * tps);
  const int ts = cfg.tile_side_log2, tm = cfg.tile_side - 1;
  I3 g;
  g.x = bi.x * cfg.vps + tx * cfg.tile_side + (c.v & tm);
  g.y = bi.y * cfg.vps + ty * cfg.tile_side + ((c.v >> ts) & tm);
  g.z = bi.z * cfg.vps + tz * cfg.tile_side + (c.v >> (2 * ts));
  c.center = voxel_center(g, cfg.voxel_size);
  return true;
}

// arg-max (first maximum wins, base.cpp:352-367) + colour hand-off (base.cpp:370-380, 172-191) of one voxel's finished row
template <int NCH>
__device__ __forceinline__ void voxel_finish_semantic(const DevCfg& cfg, const Luts* __restrict__ luts, const VoxelCtx& vc, int lane, const float (&p)[NCH]) {
  const int C = cfg.C;
  float best = -3.402823466e38f;
  int bi = 0x7fffffff;
#pragma unroll
  for (int q = 0; q < NCH; ++q) { const int c = q * 32 + lane; if (c < C && (p[q] > best || bi == 0x7fffffff)) { best = p[q]; bi = c; } }
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_down_sync(0xffffffffu, best, o);
    const int oi = __shfl_down_sync(0xffffffffu, bi, o);
    if (oi != 0x7fffffff && (bi == 0x7fffffff || ob > best || (ob == best && oi < bi))) { best = ob; bi = oi; }
  }
  best = __shfl_sync(0xffffffffu, best, 0);
  const int lab = __shfl_sync(0xffffffffu, bi, 0);
  float* prow = (float*)(vc.chunk + cfg.head_bytes) + (size_t)vc.v * C;
#pragma unroll
  for (int q = 0; q < NCH; ++q) { const int c = q * 32 + lane; if (c < C) prow[c] = p[q]; }
  if (lane == 0) {
    (vc.chunk + 4 * cfg.plane_f32)[vc.v] = (uint8_t)lab;
    const uint32_t sc = luts->label_rgba[lab];
    ((uint32_t*)(vc.chunk + 3 * cfg.plane_f32))[vc.v] = sc;
    if (cfg.color_mode == 1) ((uint32_t*)(vc.chunk + 2 * cfg.plane_f32))[vc.v] = sc;                                        // kSemantic
    else if (cfg.color_mode == 2) ((uint32_t*)(vc.chunk + 2 * cfg.plane_f32))[vc.v] = rainbow_color_map((double)expf(best));  // kSemanticProbability
  }
}

// ---------------------------------------------------------------------------------------------
// long segments: one item per role
// ---------------------------------------------------------------------------------------------
// DEEP == true: the instance for the HOT voxels only (>= kHotLen records; the voxel next to the camera has ~10^5) - their two chains are the
// critical path of the frame, and each record costs a key load -> operand load round trip, so the pipelines are twice as deep (keys 4-6
// batches ahead, operands of two batches in flight; 186 registers) and the kernel is small (one warp per chain) so that it fits beside the
// other two update kernels.  DEEP == false: everything else (skip_hot = 1 when the DEEP instance runs).
template <int NCH, bool DEEP = false>
__global__ void __launch_bounds__(256, DEEP ? 1 : 2) k_voxel_apply_long(DevCfg cfg, Xform T, Counters* cnt, MapRef map, const Luts* __restrict__ luts,
                                                            const uint64_t* __restrict__ rec, ApplySrc src, VoxelQueues q, int skip_hot) {
  __shared__ uint32_t s_ring[DEEP ? 8 : 1][128];      // DEEP: per warp, the record keys of four batches (semantic role)
  const int lane = threadIdx.x & 31;
  const int C = cfg.C;
  const int n_hot = q.counters[0], n_other = q.counters[1];
  const int n_items = DEEP ? n_hot : n_hot + n_other;
  const int first_item = (!DEEP && skip_hot) ? n_hot : 0;      // skip_hot: the hot voxels are taken by the DEEP instance
  const F3 origin = f3(T.tx, T.ty, T.tz);
  const bool keep_blend = cfg.color_mode == 0;
  const uint32_t ord_mask = (1u << kRecOrdBits) - 1u;
  const uint32_t zero_row = (uint32_t)cnt->n_cast;   // all-zero row behind the last bundle: padded lanes add +0.0f (exact)
  for (;;) {
    int it = 0;
    if (lane == 0) it = first_item + atomicAdd(&q.counters[DEEP ? 5 : 3], 1);
    it = __shfl_sync(0xffffffffu, it, 0);
    if (it >= n_items) break;
    const unsigned long long item = (it < n_hot) ? q.long_items[it] : q.long_items[q.long_cap - 1 - (it - n_hot)];
    const long long begin = (long long)(item >> 24);
    const int len = (int)((item >> 1) & 0x7FFFFFu);
    const int role = (int)(item & 1ull);       // 0: TSDF, 1: semantic
    VoxelCtx vc;
    if (!voxel_ctx(cfg, map, rec[begin], vc)) continue;
    const uint64_t* r = rec + begin;
    // hot voxel (thousands of records): the pre-pass (ksg_hot.cuh) may have finished its semantic row with the exact parallel scan,
    // and checked in parallel that the saturated TSDF state survives the frame; then there is nothing sequential left to do here
    int hot = -1;
    if (NCH == 1 && src.n_hot > 0 && len >= src.hot_thresh) {
      int a = 0, b = src.n_hot;
      while (a < b) { const int mid = (a + b) >> 1; if (src.hot_segs[mid].begin < begin) a = mid + 1; else b = mid; }
      if (a < src.n_hot && src.hot_segs[a].begin == begin && src.hot_segs[a].end == begin + len) hot = a;
    }
    if (role == 0) {
      if (hot >= 0 && src.hot_tsdf_same != nullptr && src.hot_tsdf_same[hot] != 0) continue;
      float* pd = (float*)vc.chunk + vc.v;
      float* pw = (float*)(vc.chunk + cfg.plane_f32) + vc.v;
      uint32_t* pc = (uint32_t*)(vc.chunk + 2 * cfg.plane_f32) + vc.v;
      float dist = *pd, wgt = *pw;
      uint32_t rgba = *pc;
      if (DEEP) {
        // record keys five batches ahead, their bundle parameters two batches ahead.  Three parameter and three key registers, the loop
        // unrolled by three: a rotation by register moves (a = b; b = c) would wait for the load issued in the same iteration and undo
        // the prefetch; the keys stay raw until they are used (masking at load time waits for the load, too).
        const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
        auto raw_key = [&](int idx) -> uint32_t { return (idx < len) ? (uint32_t)r[idx] : 0u; };
        float4 pr0 = (lane < len) ? src.param[raw_key(lane) & ord_mask] : z4;
        float4 pr1 = (32 + lane < len) ? src.param[raw_key(32 + lane) & ord_mask] : z4;
        float4 pr2 = z4;
        uint32_t kx2 = raw_key(64 + lane), kx0 = raw_key(96 + lane), kx1 = raw_key(128 + lane);
        const int nbatch_t = (len + 31) >> 5;
#define KSG_TSDF_STEP(S, PRU, PRL, KX)                                                                                             \
        if ((S) < nbatch_t) {                                                                                                      \
          PRL = (((S) + 2) * 32 + lane < len) ? src.param[KX & ord_mask] : z4;     /* parameters of batch S + 2 */                  \
          KX = raw_key(((S) + 5) * 32 + lane);                                                                                      \
          const int nb = (len - (S) * 32) < 32 ? (len - (S) * 32) : 32;                                                            \
          float sdf = 0.0f, uw = 0.0f;                                                                                             \
          if (lane < nb) tsdf_measure(cfg.tp, origin, f3(PRU.x, PRU.y, PRU.z), vc.center, PRU.w, sdf, uw);                         \
          tsdf_batch<true>(cfg.tp, lane, nb, sdf, uw, 0u, keep_blend, dist, wgt, rgba);                                            \
        }
        for (int j = 0; j < nbatch_t; j += 3) {
          KSG_TSDF_STEP(j, pr0, pr2, kx2)
          KSG_TSDF_STEP(j + 1, pr1, pr0, kx0)
          KSG_TSDF_STEP(j + 2, pr2, pr1, kx1)
        }
#undef KSG_TSDF_STEP
      } else {
      // parameters of the next batch are fetched one batch ahead
      float4 pr_a = (lane < len) ? src.param[(uint32_t)r[lane] & ord_mask] : make_float4(0.f, 0.f, 0.f, 0.f);
      for (int base = 0; base < len; base += 32) {
        const int nb = (len - base) < 32 ? (len - base) : 32;
        float4 pr_b = make_float4(0.f, 0.f, 0.f, 0.f);
        if (base + 32 + lane < len) pr_b = src.param[(uint32_t)r[base + 32 + lane] & ord_mask];
        float sdf = 0.0f, uw = 0.0f;
        if (lane < nb) tsdf_measure(cfg.tp, origin, f3(pr_a.x, pr_a.y, pr_a.z), vc.center, pr_a.w, sdf, uw);
        tsdf_batch(cfg.tp, lane, nb, sdf, uw, 0u, keep_blend, dist, wgt, rgba);   // merged: point colours are (0,0,0,0) (merged.cpp:70)
        pr_a = pr_b;
      }
      }
      if (lane == 0) { *pd = dist; *pw = wgt; if (keep_blend) *pc = rgba; }
    } else {
      const float* prow = (const float*)(vc.chunk + cfg.head_bytes) + (size_t)vc.v * C;
      float p[NCH];
#pragma unroll
      for (int qq = 0; qq < NCH; ++qq) { const int c = qq * 32 + lane; p[qq] = (c < C) ? prow[c] : 0.0f; }
      if (NCH == 1 && hot >= 0) {
        p[0] = (lane < C) ? src.hot_prior[(size_t)hot * 32 + lane] : 0.0f;
      } else if (NCH == 1 && DEEP) {
        // the (L * freq) rows of TWO batches are in flight while a third is added (three register buffers, loop unrolled by three so that no
        // buffer is copied); record keys are loaded six batches ahead into registers and handed to a per-warp shared-memory ring three
        // batches ahead (broadcast reads replace the 32 shuffles per batch).  The adds stay in record order; batches past the end read the
        // all-zero row: + 0.0f is exact.
        const float* lane_tmp = src.tmp + (lane < C ? lane : 0);
        uint32_t* ring = s_ring[(threadIdx.x >> 5) & 7];
        // raw keys: the order bits are masked when the key is handed to the ring, three batches after its load (zero_row < 2^23 survives the mask)
        auto key_at = [&](int idx) -> uint32_t { return (idx < len) ? (uint32_t)r[idx] : zero_row; };
        __syncwarp();
        ring[lane] = key_at(lane) & ord_mask; ring[32 + lane] = key_at(32 + lane) & ord_mask; ring[64 + lane] = key_at(64 + lane) & ord_mask;
        uint32_t k0 = key_at(96 + lane), k1 = key_at(128 + lane), k2 = key_at(160 + lane);
        __syncwarp();
        float ra[32], rb[32], rc[32];
#pragma unroll
        for (int u = 0; u < 32; ++u) ra[u] = __ldg(lane_tmp + (size_t)ring[u] * C);
#pragma unroll
        for (int u = 0; u < 32; ++u) rb[u] = __ldg(lane_tmp + (size_t)ring[32 + u] * C);
        const int nbatch = (len + 31) >> 5;
#define KSG_SEM_STEP(S, KREG, LOADBUF, ADDBUF)                                                                                     \
        {                                                                                                                          \
          ring[(((S) + 3) & 3) * 32 + lane] = KREG & ord_mask;               /* keys of batch S + 3 */                             \
          KREG = key_at(((S) + 6) * 32 + lane);                                                                                    \
          __syncwarp();                                                                                                            \
          _Pragma("unroll") for (int u = 0; u < 32; ++u) LOADBUF[u] = __ldg(lane_tmp + (size_t)ring[(((S) + 2) & 3) * 32 + u] * C);  \
          _Pragma("unroll") for (int u = 0; u < 32; ++u) p[0] += ADDBUF[u];                                                        \
        }
        for (int j = 0; j < nbatch; j += 3) {
          KSG_SEM_STEP(j, k0, rc, ra)
          KSG_SEM_STEP(j + 1, k1, ra, rb)
          KSG_SEM_STEP(j + 2, k2, rb, rc)
        }
#undef KSG_SEM_STEP
        if (lane >= C) p[0] = 0.0f;
      } else if (NCH == 1) {
        // software pipeline over batches of 32 records: keys two batches ahead, the 32 (L * freq) row values one batch ahead
        const float* lane_tmp = src.tmp + (lane < C ? lane : 0);
        uint32_t ord_a = (lane < len) ? ((uint32_t)r[lane] & ord_mask) : zero_row;
        uint32_t ord_b = (32 + lane < len) ? ((uint32_t)r[32 + lane] & ord_mask) : zero_row;
        float rv_a[32];
#pragma unroll
        for (int u = 0; u < 32; ++u) rv_a[u] = __ldg(lane_tmp + (size_t)__shfl_sync(0xffffffffu, ord_a, u) * C);
        for (int base = 0; base < len; base += 32) {
          const uint32_t ord_c = (base + 64 + lane < len) ? ((uint32_t)r[base + 64 + lane] & ord_mask) : zero_row;
          float rv_b[32];
#pragma unroll
          for (int u = 0; u < 32; ++u) rv_b[u] = __ldg(lane_tmp + (size_t)__shfl_sync(0xffffffffu, ord_b, u) * C);
#pragma unroll
          for (int u = 0; u < 32; ++u) p[0] += rv_a[u];
#pragma unroll
          for (int u = 0; u < 32; ++u) rv_a[u] = rv_b[u];
          ord_b = ord_c;
        }
        if (lane >= C) p[0] = 0.0f;
      } else {
        constexpr int kRowUnroll = (NCH <= 2) ? 8 : 2;
        for (int base = 0; base < len; base += 32) {
          const int nb = (len - base) < 32 ? (len - base) : 32;
          const uint32_t ord = (lane < nb) ? ((uint32_t)r[base + lane] & ord_mask) : zero_row;
          for (int j0 = 0; j0 < nb; j0 += kRowUnroll) {
            float rv[kRowUnroll][NCH];
#pragma unroll
            for (int u = 0; u < kRowUnroll; ++u) {
              const uint32_t o = __shfl_sync(0xffffffffu, ord, (j0 + u) & 31);
              const float* row = src.tmp + (size_t)o * C;
#pragma unroll
              for (int qq = 0; qq < NCH; ++qq) { const int cc = qq * 32 + lane; rv[u][qq] = (j0 + u < nb && cc < C) ? __ldg(row + cc) : 0.0f; }
            }
#pragma unroll
            for (int u = 0; u < kRowUnroll; ++u) {
#pragma unroll
              for (int qq = 0; qq < NCH; ++qq) p[qq] += rv[u][qq];
            }
          }
        }
      }
      voxel_finish_semantic<NCH>(cfg, luts, vc, lane, p);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// short segments: both roles by one warp
// ---------------------------------------------------------------------------------------------
template <int NCH>
__global__ void __launch_bounds__(256, 6) k_voxel_apply_short(DevCfg cfg, Xform T, Counters* cnt, MapRef map, const Luts* __restrict__ luts,
                                                             const uint64_t* __restrict__ rec, ApplySrc src, VoxelQueues q) {
  const int lane = threadIdx.x & 31;
  const int C = cfg.C;
  const int n_items = min((long long)q.counters[2], q.short_cap);
  const F3 origin = f3(T.tx, T.ty, T.tz);
  const bool keep_blend = cfg.color_mode == 0;
  const uint32_t ord_mask = (1u << kRecOrdBits) - 1u;
  for (;;) {
    int it0 = 0;
    if (lane == 0) it0 = atomicAdd(&q.counters[4], kGrab);
    it0 = __shfl_sync(0xffffffffu, it0, 0);
    if (it0 >= n_items) break;
    // the kGrab items of this round: lane g holds item g's descriptor and first record (independent loads, one round trip)
    unsigned long long my_item = 0, my_key = 0;
    if (lane < kGrab && it0 + lane < n_items) { my_item = q.short_items[it0 + lane]; my_key = rec[my_item >> 24]; }
    const int n_here = (n_items - it0) < kGrab ? (n_items - it0) : kGrab;
    for (int gi = 0; gi < n_here; ++gi) {
      const unsigned long long item = __shfl_sync(0xffffffffu, my_item, gi);
      const uint64_t key0 = __shfl_sync(0xffffffffu, my_key, gi);
      const long long begin = (long long)(item >> 24);
      const int len = (int)(item & 0xFFFFFFu);
      VoxelCtx vc;
      if (!voxel_ctx(cfg, map, key0, vc)) continue;
      const uint64_t* r = rec + begin;
      float* pd = (float*)vc.chunk + vc.v;
      float* pw = (float*)(vc.chunk + cfg.plane_f32) + vc.v;
      uint32_t* pc = (uint32_t*)(vc.chunk + 2 * cfg.plane_f32) + vc.v;
      float dist = *pd, wgt = *pw;
      uint32_t rgba = *pc;
      const float* prow = (const float*)(vc.chunk + cfg.head_bytes) + (size_t)vc.v * C;
      float p[NCH];
#pragma unroll
      for (int qq = 0; qq < NCH; ++qq) { const int c = qq * 32 + lane; p[qq] = (c < C) ? prow[c] : 0.0f; }
      for (int base = 0; base < len; base += 32) {
        const int nb = (len - base) < 32 ? (len - base) : 32;
        uint32_t ord = 0;
        float sdf = 0.0f, uw = 0.0f;
        if (lane < nb) {
          ord = (uint32_t)r[base + lane] & ord_mask;
          const float4 pr = src.param[ord];
          tsdf_measure(cfg.tp, origin, f3(pr.x, pr.y, pr.z), vc.center, pr.w, sdf, uw);
        }
        // (L * freq) rows in record order: lane c adds column c; four independent row loads in flight
        for (int j0 = 0; j0 < nb; j0 += 4) {
          float rv[4][NCH];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const uint32_t o = __shfl_sync(0xffffffffu, ord, (j0 + u) & 31);
            const float* row = src.tmp + (size_t)o * C;
#pragma unroll
            for (int qq = 0; qq < NCH; ++qq) { const int cc = qq * 32 + lane; rv[u][qq] = (j0 + u < nb && cc < C) ? __ldg(row + cc) : 0.0f; }
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
#pragma unroll
            for (int qq = 0; qq < NCH; ++qq) p[qq] += rv[u][qq];   // + 0.0f is exact for the padded tail
          }
        }
        tsdf_batch(cfg.tp, lane, nb, sdf, uw, 0u, keep_blend, dist, wgt, rgba);
      }
      if (lane == 0) { *pd = dist; *pw = wgt; if (keep_blend) *pc = rgba; }
      voxel_finish_semantic<NCH>(cfg, luts, vc, lane, p);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// short segments, C <= 32: one THREAD per voxel.
// The warp-per-voxel kernel above spends ~900 warp instructions on a voxel that has ~11 records (compute bound on bookkeeping: the
// 32-lane weight recurrence, the warp arg-max, per-voxel index arithmetic, a third of the lanes idle at C = 21).  Here a thread walks its voxel's records
// alone - the recurrences ARE sequential - and 32 voxels share every issued instruction.  Same operations in the same order per voxel as the
// warp kernels (tsdf_measure + tsdf_chain_step per record, p[c] += row[c] in record order, first maximum wins), hence the same bits.
// Rows of (L * freq) are read as 128-bit words from the zero-padded table tmp4.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256, 3) k_voxel_apply_short_t(DevCfg cfg, Xform T, Counters* cnt, MapRef map, const Luts* __restrict__ luts,
                                                               const uint64_t* __restrict__ rec, ApplySrc src, VoxelQueues q) {
  const int C = cfg.C;
  const int C4 = (C + 3) & ~3;
  const int n_items = (int)min((long long)q.counters[2], q.short_cap);
  const F3 origin = f3(T.tx, T.ty, T.tz);
  const bool keep_blend = cfg.color_mode == 0;
  const uint32_t ord_mask = (1u << kRecOrdBits) - 1u;
  const int tpb_log2 = __ffs(cfg.tiles_per_block) - 1, tps_log2 = __ffs(cfg.tiles_per_side) - 1;   // powers of two (tile_side_log2, vps - 1 masks)
  for (int it = blockIdx.x * blockDim.x + threadIdx.x; it < n_items; it += gridDim.x * blockDim.x) {
    const unsigned long long item = q.short_items[it];
    const uint64_t* r = rec + (long long)(item >> 24);
    const int len = (int)(item & 0xFFFFFFu);
    uint64_t key = r[0];
    const uint32_t tk = (uint32_t)(key >> 32);
    const int pos = (int)(tk >> tpb_log2), tile = (int)(tk & (uint32_t)(cfg.tiles_per_block - 1));
    const int slot = map.ht_slot[pos];
    if (slot < 0 || slot >= map.max_blocks) continue;
    uint8_t* chunk = map.pool + (uint64_t)slot * cfg.block_stride + (uint64_t)tile * cfg.tile_stride;
    const int v = (int)((key >> kRecOrdBits) & ((1u << kRecVoxBits) - 1u));
    const I3 bi = unpack_key(map.ht_keys[pos]);
    const int ts = cfg.tile_side_log2, tm = cfg.tile_side - 1, tpm = cfg.tiles_per_side - 1;
    I3 g;
    g.x = bi.x * cfg.vps + ((tile & tpm) << ts) + (v & tm);
    g.y = bi.y * cfg.vps + (((tile >> tps_log2) & tpm) << ts) + ((v >> ts) & tm);
    g.z = bi.z * cfg.vps + ((tile >> (2 * tps_log2)) << ts) + (v >> (2 * ts));
    const F3 center = voxel_center(g, cfg.voxel_size);
    float* pd = (float*)chunk + v;
    float* pw = (float*)(chunk + cfg.plane_f32) + v;
    uint32_t* pc = (uint32_t*)(chunk + 2 * cfg.plane_f32) + v;
    float dist = *pd, wgt = *pw;
    uint32_t rgba = *pc;
    float* prow = (float*)(chunk + cfg.head_bytes) + (size_t)v * C;
    float p[32];
#pragma unroll
    for (int c = 0; c < 32; ++c) p[c] = (c < C) ? prow[c] : 0.0f;
    for (int k = 0; k < len; ++k) {
      const uint32_t ord = (uint32_t)key & ord_mask;
      if (k + 1 < len) key = r[k + 1];                   // next key one record ahead of its use
      const float4 pr = src.param[ord];
      const float4* row = (const float4*)(src.tmp4 + (size_t)ord * C4);
      float4 rv[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) rv[j] = (4 * j < C) ? __ldg(row + j) : make_float4(0.f, 0.f, 0.f, 0.f);
      float sdf, uw;
      tsdf_measure(cfg.tp, origin, f3(pr.x, pr.y, pr.z), center, pr.w, sdf, uw);
      tsdf_chain_step(cfg.tp, sdf, uw, 0u, keep_blend, dist, wgt, rgba);   // merged: point colours are (0,0,0,0) (merged.cpp:70)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (4 * j < C) { p[4 * j] += rv[j].x; p[4 * j + 1] += rv[j].y; p[4 * j + 2] += rv[j].z; p[4 * j + 3] += rv[j].w; }   // pads add +0.0f
      }
    }
    *pd = dist; *pw = wgt;
    if (keep_blend) *pc = rgba;
    // arg-max, first maximum wins (base.cpp:352-367) + colour hand-off (base.cpp:370-380, 172-191)
    float best = p[0];
    int lab = 0;
#pragma unroll
    for (int c = 1; c < 32; ++c) if (c < C && p[c] > best) { best = p[c]; lab = c; }
#pragma unroll
    for (int c = 0; c < 32; ++c) if (c < C) prow[c] = p[c];
    (chunk + 4 * cfg.plane_f32)[v] = (uint8_t)lab;
    const uint32_t sc = luts->label_rgba[lab];
    ((uint32_t*)(chunk + 3 * cfg.plane_f32))[v] = sc;
    if (cfg.color_mode == 1) *pc = sc;                                                        // kSemantic
    else if (cfg.color_mode == 2) *pc = rainbow_color_map((double)expf(best));              // kSemanticProbability
  }
}

}  // namespace ksg
