// ksg_kernels.cuh — hand-written sm_90a kernels of the semantic TSDF integrator.
//
// Kernel family (SURVEY.md §7.4 numbering in brackets).  The `fast` frame has kernels of its own (ksg_fast.cuh, ksg_fast3.cuh);
// it shares the device structures and helpers defined here.
//   k_depth_flags / k_classify      [K1]  merged: back-projection, validity, T_G_C * p
//   k_bundle_heads / k_bundle_merge / k_bundle_alloc / k_bundle_loglik [K2] merged: bundleRays + integrateVoxel merge loop
//   k_emit_merged                   [K4]  ray cast -> update records + block-hash insertion [K5]
//   k_block_init                    [K5]  pool allocation + default construction of new voxel blocks
//   k_tile_heads / k_tile_apply     [K6]  merged: per-tile ordered TSDF + semantic update, TMA-staged
//   k_export                        [K8]  tiles -> voxblox block layout
#pragma once
#include "ksg_device.cuh"

namespace ksg {

struct DevCfg {
  float voxel_size, vsi, vps_inv;
  int vps;
  int tile_side, tile_side_log2, tiles_per_side, tiles_per_block, tile_voxels;
  uint32_t plane_f32, plane_u8;  // bytes of one float / byte plane of a tile (16 B multiples)
  uint32_t head_bytes;           // dist | weight | rgba | sem_rgba | label
  uint32_t prior_bytes;          // V * C floats, voxel-major rows (16 B multiple)
  uint32_t tile_stride;          // bytes
  int full_stage;                // 1: the whole tile chunk is staged in shared memory, 0: head only
  uint64_t block_stride;         // bytes
  TsdfParams tp;
  float min_ray, max_ray, start_inv;
  int carving, const_weight, allow_clear, maxc, anti_grazing;
  int C;
  float lm, ln;
  int color_mode;
  int type;
  int shard_rank, shard_count;   // spatial sharding: this rank applies only the tiles it owns
};

struct Luts {
  uint32_t label_rgba[256];   // 0 when unknown (color.cpp:92)
  uint8_t dynamic_label[256];
  uint32_t c2l_keys[1024];    // colour -> label open addressing table, 0xFFFFFFFF = empty
  uint8_t c2l_vals[1024];
};

struct Counters {
  int n_points;
  int n_valid;
  int n_cast;        // fast: cast rays R; merged: bundles B
  int n_new_blocks;
  int n_tiles;
  int err;
  int n_blocks_touched;
  int pool_count;    // blocks allocated in the pool (persistent across frames)
  int tile_cursor;   // dynamic tile queue of k_tile_apply
  int n_big_tiles;   // tiles with many records are queued first (front of tile_begin; the others fill it from the back)
  int n_small_tiles;
  int last_sweep;    // persistent solver: id of the converged sweep
  // observed-set solver, indexed by (sweep & 3)
  int changed[4];
  int n_truncated[4];
  unsigned long long sum_updates[4];
  unsigned long long n_records;
  unsigned long long n_skipped;   // merged anti-grazing: ray steps that emit no update
  unsigned long long n_cand_ext;
  unsigned long long ray_steps;
  int n_nonclear;    // merged, KSG_BUNDLE_ORDER_LIBSTDCXX: bundles of the non-clearing map (they precede the clearing ones)
  int pad0;
};

static constexpr int kH0 = 16;           // ray steps materialised before the first observed-set sweep
static constexpr int kExtSegs = 12;      // horizon doubles per extension: 16, 32, ..., 65536
static constexpr int kOrderStepBits = 16;
static constexpr int kRecVoxBits = 9, kRecOrdBits = 23;

__device__ __forceinline__ void set_err(Counters* c, int e) { atomicCAS(&c->err, 0, e); }

// Warp-aggregated bump allocation: every lane of a converged warp asks for `n` items (0 allowed) and receives its base;
// one atomic per warp instead of 32 atomics on one address (same-address atomics serialise in L2).
__device__ __forceinline__ unsigned long long warp_alloc(unsigned long long* counter, unsigned long long n) {
  const int lane = threadIdx.x & 31;
  unsigned long long incl = n;
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  const unsigned long long total = __shfl_sync(0xffffffffu, incl, 31);
  unsigned long long base = 0;
  if (lane == 0 && total) base = atomicAdd(counter, total);
  base = __shfl_sync(0xffffffffu, base, 0);
  return base + incl - n;
}
__device__ __forceinline__ void warp_add(unsigned long long* counter, unsigned long long n) {
  for (int o = 16; o > 0; o >>= 1) n += __shfl_down_sync(0xffffffffu, n, o);
  if ((threadIdx.x & 31) == 0 && n) atomicAdd(counter, n);
}

// ---------------------------------------------------------------------------------------------
// frame set-up
// ---------------------------------------------------------------------------------------------
// The per-frame counters at the start of a frame of n_points points.
__device__ __forceinline__ void frame_counters_reset(Counters* c, int n_points) {
  c->n_points = n_points; c->n_valid = 0; c->n_cast = 0;
  c->n_new_blocks = 0; c->n_tiles = 0; c->n_blocks_touched = 0; c->tile_cursor = 0; c->n_big_tiles = 0; c->n_small_tiles = 0;
  for (int i = 0; i < 4; ++i) { c->changed[i] = 0; c->n_truncated[i] = 0; c->sum_updates[i] = 0; }
  c->n_records = 0; c->n_skipped = 0; c->n_cand_ext = 0; c->ray_steps = 0;
}
__global__ void k_frame_reset(Counters* c, int n_points) { frame_counters_reset(c, n_points); }

// depth_map_to_pointcloud.h:259: DepthTraits<float>::valid = isfinite
__global__ void k_depth_flags(const float* __restrict__ depth, int n, uint8_t* __restrict__ flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flags[i] = isfinite(depth[i]) ? 1 : 0;
}

__device__ __forceinline__ int mixed_index(int seq, int n) {  // voxblox MixedThreadSafeIndex (A.3)
  const int groups = n / 1024;
  if (groups * 1024 <= seq) return seq;
  return (seq % groups) * 1024 + seq / groups;
}

struct FrameIn {
  const float* xyz;         // n*3 or NULL
  const uint8_t* rgba;      // n*4 or NULL
  const uint8_t* labels;    // n or NULL
  const float* depth;       // image or NULL
  const uint8_t* label_img; // image or NULL
  const int* pix_list;      // finite pixels (depth entry)
  const int* point_of_seq;  // "sorted" order mode, else NULL
  int width;
  float cx, cy, constant_x, constant_y;
  float z_scale;            // z = depth * z_scale: 1 for float32 metres, 0.001f for uint16 millimetres (DepthTraits<T>::toMeters)
  const uint32_t* color_img; // per-pixel point colour (RGB semantic image entry) or NULL: colour of the label
  int freespace;
};

// The per-point rules of the reference's front end, shared by the classify kernels of both integrators and the "sorted" order keys.
//
// SemanticLabel2Color::getSemanticLabelFromColor (color.cpp:69-82): Luts::c2l_keys / c2l_vals is an open addressing table of 1024 slots,
// probed linearly from the colour's home slot.  ksg_set_color_to_label inserts with the same home slot and probe.
__host__ __device__ __forceinline__ uint32_t color_home_slot(uint32_t rgb) { return (rgb * 2654435761u) >> 22; }
// label of the colour rgb = R | G << 8 | B << 16 (the alpha is forced to 255 by fast.cpp:157 / merged.cpp:87, so it is not part of the key),
// 0 when the table does not hold it
__device__ __forceinline__ uint8_t label_of_color(const Luts* __restrict__ luts, uint32_t rgb) {
  uint32_t h = color_home_slot(rgb);
  for (int p = 0; p < 1024; ++p) {
    const uint32_t k = luts->c2l_keys[h];
    if (k == rgb) return luts->c2l_vals[h];
    if (k == 0xFFFFFFFFu) break;
    h = (h + 1) & 1023;
  }
  return 0;
}

// Points entry, input point i: its position, its colour (the packed RGBA; without RGBA, the colour of the label) and its label (the
// explicit label; else the label of the colour; else 0).
__device__ __forceinline__ void point_input(const FrameIn& in, const Luts* __restrict__ luts, int i, F3& pC, uint32_t& color, uint8_t& label) {
  pC = f3(in.xyz[3 * i], in.xyz[3 * i + 1], in.xyz[3 * i + 2]);
  color = 0;
  label = 0;
  if (in.rgba) color = (uint32_t)in.rgba[4 * i] | ((uint32_t)in.rgba[4 * i + 1] << 8) | ((uint32_t)in.rgba[4 * i + 2] << 16) | ((uint32_t)in.rgba[4 * i + 3] << 24);
  if (in.labels) label = in.labels[i];
  else if (in.rgba) label = label_of_color(luts, color & 0x00FFFFFFu);
  if (!in.rgba) color = luts->label_rgba[label];
}

// Depth entry, pixel pix = v * width + u of depth value d: the camera-frame point (depth_map_to_pointcloud.h:222-230)
__device__ __forceinline__ F3 backproject(const FrameIn& in, int pix, float d) {
  const int v = pix / in.width, u = pix - v * in.width;
  return f3(((float)u - in.cx) * d * in.constant_x, ((float)v - in.cy) * d * in.constant_y, d * in.z_scale);
}

// The point test: a label >= C is an error (CHECK_LT fast.cpp:134) and becomes 0; isPointValid (A.6) decides whether the point is
// integrated and whether it only clears.
__device__ __forceinline__ void point_test(const DevCfg& cfg, int freespace, Counters* cnt, F3 pC, uint8_t& label, bool& valid, bool& clearing) {
  if ((int)label >= cfg.C) { set_err(cnt, 1 /*KSG_ERR_INVALID_ARGUMENT*/); label = 0; }
  const float ray_distance = norm3(pC);
  valid = true;
  clearing = false;
  if (ray_distance < cfg.min_ray) valid = false;
  else if (ray_distance > cfg.max_ray) { if (cfg.allow_clear || freespace) clearing = true; else valid = false; }
  else clearing = freespace != 0;
  if (!(ray_distance == ray_distance)) valid = false;  // NaN points never pass the comparisons upstream either way
}
// getVoxelWeight (A.6)
__device__ __forceinline__ float point_weight(const DevCfg& cfg, F3 pC) {
  if (cfg.const_weight) return 1.0f;
  const float z = fabsf(pC.z);
  return (z > kEps) ? 1.0f / (z * z) : 0.0f;
}

// depth_map_to_pointcloud.h:213-266 for uint16 depth (DepthTraits<uint16_t>: valid = depth != 0, metres = depth * 0.001f): the raw value as
// float (exact), invalid -> NaN, so that the float pipeline (finite test, (u - cx) * depth * constant_x with constant_x = 0.001 / fx) applies
__global__ void k_u16_to_f32(const uint16_t* __restrict__ raw, int n, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { const uint16_t d = raw[i]; out[i] = d ? (float)d : __int_as_float(0x7fc00000); }
}

// RGB semantic image: the label and the colour (alpha 255) of every pixel
__global__ void k_rgb_to_label(const uint8_t* __restrict__ rgb, int n, const Luts* __restrict__ luts, uint8_t* __restrict__ label, uint32_t* __restrict__ color) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t c = (uint32_t)rgb[3 * i] | ((uint32_t)rgb[3 * i + 1] << 8) | ((uint32_t)rgb[3 * i + 2] << 16);
  label[i] = label_of_color(luts, c);
  color[i] = c | 0xFF000000u;
}

// merged, "sorted" integration order (voxblox SortedThreadSafeIndex, A.3): key = squared norm of the point
__global__ void k_sqnorm(FrameIn in, const Counters* cnt, int capacity, uint32_t* keys) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= capacity) return;
  if (i >= cnt->n_points) { keys[i] = 0xFFFFFFFFu; return; }
  F3 pC;
  if (in.depth) { const int pix = in.pix_list[i]; pC = backproject(in, pix, in.depth[pix]); }
  else pC = f3(in.xyz[3 * i], in.xyz[3 * i + 1], in.xyz[3 * i + 2]);
  keys[i] = __float_as_uint(dot3(pC, pC));
}

// One thread per sequence position (the order in which the reference's ThreadSafeIndex hands out points).
// merged: colour->label, validity, transform and bundleRays' per-point part (A.5).
__global__ void k_classify(DevCfg cfg, Xform T, FrameIn in, const Luts* __restrict__ luts,
                           int capacity, Counters* cnt, float4* __restrict__ pt_pC, float4* __restrict__ pt_pG,
                           uint8_t* __restrict__ pt_label, uint8_t* __restrict__ pt_flags, uint32_t* __restrict__ pt_color,
                           uint64_t* __restrict__ pt_key) {
  const int seq = blockIdx.x * blockDim.x + threadIdx.x;
  if (seq >= capacity) return;
  const int n = cnt->n_points;
  if (seq >= n) { pt_key[seq] = ~0ull; pt_flags[seq] = 0; return; }
  const int i = in.point_of_seq ? in.point_of_seq[seq] : mixed_index(seq, n);
  F3 pC;
  uint8_t label;
  uint32_t color;
  if (in.depth) {
    const int pix = in.pix_list[i];
    pC = backproject(in, pix, in.depth[pix]);
    label = in.label_img[pix];
    color = in.color_img ? in.color_img[pix] : luts->label_rgba[label];
  } else point_input(in, luts, i, pC, color, label);
  bool valid, clearing;
  point_test(cfg, in.freespace, cnt, pC, label, valid, clearing);
  const float w = point_weight(cfg, pC);
  const F3 pG = xform_apply(T, pC);
  pt_pC[seq] = make_float4(pC.x, pC.y, pC.z, w);
  pt_pG[seq] = make_float4(pG.x, pG.y, pG.z, w);
  pt_label[seq] = label;
  pt_color[seq] = color;
  pt_flags[seq] = (valid ? 1 : 0) | (clearing ? 2 : 0);
  uint64_t key = ~0ull;
  if (valid) {
    const I3 g = grid_index(pG, cfg.vsi);          // bundleRays (A.5)
    if (!key_in_range(g) || !index_in_range(mul(pG, cfg.vsi))) { set_err(cnt, 5); }
    else key = pack_key(g) | (clearing ? (1ull << 63) : 0ull);
  }
  pt_key[seq] = key;
  {  // count valid points: one atomic per warp
    const unsigned am = __activemask();
    const unsigned m = __ballot_sync(am, valid);
    if (m && (int)(threadIdx.x & 31) == (__ffs(am) - 1)) atomicAdd(&cnt->n_valid, __popc(m));
  }
}

// ---------------------------------------------------------------------------------------------
// state shared with the `fast` observed-set solver (ksg_fast3.cuh) and ksg_voxel.cuh
// ---------------------------------------------------------------------------------------------
struct RayState {      // saved DDA state after the materialised steps
  int cx, cy, cz, sg;  // sg: 2 bits per axis (0,1,2 = -1,0,+1)
  float tn0, tn1, tn2, ts0, ts1, ts2;
};
__device__ __forceinline__ void save_state(RayState& s, const Dda& d) {
  s.cx = d.cur.x; s.cy = d.cur.y; s.cz = d.cur.z;
  s.sg = (d.sg[0] + 1) | ((d.sg[1] + 1) << 2) | ((d.sg[2] + 1) << 4);
  s.tn0 = d.tn[0]; s.tn1 = d.tn[1]; s.tn2 = d.tn[2]; s.ts0 = d.ts[0]; s.ts1 = d.ts[1]; s.ts2 = d.ts[2];
}
__device__ __forceinline__ void load_state(Dda& d, const RayState& s) {
  d.cur.x = s.cx; d.cur.y = s.cy; d.cur.z = s.cz;
  d.sg[0] = (s.sg & 3) - 1; d.sg[1] = ((s.sg >> 2) & 3) - 1; d.sg[2] = ((s.sg >> 4) & 3) - 1;
  d.tn[0] = s.tn0; d.tn[1] = s.tn1; d.tn[2] = s.tn2; d.ts[0] = s.ts0; d.ts[1] = s.ts1; d.ts[2] = s.ts2;
}

// observed-set bucket entry: [performed:1][order = (rank << 16) | step : 39][value >> 20 : 13]
static constexpr uint64_t kEntPerf = 1ull << 63;
static constexpr int kEntOrderBits = 23 + kOrderStepBits;  // rank < 2^23, step < 2^16

// ---------------------------------------------------------------------------------------------
// spatial block hash (Layer<>::BlockHashMap replacement): open addressing, 64-bit packed keys
// ---------------------------------------------------------------------------------------------
struct MapRef {
  uint64_t* ht_keys;
  int* ht_slot;          // pool slot of the entry, -1 until k_block_init ran
  uint32_t ht_mask;
  int* new_list;         // hash positions inserted this frame
  int new_cap;
  uint8_t* pool;
  uint64_t* slot_key;    // block key of every pool slot
  int max_blocks;
  int* touched_stamp;    // per hash position: frame stamp of the last touch
  int* touched_list;
};

// Read-side helpers of the map (mesher, point queries): pool slot of a block key (-1: not in the hash) ...
__device__ __forceinline__ int ht_lookup_slot(const MapRef& m, uint64_t key) {
  uint32_t pos = mix64(key) & m.ht_mask;
  for (uint32_t probe = 0; probe <= m.ht_mask; ++probe) {
    const uint64_t k = m.ht_keys[pos];
    if (k == key) { const int s = m.ht_slot[pos]; return (s >= 0 && s < m.max_blocks) ? s : -1; }
    if (k == kEmptyKey) return -1;
    pos = (pos + 1) & m.ht_mask;
  }
  return -1;
}

// ... and the tile chunk holding voxel (lx, ly, lz) of the block in `slot`, with the voxel's index inside the tile in `vox`
__device__ __forceinline__ const uint8_t* mesh_voxel_chunk(const DevCfg& cfg, const MapRef& map, int slot, int lx, int ly, int lz, int& vox) {
  const int ts = cfg.tile_side_log2, tm = cfg.tile_side - 1;
  const int tile = (lx >> ts) + cfg.tiles_per_side * ((ly >> ts) + cfg.tiles_per_side * (lz >> ts));
  vox = (lx & tm) + cfg.tile_side * ((ly & tm) + cfg.tile_side * (lz & tm));
  return map.pool + (uint64_t)slot * cfg.block_stride + (uint64_t)tile * cfg.tile_stride;
}

__device__ __forceinline__ int ht_find_or_insert_raw(uint64_t* ht_keys, uint32_t ht_mask, int* new_list, int new_cap, uint64_t key, Counters* cnt) {
  uint32_t pos = mix64(key) & ht_mask;
  for (uint32_t probe = 0; probe <= ht_mask; ++probe) {
    const uint64_t k = ((volatile uint64_t*)ht_keys)[pos];
    if (k == key) return (int)pos;
    if (k == kEmptyKey) {
      const uint64_t old = atomicCAS((unsigned long long*)&ht_keys[pos], (unsigned long long)kEmptyKey, (unsigned long long)key);
      if (old == kEmptyKey) {
        const int i = atomicAdd(&cnt->n_new_blocks, 1);
        if (i < new_cap) new_list[i] = (int)pos; else set_err(cnt, 3);
        return (int)pos;
      }
      if (old == key) return (int)pos;
    }
    pos = (pos + 1) & ht_mask;
  }
  set_err(cnt, 3);
  return -1;
}
__device__ __forceinline__ int ht_find_or_insert(const MapRef& m, uint64_t key, Counters* cnt) {
  return ht_find_or_insert_raw(m.ht_keys, m.ht_mask, m.new_list, m.new_cap, key, cnt);
}

// update record: [hash position * tiles_per_block + tile : 32][voxel in tile : 9][order : 23]
__device__ __forceinline__ uint64_t make_record(const DevCfg& cfg, int htpos, I3 g, uint32_t order) {
  const int m = cfg.vps - 1;
  const int lx = g.x & m, ly = g.y & m, lz = g.z & m;  // getLocalFromGlobalVoxelIndex (A.2)
  const int ts = cfg.tile_side_log2, tm = cfg.tile_side - 1;
  const int tile = (lx >> ts) + cfg.tiles_per_side * ((ly >> ts) + cfg.tiles_per_side * (lz >> ts));
  const int vox = (lx & tm) + cfg.tile_side * ((ly & tm) + cfg.tile_side * (lz & tm));
  const uint64_t tk = (uint64_t)htpos * (uint64_t)cfg.tiles_per_block + (uint64_t)tile;
  return (tk << 32) | ((uint64_t)vox << kRecOrdBits) | (uint64_t)order;
}

// ---------------------------------------------------------------------------------------------
// merged: bundles (A.5 bundleRays + merged.cpp:235-294)
// ---------------------------------------------------------------------------------------------
// sorted (key, seq) pairs: a bundle = run of equal keys; its points are in sequence order (stable sort of a
// sequence-ordered array); its rank = first sequence position (canonical first-insertion order).
__global__ void k_bundle_heads(const uint64_t* __restrict__ ks, const uint32_t* __restrict__ seq_sorted, int capacity,
                               uint8_t* __restrict__ bflag, int* __restrict__ bstart) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= capacity) return;
  const uint64_t k = ks[i];
  if (k == ~0ull) return;
  if (i > 0 && ks[i - 1] == k) return;
  const size_t f = (size_t)(k >> 63) * (size_t)capacity + seq_sorted[i];  // non-clearing pass first (merged.cpp:126-144)
  bflag[f] = 1;
  bstart[f] = i;
}

// One warp per bundle (grid-stride).  The points of a bundle are gathered 32 at a time (lane = point); the weighted-mean
// recurrence of merged.cpp:271-275 runs over them in sequence order (uniform across lanes, operands by shuffle) because it
// is order dependent in floating point; the label histogram (merged.cpp:277-279) has lanes = classes.
__global__ void k_bundle_merge(DevCfg cfg, Xform T, Counters* cnt, const int* __restrict__ bundle_f, const int* __restrict__ bstart,
                               const uint64_t* __restrict__ ks, const uint32_t* __restrict__ seq_sorted, int capacity,
                               const float4* __restrict__ pt_pC, const uint8_t* __restrict__ pt_label, float* __restrict__ hist,
                               float4* __restrict__ b_param, uint8_t* __restrict__ b_flags, uint64_t* __restrict__ b_key,
                               int* __restrict__ b_nsteps) {
  const int lane = threadIdx.x & 31;
  const int warps_total = (gridDim.x * blockDim.x) >> 5;
  const int n_bundles = cnt->n_cast;
  const int C = cfg.C;
  unsigned long long steps = 0;
  for (int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < n_bundles; b += warps_total) {
    const int f = bundle_f[b];
    const int i0 = bstart[f];
    const uint64_t key = ks[i0];
    const bool clearing = (key >> 63) != 0;
    float hcount[8];   // classes lane, lane+32, ... (C <= 256)
#pragma unroll
    for (int q = 0; q < 8; ++q) hcount[q] = 0.0f;
    F3 mp = f3(0.0f, 0.0f, 0.0f);
    float mw = 0.0f;
    bool done = false;
    for (int base = i0; !done; base += 32) {
      const int idx = base + lane;
      const bool in = idx < capacity && ks[idx] == key;
      const unsigned m = __ballot_sync(0xffffffffu, in);
      const int nb = (m == 0xffffffffu) ? 32 : (__ffs(~m) - 1);   // the bundle's points are contiguous in the sorted array
      if (nb < 32) done = true;
      float4 pc = make_float4(0.f, 0.f, 0.f, 0.f);
      int lab = 0;
      if (lane < nb) { const uint32_t seq = seq_sorted[idx]; pc = pt_pC[seq]; lab = pt_label[seq]; }
      for (int jj = 0; jj < nb; ++jj) {
        const float pw = __shfl_sync(0xffffffffu, pc.w, jj);
        if (pw < kEps) continue;                                   // merged.cpp:268-270
        const float px = __shfl_sync(0xffffffffu, pc.x, jj), py = __shfl_sync(0xffffffffu, pc.y, jj), pz = __shfl_sync(0xffffffffu, pc.z, jj);
        const int l = __shfl_sync(0xffffffffu, lab, jj);
        const float tot = mw + pw;
        mp = f3((mp.x * mw + px * pw) / tot, (mp.y * mw + py * pw) / tot, (mp.z * mw + pz * pw) / tot);
        mw += pw;
#pragma unroll
        for (int q = 0; q < 8; ++q) if (q * 32 + lane == l) hcount[q] += 1.0f;
        if (clearing) { done = true; break; }                      // only take first point when clearing (merged.cpp:282-284)
      }
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) { const int c = q * 32 + lane; if (c < C) hist[(size_t)b * C + c] = hcount[q]; }
    if (lane == 0) {
      const F3 pG = xform_apply(T, mp);
      b_param[b] = make_float4(pG.x, pG.y, pG.z, mw);
      b_flags[b] = clearing ? 2 : 0;
      b_key[b] = key & ~(1ull << 63);
      Dda d;
      raycaster_init(d, f3(T.tx, T.ty, T.tz), pG, clearing, cfg.carving != 0, cfg.max_ray, cfg.vsi, cfg.tp.trunc, true);
      int n = d.length_in_steps + 1;
      if (!d.in_range) { set_err(cnt, 5); n = 0; }
      b_nsteps[b] = n;
      steps += (unsigned long long)n;
    }
  }
  warp_add(&cnt->ray_steps, steps);
}

// record ranges of the bundles: one warp-aggregated bump allocation per 32 bundles
__global__ void k_bundle_alloc(Counters* cnt, int* __restrict__ b_nsteps, long long* __restrict__ b_base, long long rec_cap) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = b < cnt->n_cast;
  const int n = live ? b_nsteps[b] : 0;
  const long long base = (long long)warp_alloc(&cnt->n_records, (unsigned long long)n);
  if (live) {
    if (base + n > rec_cap) { set_err(cnt, 4); b_nsteps[b] = 0; }
    b_base[b] = base;
  }
}

// tmp[b][i] = sum_j L[i][j] * freq[j]  (base.cpp:306-307) with L[i][j] = log_match on the diagonal, log_non_match
// elsewhere, column 0 zero (base.cpp:108-127); summation fixed as j ascending, one multiply + one add per term (A.9).
// tmp4 (optional): the same rows at a stride of C rounded up to a multiple of 4, padded with zeros, for 128-bit row loads.
__global__ void k_bundle_loglik(DevCfg cfg, const Counters* cnt, const float* __restrict__ hist, float* __restrict__ tmp, float* __restrict__ tmp4) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)cnt->n_cast * cfg.C;
  const int C4 = (cfg.C + 3) & ~3;
  if (t >= total) {   // row n_cast = zeros: target of padded row loads
    if (t < total + cfg.C) { tmp[t] = 0.0f; if (tmp4) { const long long b = t / cfg.C; const int i = (int)(t % cfg.C); tmp4[b * C4 + i] = 0.0f; if (i == 0) for (int k = cfg.C; k < C4; ++k) tmp4[b * C4 + k] = 0.0f; } }
    return;
  }
  const int i = (int)(t % cfg.C);
  const float* h = hist + (t - i);
  float acc = 0.0f;
  for (int j = 1; j < cfg.C; ++j) acc = acc + ((i == j) ? cfg.lm : cfg.ln) * h[j];
  tmp[t] = acc;
  if (tmp4) {
    const long long b = t / cfg.C;
    tmp4[b * C4 + i] = acc;
    if (i == 0) for (int k = cfg.C; k < C4; ++k) tmp4[b * C4 + k] = 0.0f;
  }
}

__global__ void k_emit_merged(DevCfg cfg, Xform T, Counters* cnt, MapRef map, const float4* __restrict__ b_param,
                              const uint8_t* __restrict__ b_flags, const uint64_t* __restrict__ b_key,
                              const int* __restrict__ b_nsteps, const long long* __restrict__ b_base,
                              const uint64_t* __restrict__ ks, int capacity, uint64_t* __restrict__ records) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = (b < cnt->n_cast) ? b_nsteps[b] : 0;
  unsigned long long skipped = 0;      // one atomic per warp at the end (one per skipped record was ~5 x 10^5 same-address atomics per frame)
  if (n > 0) {
  const float4 p = b_param[b];
  const bool clearing = (b_flags[b] & 2) != 0;
  Dda d;
  raycaster_init(d, f3(T.tx, T.ty, T.tz), f3(p.x, p.y, p.z), clearing, cfg.carving != 0, cfg.max_ray, cfg.vsi, cfg.tp.trunc, true);
  const long long base = b_base[b];
  I3 last_b; last_b.x = last_b.y = last_b.z = 0x7fffffff;
  int htpos = -1;
  const uint64_t own = b_key[b];
  for (int s = 0; s < n; ++s) {
    const I3 g = dda_next(d);
    bool skip = false;
    if (cfg.anti_grazing) {  // merged.cpp:306-313: skip voxels that are some bundle's end voxel
      if (!key_in_range(g)) skip = false;
      else {
        const uint64_t gk = pack_key(g);
        if (clearing || gk != own) {
          int lo = 0, hi = capacity;
          while (lo < hi) { const int mid = (lo + hi) >> 1; if (ks[mid] < gk) lo = mid + 1; else hi = mid; }
          skip = (lo < capacity && ks[lo] == gk);
        }
      }
    }
    if (skip) { records[base + s] = ~0ull; ++skipped; continue; }
    const I3 bi = block_of_voxel(g, cfg.vps_inv);
    if (bi.x != last_b.x || bi.y != last_b.y || bi.z != last_b.z) {
      last_b = bi;
      if (!key_in_range(bi)) { set_err(cnt, 5); htpos = -1; }
      else htpos = ht_find_or_insert(map, pack_key(bi), cnt);
    }
    records[base + s] = (htpos >= 0) ? make_record(cfg, htpos, g, (uint32_t)b) : ~0ull;
  }
  }
  warp_add(&cnt->n_skipped, skipped);
}

// ---------------------------------------------------------------------------------------------
// merged, KSG_BUNDLE_ORDER_LIBSTDCXX: bundle order = iteration order of the reference's std::unordered_map (merged.cpp:210-231)
// ---------------------------------------------------------------------------------------------
// libstdc++ keeps one singly linked node list; inserting into an empty bucket puts the node at the list FRONT, into a non-empty
// bucket at the front of that bucket's run, and a rehash re-inserts all nodes in list order by the same two rules.  Hence every
// phase (rehash + the insertions up to the next rehash) is one sort of the nodes by
//     (arrival of the FIRST node of the node's bucket, descending ; own arrival, descending)
// with arrival = position in the old list for rehashed nodes, then insertion time.  Prototype + proof against the real container:
// tools/libstdcxx_order.py, tests/test_unordered_map_order.py.  All phases run in one launch: k_bundle_order (ksg_bundle_order.cuh).
__global__ void k_bord_hash(Counters* cnt, const int* __restrict__ bundle_f, const int* __restrict__ bstart,
                            const uint64_t* __restrict__ ks, int capacity, uint32_t* __restrict__ hash) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  const int nb = cnt->n_cast;
  if (b >= nb) return;
  const int f = bundle_f[b];
  hash[b] = index_hash(unpack_key(ks[bstart[f]]));              // LongIndexHash of the bundle's voxel (A.2); bit 63 = clearing flag
  const bool clr = f >= capacity;
  if (clr && (b == 0 || bundle_f[b - 1] < capacity)) cnt->n_nonclear = b;   // bundle_f is ascending: non-clearing heads first
  if (!clr && b == nb - 1) cnt->n_nonclear = nb;
}

// ---------------------------------------------------------------------------------------------
// block pool
// ---------------------------------------------------------------------------------------------
// SemanticVoxel / TsdfVoxel default construction (semantic_voxel.h:14-27; TsdfVoxel A.0)
__global__ void k_block_init(DevCfg cfg, Counters* cnt, MapRef map) {
  const int n_new = cnt->n_new_blocks < map.new_cap ? cnt->n_new_blocks : map.new_cap;
  const int per_block = cfg.tiles_per_block;
  for (long long w = blockIdx.x; w < (long long)n_new * per_block; w += gridDim.x) {
    const int i = (int)(w / per_block), tile = (int)(w % per_block);
    const int slot = cnt->pool_count + i;
    if (slot >= map.max_blocks) { if (tile == 0 && threadIdx.x == 0) set_err(cnt, 3); continue; }
    if (tile == 0 && threadIdx.x == 0) {   // k_block_assign: hash entry -> pool slot
      const int pos = map.new_list[i];
      map.ht_slot[pos] = slot;
      map.slot_key[slot] = map.ht_keys[pos];
    }
    uint8_t* chunk = map.pool + (uint64_t)slot * cfg.block_stride + (uint64_t)tile * cfg.tile_stride;
    float* dist = (float*)chunk;
    float* wgt = (float*)(chunk + cfg.plane_f32);
    uint32_t* rgba = (uint32_t*)(chunk + 2 * cfg.plane_f32);
    uint32_t* srgba = (uint32_t*)(chunk + 3 * cfg.plane_f32);
    uint8_t* label = chunk + 4 * cfg.plane_f32;
    float* prior = (float*)(chunk + cfg.head_bytes);
    const int V = cfg.tile_voxels;
    for (int v = threadIdx.x; v < V; v += blockDim.x) {
      dist[v] = 0.0f; wgt[v] = 0.0f; rgba[v] = 0u; srgba[v] = 0xFF7F7F7Fu; label[v] = 0;
    }
    for (int t = threadIdx.x; t < cfg.C * V; t += blockDim.x) prior[t] = (float)-0.60205999132;
  }
}
__global__ void k_frame_finish(Counters* cnt, MapRef map) {
  int n_new = cnt->n_new_blocks < map.new_cap ? cnt->n_new_blocks : map.new_cap;
  if (cnt->pool_count + n_new > map.max_blocks) n_new = map.max_blocks - cnt->pool_count;
  cnt->pool_count += n_new;
}

// ---------------------------------------------------------------------------------------------
// tile apply
// ---------------------------------------------------------------------------------------------
static constexpr int kBigTileRecords = 8192;
__global__ void k_tile_heads(DevCfg cfg, Counters* cnt, MapRef map, const uint64_t* __restrict__ rec, long long n, int stamp,
                             long long* __restrict__ tile_begin, long long tile_cap) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t k = rec[i];
  if (k == ~0ull) return;
  const uint32_t tk = (uint32_t)(k >> 32);
  if (i > 0 && (uint32_t)(rec[i - 1] >> 32) == tk) return;
  const int pos = (int)(tk / (uint32_t)cfg.tiles_per_block);
  {   // updated() bookkeeping is replicated on every shard
    const int old = atomicExch(&map.touched_stamp[pos], stamp);
    if (old != stamp) map.touched_list[atomicAdd(&cnt->n_blocks_touched, 1)] = pos;
  }
  if (cfg.shard_count > 1 && tile_owner(map.ht_keys[pos], (int)(tk % (uint32_t)cfg.tiles_per_block), cfg.shard_count) != cfg.shard_rank) return;
  // does the tile hold more than kBigTileRecords records? (longest-processing-time-first scheduling)
  const long long probe = i + kBigTileRecords;
  const bool big = probe < n && (uint32_t)(rec[probe] >> 32) == tk;
  atomicAdd(&cnt->n_tiles, 1);
  if (big) { const int j = atomicAdd(&cnt->n_big_tiles, 1); if (j < tile_cap) tile_begin[j] = i; }
  else {
    const int j = atomicAdd(&cnt->n_small_tiles, 1);
    if (j < tile_cap) tile_begin[tile_cap - 1 - j] = i;
  }
  if (cnt->n_tiles > tile_cap) set_err(cnt, 4);
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  } while (!ok);
}
// TMA 1-D bulk copies (cp.async.bulk -> SASS UBLKCP)
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_store_1d(void* gmem_dst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_store_commit_wait() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// A "hot" voxel of a merged frame (ksg_hot.cuh): a run of >= kHotThresh records whose log-probability row was finished by the
// pre-pass, so that the tile kernel's semantic warp can skip the run.
struct HotSeg {
  long long begin, end;   // record range in the sorted array
  long long prior_off;    // byte offset of the voxel's log-probability row in the tile pool
  long long tile_off;     // byte offset of the voxel's tile chunk (distance plane first, then weight, ...)
  int first_chunk, n_chunks;
  int vox;                // voxel index inside the tile
  float cx, cy, cz;       // voxel centre (A.2 getCenterPointFromGridIndex)
};

struct ApplySrc {
  const float4* param;   // per order id: (point_G xyz, weight)
  const uint8_t* label;  // fast: measured label (one-hot frequencies, fast.cpp:132-135); NULL for merged
  const uint32_t* color; // fast: point colour; NULL -> (0,0,0,0) (merged.cpp:70 unfilled hash_colors)
  const float* tmp;      // merged: C floats per bundle = L * freq; NULL for fast
  const float* tmp4;     // merged, C <= 32: the same rows at stride ((C + 3) & ~3), zero padded (128-bit loads of k_voxel_apply_short_t)
  // HOTSEM instantiation only: segments sorted by begin, and their finished rows (32 floats per segment)
  const HotSeg* hot_segs;
  const float* hot_prior;
  const int* hot_tsdf_same;   // hot_voxel_mode 2: 1 = the frame provably leaves the voxel's (distance, weight, colour) untouched
  int n_hot;
  int hot_thresh;
};

static constexpr int kApplyThreads = 256;


// TSDF recurrence of one batch (<= 32 records, lane j holds record j's sdf / weight / colour) in record order (A.6).
// The weight chain does not depend on the distance, so it runs first (uniform over the lanes, each lane keeps the weight
// seen by ITS record; skipped when the voxel already sits at max_weight: min(max_weight, max_weight + uw) = max_weight for
// uw >= 0); then every lane evaluates its record assuming the distance did not change before it.  Free-space voxels stay
// pinned at +truncation, so whole batches commit without a sequential pass; the first record that moves the distance ends
// the speculation and the rest of the batch is replayed in order.
// WIDE (the hot-voxel kernel only, it has the registers): all 32 weights are shuffled into registers BEFORE the addition chain starts -
// interleaved, every FADD of the chain waits ~23 cycles for its own shuffle (ncu: 1972 of 2183 samples on that FADD were short-scoreboard
// stalls), 4x the latency of the addition itself.
template <bool WIDE = false>
__device__ __forceinline__ void tsdf_batch(const TsdfParams& tp, int lane, int nb, float sdf, float uw, uint32_t col, bool keep_blend,
                                           float& dist, float& wgt, uint32_t& rgba) {
  float w_before = wgt, wc = wgt;
  const unsigned negative = __ballot_sync(0xffffffffu, lane < nb && !(uw >= 0.0f));
  const bool saturated = (wgt == tp.max_weight) && negative == 0u;
  if (!saturated) {
    // The weight recurrence w <- min(max_weight, fl(w + u)), skipped while fl(w + u) < 1e-6, is sequential by definition.  When the
    // batch provably neither skips nor clamps - all u >= 0, w already >= 1e-6 (the sums only grow), and a generous bound of the final
    // sum stays below max_weight - it is a bare chain of float additions in record order (one dependent FADD per record instead of
    // FADD + compare + min + select); the hot voxels next to a MOVING camera are new every frame and never saturated.
    float usum = (lane < nb) ? uw : 0.0f;
    for (int o = 16; o > 0; o >>= 1) usum += __shfl_xor_sync(0xffffffffu, usum, o);
    // sequential partial sums <= (1 + 2^-24)^32 x the exact sum; the tree sum >= (1 - 2^-24)^6 x it: a 0.1 % margin is ample
    const bool plain = negative == 0u && wgt >= kEps && (wgt + usum) * 1.001f < tp.max_weight;
    if (WIDE && plain && nb == 32) {
      float u[32];
#pragma unroll
      for (int jj = 0; jj < 32; ++jj) u[jj] = __shfl_sync(0xffffffffu, uw, jj);
#pragma unroll
      for (int jj = 0; jj < 32; ++jj) {     // one dependent FADD per record
        w_before = (jj == lane) ? wc : w_before;
        wc = wc + u[jj];
      }
    } else if (plain && nb == 32) {
#pragma unroll
      for (int jj = 0; jj < 32; ++jj) {     // no loop overhead: shuffle, select, one dependent FADD per record
        const float uj = __shfl_sync(0xffffffffu, uw, jj);
        w_before = (jj == lane) ? wc : w_before;
        wc = wc + uj;
      }
    } else if (plain) {
      for (int jj = 0; jj < nb; ++jj) {
        const float uj = __shfl_sync(0xffffffffu, uw, jj);
        if (jj == lane) w_before = wc;
        wc = wc + uj;
      }
    } else {
      for (int jj = 0; jj < nb; ++jj) {
        const float uj = __shfl_sync(0xffffffffu, uw, jj);
        if (jj == lane) w_before = wc;
        const float nw = wc + uj;
        if (!(nw < kEps)) wc = fminf(tp.max_weight, nw);
      }
    }
  }
  bool applies = false;
  float dn = dist;
  if (lane < nb) {
    const float nw = w_before + uw;
    if (!(nw < kEps)) {
      applies = true;
      const float nd = (sdf * uw + dist * w_before) / nw;
      dn = (nd > 0.0f) ? fminf(tp.trunc, nd) : fmaxf(-tp.trunc, nd);
    }
  }
  if (keep_blend) {   // colour blending only near the surface, in record order (needs only the weight chain)
    unsigned m = __ballot_sync(0xffffffffu, applies && fabsf(sdf) < tp.trunc);
    while (m) {
      const int jj = __ffs(m) - 1;
      m &= m - 1;
      rgba = blend_two_colors(rgba, __shfl_sync(0xffffffffu, w_before, jj), __shfl_sync(0xffffffffu, col, jj),
                              __shfl_sync(0xffffffffu, uw, jj));
    }
  }
  const unsigned moved = __ballot_sync(0xffffffffu, applies && (__float_as_uint(dn) != __float_as_uint(dist)));
  if (moved) {
    const int f = __ffs(moved) - 1;
    dist = __shfl_sync(0xffffffffu, dn, f);
    for (int jj = f + 1; jj < nb; ++jj) {
      const float sj = __shfl_sync(0xffffffffu, sdf, jj);
      const float uj = __shfl_sync(0xffffffffu, uw, jj);
      const float wb = __shfl_sync(0xffffffffu, w_before, jj);
      const float nw = wb + uj;
      if (!(nw < kEps)) {
        const float nd = (sj * uj + dist * wb) / nw;
        dist = (nd > 0.0f) ? fminf(tp.trunc, nd) : fmaxf(-tp.trunc, nd);
      }
    }
  }
  wgt = wc;
}

// merged: one CTA per touched tile, tiles handed out through a device-side queue.  The tile's voxel planes (and, when
// they fit, its log-probability rows) are staged in shared memory with ONE TMA bulk copy (cooperative copy when
// USE_TMA == false) that overlaps the record-segment scan.  Each warp then takes voxels from a CTA-local queue;
// a voxel's update records (sorted by (voxel, order)) are applied in the reference's order:
//   * lanes = records : the state-independent half of updateTsdfVoxel (sdf, weight drop-off; A.6) for 32 records
//   * all lanes       : the (distance, weight, colour) recurrence, one record after the other
//   * lanes = classes : semantic log-probability rows, prior[c] += (L * freq)[c]  (base.cpp:283-314)
// followed by the arg-max label (base.cpp:352-367) and the colour hand-off (base.cpp:370-191).  The tile is
// written back once with a TMA bulk store.  NCH = ceil(C / 32) register chunks per lane.
template <bool USE_TMA, int NCH, bool HOTSEM = false>
__global__ void __launch_bounds__(512, 1) k_tile_apply(DevCfg cfg, Xform T, Counters* cnt, MapRef map,
                                                               const Luts* __restrict__ luts, const uint64_t* __restrict__ rec,
                                                               long long n_rec, const long long* __restrict__ tile_begin,
                                                               long long tile_cap, ApplySrc src,
                                                               long long* __restrict__ tile_debug) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int V = cfg.tile_voxels;
  const int C = cfg.C;
  float* s_dist = (float*)smem;
  float* s_wgt = (float*)(smem + cfg.plane_f32);
  uint32_t* s_rgba = (uint32_t*)(smem + 2 * cfg.plane_f32);
  uint32_t* s_srgba = (uint32_t*)(smem + 3 * cfg.plane_f32);
  uint8_t* s_label = smem + 4 * cfg.plane_f32;
  float* s_prior = (float*)(smem + cfg.head_bytes);             // only when cfg.full_stage
  const uint32_t stage_bytes = cfg.head_bytes + (cfg.full_stage ? cfg.prior_bytes : 0u);
  uint8_t* aux = smem + stage_bytes;
  int* s_seg_lo = (int*)aux;                 // [V]
  int* s_seg_hi = s_seg_lo + V;              // [V]
  uint64_t* s_bar = (uint64_t*)(s_seg_hi + V + (V & 1));
  __shared__ long long s_begin, s_end;
  __shared__ uint8_t* s_chunk;
  __shared__ int s_g0x, s_g0y, s_g0z, s_tile, s_vox_cursor;

  const int tid = threadIdx.x, lane = tid & 31;
  const int nthreads = blockDim.x;
  uint32_t phase = 0;
  if (USE_TMA && tid == 0) { mbar_init(s_bar, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
  __syncthreads();
  const int n_tiles = cnt->n_tiles, n_big = cnt->n_big_tiles;
  const F3 origin = f3(T.tx, T.ty, T.tz);
  const bool keep_blend = cfg.color_mode == 0;  // kColor: the blended colour survives; otherwise base.cpp:177-185 overwrites it
  const uint32_t ord_mask = (1u << kRecOrdBits) - 1u, vox_mask = (1u << kRecVoxBits) - 1u;

  for (;;) {
    if (tid == 0) s_tile = atomicAdd(&cnt->tile_cursor, 1);
    __syncthreads();
    const int j = s_tile;
    if (j >= n_tiles) break;
    const long long t_start = tile_debug ? clock64() : 0;
    if (tid == 0) {
      const long long b = (j < n_big) ? tile_begin[j] : tile_begin[tile_cap - 1 - (j - n_big)];
      const uint32_t tk = (uint32_t)(rec[b] >> 32);
      long long lo = b, hi = n_rec;  // first record whose tile key is greater
      while (lo < hi) { const long long mid = (lo + hi) >> 1; if ((uint32_t)(rec[mid] >> 32) <= tk) lo = mid + 1; else hi = mid; }
      s_begin = b; s_end = lo;
      const int pos = (int)(tk / (uint32_t)cfg.tiles_per_block), tile = (int)(tk % (uint32_t)cfg.tiles_per_block);
      const int slot = map.ht_slot[pos];
      uint8_t* chunk = (slot >= 0 && slot < map.max_blocks) ? map.pool + (uint64_t)slot * cfg.block_stride + (uint64_t)tile * cfg.tile_stride : nullptr;
      s_chunk = chunk;
      const I3 bi = unpack_key(map.ht_keys[pos]);
      const int tps = cfg.tiles_per_side;
      const int tx = tile % tps, ty = (tile / tps) % tps, tz = tile / (tps * tps);
      s_g0x = bi.x * cfg.vps + tx * cfg.tile_side;
      s_g0y = bi.y * cfg.vps + ty * cfg.tile_side;
      s_g0z = bi.z * cfg.vps + tz * cfg.tile_side;
      s_vox_cursor = 0;
      if (USE_TMA && chunk) { mbar_expect_tx(s_bar, stage_bytes); tma_load_1d(smem, chunk, stage_bytes, s_bar); }
    }
    for (int v = tid; v < V; v += nthreads) { s_seg_lo[v] = 0; s_seg_hi[v] = 0; }
    __syncthreads();
    uint8_t* chunk = s_chunk;
    if (chunk == nullptr) continue;  // pool overflow already flagged; the loop-top barrier keeps the CTA in step
    const long long begin = s_begin, end = s_end;
    // per-voxel record segments (overlaps the bulk load)
    for (long long i = begin + tid; i < end; i += nthreads) {
      const int vx = (int)((rec[i] >> kRecOrdBits) & vox_mask);
      if (i == begin || (int)((rec[i - 1] >> kRecOrdBits) & vox_mask) != vx) s_seg_lo[vx] = (int)(i - begin);
      if (i + 1 == end || (int)((rec[i + 1] >> kRecOrdBits) & vox_mask) != vx) s_seg_hi[vx] = (int)(i + 1 - begin);
    }
    if (USE_TMA) { mbar_wait(s_bar, phase); phase ^= 1; }
    else for (uint32_t t = tid; t < stage_bytes / 16; t += nthreads) ((uint4*)smem)[t] = ((const uint4*)chunk)[t];
    __syncthreads();
    float* g_prior = (float*)(chunk + cfg.head_bytes);

    // Work items of the CTA's warps: (voxel, role).  A voxel's TSDF recurrence and its semantic recurrences are
    // independent (DESIGN.md §3), so long segments are handled by two warps, one per role, with lean loops; short
    // segments by one warp doing both.
    constexpr int kSplitLen = 96;
    for (;;) {
      int item = 0;
      if (lane == 0) item = atomicAdd(&s_vox_cursor, 1);
      item = __shfl_sync(0xffffffffu, item, 0);
      if (item >= 2 * V) break;
      const int v = item >> 1;
      const int lo = s_seg_lo[v], hi = s_seg_hi[v];
      if (lo >= hi) continue;
      const bool split = NCH == 1 && (hi - lo) >= kSplitLen;
      const int role = item & 1;                 // 0: TSDF (+ everything for short segments), 1: semantic half of a split voxel
      if (role == 1 && !split) continue;
      const bool do_tsdf = !split || role == 0;
      const bool do_sem = !split || role == 1;
      const int ts = cfg.tile_side_log2, tm = cfg.tile_side - 1;
      I3 g; g.x = s_g0x + (v & tm); g.y = s_g0y + ((v >> ts) & tm); g.z = s_g0z + (v >> (2 * ts));
      const F3 center = voxel_center(g, cfg.voxel_size);
      float dist = s_dist[v], wgt = s_wgt[v];
      uint32_t rgba = s_rgba[v];
      float* prow = (cfg.full_stage ? s_prior : g_prior) + (size_t)v * C;
      float p[NCH];
#pragma unroll
      for (int q = 0; q < NCH; ++q) { const int c = q * 32 + lane; p[q] = (c < C) ? prow[c] : 0.0f; }

      bool hot_done = false;
      if (HOTSEM && NCH == 1 && split && (hi - lo) >= src.hot_thresh) {
        // the pre-pass may have dealt with this voxel: look the run up by its first record
        const long long first = begin + lo;
        int a = 0, b = src.n_hot;
        while (a < b) { const int mid = (a + b) >> 1; if (src.hot_segs[mid].begin < first) a = mid + 1; else b = mid; }
        if (a < src.n_hot && src.hot_segs[a].begin == first && src.hot_segs[a].end == begin + hi) {
          if (role == 1) {                       // semantic role: the finished log-probability row
            p[0] = (lane < C) ? src.hot_prior[(size_t)a * 32 + lane] : 0.0f;
            hot_done = true;
          } else if (src.hot_tsdf_same != nullptr && src.hot_tsdf_same[a] != 0) {
            hot_done = true;                     // TSDF role: every record was checked to leave the saturated state as it is
          }
        }
      }
      if (hot_done) {
        // nothing to accumulate
      } else if (NCH == 1) {
        // software pipeline over batches of 32 records: record keys are fetched two batches ahead, the parameters and the
        // 32 (L * freq) row values of the next batch one batch ahead, so that the recurrences below never wait on L2.
        // Padded lanes / rows point at the all-zero row behind the last bundle (adds +0.0f, exact).
        const int nbatches = (hi - lo + 31) >> 5;
        const uint32_t zero_row = (uint32_t)cnt->n_cast;
        const float* lane_tmp = src.tmp + (lane < C ? lane : 0);
        const bool lane_live = lane < C;
        uint32_t ord_a = (lo + lane < hi) ? ((uint32_t)rec[begin + lo + lane] & ord_mask) : zero_row;
        uint32_t ord_b = (lo + 32 + lane < hi) ? ((uint32_t)rec[begin + lo + 32 + lane] & ord_mask) : zero_row;
        float4 pr_a = (do_tsdf && lo + lane < hi) ? src.param[ord_a] : make_float4(0.f, 0.f, 0.f, 0.f);
        float rv_a[32];
        if (do_sem) {
#pragma unroll
          for (int u = 0; u < 32; ++u) rv_a[u] = __ldg(lane_tmp + (size_t)__shfl_sync(0xffffffffu, ord_a, u) * C);
        }
        for (int bi = 0; bi < nbatches; ++bi) {
          const int base = lo + (bi << 5);
          const int nb = (hi - base) < 32 ? (hi - base) : 32;
          // ---- issue the loads of the following batches
          const uint32_t ord_c = (base + 64 + lane < hi) ? ((uint32_t)rec[begin + base + 64 + lane] & ord_mask) : zero_row;
          float4 pr_b = make_float4(0.f, 0.f, 0.f, 0.f);
          if (do_tsdf && base + 32 + lane < hi) pr_b = src.param[ord_b];
          float rv_b[32];
          if (do_sem) {
#pragma unroll
            for (int u = 0; u < 32; ++u) rv_b[u] = __ldg(lane_tmp + (size_t)__shfl_sync(0xffffffffu, ord_b, u) * C);
          }
          // ---- this batch
          if (do_sem) {
#pragma unroll
            for (int u = 0; u < 32; ++u) p[0] += rv_a[u];
#pragma unroll
            for (int u = 0; u < 32; ++u) rv_a[u] = rv_b[u];
          }
          if (do_tsdf) {
            float sdf = 0.0f, uw = 0.0f;
            if (lane < nb) tsdf_measure(cfg.tp, origin, f3(pr_a.x, pr_a.y, pr_a.z), center, pr_a.w, sdf, uw);
            tsdf_batch(cfg.tp, lane, nb, sdf, uw, 0u, keep_blend, dist, wgt, rgba);
            pr_a = pr_b;
          }
          ord_b = ord_c;
        }
        if (!lane_live) p[0] = 0.0f;
      } else {
      for (int base = lo; base < hi; base += 32) {
        const int k = base + lane;
        uint32_t ord = 0, col = 0;
        float sdf = 0.0f, uw = 0.0f;
        if (k < hi) {
          ord = (uint32_t)(rec[begin + k]) & ord_mask;
          const float4 pr = src.param[ord];
          tsdf_measure(cfg.tp, origin, f3(pr.x, pr.y, pr.z), center, pr.w, sdf, uw);
          if (src.color && keep_blend) col = src.color[ord];
        }
        const int nb = (hi - base) < 32 ? (hi - base) : 32;
        // (L * freq) rows, lanes = classes: lane c adds column c of the records' rows in record order; kRowUnroll rows are
        // loaded (coalesced, independent) before the first add so that the L2 latency is paid once per group
        constexpr int kRowUnroll = (NCH <= 2) ? 16 / NCH : 2;
        for (int j0 = 0; j0 < nb; j0 += kRowUnroll) {
          float rv[kRowUnroll][NCH];
#pragma unroll
          for (int u = 0; u < kRowUnroll; ++u) {
            const uint32_t o = __shfl_sync(0xffffffffu, ord, (j0 + u) & 31);
            const float* row = src.tmp + (size_t)o * C;
#pragma unroll
            for (int q = 0; q < NCH; ++q) { const int cc = q * 32 + lane; rv[u][q] = (j0 + u < nb && cc < C) ? __ldg(row + cc) : 0.0f; }
          }
#pragma unroll
          for (int u = 0; u < kRowUnroll; ++u) {
#pragma unroll
            for (int q = 0; q < NCH; ++q) p[q] += rv[u][q];   // + 0.0f is exact for the padded tail
          }
        }
        tsdf_batch(cfg.tp, lane, nb, sdf, uw, col, keep_blend, dist, wgt, rgba);
      }
      }
      int bi_lab = 0;
      float best = 0.0f;
      if (do_sem) {
        // arg-max, first maximum wins (base.cpp:352-367)
        best = -3.402823466e38f;
        int bi = 0x7fffffff;
#pragma unroll
        for (int q = 0; q < NCH; ++q) { const int c = q * 32 + lane; if (c < C && (p[q] > best || bi == 0x7fffffff)) { best = p[q]; bi = c; } }
        for (int o = 16; o > 0; o >>= 1) {
          const float ob = __shfl_down_sync(0xffffffffu, best, o);
          const int oi = __shfl_down_sync(0xffffffffu, bi, o);
          if (oi != 0x7fffffff && (bi == 0x7fffffff || ob > best || (ob == best && oi < bi))) { best = ob; bi = oi; }
        }
        best = __shfl_sync(0xffffffffu, best, 0);
        bi_lab = __shfl_sync(0xffffffffu, bi, 0);
#pragma unroll
        for (int q = 0; q < NCH; ++q) { const int c = q * 32 + lane; if (c < C) prow[c] = p[q]; }
      }
      if (lane == 0) {
        if (do_tsdf) { s_dist[v] = dist; s_wgt[v] = wgt; }
        if (do_sem) {
          s_label[v] = (uint8_t)bi_lab;
          const uint32_t sc = luts->label_rgba[bi_lab];          // base.cpp:370-380
          s_srgba[v] = sc;
          if (cfg.color_mode == 1) s_rgba[v] = sc;               // kSemantic (base.cpp:177-180)
          else if (cfg.color_mode == 2) s_rgba[v] = rainbow_color_map((double)expf(best));  // base.cpp:181-185
        }
        if (do_tsdf && cfg.color_mode == 0) s_rgba[v] = rgba;    // kColor: the blended colour is the result
      }
    }
    // ---- write the tile back
    if (USE_TMA) {
      fence_proxy_async();
      __syncthreads();
      if (tid == 0) { tma_store_1d(chunk, smem, stage_bytes); tma_store_commit_wait(); }
    } else {
      __syncthreads();
      for (uint32_t t = tid; t < stage_bytes / 16; t += nthreads) ((uint4*)chunk)[t] = ((const uint4*)smem)[t];
    }
    if (tile_debug && tid == 0) { tile_debug[2 * j] = end - begin; tile_debug[2 * j + 1] = clock64() - t_start; }
    // the loop-top barrier orders the store's completion before the next tile's load
  }
}

// ---------------------------------------------------------------------------------------------
// import: voxblox block layout -> tiles (inverse of k_export); `fresh[bi]` = 1: default-construct the block first
// ---------------------------------------------------------------------------------------------
__global__ void k_import(DevCfg cfg, MapRef map, const int* __restrict__ slots, const uint8_t* __restrict__ fresh, int nb,
                         const float* __restrict__ i_dist, const float* __restrict__ i_wgt, const uint32_t* __restrict__ i_rgba,
                         const uint8_t* __restrict__ i_label, const float* __restrict__ i_prior, const uint32_t* __restrict__ i_srgba) {
  const int per_block = cfg.tiles_per_block;
  const int V = cfg.tile_voxels;
  const size_t VB = (size_t)cfg.vps * cfg.vps * cfg.vps;
  for (long long w = blockIdx.x; w < (long long)nb * per_block; w += gridDim.x) {
    const int bi = (int)(w / per_block), tile = (int)(w % per_block);
    uint8_t* chunk = map.pool + (uint64_t)slots[bi] * cfg.block_stride + (uint64_t)tile * cfg.tile_stride;
    float* dist = (float*)chunk;
    float* wgt = (float*)(chunk + cfg.plane_f32);
    uint32_t* rgba = (uint32_t*)(chunk + 2 * cfg.plane_f32);
    uint32_t* srgba = (uint32_t*)(chunk + 3 * cfg.plane_f32);
    uint8_t* label = chunk + 4 * cfg.plane_f32;
    float* prior = (float*)(chunk + cfg.head_bytes);
    const int tps = cfg.tiles_per_side, ts = cfg.tile_side_log2, tm = cfg.tile_side - 1;
    const int tx = tile % tps, ty = (tile / tps) % tps, tz = tile / (tps * tps);
    const bool fr = fresh[bi] != 0;
    for (int v = threadIdx.x; v < V; v += blockDim.x) {
      const int lx = tx * cfg.tile_side + (v & tm), ly = ty * cfg.tile_side + ((v >> ts) & tm), lz = tz * cfg.tile_side + (v >> (2 * ts));
      const size_t lin = (size_t)bi * VB + (size_t)lx + (size_t)cfg.vps * ((size_t)ly + (size_t)cfg.vps * lz);
      if (i_dist) dist[v] = i_dist[lin]; else if (fr) dist[v] = 0.0f;
      if (i_wgt) wgt[v] = i_wgt[lin]; else if (fr) wgt[v] = 0.0f;
      if (i_rgba) rgba[v] = i_rgba[lin]; else if (fr) rgba[v] = 0u;
      if (i_srgba) srgba[v] = i_srgba[lin]; else if (fr) srgba[v] = 0xFF7F7F7Fu;
      if (i_label) label[v] = i_label[lin]; else if (fr) label[v] = 0;
      for (int c = 0; c < cfg.C; ++c) {
        if (i_prior) prior[(size_t)v * cfg.C + c] = i_prior[lin * cfg.C + c];
        else if (fr) prior[(size_t)v * cfg.C + c] = (float)-0.60205999132;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// export: tiles -> voxblox block layout (linear index x + vps*(y + vps*z))
// ---------------------------------------------------------------------------------------------
__global__ void k_export(DevCfg cfg, MapRef map, const int* __restrict__ slots, int nb, float* __restrict__ o_dist,
                         float* __restrict__ o_wgt, uint32_t* __restrict__ o_rgba, uint8_t* __restrict__ o_label,
                         float* __restrict__ o_prior, uint32_t* __restrict__ o_srgba) {
  const int per_block = cfg.tiles_per_block;
  const int V = cfg.tile_voxels;
  const size_t VB = (size_t)cfg.vps * cfg.vps * cfg.vps;
  for (long long w = blockIdx.x; w < (long long)nb * per_block; w += gridDim.x) {
    const int bi = (int)(w / per_block), tile = (int)(w % per_block);
    const uint8_t* chunk = map.pool + (uint64_t)slots[bi] * cfg.block_stride + (uint64_t)tile * cfg.tile_stride;
    const float* dist = (const float*)chunk;
    const float* wgt = (const float*)(chunk + cfg.plane_f32);
    const uint32_t* rgba = (const uint32_t*)(chunk + 2 * cfg.plane_f32);
    const uint32_t* srgba = (const uint32_t*)(chunk + 3 * cfg.plane_f32);
    const uint8_t* label = chunk + 4 * cfg.plane_f32;
    const float* prior = (const float*)(chunk + cfg.head_bytes);
    const int tps = cfg.tiles_per_side, ts = cfg.tile_side_log2, tm = cfg.tile_side - 1;
    const int tx = tile % tps, ty = (tile / tps) % tps, tz = tile / (tps * tps);
    for (int v = threadIdx.x; v < V; v += blockDim.x) {
      const int lx = tx * cfg.tile_side + (v & tm), ly = ty * cfg.tile_side + ((v >> ts) & tm), lz = tz * cfg.tile_side + (v >> (2 * ts));
      const size_t lin = (size_t)bi * VB + (size_t)lx + (size_t)cfg.vps * ((size_t)ly + (size_t)cfg.vps * lz);
      if (o_dist) o_dist[lin] = dist[v];
      if (o_wgt) o_wgt[lin] = wgt[v];
      if (o_rgba) o_rgba[lin] = rgba[v];
      if (o_srgba) o_srgba[lin] = srgba[v];
      if (o_label) o_label[lin] = label[v];
      if (o_prior) for (int c = 0; c < cfg.C; ++c) o_prior[lin * cfg.C + c] = prior[(size_t)v * cfg.C + c];
    }
  }
}

}  // namespace ksg
