// ksg_fast.cuh — the `fast` integrator's frame: six launches and no host read-back inside the frame.
//
//   k_fast_count       depth image, 128-bit loads: finite pixels per 1024-pixel block; the last block to finish scans the
//                      block counts (ticket) and resets the frame counters                      (depth entry only)
//   k_fast_classify    image order, 4 pixels / thread (float4 depth + uchar4 label): back-projection, validity, dynamic
//                      labels, T_G_C * p, start cell; the sequence position (voxblox ThreadSafeIndex, A.3) comes from the
//                      inverse of the mixed permutation; the start-set visits merged per slot into the slot's record, and
//                      the slots the frame touched listed                                                    (fast.cpp:75-92)
//   k_fast_start_slots start_voxel_approx_set_ decision once per touched slot: cast bit of the first visitor + table commit
//                      where one start cell visited the slot; slots shared by several cells listed for k_fast_solve3 (fast.cpp:90)
//   k_fast_solve3      ONE persistent cooperative kernel, grid barriers between its phases: start-set slots shared by
//                      several cells, compaction of the cast rays, ray set-up, the observed-set fixpoint sweeps to convergence
//                      (device-side test), table commit, and the distribution of the update keys to per-tile segments
//                      (count, allocate, scatter) + new-block construction               (ksg_fast3.cuh, fast.cpp:110-141)
//   k_fast_group       one CTA per touched 8^3 tile: the tile's keys sorted by (voxel, ray rank) in place (the reference's
//                      per-voxel update order), one work item per touched voxel into a frame-wide array
//   k_fast_apply       one warp per work item: the voxel's state read from the pool, its records applied (TSDF + semantic
//                      update), the voxel written back
// The "sorted" integration order adds k_fast_sqnorm(_points), k_fast_pad_keys, a radix sort and k_fast_invert_perm before k_fast_classify.
#pragma once
#include "ksg_kernels.cuh"

namespace ksg {

static constexpr int kCountBlock = 1024;      // pixels per block of k_fast_count / k_fast_classify (256 threads x 4)
static constexpr int kSolveThreads = 1024;     // default block size of k_fast_solve3 (KSG_SOLVE_THREADS)
static constexpr int kFastKeyCap = 4096;      // update records of one tile sorted in shared memory (more: sorted in place in global memory)
static constexpr int kGroupThreads = 512;      // block size of k_fast_group
static constexpr int kFastApplyThreads = 256;  // block size of k_fast_apply
static constexpr int kRecVoxMax = 1 << kRecVoxBits;   // voxels of one tile
static constexpr int kTimelineSlots = 64;

struct FastCounters {      // device-resident state of the frame driver (persistent across frames)
  unsigned int ticket_count;                 // "last block done" ticket of k_fast_count
  unsigned int gridbar;                      // grid barrier of k_fast_solve3
  int sweep_base;                            // id of the last observed-set sweep ever run (sweep ids are monotonic: slot stamps)
  int sweeps_last;                           // sweeps of the last frame
  int tile_cursor;
  int n_tile_list;
  int pool_base;                             // pool_count before this frame's new blocks
  unsigned long long rec_cursor;             // allocation cursor of the per-tile key segments
  int ovf_count;                             // overflow pool cursor of the observed-set buckets
  unsigned long long n_touched;              // start-set slots visited this frame (k_fast_classify)
  int n_mixed;                               // start-set slots visited by more than one start cell this frame
  int m_cursor;                              // allocation cursor of their visitor lists
  int log_count;                             // work items of k_fast_apply = update-log entries of the frame (may exceed the log's capacity:
                                             // then the log is incomplete)
  int item_cursor;                           // claim cursor of k_fast_apply (zeroed by k_fast_group)
  int wl_claim[4];                           // slot sweep & 3: next item of the sweep's scan list claimed by a warp
  int wl_count[4];                           // ... rays on the sweep's scan list
  long long timeline[kTimelineSlots];        // clock64 of block 0 at the phase boundaries of k_fast_solve3 (profiling)
  long long dbg[16];                         // profiling only: maxima / counts gathered inside the solve kernel (see ksg_debug_fast_timeline)
};

struct TileDesc { uint32_t tk; int n; long long off; };
// what k_fast_apply needs of a tile (k_fast_group, index = the tile's index in tile_list) and of a touched voxel
struct __align__(16) FastTile { long long off; int slot, tile, bx, by, bz, pad; };
struct __align__(16) FastItem { int tile, vox, lo, len; };   // lo: first key of the voxel's run, relative to the tile's segment

// update log (eager host-layer sync of the C++ drop-in classes): one entry per voxel the frame updated, its final state
struct VoxelUpdate { int bx, by, bz; uint32_t lin_label; float dist, wgt; uint32_t rgba, srgba; };   // lin_label = linear voxel index | label << 24

// start set: the persistent table and one record per slot of the frame's visits.  k_fast_classify fills the records of the slots
// it visits and lists those slots; whoever decides a slot (k_fast_start_slots, or phase 0b of k_fast_solve3 for a slot shared by
// several cells) empties its record again, so no record needs a clear per frame.
struct __align__(16) StartRec {
  uint32_t first;        // smallest sequence position that visited the slot; for a shared slot, once k_fast_start_slots has listed
                         // it: the cursor of its visitor list in m_list (phase 0a)
  uint32_t hmin, hmax;   // smallest / largest (value >> 20) among the visitors: different <=> several cells share the slot
  uint32_t visits;       // visitors this frame
};
__device__ __forceinline__ uint4 start_rec_empty() { return make_uint4(~0u, ~0u, 0u, 0u); }
struct StartBuf {
  StartRec* rec;            // [2^20]
  uint32_t* table;          // [2^20] persistent: value >> 20 of the slot's last visitor
  int* touched;             // slots visited this frame (FastCounters::n_touched)
  const int* i_of_seq;      // "sorted" order mode: input index of sequence position s, else NULL (mixed: closed form)
};

// observed-set solver (ksg_fast3.cuh)
struct Cand;
struct OvfEnt;
struct RayRec;
struct Obs3 {
  Cand* cand;              // one 16-byte record per materialised ray step
  long long ext_base, cand_cap;
  int* slot_cnt;           // [2^20] performed-ever candidates of the slot this frame (cleared per frame)
  uint64_t* bkt;           // [2^20][kBkt3] entries [performed:1][order:39][value >> 20 : 13]
  int* head;               // [2^20] overflow list head (cleared to -1 per frame)
  OvfEnt* ovf;             // overflow pool (slots with more than kBkt3 performed-ever candidates)
  int ovf_cap;
  uint64_t* stamp_max;     // [2^20] max over the toggles of the slot of (sweep << 32 | ray)
  uint64_t* stamp_min;     // [2^20] min over the toggles of ((~sweep) << 32 | ray)
  uint32_t* table;         // persistent compact table: value >> 20
};

// everything the fast frame kernels need (passed by value)
struct FastFrame {
  DevCfg cfg;
  Xform T;
  FrameIn in;
  const Luts* luts;
  Counters* cnt;
  FastCounters* fc;
  MapRef map;
  StartBuf sb;
  uint64_t set_offset;
  int capacity;              // host upper bound of the point count (pixels or points)
  int n_count_blocks;        // blocks of k_fast_count / k_fast_classify (depth entry)
  int vec_ok;                // depth / label pointers allow 128-bit / 32-bit vector loads
  int frame_stamp;
  int profile;               // per-ray / per-slot probes of the solve kernel (FastCounters::dbg): same-address atomics that slow the
                             // phases they probe, the ray set-up the most
  int prof_marks;            // block 0 of the solve kernel stamps clock64 at every phase boundary (FastCounters::timeline)
  const int* seq_of_i;       // "sorted" order mode: sequence position of input index i, else NULL (mixed: closed form)
  int* block_cnt; int* block_off;     // finite pixels per 1024-pixel block
  uint32_t* cast_bits;                // one bit per sequence position: cast (empty between frames: phase 0c clears what it reads)
  int* warp_off;                      // cast points before each word of cast_bits
  // per input index (image order): start-set value (hash + offset), ~0 for a point that is not valid; depth entry: the pixel
  uint64_t* pt_key; int* pt_pix;
  // per cast ray
  int* cast_seq; float4* ray_param; uint8_t* ray_label; uint8_t* ray_flags; uint32_t* ray_color;
  RayState* ray_state; long long* ext_off;
  // update keys
  long long rec_cap;
  uint32_t* keys;            // per-tile segments of (voxel << 23 | ray rank)
  int* tile_cnt;             // [hash capacity * tiles_per_block] records of the tile this frame (returns to 0 by itself)
  int* tile_slot;            // ... index of the tile in tile_list
  TileDesc* tile_list; long long tile_cap;
  // observed-set solver
  Obs3 o3;
  RayRec* rayrec;
  int* blk_run;              // consecutive-collision count at the start of every evaluation block (index: candidate index / 16)
  int* wl_listed;            // per ray: the latest sweep whose scan list holds it (sweep ids are monotonic: never cleared per frame)
  int* wl_list[2];           // scan lists of the sweeps after the second, slot sweep & 1
  // update log (NULL: off)
  VoxelUpdate* log_head; float* log_prior; int log_cap;
  // start-set slots shared by several cells
  int* mixed_list;           // such slots
  int* m_list;               // their visitors (sequence positions), grouped by slot
};

__device__ __forceinline__ int inv_mixed_index(int i, int n) {   // inverse of mixed_index (voxblox MixedThreadSafeIndex, A.3)
  const int groups = n / 1024;
  if (groups * 1024 <= i) return i;
  return (i % 1024) * groups + i / 1024;
}

// exclusive scan of a[0..n) into out[0..n) by ONE block (every thread of the block calls it); returns the total.  a and out are
// 16-byte aligned; every thread owns a contiguous run whose length is a multiple of four (128-bit loads and stores, all independent).
// POPC: the scan of the bit counts of a[].
template <bool POPC = false>
__device__ __forceinline__ int block_scan_array(const int* a, int* out, int n) {
  auto val = [](int x) { return POPC ? __popc(x) : x; };
  __shared__ int s_w[32];
  __shared__ int s_total;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int nthreads = blockDim.x, nwarps = nthreads >> 5;
  const int per = (((n + nthreads - 1) / nthreads) + 3) & ~3;
  const int i0 = min(n, tid * per), i1 = min(n, i0 + per);
  int local = 0;
  {
    int i = i0;
    for (; i + 4 <= i1; i += 4) { const int4 v = __ldcg((const int4*)(a + i)); local += val(v.x) + val(v.y) + val(v.z) + val(v.w); }
    for (; i < i1; ++i) local += val(__ldcg(&a[i]));
  }
  int incl = local;
  for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
  if (lane == 31) s_w[wid] = incl;
  __syncthreads();
  if (tid == 0) { int t = 0; for (int w = 0; w < nwarps; ++w) { const int v = s_w[w]; s_w[w] = t; t += v; } s_total = t; }
  __syncthreads();
  int run = s_w[wid] + incl - local;
  {
    int i = i0;
    for (; i + 4 <= i1; i += 4) {
      const int4 v = __ldcg((const int4*)(a + i));
      int4 r; r.x = run; r.y = run + val(v.x); r.z = r.y + val(v.y); r.w = r.z + val(v.z);
      *(int4*)(out + i) = r;
      run = r.w + val(v.w);
    }
    for (; i < i1; ++i) { const int v = val(__ldcg(&a[i])); out[i] = run; run += v; }
  }
  return s_total;
}

// ---------------------------------------------------------------------------------------------
// k_fast_count: finite pixels per block (depth_map_to_pointcloud.h:259: DepthTraits<float>::valid = isfinite)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void load_depth4(const float* __restrict__ depth, int p0, int P, int vec_ok, float d[4], int& npx) {
  npx = P - p0; if (npx > 4) npx = 4; if (npx < 0) npx = 0;
  if (npx == 4 && vec_ok) { const float4 v = __ldg((const float4*)(depth + p0)); d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w; }
  else { for (int k = 0; k < 4; ++k) d[k] = (k < npx) ? __ldg(depth + p0 + k) : 0.0f; }
}
// Index among all finite pixels of the first finite one of this thread's pixels d[0 .. npx) (load_depth4): the finite pixels of the
// block's earlier threads (warp scan, then the earlier warps) after the block's offset from k_fast_count.  Every thread of the block
// calls it.
__device__ __forceinline__ int first_finite_index(const FastFrame& f, const float d[4], int npx) {
  __shared__ int s_w[8];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  int c = 0;
  for (int k = 0; k < 4; ++k) c += (k < npx && isfinite(d[k])) ? 1 : 0;
  int incl = c;
  for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
  if (lane == 31) s_w[wid] = incl;
  __syncthreads();
  int base = f.block_off[blockIdx.x];
  for (int w = 0; w < wid; ++w) base += s_w[w];
  return base + incl - c;
}

__global__ void __launch_bounds__(256) k_fast_count(FastFrame f) {
  __shared__ int s_w[8];
  __shared__ int s_last;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int p0 = blockIdx.x * kCountBlock + tid * 4;
  float d[4]; int npx;
  load_depth4(f.in.depth, p0, f.capacity, f.vec_ok, d, npx);
  int c = 0;
  for (int k = 0; k < 4; ++k) c += (k < npx && isfinite(d[k])) ? 1 : 0;
  for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
  if (lane == 0) s_w[wid] = c;
  __syncthreads();
  if (tid == 0) {
    int t = 0; for (int w = 0; w < 8; ++w) t += s_w[w];
    __stcg(&f.block_cnt[blockIdx.x], t);
    __threadfence();
    s_last = (atomicAdd(&f.fc->ticket_count, 1u) == (unsigned)(f.n_count_blocks - 1));
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const int total = block_scan_array(f.block_cnt, f.block_off, f.n_count_blocks);
  if (tid == 0) { frame_counters_reset(f.cnt, total); f.fc->ticket_count = 0; }
}
// points entry: every point counts
__global__ void k_fast_reset(FastFrame f) { frame_counters_reset(f.cnt, f.capacity); }

// ---------------------------------------------------------------------------------------------
// k_fast_classify: per input point (image order) — fast.cpp:152-158, :75-81, :87-89 — + start-set visits
// ---------------------------------------------------------------------------------------------
// What `fast` takes of input point `pix` (depth entry: the pixel, of depth d; points entry: the input index, d unused).
// k_fast_classify and the ray set-up of k_fast_solve3 both call it, so a cast ray's point is the classified point, bit for bit,
// and no per-point state has to be stored for the ray set-up.
struct FastPoint { F3 pG; float w; uint32_t color; uint8_t label; bool valid, clearing; };
__device__ __forceinline__ FastPoint fast_point(const FastFrame& f, int pix, float d) {
  const DevCfg& cfg = f.cfg;
  FastPoint p;
  F3 pC;
  if (f.in.depth) {
    pC = backproject(f.in, pix, d);
    p.label = __ldg(f.in.label_img + pix);
    p.color = f.in.color_img ? f.in.color_img[pix] : f.luts->label_rgba[p.label];
  } else {
    point_input(f.in, f.luts, pix, pC, p.color, p.label);
  }
  point_test(cfg, f.in.freespace, f.cnt, pC, p.label, p.valid, p.clearing);
  if (f.luts->dynamic_label[p.label]) p.valid = false;       // isSemanticLabelValid (base.h:170-175): fast only (fast.cpp:76)
  p.w = point_weight(cfg, pC);
  p.pG = xform_apply(f.T, pC);
  return p;
}
// the start-set value (hash + offset) of a point, ~0 when it is not valid
__device__ __forceinline__ uint64_t fast_start_key(const FastFrame& f, const FastPoint& p) {
  if (!p.valid) return ~0ull;
  const F3 sc = mul(p.pG, f.cfg.start_inv);
  if (!index_in_range(sc)) set_err(f.cnt, 5);
  const I3 g = grid_index(p.pG, f.cfg.start_inv);            // fast.cpp:88-89
  return (uint64_t)index_hash(g) + f.set_offset;             // ApproxHashSet value = hash + offset_
}

// The start-set visits of a thread's K points (key ~0: not valid) into the slots' records.  A run of the thread's valid points
// that share a slot makes one set of updates; the thread that brings a slot its first visitors lists the slot (one allocation per
// warp).  No other result of the atomics steers the thread, so the runs overlap.  Every lane of the warp calls it.
template <int K>
__device__ __forceinline__ void start_visits(const FastFrame& f, const uint64_t (&key)[K], const int (&seq)[K]) {
  uint32_t slot[K];
  bool head[K], fresh[K];
  uint32_t prev = ~0u;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    slot[k] = (uint32_t)key[k] & kSetMask;
    head[k] = key[k] != ~0ull && slot[k] != prev;
    if (key[k] != ~0ull) prev = slot[k];
    fresh[k] = false;
  }
#pragma unroll
  for (int k = 0; k < K; ++k) {
    if (!head[k]) continue;
    uint32_t first = (uint32_t)seq[k], hmin = (uint32_t)(key[k] >> kSetBits), hmax = hmin, n = 1;
    bool run = true;
#pragma unroll
    for (int j = k + 1; j < K; ++j) {
      if (!run || key[j] == ~0ull) continue;
      if (slot[j] != slot[k]) { run = false; continue; }
      const uint32_t hi = (uint32_t)(key[j] >> kSetBits);
      first = min(first, (uint32_t)seq[j]); hmin = min(hmin, hi); hmax = max(hmax, hi); ++n;
    }
    StartRec* r = &f.sb.rec[slot[k]];
    atomicMin(&r->first, first);
    atomicMin(&r->hmin, hmin);
    atomicMax(&r->hmax, hmax);
    fresh[k] = atomicAdd(&r->visits, n) == 0;
  }
  int n_fresh = 0;
#pragma unroll
  for (int k = 0; k < K; ++k) n_fresh += fresh[k] ? 1 : 0;
  int at = (int)warp_alloc(&f.fc->n_touched, (unsigned long long)n_fresh);
#pragma unroll
  for (int k = 0; k < K; ++k)
    if (fresh[k]) f.sb.touched[at++] = (int)slot[k];
}

template <bool DEPTH>
__global__ void __launch_bounds__(256) k_fast_classify(FastFrame f) {
  const int tid = threadIdx.x, lane = tid & 31;
  const int n = f.cnt->n_points;
  int nvalid = 0;
  if (DEPTH) {
    const int p0 = blockIdx.x * kCountBlock + tid * 4;
    float d[4]; int npx;
    load_depth4(f.in.depth, p0, f.capacity, f.vec_ok, d, npx);
    int i = first_finite_index(f, d, npx);
    uint64_t key[4];
    int seq[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      key[k] = ~0ull; seq[k] = 0;
      if (k >= npx || !isfinite(d[k])) continue;
      const int pix = p0 + k;
      const FastPoint p = fast_point(f, pix, d[k]);
      seq[k] = f.seq_of_i ? f.seq_of_i[i] : inv_mixed_index(i, n);
      key[k] = fast_start_key(f, p);
      f.pt_key[i] = key[k];
      f.pt_pix[i] = pix;
      nvalid += p.valid ? 1 : 0;
      ++i;
    }
    start_visits<4>(f, key, seq);
  } else {
    const int i = blockIdx.x * blockDim.x + tid;
    uint64_t key[1] = {~0ull};
    int seq[1] = {0};
    if (i < n) {
      const FastPoint p = fast_point(f, i, 0.0f);
      seq[0] = f.seq_of_i ? f.seq_of_i[i] : inv_mixed_index(i, n);
      key[0] = fast_start_key(f, p);
      f.pt_key[i] = key[0];
      nvalid = p.valid ? 1 : 0;
    }
    start_visits<1>(f, key, seq);
  }
  for (int o = 16; o > 0; o >>= 1) nvalid += __shfl_down_sync(0xffffffffu, nvalid, o);
  if (lane == 0 && nvalid) atomicAdd(&f.cnt->n_valid, nvalid);
}

// "sorted" order mode (voxblox SortedThreadSafeIndex, A.3): squared norm per input index, image order
__global__ void __launch_bounds__(256) k_fast_sqnorm(FastFrame f, uint32_t* __restrict__ keys) {
  const int p0 = blockIdx.x * kCountBlock + threadIdx.x * 4;
  float d[4]; int npx;
  load_depth4(f.in.depth, p0, f.capacity, f.vec_ok, d, npx);
  int i = first_finite_index(f, d, npx);
  for (int k = 0; k < npx; ++k) {
    if (!isfinite(d[k])) continue;
    const F3 pC = backproject(f.in, p0 + k, d[k]);
    keys[i++] = __float_as_uint(dot3(pC, pC));
  }
}
__global__ void k_fast_sqnorm_points(FastFrame f, uint32_t* __restrict__ keys) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= f.capacity) return;
  const F3 pC = f3(f.in.xyz[3 * i], f.in.xyz[3 * i + 1], f.in.xyz[3 * i + 2]);
  keys[i] = __float_as_uint(dot3(pC, pC));
}
__global__ void k_fast_pad_keys(const Counters* cnt, int capacity, uint32_t* __restrict__ keys) {   // positions behind the finite count sort last
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < capacity && i >= cnt->n_points) keys[i] = 0xFFFFFFFFu;
}
__global__ void k_fast_invert_perm(const Counters* cnt, const uint32_t* __restrict__ point_of_seq, int* __restrict__ seq_of_i) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < cnt->n_points) seq_of_i[point_of_seq[s]] = s;
}

// ---------------------------------------------------------------------------------------------
// k_fast_start_slots: start_voxel_approx_set_.replaceHash (fast.cpp:90, A.4) + table commit, once per slot the frame visited.
// The set's state is the value of the last visit: a point is cast iff the previous visitor of its slot (sequence order; before
// the first visitor: the persistent table) carried a different value, and after the frame the table holds the last visitor's
// value.  A slot visited by ONE start cell (the normal case) is decided here: only its first visitor can be cast, and its record
// is emptied.  A slot shared by several cells (20-bit aliasing, a few thousand per frame) needs every visitor's predecessor in
// sequence order: it gets a visitor list and k_fast_solve3 fills, sorts and decides it with one warp per slot (a per-slot linked
// list walked by every visitor made the longest list the critical path).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_fast_start_slots(FastFrame f) {
  if (blockIdx.x == 0 && threadIdx.x == 0) f.fc->gridbar = 0;
  const int n = (int)f.fc->n_touched;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
    const uint32_t slot = (uint32_t)f.sb.touched[t];
    StartRec* r = &f.sb.rec[slot];
    const uint4 v = *(const uint4*)r;            // first, hmin, hmax, visits
    if (v.y == v.z) {
      if (f.sb.table[slot] != v.y) atomicOr(&f.cast_bits[v.x >> 5], 1u << (v.x & 31));
      f.sb.table[slot] = v.y;
      *(uint4*)r = start_rec_empty();
    } else {
      r->first = (uint32_t)atomicAdd(&f.fc->m_cursor, (int)v.w);
      f.mixed_list[atomicAdd(&f.fc->n_mixed, 1)] = (int)slot;
    }
  }
}

// ascending sort of a[0..n) by one warp (same network as cta_sort_u32 below)
__device__ __forceinline__ void warp_sort_i32(int* a, int n, int lane) {
  int n2 = 1;
  while (n2 < n) n2 <<= 1;
  const int half = n2 >> 1;
  for (int k = 2; k <= n2; k <<= 1) {
    const int hk = k >> 1;
    for (int t = lane; t < half; t += 32) {
      const int blk = t / hk, o = t - blk * hk;
      const int i = blk * k + o, p = blk * k + (k - 1 - o);
      if (p < n) { const int x = a[i], y = a[p]; if (x > y) { a[i] = y; a[p] = x; } }
    }
    __syncwarp();
    for (int j = k >> 2; j > 0; j >>= 1) {
      for (int t = lane; t < half; t += 32) {
        const int i = (t / j) * 2 * j + (t % j), p = i + j;
        if (p < n) { const int x = a[i], y = a[p]; if (x > y) { a[i] = y; a[p] = x; } }
      }
      __syncwarp();
    }
  }
}

// ---------------------------------------------------------------------------------------------
// k_fast_solve3 helpers (ksg_fast3.cuh): grid barrier, profiling marks, new-block construction
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void solve_barrier(unsigned int* bar, unsigned int& epoch) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned int target = (++epoch) * gridDim.x;
    atomicAdd(bar, 1u);
    while (((volatile unsigned int*)bar)[0] < target) {}
    __threadfence();
  }
  __syncthreads();
}
__device__ __forceinline__ void dbg_max(const FastFrame& f, int k, long long v) { if (f.profile) atomicMax((unsigned long long*)&f.fc->dbg[k], (unsigned long long)v); }
__device__ __forceinline__ void dbg_add(const FastFrame& f, int k, long long v) { if (f.profile) atomicAdd((unsigned long long*)&f.fc->dbg[k], (unsigned long long)v); }
__device__ __forceinline__ void timeline_mark(const FastFrame& f, int slot) {
  if (f.prof_marks && blockIdx.x == 0 && threadIdx.x == 0 && slot < kTimelineSlots) f.fc->timeline[slot] = clock64();
}

// SemanticVoxel / TsdfVoxel default construction of the frame's new blocks (semantic_voxel.h:14-27), all CTAs
__device__ __forceinline__ void fast_block_init(const FastFrame& f, int n_new, int pool_base) {
  const DevCfg& cfg = f.cfg;
  const MapRef& map = f.map;
  const int per_block = cfg.tiles_per_block;
  for (long long w = blockIdx.x; w < (long long)n_new * per_block; w += gridDim.x) {
    const int i = (int)(w / per_block), tile = (int)(w % per_block);
    const int slot = pool_base + i;
    if (slot >= map.max_blocks) { if (tile == 0 && threadIdx.x == 0) set_err(f.cnt, 3); continue; }
    if (tile == 0 && threadIdx.x == 0) {
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
    for (int v = threadIdx.x; v < V; v += blockDim.x) { dist[v] = 0.0f; wgt[v] = 0.0f; rgba[v] = 0u; srgba[v] = 0xFF7F7F7Fu; label[v] = 0; }
    for (int t = threadIdx.x; t < cfg.C * V; t += blockDim.x) prior[t] = (float)-0.60205999132;
  }
}

// ---------------------------------------------------------------------------------------------
// k_fast_group / k_fast_apply
// ---------------------------------------------------------------------------------------------
// ascending sort of a[0..n) by one CTA; bitonic network in its "flip" form (every compare-exchange puts the minimum at the lower
// index), so the virtual +inf padding behind n never has to move and pairs that reach past n are skipped
__device__ __forceinline__ void cta_sort_u32(uint32_t* a, int n) {
  int n2 = 1;
  while (n2 < n) n2 <<= 1;
  const int half = n2 >> 1;
  for (int k = 2; k <= n2; k <<= 1) {
    const int hk = k >> 1;
    for (int t = threadIdx.x; t < half; t += blockDim.x) {
      const int blk = t / hk, o = t - blk * hk;
      const int i = blk * k + o, p = blk * k + (k - 1 - o);
      if (p < n) { const uint32_t x = a[i], y = a[p]; if (x > y) { a[i] = y; a[p] = x; } }
    }
    __syncthreads();
    for (int j = k >> 2; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < half; t += blockDim.x) {
        const int i = (t / j) * 2 * j + (t % j), p = i + j;
        if (p < n) { const uint32_t x = a[i], y = a[p]; if (x > y) { a[i] = y; a[p] = x; } }
      }
      __syncthreads();
    }
  }
}

// ---------------------------------------------------------------------------------------------
// k_fast_group: one CTA per touched tile.  The tile's keys (voxel << kRecOrdBits | ray rank) are sorted ascending in place in their
// segment of f.keys - ascending key order is the reference's per-voxel update order - and every touched voxel becomes one work
// item of k_fast_apply: the tile, the voxel, and where its run of keys starts and ends.  Tiles another shard owns (n < 0) and tiles
// without a pool slot (the pool overflow is flagged by the block construction) give no items.  Items land in one frame-wide array
// in the order the CTAs reserve them; fc->log_count counts them (and is the update log's entry count: entry i = item i).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kGroupThreads, 2) k_fast_group(FastFrame f, FastItem* __restrict__ items, FastTile* __restrict__ tiles,
                                                              int item_cap) {
  __shared__ uint32_t s_keys[kFastKeyCap];    // the tile's keys, sorted
  __shared__ uint32_t s_keys2[kFastKeyCap];   // ... grouped by voxel
  __shared__ int s_seg_lo[kRecVoxMax], s_seg_hi[kRecVoxMax];
  __shared__ int s_w[kGroupThreads / 32];
  __shared__ int s_tile, s_n, s_base;
  __shared__ long long s_off;
  const DevCfg& cfg = f.cfg;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (blockIdx.x == 0 && tid == 0) f.fc->item_cursor = 0;   // k_fast_apply's claim cursor (stream order: it runs after this kernel)
  const int n_tiles = f.cnt->n_tiles;
  for (;;) {
    __syncthreads();                           // every thread has read the previous claim
    if (tid == 0) {
      const int j = atomicAdd(&f.fc->tile_cursor, 1);
      int n = 0;
      if (j < n_tiles) {
        const TileDesc td = f.tile_list[j];
        const int pos = (int)(td.tk / (uint32_t)cfg.tiles_per_block), tile = (int)(td.tk % (uint32_t)cfg.tiles_per_block);
        const int slot = f.map.ht_slot[pos];
        if (td.n > 0 && slot >= 0 && slot < f.map.max_blocks) {
          n = td.n;
          const I3 bi = unpack_key(f.map.ht_keys[pos]);
          FastTile t;
          t.off = td.off; t.slot = slot; t.tile = tile; t.bx = bi.x; t.by = bi.y; t.bz = bi.z; t.pad = 0;
          tiles[j] = t;
          s_off = td.off;
        }
      }
      s_tile = j; s_n = n;
    }
    __syncthreads();
    const int j = s_tile, n = s_n;
    if (j >= n_tiles) break;
    if (n == 0) continue;
    uint32_t* g_keys = f.keys + s_off;
    const bool in_smem = n <= kFastKeyCap;
    uint32_t* keys = in_smem ? s_keys : g_keys;
    if (in_smem) {
      // counting sort by voxel (histogram, scan, scatter), then every key finds its place in its voxel's run by counting the
      // smaller keys there (runs are short: tens of keys; the work grows with the square of a run's length)
      for (int v = tid; v < kRecVoxMax; v += kGroupThreads) s_seg_hi[v] = 0;
      for (int i = tid; i < n; i += kGroupThreads) s_keys[i] = g_keys[i];
      __syncthreads();
      for (int i = tid; i < n; i += kGroupThreads) atomicAdd(&s_seg_hi[s_keys[i] >> kRecOrdBits], 1);
      __syncthreads();
      if (tid < 32) {        // exclusive scan of the counts by one warp
        constexpr int per = kRecVoxMax / 32;
        const int v0 = lane * per;
        int local = 0;
        for (int v = v0; v < v0 + per; ++v) local += s_seg_hi[v];
        int incl = local;
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
        int run = incl - local;
        for (int v = v0; v < v0 + per; ++v) { const int c = s_seg_hi[v]; s_seg_lo[v] = run; s_seg_hi[v] = run; run += c; }
      }
      __syncthreads();
      for (int i = tid; i < n; i += kGroupThreads) { const uint32_t k = s_keys[i]; s_keys2[atomicAdd(&s_seg_hi[k >> kRecOrdBits], 1)] = k; }
      __syncthreads();
      for (int i = tid; i < n; i += kGroupThreads) {
        const uint32_t k = s_keys2[i];
        const int vx = (int)(k >> kRecOrdBits), lo = s_seg_lo[vx], hi = s_seg_hi[vx];
        int r = lo;
        for (int q = lo; q < hi; ++q) r += s_keys2[q] < k ? 1 : 0;
        s_keys[r] = k;
      }
      __syncthreads();
      for (int i = tid; i < n; i += kGroupThreads) g_keys[i] = s_keys[i];
    } else {
      __syncthreads();
      cta_sort_u32(keys, n);                   // ends with a barrier
      for (int i = tid; i < n; i += kGroupThreads) {
        const int vx = (int)(keys[i] >> kRecOrdBits);
        if (i + 1 == n || (int)(keys[i + 1] >> kRecOrdBits) != vx) s_seg_hi[vx] = i + 1;
      }
    }
    __syncthreads();
    const int rounds = (n + kGroupThreads - 1) / kGroupThreads;
    for (int r = 0; r < rounds; ++r) {
      const int i = r * kGroupThreads + tid;
      const int vx = i < n ? (int)(keys[i] >> kRecOrdBits) : -1;
      const bool head = i < n && (i == 0 || (int)(keys[i - 1] >> kRecOrdBits) != vx);
      const unsigned m = __ballot_sync(0xffffffffu, head);
      if (lane == 0) s_w[wid] = __popc(m);
      __syncthreads();
      if (tid == 0) {                          // one reservation per round of the tile
        int t = 0;
        for (int w = 0; w < kGroupThreads / 32; ++w) { const int c = s_w[w]; s_w[w] = t; t += c; }
        s_base = t ? atomicAdd(&f.fc->log_count, t) : 0;
      }
      __syncthreads();
      if (head) {
        const int at = s_base + s_w[wid] + __popc(m & ((1u << lane) - 1u));
        if (at < item_cap) { FastItem it; it.tile = j; it.vox = vx; it.lo = i; it.len = s_seg_hi[vx] - i; items[at] = it; }
        else set_err(f.cnt, 4);
      }
      __syncthreads();
    }
  }
}

// k_fast_apply: one warp per item (touched voxel); warps claim items from a cursor (the first one by warp index).  The voxel's
// distance, weight, colour and label fields and its C-float log-probability row (lanes = classes) are read from the pool, its
// sorted keys applied 32 at a time - TSDF recurrence (tsdf_batch), one-hot rows (fast.cpp:132-135), first-max arg-max
// (base.cpp:352-367), colour hand-off (base.cpp:370-380) - and the voxel alone is written back.  When the frame has more items than
// the item array holds, k_fast_group flagged it and nothing is applied.  NCH = ceil(C / 32) register chunks per lane.
template <int NCH>
__global__ void __launch_bounds__(kFastApplyThreads, NCH <= 4 ? 4 : 2) k_fast_apply(FastFrame f, ApplySrc src, const FastItem* __restrict__ items,
                                                                  const FastTile* __restrict__ tiles, int item_cap) {
  const DevCfg& cfg = f.cfg;
  const int C = cfg.C;
  const int lane = threadIdx.x & 31;
  const int n_items = f.fc->log_count;
  if (n_items > item_cap) return;
  const int warps_total = (gridDim.x * blockDim.x) >> 5;
  const F3 origin = f3(f.T.tx, f.T.ty, f.T.tz);
  const bool keep_blend = cfg.color_mode == 0;
  const uint32_t ord_mask = (1u << kRecOrdBits) - 1u;
  const int ts = cfg.tile_side_log2, tm = cfg.tile_side - 1, tps = cfg.tiles_per_side;
  for (int item = (int)(blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)); item < n_items;) {
    const FastItem it = items[item];
    const FastTile t = tiles[it.tile];
    const int v = it.vox;
    uint8_t* chunk = f.map.pool + (uint64_t)t.slot * cfg.block_stride + (uint64_t)t.tile * cfg.tile_stride;
    float* g_dist = (float*)chunk;
    float* g_wgt = (float*)(chunk + cfg.plane_f32);
    uint32_t* g_rgba = (uint32_t*)(chunk + 2 * cfg.plane_f32);
    uint32_t* g_srgba = (uint32_t*)(chunk + 3 * cfg.plane_f32);
    uint8_t* g_label = chunk + 4 * cfg.plane_f32;
    float* prow = (float*)(chunk + cfg.head_bytes) + (size_t)v * C;
    const uint32_t* keys = f.keys + t.off + it.lo;
    const int len = it.len;
    I3 g;
    g.x = t.bx * cfg.vps + (t.tile % tps) * cfg.tile_side + (v & tm);
    g.y = t.by * cfg.vps + ((t.tile / tps) % tps) * cfg.tile_side + ((v >> ts) & tm);
    g.z = t.bz * cfg.vps + (t.tile / (tps * tps)) * cfg.tile_side + (v >> (2 * ts));
    const F3 center = voxel_center(g, cfg.voxel_size);
    float dist = g_dist[v], wgt = g_wgt[v];
    uint32_t rgba = g_rgba[v];
    float p[NCH];
#pragma unroll
    for (int q = 0; q < NCH; ++q) { const int c = q * 32 + lane; p[q] = (c < C) ? prow[c] : 0.0f; }
    for (int base = 0; base < len; base += 32) {
      uint32_t col = 0;
      int lab = 0;
      float sdf = 0.0f, uw = 0.0f;
      if (base + lane < len) {
        const uint32_t ord = keys[base + lane] & ord_mask;
        const float4 pr = src.param[ord];
        tsdf_measure(cfg.tp, origin, f3(pr.x, pr.y, pr.z), center, pr.w, sdf, uw);
        if (keep_blend) col = src.color[ord];
        lab = (int)src.label[ord];
      }
      const int nb = (len - base) < 32 ? (len - base) : 32;
      for (int jj = 0; jj < nb; ++jj) {      // semantic rows: lanes = classes, one-hot frequencies (fast.cpp:132-135)
        const int l = __shfl_sync(0xffffffffu, lab, jj);
        if (l != 0) {   // label 0: column 0 of the likelihood is zero (base.cpp:127)
#pragma unroll
          for (int q = 0; q < NCH; ++q) p[q] += ((q * 32 + lane) == l) ? cfg.lm : cfg.ln;
        }
      }
      tsdf_batch(cfg.tp, lane, nb, sdf, uw, col, keep_blend, dist, wgt, rgba);
    }
    // arg-max, first maximum wins (base.cpp:352-367)
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
    const int bi_lab = __shfl_sync(0xffffffffu, bi, 0);
#pragma unroll
    for (int q = 0; q < NCH; ++q) { const int c = q * 32 + lane; if (c < C) prow[c] = p[q]; }
    const uint32_t sc = f.luts->label_rgba[bi_lab];          // base.cpp:370-380
    uint32_t out_rgba = rgba;                                 // kColor: the blended colour is the result
    if (cfg.color_mode == 1) out_rgba = sc;                   // kSemantic (base.cpp:177-180)
    else if (cfg.color_mode == 2) out_rgba = rainbow_color_map((double)expf(best));  // base.cpp:181-185
    if (lane == 0) { g_dist[v] = dist; g_wgt[v] = wgt; g_label[v] = (uint8_t)bi_lab; g_srgba[v] = sc; g_rgba[v] = out_rgba; }
    if (f.log_head != nullptr && item < f.log_cap) {
      if (lane == 0) {
        const int m = cfg.vps - 1;
        VoxelUpdate u;
        u.bx = t.bx; u.by = t.by; u.bz = t.bz;
        u.lin_label = (uint32_t)((g.x & m) + cfg.vps * ((g.y & m) + cfg.vps * (g.z & m))) | ((uint32_t)bi_lab << 24);
        u.dist = dist; u.wgt = wgt; u.rgba = out_rgba; u.srgba = sc;
        f.log_head[item] = u;
      }
#pragma unroll
      for (int q = 0; q < NCH; ++q) { const int c = q * 32 + lane; if (c < C) f.log_prior[(size_t)item * C + c] = p[q]; }
    }
    int next = 0;
    if (lane == 0) next = warps_total + atomicAdd(&f.fc->item_cursor, 1);
    item = __shfl_sync(0xffffffffu, next, 0);
  }
}

}  // namespace ksg
