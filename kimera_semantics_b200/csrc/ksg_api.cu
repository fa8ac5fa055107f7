// ksg_api.cu — host side of the C-ABI in include/ksg.h: owns the device-resident map (spatial block hash +
// tile pool), the per-frame scratch, and enqueues the kernel family of ksg_kernels.cuh.
// Compiled for sm_90a (H100) only, with -fmad=false (bit-exact index arithmetic, see ksg_device.cuh).
#include <cuda_runtime.h>
#include <cub/cub.cuh>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <numeric>
#include <string>
#include <type_traits>
#include <unordered_map>
#include <unordered_set>
#include <utility>
#include <vector>

#include "../../include/ksg.h"
#include "ksg_kernels.cuh"
#include "ksg_chain.cuh"
#include "ksg_hot.cuh"
#include "ksg_bundle_order.cuh"
#include "ksg_fast.cuh"
#include "ksg_fast3.cuh"
#include "ksg_voxel.cuh"
#include "ksg_log.cuh"
#include "ksg_merge.cuh"
#include "ksg_eval.cuh"
#include "ksg_mesh.cuh"
#include "ksg_query.cuh"
#include "ksg_render.cuh"
#include "ksg_esdf.cuh"

using namespace ksg;

namespace {

thread_local std::string g_last_error;

// Every caller names its integrator `h`.
#define KSG_CUDA(call)                                                                              \
  do {                                                                                              \
    cudaError_t e_ = (call);                                                                        \
    if (e_ != cudaSuccess) {                                                                        \
      char buf_[512];                                                                               \
      snprintf(buf_, sizeof(buf_), "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
      return h->fail(KSG_ERR_CUDA, buf_);                                                           \
    }                                                                                               \
  } while (0)

inline int ilog2(int v) { int l = 0; while ((1 << l) < v) ++l; return l; }
inline uint32_t round_up(uint32_t v, uint32_t m) { return (v + m - 1) / m * m; }
inline int grid_for(long long n, int block) { return (int)std::max<long long>(1, (n + block - 1) / block); }

// f(std::integral_constant<int, NCH>) for the template instance that serves `nch` label chunks (1, 2, 4, otherwise 8)
template <typename F> auto with_nch(int nch, F&& f) {
  switch (nch) {
    case 1: return f(std::integral_constant<int, 1>{});
    case 2: return f(std::integral_constant<int, 2>{});
    case 4: return f(std::integral_constant<int, 4>{});
    default: return f(std::integral_constant<int, 8>{});
  }
}
// f for every instance, in the order 1, 2, 4, 8; stops at the first non-zero result
template <typename F> int for_each_nch(F&& f) {
  for (int nch : {1, 2, 4, 8}) if (const int rc = with_nch(nch, f)) return rc;
  return 0;
}
template <typename F> auto with_tma(bool tma, F&& f) { return tma ? f(std::true_type{}) : f(std::false_type{}); }
// f(tma, nch) for every (TMA staging, label chunks) instance, TMA first; stops at the first non-zero result
template <typename F> int for_each_tma_nch(F&& f) {
  for (const bool tma : {true, false})
    if (const int rc = with_tma(tma, [&](auto t) { return for_each_nch([&](auto nch) { return f(t, nch); }); })) return rc;
  return 0;
}

// Owner of device memory, pinned host memory, streams and events: it remembers what it made and releases what it still holds
// in reverse order when it is destroyed.  The caller selects the device.
class Resources {
 public:
  Resources() = default;
  Resources(const Resources&) = delete;
  Resources& operator=(const Resources&) = delete;
  ~Resources() { for (auto it = held_.rbegin(); it != held_.rend(); ++it) destroy(*it); }

  // (the call is made before *p is read: keep() takes the result, not the call)
  template <typename Tp> cudaError_t device(Tp** p, size_t count) { return alloc(p, count, kDevice); }
  template <typename Tp> cudaError_t pinned(Tp** p, size_t count) { return alloc(p, count, kPinned); }
  cudaError_t stream(cudaStream_t* s) {
    const cudaError_t e = cudaStreamCreateWithFlags(s, cudaStreamNonBlocking);
    return keep(e, kStream, (void*)*s);
  }
  cudaError_t stream(cudaStream_t* s, int priority) {
    const cudaError_t e = cudaStreamCreateWithPriority(s, cudaStreamNonBlocking, priority);
    return keep(e, kStream, (void*)*s);
  }
  cudaError_t event(cudaEvent_t* ev, unsigned flags) {
    const cudaError_t e = cudaEventCreateWithFlags(ev, flags);
    return keep(e, kEvent, (void*)*ev);
  }

  // Releases one allocation before the owner goes (nullptr: nothing to do).
  void release(void* p) {
    if (!p) return;
    for (size_t i = held_.size(); i-- > 0;)
      if (held_[i].p == p) { destroy(held_[i]); held_.erase(held_.begin() + (ptrdiff_t)i); return; }
  }
  // A buffer that grows: *p is released and replaced by `count` fresh elements (the contents are not kept).  *cap records the
  // new capacity, or 0 when the allocation fails.
  template <typename Tp, typename Cap> cudaError_t regrow(Tp** p, Cap* cap, size_t count) { return replace(p, cap, count, kDevice); }
  template <typename Tp, typename Cap> cudaError_t regrow_pinned(Tp** p, Cap* cap, size_t count) { return replace(p, cap, count, kPinned); }

 private:
  enum Kind { kDevice, kPinned, kStream, kEvent };
  struct Item { Kind kind; void* p; };
  template <typename Tp> cudaError_t alloc(Tp** p, size_t count, Kind kind) {
    const size_t bytes = std::max<size_t>(count, 1) * sizeof(Tp);
    const cudaError_t e = kind == kPinned ? cudaMallocHost((void**)p, bytes) : cudaMalloc((void**)p, bytes);
    return keep(e, kind, (void*)*p);
  }
  template <typename Tp, typename Cap> cudaError_t replace(Tp** p, Cap* cap, size_t count, Kind kind) {
    release(*p); *p = nullptr; *cap = 0;
    const cudaError_t e = alloc(p, count, kind);
    if (e == cudaSuccess) *cap = (Cap)count;
    return e;
  }
  cudaError_t keep(cudaError_t e, Kind kind, void* p) {
    if (e == cudaSuccess && p) held_.push_back(Item{kind, p});
    return e;
  }
  static void destroy(const Item& it) {
    switch (it.kind) {
      case kDevice: cudaFree(it.p); break;
      case kPinned: cudaFreeHost(it.p); break;
      case kStream: cudaStreamDestroy(static_cast<cudaStream_t>(it.p)); break;
      case kEvent: cudaEventDestroy(static_cast<cudaEvent_t>(it.p)); break;
    }
  }
  std::vector<Item> held_;
};

// Development knobs (environment), read once when an integrator is created.  They reshape launches that were measured against
// the defaults; ksg_create applies each one only where it mattered before (see there).
//
// The short-segment kernel is capped at short_ctas CTAs per SM through a dynamic shared-memory reservation so that a CTA of the
// long-segment kernel (128 registers per thread) always finds room beside it - otherwise the two kernels run back to back.
// short_t_ctas: the frame is bound by the long-segment kernel (128 registers per thread); whatever the short kernel takes from it
// costs more than it gains.  Re-measured on an H100 80GB HBM3 (400 W, merged2, bench.py --quick, two alternating passes):
// KSG_SHORT_T_CTAS 1 -> 164 frames/s, 2 -> 181-182, 3 -> 171-173, 4 -> 177-178; KSG_LONG_THREADS=128 172-176,
// KSG_DEEP_THREADS=64 180-182 - the defaults below stay.  The non-hot long segments of C <= 32 run behind the short kernel, not
// beside it: 181-182 against 176-178 frames/s in the same passes.
struct Knobs {
  bool tile_apply = false;        // KSG_MERGED_TILE_APPLY=1: merged uses the tile kernel instead of the per-voxel kernels
  int long_len = 0;               // KSG_LONG_LEN: records from which a voxel is long under k_voxel_apply_short_t (0: kLongLenThread)
  int long_threads = 256;         // KSG_LONG_THREADS: 64, 128 or 256
  int long_grid = 0;              // KSG_LONG_GRID (0: one CTA per SM)
  int deep_threads = 128;         // KSG_DEEP_THREADS: block size of the hot-voxel instance (32, 64, 128 or 256), one warp per chain
  int short_t_ctas = 2;           // KSG_SHORT_T_CTAS: CTAs per SM of k_voxel_apply_short_t, 1 to 8
  int short_ctas = 3;             // KSG_SHORT_CTAS: CTAs per SM of k_voxel_apply_short, 1 to 6
  int solve_threads = kSolveThreads;   // KSG_SOLVE_THREADS: 256, 512 or 1024
  int solve_ctas_per_sm = INT_MAX;     // KSG_SOLVE_CTAS_PER_SM, at least 1 and at most what the occupancy allows
  bool profile_marks_only = false;     // KSG_PROFILE_MARKS_ONLY=1: fast, the solve kernel's phase marks without its per-ray probes
};

Knobs read_knobs() {
  Knobs k;
  auto env = [](const char* name, int* v) { const char* e = std::getenv(name); if (e) *v = std::atoi(e); return e != nullptr; };
  int v = 0;
  if (env("KSG_MERGED_TILE_APPLY", &v) && v != 0) k.tile_apply = true;
  if (env("KSG_LONG_LEN", &v)) k.long_len = std::max(kLongLen, std::min(1 << 20, v));
  if (env("KSG_LONG_THREADS", &v) && (v == 64 || v == 128 || v == 256)) k.long_threads = v;
  if (env("KSG_LONG_GRID", &v)) k.long_grid = std::max(1, v);
  if (env("KSG_DEEP_THREADS", &v) && (v == 32 || v == 64 || v == 128 || v == 256)) k.deep_threads = v;
  if (env("KSG_SHORT_T_CTAS", &v)) k.short_t_ctas = std::max(1, std::min(8, v));
  if (env("KSG_SHORT_CTAS", &v)) k.short_ctas = std::max(1, std::min(6, v));
  if (env("KSG_SOLVE_THREADS", &v) && (v == 256 || v == 512 || v == 1024)) k.solve_threads = v;
  if (env("KSG_SOLVE_CTAS_PER_SM", &v)) k.solve_ctas_per_sm = v;
  if (env("KSG_PROFILE_MARKS_ONLY", &v)) k.profile_marks_only = v != 0;
  return k;
}

}  // namespace

struct ksg_integrator {
  ksg_config cfg{};
  DevCfg dc{};
  int device = 0;
  int sm_count = 132;
  cudaStream_t own_stream = nullptr;
  std::string err;
  int deferred_status = 0;

  // map
  MapRef map{};
  uint32_t ht_cap = 0;
  Luts h_luts{};
  Luts* d_luts = nullptr;
  Counters* d_cnt = nullptr;
  Counters* h_cnt = nullptr;  // pinned
  int frame_stamp = 0;
  int64_t num_blocks = 0;
  int64_t last_blocks_touched = 0;

  // per-frame scratch
  int cap_points = 0;
  float4 *pt_pC = nullptr, *pt_pG = nullptr;
  uint8_t *pt_label = nullptr, *pt_flags = nullptr;
  uint32_t* pt_color = nullptr;
  uint64_t* pt_key = nullptr;
  uint8_t* flags8 = nullptr;  // 2*cap bytes
  int* pix_list = nullptr;
  int* point_of_seq = nullptr;
  uint32_t *sq_keys = nullptr, *sq_keys_out = nullptr;
  uint32_t *iota = nullptr;

  // fast
  StartRec* start_rec = nullptr;     // [2^20] empty between frames (StartBuf)
  uint32_t *start_table = nullptr;
  int* start_touched = nullptr;
  uint64_t set_offset = 0;  // both ApproxHashSets share reset times, hence one offset (fast.cpp:165-170)
  int64_t reset_counter = 0;
  int* cast_seq = nullptr;
  float4* ray_param = nullptr;
  uint8_t *ray_label = nullptr, *ray_flags = nullptr;
  uint32_t* ray_color = nullptr;
  int* nsteps = nullptr;
  RayState* ray_state = nullptr;
  long long* ext_off = nullptr;
  Obs3 o3{};                         // observed-set solver (ksg_fast3.cuh)

  // merged
  uint64_t* ks_sorted = nullptr;
  uint32_t* seq_sorted = nullptr;
  int *bstart = nullptr, *bundle_f = nullptr;
  float *hist = nullptr, *tmp = nullptr, *tmp4 = nullptr;   // tmp4: rows of tmp at a 4-float stride (k_voxel_apply_short_t)
  uint64_t* b_key = nullptr;
  long long* b_base = nullptr;
  // merged, KSG_BUNDLE_ORDER_LIBSTDCXX
  std::vector<std::pair<int, uint32_t>> bord_phases;   // (first insertion index, bucket count) of every rehash phase
  uint32_t* bord_hash = nullptr;
  int* bundle_f2 = nullptr;
  int* bord_scratch = nullptr;       // one allocation behind every array of BordBuf
  unsigned long long* d_scan_tot = nullptr;   // per-CTA totals of k_bundle_scan
  BordBuf bord{};

  // merged, hot_voxel_mode = 1 (ksg_hot.cuh)
  bool hot_enabled = false;
  HotSeg* d_hot_segs = nullptr;
  HotSeg* h_hot_segs = nullptr;      // pinned
  int *d_hot_counts = nullptr;       // [0] segments found, [1] chunks that fell back to the plain loop (accumulated)
  int *d_hot_chunk_seg = nullptr, *h_hot_chunk_seg = nullptr, *d_hot_guess = nullptr;
  double* d_hot_sums = nullptr;
  ChainTable* d_hot_tables = nullptr;
  float* d_hot_prior = nullptr;
  int* d_hot_same = nullptr;          // hot_voxel_mode 2
  long long hot_chunk_cap = 0;
  int64_t hot_segments_total = 0, hot_chunks_total = 0;
  int last_hot_segments = 0;          // segments of the last frame's pre-pass (ksg_debug_apply_routes)
  bool last_frame_queued = false;     // the last frame filled the per-voxel queues

  // records
  uint64_t *rec_a = nullptr, *rec_b = nullptr;
  long long rec_cap = 0;
  long long* tile_begin = nullptr;
  long long tile_cap = 0;
  uint8_t* cub_temp = nullptr;
  size_t cub_temp_bytes = 0;

  // host staging (pinned) + device input buffers for the host-buffer entry points
  uint8_t* h_stage = nullptr;
  size_t h_stage_bytes = 0;
  uint8_t* d_in = nullptr;
  size_t d_in_bytes = 0;

  // export staging
  uint8_t* d_exp = nullptr;
  size_t d_exp_bytes = 0;
  int* d_exp_slots = nullptr;
  int exp_slots_cap = 0;

  // fast frame driver (ksg_fast.cuh): no host read-back inside the frame
  FastCounters* d_fc = nullptr;
  FastCounters* h_fc = nullptr;      // pinned
  int *blk_cnt = nullptr, *blk_off = nullptr, *warp_off = nullptr, *seq_of_i = nullptr;
  uint32_t* cast_bits = nullptr;     // empty between frames (FastFrame)
  uint32_t* keys32 = nullptr;
  int *tile_cnt = nullptr, *tile_slot = nullptr;
  TileDesc* tile_list = nullptr;
  FastTile* fast_tiles = nullptr;    // [tile_cap]
  FastItem* fast_items = nullptr;    // [item_cap] touched voxels of the frame
  int item_cap = 0;
  int solve_grid = 0, group_grid = 0, fast_apply_grid = 0;
  int solve_threads = 0;             // Knobs
  RayRec* rayrec = nullptr;
  int* wl = nullptr;                 // [3][max_points] per-ray listed sweep, two scan lists
  int *mixed_list = nullptr, *m_list = nullptr, *blk_run = nullptr;
  // update log (ksg_set_update_log): one entry per voxel the last frame updated
  VoxelUpdate *d_log_head = nullptr, *h_log_head = nullptr;
  float *d_log_prior = nullptr, *h_log_prior = nullptr;
  int log_cap = 0;
  int64_t merged_log_count = 0;      // merged: entries of the last integrate call (ksg_merge_*_device reuse Counters, so it is kept here)
  int solve_smem = 0;
  double clock_khz = 1980000.0;
  // frames whose counters have not been read back yet (at most two: the counter copies land in two pinned slots)
  Counters* h_cnt_base = nullptr;    // [2] pinned; h_cnt points at the slot read last
  FastCounters* h_fc_base = nullptr; // [2] pinned
  cudaEvent_t ev_frame_s[2] = {nullptr, nullptr};   // recorded behind the frame's counter copy
  int pend[2] = {0, 0};
  int n_pend = 0, next_slot = 0;
  // pipelined host-buffer entry (ksg_integrate_depth_async): the H2D copy of frame t+1 overlaps the kernels of frame t
  cudaStream_t copy_stream = nullptr;
  uint8_t* d_in2[2] = {nullptr, nullptr};
  uint8_t* h_stage2[2] = {nullptr, nullptr};
  size_t in2_bytes[2] = {0, 0};
  cudaEvent_t ev_copy[2] = {nullptr, nullptr}, ev_free[2] = {nullptr, nullptr};
  bool in2_used[2] = {false, false};
  int in_slot = 0;
  ksg_frame_stats stash[4];
  int n_stash = 0;

  // merged, round-2 per-voxel apply (ksg_voxel.cuh)
  bool voxel_apply = false;
  VoxelQueues vq{};
  cudaStream_t aux_stream = nullptr;  // high priority, one kernel of the per-voxel apply per frame (merged_apply_voxels)
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  // shape of the per-voxel kernels: development knobs (Knobs), set by ksg_create for the per-voxel apply only
  int long_threads = 0, long_grid = 0, short_ctas = 0, short_smem = 0;
  int deep_threads = 0;
  int short_t_ctas = 0;

  // device ESDF layer (ksg_update_esdf, ksg_esdf.cuh): rows by pool slot, max_blocks of them, allocated by the first update
  float* esdf_dist = nullptr;
  uint8_t *esdf_flags = nullptr, *esdf_site = nullptr;
  bool esdf_full = true;              // the next update recomputes everything: no update yet, or a clear / reset / import since the last
  bool esdf_valid = false;            // the layer describes slots [0, esdf_blocks) of the map (export and query allowed)
  float esdf_min_weight = 0.0f, esdf_max_distance = 0.0f;
  int esdf_stamp = 0;                 // frame_stamp at the last update: blocks stamped after it changed
  int64_t esdf_blocks = 0;
  std::vector<uint64_t> esdf_keys;    // key of each slot of the layer
  std::vector<uint8_t> esdf_has_site; // per slot: the row holds a site
  std::vector<int> esdf_rewritten;    // slots whose output the last update rewrote, in (z, y, x) order

  // device mesh layer (ksg_update_mesh, ksg_mesh.cuh): per pool slot a vertex range of the arena, in slot order
  unsigned* mesh_mark = nullptr;      // [max_blocks] 0 between updates
  int *mesh_rpos = nullptr, *mesh_list = nullptr, *mesh_count = nullptr;   // [max_blocks]: list position of a marked slot, R, R's counts
  long long* mesh_lfirst = nullptr;   // [max_blocks] first vertex of R's entries in the new arena
  long long* mesh_first[2] = {nullptr, nullptr};   // [max_blocks + 1] per slot, of arena 0 / 1
  MeshBuf mesh_arena[2] = {};
  int64_t mesh_cap[2] = {0, 0};       // vertices each arena holds
  MeshCounters *d_mesh_ctr = nullptr, *h_mesh_ctr = nullptr;   // h_: pinned
  int mesh_cur = 0;                   // the arena of the layer
  bool mesh_full = true;              // as esdf_full
  bool mesh_valid = false;            // as esdf_valid: the layer describes slots [0, mesh_blocks)
  bool mesh_far = false;              // a block of the layer lies beyond the window bound: every update is full
  float mesh_min_weight = 0.0f;
  int mesh_stamp = 0;
  int64_t mesh_blocks = 0, mesh_vertices = 0, mesh_remeshed = 0;   // mesh_remeshed = |R| of the last update, listed in mesh_list

  long long* tile_debug = nullptr;  // optional per-tile (records, cycles) trace
  int apply_smem = 0;
  int apply_nch = 1;
  bool use_tma = true;

  // profiling
  bool profiling = false;
  bool profile_marks_only = false;   // fast (Knobs): the solve kernel's phase marks without its per-ray probes
  cudaEvent_t ev[KSG_NUM_PHASES + 1] = {};
  double phase_ms[KSG_NUM_PHASES] = {};
  int64_t prof_frames = 0;
  int64_t n_launches = 0, n_libcalls = 0;

  Resources res;                     // every device / pinned buffer, stream and event above that is not an alias into another

  ~ksg_integrator() { cudaSetDevice(device); }   // then `res` releases
  int fail(int code, const char* msg) { err = msg; g_last_error = msg; return code; }
};

namespace {

int validate(const ksg_config* c, std::string& why) {
  if (!c) { why = "null config"; return KSG_ERR_INVALID_ARGUMENT; }
  if (c->abi_version != KSG_ABI_VERSION) { why = "abi_version mismatch"; return KSG_ERR_INVALID_ARGUMENT; }
  if (c->integrator_type != KSG_INTEGRATOR_FAST && c->integrator_type != KSG_INTEGRATOR_MERGED) {
    why = "Unknown Semantic/TSDF integrator type (factory.cpp:83)"; return KSG_ERR_INVALID_ARGUMENT; }
  const int v = c->voxels_per_side;
  if (v <= 0 || (v & (v - 1)) || v > 64) { why = "voxels_per_side must be a power of two <= 64"; return KSG_ERR_INVALID_ARGUMENT; }
  if (!(c->voxel_size > 0.0f)) { why = "voxel_size must be positive"; return KSG_ERR_INVALID_ARGUMENT; }
  if (c->num_labels < 2 || c->num_labels > 256) { why = "num_labels must be in [2, 256]"; return KSG_ERR_INVALID_ARGUMENT; }
  const float p = c->semantic_measurement_probability;  // base.cpp:98-107
  if (!(p > 0.0f && p < 1.0f) || !((1.0f - p) > 0.0f) || !(std::log(p) > std::log(1.0f - p))) {
    why = "semantic_measurement_probability must satisfy 0 < 1-p < p < 1 (base.cpp:98-107)"; return KSG_ERR_INVALID_ARGUMENT; }
  if (c->integration_order_mode != KSG_ORDER_MIXED && c->integration_order_mode != KSG_ORDER_SORTED) {
    why = "unknown integration_order_mode"; return KSG_ERR_INVALID_ARGUMENT; }
  if (c->color_mode < 0 || c->color_mode > 2) { why = "Unknown semantic color mode (base.cpp:186-190)"; return KSG_ERR_INVALID_ARGUMENT; }
  if (c->max_points <= 0 || c->max_points > (1 << kRecOrdBits)) { why = "max_points must be in (0, 2^23]"; return KSG_ERR_INVALID_ARGUMENT; }
  if (c->max_blocks <= 0) { why = "max_blocks must be positive"; return KSG_ERR_INVALID_ARGUMENT; }
  if (c->shard_count < 0 || (c->shard_count > 1 && (c->shard_rank < 0 || c->shard_rank >= c->shard_count))) {
    why = "shard_rank must be in [0, shard_count)"; return KSG_ERR_INVALID_ARGUMENT; }
  if (c->max_consecutive_ray_collisions < 0) { why = "max_consecutive_ray_collisions < 0"; return KSG_ERR_INVALID_ARGUMENT; }
  if (c->merged_bundle_order != KSG_BUNDLE_ORDER_CANONICAL && c->merged_bundle_order != KSG_BUNDLE_ORDER_LIBSTDCXX) {
    why = "unknown merged_bundle_order"; return KSG_ERR_INVALID_ARGUMENT; }
  if (c->hot_voxel_mode < 0 || c->hot_voxel_mode > 2) { why = "unknown hot_voxel_mode"; return KSG_ERR_INVALID_ARGUMENT; }
  return KSG_OK;
}

__global__ void k_iota(uint32_t* p, int n) { const int i = blockIdx.x * blockDim.x + threadIdx.x; if (i < n) p[i] = (uint32_t)i; }

int reset_map(ksg_integrator* h, cudaStream_t s) {
  KSG_CUDA(cudaMemsetAsync(h->map.ht_keys, 0xFF, sizeof(uint64_t) * h->ht_cap, s));
  KSG_CUDA(cudaMemsetAsync(h->map.ht_slot, 0xFF, sizeof(int) * h->ht_cap, s));
  KSG_CUDA(cudaMemsetAsync(h->map.touched_stamp, 0, sizeof(int) * h->ht_cap, s));
  KSG_CUDA(cudaMemsetAsync(h->d_cnt, 0, sizeof(Counters), s));
  if (h->start_table) KSG_CUDA(cudaMemsetAsync(h->start_table, 0xFF, sizeof(uint32_t) * kSetSize, s));
  if (h->o3.table) KSG_CUDA(cudaMemsetAsync(h->o3.table, 0xFF, sizeof(uint32_t) * kSetSize, s));
  if (h->d_fc) KSG_CUDA(cudaMemsetAsync(h->d_fc, 0, sizeof(FastCounters), s));
  if (h->start_rec) {   // every consumer empties what it decided; a reset does not rely on it
    KSG_CUDA(cudaMemset2DAsync(&h->start_rec->first, sizeof(StartRec), 0xFF, 2 * sizeof(uint32_t), kSetSize, s));   // first, hmin
    KSG_CUDA(cudaMemset2DAsync(&h->start_rec->hmax, sizeof(StartRec), 0x00, 2 * sizeof(uint32_t), kSetSize, s));    // hmax, visits
  }
  if (h->cast_bits) KSG_CUDA(cudaMemsetAsync(h->cast_bits, 0, sizeof(uint32_t) * ((size_t)h->cap_points / 32 + 64), s));
  if (h->o3.stamp_max) {   // (sweep 0, nobody): max word 0, min word all ones
    KSG_CUDA(cudaMemsetAsync(h->o3.stamp_max, 0x00, sizeof(uint64_t) * kSetSize, s));
    KSG_CUDA(cudaMemsetAsync(h->o3.stamp_min, 0xFF, sizeof(uint64_t) * kSetSize, s));
  }
  if (h->wl) KSG_CUDA(cudaMemsetAsync(h->wl, 0, sizeof(int) * (size_t)h->cap_points, s));   // listed sweeps: sweep ids restart at 0
  if (h->tile_cnt) KSG_CUDA(cudaMemsetAsync(h->tile_cnt, 0, sizeof(int) * (size_t)h->ht_cap * h->dc.tiles_per_block, s));
  h->n_pend = 0; h->n_stash = 0;
  std::memset(h->h_cnt_base, 0, 2 * sizeof(Counters));
  h->set_offset = 0;
  h->reset_counter = 0;
  h->num_blocks = 0;
  h->frame_stamp = 0;
  h->last_blocks_touched = 0;
  h->deferred_status = 0;
  h->merged_log_count = 0;
  h->esdf_full = true;
  h->esdf_valid = false;
  h->mesh_full = true;
  h->mesh_valid = false;
  KSG_CUDA(cudaStreamSynchronize(s));
  return KSG_OK;
}

struct InputDesc {
  const float* d_xyz = nullptr;
  const uint8_t* d_rgba = nullptr;
  const uint8_t* d_labels = nullptr;
  const float* d_depth = nullptr;
  const uint8_t* d_label_img = nullptr;
  int width = 0, height = 0;
  double K[4] = {0, 0, 0, 0};   // fx fy cx cy as the reference holds them (sensor_msgs/CameraInfo: float64)
  double unit_scaling = 1.0;    // DepthTraits<T>::toMeters(T(1)) as double: 1 (float32 metres) or double(0.001f) (uint16 millimetres)
  float z_scale = 1.0f;
  const uint32_t* d_color_img = nullptr;
  int64_t n = 0;  // points (points entry) or pixels (depth entry)
  int freespace = 0;
};

int fetch_counters(ksg_integrator* h, cudaStream_t s) {
  KSG_CUDA(cudaMemcpyAsync(h->h_cnt, h->d_cnt, sizeof(Counters), cudaMemcpyDeviceToHost, s));
  KSG_CUDA(cudaStreamSynchronize(s));
  return KSG_OK;
}

const char* err_text(int e) {
  switch (e) {
    case 1: return "invalid argument: a semantic label >= num_labels (CHECK_LT fast.cpp:134 / merged.cpp:278)";
    case 2: return "observed-set solver did not converge within its sweep budget";
    case 3: return "block pool / hash table full: raise ksg_config.max_blocks";
    case 4: return "per-frame scratch full: raise ksg_config.max_ray_steps / max_updates";
    case 5: return "voxel or block index outside the supported range";
    default: return "device-side error";
  }
}

// hot_voxel_mode = 1: finish the log-probability rows of the frame's hot voxels ahead of the apply kernels (ksg_hot.cuh).
// Returns the number of hot segments (0: nothing to do) through *n_hot.
int hot_voxel_rows(ksg_integrator* h, cudaStream_t s, const Xform& T, const float4* bundle_param, long long n_records, int* n_hot) {
  const DevCfg& dc = h->dc;
  KSG_CUDA(cudaMemsetAsync(h->d_hot_counts, 0, sizeof(int), s));
  ++h->n_launches;
  k_hot_find<<<grid_for(n_records, 256), 256, 0, s>>>(dc, h->map, h->rec_b, n_records, h->d_hot_segs, h->d_hot_counts);
  int found = 0;
  KSG_CUDA(cudaMemcpyAsync(&found, h->d_hot_counts, sizeof(int), cudaMemcpyDeviceToHost, s));
  KSG_CUDA(cudaStreamSynchronize(s));
  const int n = std::min(found, kHotMaxSegs);
  if (n <= 0) return KSG_OK;
  KSG_CUDA(cudaMemcpyAsync(h->h_hot_segs, h->d_hot_segs, sizeof(HotSeg) * (size_t)n, cudaMemcpyDeviceToHost, s));
  KSG_CUDA(cudaStreamSynchronize(s));
  std::sort(h->h_hot_segs, h->h_hot_segs + n, [](const HotSeg& a, const HotSeg& b) { return a.begin < b.begin; });
  long long chunks = 0;
  int kept = 0;
  for (int i = 0; i < n; ++i) {                       // segments that do not fit the chunk scratch stay on the ordinary path
    HotSeg& g = h->h_hot_segs[i];
    if (chunks + g.n_chunks > h->hot_chunk_cap) break;
    g.first_chunk = (int)chunks;
    for (int k = 0; k < g.n_chunks; ++k) h->h_hot_chunk_seg[chunks + k] = i;
    chunks += g.n_chunks;
    ++kept;
  }
  if (kept == 0) return KSG_OK;
  KSG_CUDA(cudaMemcpyAsync(h->d_hot_segs, h->h_hot_segs, sizeof(HotSeg) * (size_t)kept, cudaMemcpyHostToDevice, s));
  KSG_CUDA(cudaMemcpyAsync(h->d_hot_chunk_seg, h->h_hot_chunk_seg, sizeof(int) * (size_t)chunks, cudaMemcpyHostToDevice, s));
  const int nch = (int)chunks;
  h->n_launches += 4;
  k_hot_chunk_sums<<<grid_for((long long)nch * 32, 128), 128, 0, s>>>(dc.C, h->d_hot_segs, h->d_hot_chunk_seg, nch, h->rec_b, h->tmp, h->d_hot_sums);
  k_hot_guess<<<grid_for((long long)kept * 32, 128), 128, 0, s>>>(dc.C, h->d_hot_segs, kept, h->map.pool, h->d_hot_sums, h->d_hot_guess);
  k_hot_chunk_tables<<<nch, 128, sizeof(float) * (size_t)dc.C * kHotColStride, s>>>(dc.C, h->d_hot_segs, h->d_hot_chunk_seg, h->rec_b, h->tmp,
                                                                                  h->d_hot_guess, h->d_hot_tables);
  k_hot_apply<<<grid_for((long long)kept * 32, 128), 128, 0, s>>>(dc.C, h->d_hot_segs, kept, h->map.pool, h->rec_b, h->tmp, h->d_hot_guess,
                                                                  h->d_hot_tables, h->d_hot_prior, h->d_hot_counts + 1);
  if (h->cfg.hot_voxel_mode == 2) {
    KSG_CUDA(cudaMemsetAsync(h->d_hot_same, 0x01, sizeof(int) * (size_t)kept, s));   // 0x01010101: non-zero = "same" until refuted
    ++h->n_launches;
    k_hot_tsdf_same<<<nch, 128, 0, s>>>(dc, T, h->d_hot_segs, h->d_hot_chunk_seg, h->map.pool, h->rec_b, bundle_param, h->d_hot_same);
  }
  KSG_CUDA(cudaGetLastError());
  h->hot_segments_total += kept;
  h->hot_chunks_total += chunks;
  *n_hot = kept;
  return KSG_OK;
}
// The pre-pass, with `src` pointed at its results for the apply kernels.
int hot_voxel_prepass(ksg_integrator* h, cudaStream_t s, const Xform& T, long long n_records, ApplySrc* src, int* n_hot) {
  *n_hot = 0;
  const int rc = hot_voxel_rows(h, s, T, src->param, n_records, n_hot);
  if (rc) return rc;
  src->hot_segs = h->d_hot_segs; src->hot_prior = h->d_hot_prior; src->n_hot = *n_hot; src->hot_thresh = kHotThresh;
  src->hot_tsdf_same = (h->cfg.hot_voxel_mode == 2) ? h->d_hot_same : nullptr;
  return KSG_OK;
}


void fill_stats(ksg_integrator* h, ksg_frame_stats* stats) {
  std::memset(stats, 0, sizeof(*stats));
  stats->points_in = h->h_cnt->n_points;
  stats->points_valid = h->h_cnt->n_valid;
  stats->rays_cast = h->h_cnt->n_cast;
  stats->ray_steps = (int64_t)h->h_cnt->ray_steps;
  stats->voxel_updates = (int64_t)h->h_cnt->n_records - (int64_t)h->h_cnt->n_skipped;
  stats->blocks_allocated = h->num_blocks;
  stats->blocks_touched = h->h_cnt->n_blocks_touched;
  stats->tiles_touched = h->h_cnt->n_tiles;
  stats->fixpoint_iterations = h->h_fc ? h->h_fc->sweeps_last : 0;
}

// The end of every frame, once its counters are on the host: the map's size mirrored, and a device-side error turned into
// the integrator's deferred status.
void mirror_counters(ksg_integrator* h) {
  h->num_blocks = h->h_cnt->pool_count;
  h->last_blocks_touched = h->h_cnt->n_blocks_touched;
}
int device_error(ksg_integrator* h) {
  const int dev_err = h->h_cnt->err;
  if (dev_err) {
    h->deferred_status = dev_err;  // the map may be inconsistent from here on
    return h->fail(dev_err, err_text(dev_err));
  }
  return KSG_OK;
}
// The synchronous epilogue of the map-merge entries
int finish_sync(ksg_integrator* h, cudaStream_t s) {
  KSG_CUDA(cudaGetLastError());
  const int rc = fetch_counters(h, s);
  if (rc) return rc;
  mirror_counters(h);
  return device_error(h);
}

// Completes the OLDEST frame whose counters are still in flight (fast): waits for its counter copy, mirrors the
// counters on the host and reports a device-side error.
int finish_oldest(ksg_integrator* h, ksg_frame_stats* stats) {
  if (h->n_pend <= 0) return KSG_OK;
  const int slot = h->pend[0];
  h->pend[0] = h->pend[1];
  --h->n_pend;
  KSG_CUDA(cudaEventSynchronize(h->ev_frame_s[slot]));
  h->h_cnt = h->h_cnt_base + slot;
  if (h->h_fc_base) h->h_fc = h->h_fc_base + slot;
  mirror_counters(h);
  if (h->profiling && h->h_fc) {
    // events: 0 frame start, 1 before the solve kernel, 2 after it, 3 after the tile kernel; the solve kernel's own phases come from
    // the clock64 marks block 0 left in FastCounters::timeline
    float a = 0, b = 0, c = 0, tot = 0;
    cudaEventElapsedTime(&a, h->ev[0], h->ev[1]); cudaEventElapsedTime(&b, h->ev[1], h->ev[2]);
    cudaEventElapsedTime(&c, h->ev[2], h->ev[3]); cudaEventElapsedTime(&tot, h->ev[0], h->ev[3]);
    const long long* tl = h->h_fc->timeline;
    const int sweeps_end = (int)tl[kTimelineSlots - 1];
    const int tb = kTimelineSlots - 12;
    const double span = (double)(tl[tb + 4] - tl[0]);
    if (span > 0 && sweeps_end >= 3 && sweeps_end <= tb) {
      const double k = (double)b / span;
      h->phase_ms[0] += a + k * (double)(tl[2] - tl[0]);                 // count + classify + start set + compaction + ray set-up
      h->phase_ms[1] += k * (double)(tl[tb] - tl[2]);                    // observed-set sweeps
      h->phase_ms[2] += k * (double)(tl[tb + 1] - tl[tb]);               // table commit + ray emit / block allocation
      h->phase_ms[3] += k * (double)(tl[tb + 4] - tl[tb + 1]);           // records -> tile segments (count, allocate + new blocks, scatter)
    } else { h->phase_ms[0] += a; h->phase_ms[1] += b; }
    h->phase_ms[5] += c;
    h->phase_ms[6] += tot;
    h->prof_frames += 1;
  }
  if (stats) fill_stats(h, stats);
  return device_error(h);
}
// Completes every outstanding frame; `stats` receives the newest frame's counters.
int finish_frame(ksg_integrator* h, ksg_frame_stats* stats) {
  while (h->n_pend > 1) { const int rc = finish_oldest(h, nullptr); if (rc) return rc; }
  if (h->n_pend == 1) return finish_oldest(h, stats);
  if (stats) fill_stats(h, stats);
  if (h->deferred_status) return h->fail(h->deferred_status, err_text(h->deferred_status));
  return KSG_OK;
}
// The prologue of a host-buffer entry, which sees the map only once every submitted frame has completed: the device idle, the pending
// frames completed, and their status.
int complete_frames(ksg_integrator* h) {
  KSG_CUDA(cudaSetDevice(h->device));
  KSG_CUDA(cudaDeviceSynchronize());
  return finish_frame(h, nullptr);
}

// fast: ApproxHashSet resets (fast.cpp:165-170, A.4), once per frame before any point is looked at
int advance_sets(ksg_integrator* h, cudaStream_t s) {
  if ((++h->reset_counter) >= h->cfg.clear_checks_every_n_frames) {
    h->reset_counter = 0;
    if (++h->set_offset >= 10000) {
      h->set_offset = 0;
      KSG_CUDA(cudaMemsetAsync(h->start_table, 0xFF, sizeof(uint32_t) * kSetSize, s));
      KSG_CUDA(cudaMemsetAsync(h->o3.table, 0xFF, sizeof(uint32_t) * kSetSize, s));
    }
  }
  return KSG_OK;
}

// `fast` frame driver: six launches, no host read-back inside the frame (ksg_fast.cuh).
int integrate_fast(ksg_integrator* h, const InputDesc& in, const FrameIn& fin, const Xform& T, int cap, cudaStream_t s,
                   ksg_frame_stats* stats) {
  const bool sorted = h->cfg.integration_order_mode == KSG_ORDER_SORTED;
  { const int rcs = advance_sets(h, s); if (rcs) return rcs; }
  FastFrame f{};
  f.cfg = h->dc; f.T = T; f.in = fin; f.in.pix_list = nullptr; f.in.point_of_seq = nullptr;
  f.luts = h->d_luts; f.cnt = h->d_cnt; f.fc = h->d_fc; f.map = h->map;
  f.sb = StartBuf{h->start_rec, h->start_table, h->start_touched, sorted ? h->point_of_seq : nullptr};
  f.set_offset = h->set_offset;
  f.capacity = cap;
  f.n_count_blocks = (cap + kCountBlock - 1) / kCountBlock;
  f.vec_ok = in.d_depth ? (((uintptr_t)in.d_depth % 16 == 0 && (uintptr_t)in.d_label_img % 4 == 0) ? 1 : 0) : 0;
  f.frame_stamp = h->frame_stamp;
  f.profile = (h->profiling && !h->profile_marks_only) ? 1 : 0;
  f.prof_marks = h->profiling ? 1 : 0;
  f.seq_of_i = sorted ? h->seq_of_i : nullptr;
  f.block_cnt = h->blk_cnt; f.block_off = h->blk_off; f.cast_bits = h->cast_bits; f.warp_off = h->warp_off;
  f.pt_key = h->pt_key; f.pt_pix = h->pix_list;
  f.cast_seq = h->cast_seq; f.ray_param = h->ray_param; f.ray_label = h->ray_label; f.ray_flags = h->ray_flags; f.ray_color = h->ray_color;
  f.ray_state = h->ray_state; f.ext_off = h->ext_off;
  f.rec_cap = h->rec_cap; f.keys = h->keys32;
  f.tile_cnt = h->tile_cnt; f.tile_slot = h->tile_slot; f.tile_list = h->tile_list; f.tile_cap = h->tile_cap;
  f.o3 = h->o3;
  f.rayrec = h->rayrec; f.blk_run = h->blk_run;
  f.wl_listed = h->wl;
  f.wl_list[0] = h->wl + h->cap_points; f.wl_list[1] = h->wl + 2 * (size_t)h->cap_points;
  f.log_head = h->d_log_head; f.log_prior = h->d_log_prior; f.log_cap = h->log_cap;
  f.mixed_list = h->mixed_list; f.m_list = h->m_list;

  if (h->profiling) {
    cudaEventRecord(h->ev[0], s);
    KSG_CUDA(cudaMemsetAsync(h->d_fc->dbg, 0, sizeof(h->d_fc->dbg), s));
  }
  KSG_CUDA(cudaMemsetAsync(h->o3.head, 0xFF, sizeof(int) * kSetSize, s));
  KSG_CUDA(cudaMemsetAsync(h->o3.slot_cnt, 0x00, sizeof(int) * kSetSize, s));
  const int B = 256;
  ++h->n_launches;
  if (in.d_depth) k_fast_count<<<f.n_count_blocks, 256, 0, s>>>(f);
  else k_fast_reset<<<1, 1, 0, s>>>(f);
  if (sorted) {   // voxblox SortedThreadSafeIndex (A.3): stable order by squared norm
    h->n_launches += 3;
    if (in.d_depth) k_fast_sqnorm<<<f.n_count_blocks, 256, 0, s>>>(f, h->sq_keys);
    else k_fast_sqnorm_points<<<grid_for(cap, B), B, 0, s>>>(f, h->sq_keys);
    k_fast_pad_keys<<<grid_for(cap, B), B, 0, s>>>(h->d_cnt, cap, h->sq_keys);
    size_t tb = h->cub_temp_bytes;
    ++h->n_libcalls;
    KSG_CUDA(cub::DeviceRadixSort::SortPairs(h->cub_temp, tb, h->sq_keys, h->sq_keys_out, h->iota, (uint32_t*)h->point_of_seq, cap, 0, 32, s));
    k_fast_invert_perm<<<grid_for(cap, B), B, 0, s>>>(h->d_cnt, (const uint32_t*)h->point_of_seq, h->seq_of_i);
  }
  ++h->n_launches;
  if (in.d_depth) k_fast_classify<true><<<f.n_count_blocks, 256, 0, s>>>(f);
  else k_fast_classify<false><<<grid_for(cap, B), B, 0, s>>>(f);
  ++h->n_launches;
  k_fast_start_slots<<<std::min(grid_for(cap, B), 4 * h->sm_count), B, 0, s>>>(f);
  if (h->profiling) cudaEventRecord(h->ev[1], s);
  {
    // The fixpoint is reached within rays + 1 sweeps, plus one that changes nothing (DESIGN.md section 4), and a frame casts at
    // most max_points rays: past this budget the solver is wrong, not slow, and the kernel flags an error rather than spin.
    int max_sweeps = h->cap_points + 2;
    void* args[] = {(void*)&f, (void*)&max_sweeps};
    ++h->n_launches;
    KSG_CUDA(cudaLaunchCooperativeKernel((const void*)k_fast_solve3, dim3(h->solve_grid), dim3(h->solve_threads), args,
                                         (size_t)h->solve_smem, s));
  }
  if (h->profiling) cudaEventRecord(h->ev[2], s);
  {
    ApplySrc src{};
    src.param = h->ray_param; src.label = h->ray_label; src.color = h->ray_color; src.tmp = nullptr;
    h->n_launches += 2;
    k_fast_group<<<h->group_grid, kGroupThreads, 0, s>>>(f, h->fast_items, h->fast_tiles, h->item_cap);
    with_nch(h->apply_nch, [&](auto nch) {
      k_fast_apply<decltype(nch)::value><<<h->fast_apply_grid, kFastApplyThreads, 0, s>>>(f, src, h->fast_items, h->fast_tiles, h->item_cap);
    });
  }
  if (h->profiling) cudaEventRecord(h->ev[3], s);
  KSG_CUDA(cudaGetLastError());
  if (h->n_pend == 2) {   // both counter slots in flight: complete the older frame first (its statistics stay retrievable)
    ksg_frame_stats old_stats;
    const int rco = finish_oldest(h, &old_stats);
    if (h->n_stash < 4) h->stash[h->n_stash++] = old_stats;
    if (rco) return rco;
  }
  const int slot = h->next_slot;
  KSG_CUDA(cudaMemcpyAsync(h->h_cnt_base + slot, h->d_cnt, sizeof(Counters), cudaMemcpyDeviceToHost, s));
  KSG_CUDA(cudaMemcpyAsync(h->h_fc_base + slot, h->d_fc, sizeof(FastCounters), cudaMemcpyDeviceToHost, s));
  KSG_CUDA(cudaEventRecord(h->ev_frame_s[slot], s));
  h->pend[h->n_pend++] = slot;
  h->next_slot ^= 1;
  if (stats || h->profiling) return finish_frame(h, stats);
  return KSG_OK;
}

// `merged` frame: what one stage of the driver hands to the next
struct MergedFrame {
  const InputDesc& in;
  FrameIn fin;
  Xform T;
  int cap;                 // host upper bound of the point count
  cudaStream_t s;
  long long n_records = 0;
  int n_hot = 0;           // hot segments of the pre-pass (hot_voxel_mode >= 1)
  ApplySrc src{};
};

// Bundling: the points classified and grouped into bundles (one ray each), the bundles' record ranges; ends with the counters
// on the host.
int merged_bundles(ksg_integrator* h, MergedFrame& m) {
  const DevCfg& dc = h->dc;
  const int cap = m.cap, B = 256;
  cudaStream_t s = m.s;
  ++h->n_launches;
  k_frame_reset<<<1, 1, 0, s>>>(h->d_cnt, m.in.d_depth ? 0 : cap);
  if (m.in.d_depth) {
    ++h->n_launches;
    k_depth_flags<<<grid_for(cap, B), B, 0, s>>>(m.in.d_depth, cap, h->flags8);
    size_t tb = h->cub_temp_bytes;
    ++h->n_libcalls;
    KSG_CUDA(cub::DeviceSelect::Flagged(h->cub_temp, tb, cub::CountingInputIterator<int>(0), h->flags8, h->pix_list,
                                        &h->d_cnt->n_points, cap, s));
  }
  if (h->cfg.integration_order_mode == KSG_ORDER_SORTED) {
    ++h->n_launches;
    k_sqnorm<<<grid_for(cap, B), B, 0, s>>>(m.fin, h->d_cnt, cap, h->sq_keys);
    size_t tb = h->cub_temp_bytes;
    ++h->n_libcalls;
    KSG_CUDA(cub::DeviceRadixSort::SortPairs(h->cub_temp, tb, h->sq_keys, h->sq_keys_out, h->iota, (uint32_t*)h->point_of_seq,
                                             cap, 0, 32, s));
    m.fin.point_of_seq = h->point_of_seq;
  }
  ++h->n_launches;
  k_classify<<<grid_for(cap, B), B, 0, s>>>(dc, m.T, m.fin, h->d_luts, cap, h->d_cnt, h->pt_pC, h->pt_pG, h->pt_label,
                                            h->pt_flags, h->pt_color, h->pt_key);
  if (h->profiling) cudaEventRecord(h->ev[1], s);
  {
    size_t tb = h->cub_temp_bytes;
    ++h->n_libcalls;
    KSG_CUDA(cub::DeviceRadixSort::SortPairs(h->cub_temp, tb, h->pt_key, h->ks_sorted, h->iota, h->seq_sorted, cap, 0, 64, s));
  }
  KSG_CUDA(cudaMemsetAsync(h->flags8, 0, 2 * (size_t)cap, s));
  ++h->n_launches;
  k_bundle_heads<<<grid_for(cap, B), B, 0, s>>>(h->ks_sorted, h->seq_sorted, cap, h->flags8, h->bstart);
  {
    size_t tb = h->cub_temp_bytes;
    ++h->n_libcalls;
    KSG_CUDA(cub::DeviceSelect::Flagged(h->cub_temp, tb, cub::CountingInputIterator<int>(0), h->flags8, h->bundle_f,
                                        &h->d_cnt->n_cast, 2 * cap, s));
  }
  const int* bundle_heads = h->bundle_f;   // canonical: first-insertion order
  if (h->cfg.merged_bundle_order == KSG_BUNDLE_ORDER_LIBSTDCXX) {
    h->n_launches += 2;
    k_bord_hash<<<grid_for(cap, B), B, 0, s>>>(h->d_cnt, h->bundle_f, h->bstart, h->ks_sorted, cap, h->bord_hash);
    // every rehash phase of both maps (voxel_map merged.cpp:126-134, clear_map :138-145) in one launch: one cluster per map
    k_bundle_order<<<2 * kBordCluster, kBordThreads, 0, s>>>(h->d_cnt, h->bord, h->bundle_f, h->bundle_f2);
    bundle_heads = h->bundle_f2;
  }
  ++h->n_launches;
  k_bundle_merge<<<h->sm_count * 8, 256, 0, s>>>(dc, m.T, h->d_cnt, bundle_heads, h->bstart, h->ks_sorted, h->seq_sorted, cap, h->pt_pC,
                                                 h->pt_label, h->hist, h->ray_param, h->ray_flags, h->b_key, h->nsteps);
  ++h->n_launches;
  k_bundle_scan<<<kBordCluster, kBordThreads, 0, s>>>(h->d_cnt, h->nsteps, h->b_base, h->rec_cap, h->d_scan_tot);
  return fetch_counters(h, s);
}

// The bundles' log-likelihood rows and their update records
void merged_emit(ksg_integrator* h, MergedFrame& m) {
  const DevCfg& dc = h->dc;
  const int B = 256;
  cudaStream_t s = m.s;
  const int nb = std::max(1, h->h_cnt->n_cast);
  m.n_records = (long long)h->h_cnt->n_records;
  ++h->n_launches;
  k_bundle_loglik<<<grid_for((long long)(nb + 1) * dc.C, B), B, 0, s>>>(dc, h->d_cnt, h->hist, h->tmp, h->tmp4);
  ++h->n_launches;
  k_emit_merged<<<grid_for(nb, 128), 128, 0, s>>>(dc, m.T, h->d_cnt, h->map, h->ray_param, h->ray_flags, h->b_key, h->nsteps,
                                                  h->b_base, h->ks_sorted, m.cap, h->rec_a);
}

// The update records in (tile, voxel, order) order: per-voxel application order = reference order; then the frame's new blocks
int merged_sort_records(ksg_integrator* h, MergedFrame& m) {
  const DevCfg& dc = h->dc;
  cudaStream_t s = m.s;
  size_t tb = h->cub_temp_bytes;
  ++h->n_libcalls;
  // significant key bits: [order 23][voxel 9][tile key < ht_cap * tiles_per_block]
  int end_bit = 32;
  while (end_bit < 64 && (1ull << (end_bit - 32)) < (unsigned long long)h->ht_cap * (unsigned long long)dc.tiles_per_block) ++end_bit;
  // the records were laid out by (bundle rank, step), so a stable sort on the voxel bits [23, end) keeps the rank order
  KSG_CUDA(cub::DeviceRadixSort::SortKeys(h->cub_temp, tb, h->rec_a, h->rec_b, m.n_records, kRecOrdBits, end_bit, s));
  if (h->profiling) cudaEventRecord(h->ev[4], s);
  ++h->n_launches;
  k_block_init<<<h->sm_count * 4, 256, 0, s>>>(dc, h->d_cnt, h->map);
  return KSG_OK;
}

// Per-voxel update (ksg_voxel.cuh): segment heads -> two queues; then one kernel on the high-priority side stream and the short
// kernel on the frame's stream.  C <= 32: the hot voxels' chains (the DEEP instance, one warp per chain) beside the thread-per-voxel
// short kernel, and the remaining long segments, little work, behind it.  C > 32: the long kernel beside the warp-per-voxel one.
int merged_apply_voxels(ksg_integrator* h, MergedFrame& m) {
  const DevCfg& dc = h->dc;
  const Xform& T = m.T;
  cudaStream_t s = m.s;
  KSG_CUDA(cudaMemsetAsync(h->vq.counters, 0, sizeof(int) * 8, s));
  ++h->n_launches;
  k_voxel_heads<<<grid_for(m.n_records, kHeadsBlock), 256, 0, s>>>(dc, h->d_cnt, h->map, h->rec_b, m.n_records, h->frame_stamp, h->vq);
  if (h->profiling) cudaEventRecord(h->ev[5], s);
  if (h->hot_enabled) { const int rch = hot_voxel_prepass(h, s, T, m.n_records, &m.src, &m.n_hot); if (rch) return rch; }
  const ApplySrc& src = m.src;
  KSG_CUDA(cudaEventRecord(h->ev_fork, s));
  KSG_CUDA(cudaStreamWaitEvent(h->aux_stream, h->ev_fork, 0));
  if (h->apply_nch == 1) {
    h->n_launches += 3;
    k_voxel_apply_long<1, true><<<h->sm_count, h->deep_threads, 0, h->aux_stream>>>(dc, T, h->d_cnt, h->map, h->d_luts, h->rec_b, src, h->vq, 0);
    k_voxel_apply_short_t<<<h->sm_count * h->short_t_ctas, 256, 0, s>>>(dc, T, h->d_cnt, h->map, h->d_luts, h->rec_b, src, h->vq);
    k_voxel_apply_long<1><<<h->long_grid, h->long_threads, 0, s>>>(dc, T, h->d_cnt, h->map, h->d_luts, h->rec_b, src, h->vq, 1);
  } else {
    h->n_launches += 2;
    with_nch(h->apply_nch, [&](auto nch) {
      constexpr int NCH = decltype(nch)::value;
      k_voxel_apply_long<NCH><<<h->long_grid, h->long_threads, 0, h->aux_stream>>>(dc, T, h->d_cnt, h->map, h->d_luts, h->rec_b, src, h->vq, 0);
      k_voxel_apply_short<NCH><<<h->sm_count * h->short_ctas, 256, h->short_smem, s>>>(dc, T, h->d_cnt, h->map, h->d_luts, h->rec_b, src, h->vq);
    });
  }
  KSG_CUDA(cudaEventRecord(h->ev_join, h->aux_stream));
  KSG_CUDA(cudaStreamWaitEvent(s, h->ev_join, 0));
  return KSG_OK;
}

// Tile update (apply_mode 1, KSG_MERGED_TILE_APPLY=1): one CTA walks the records of a tile
int merged_apply_tiles(ksg_integrator* h, MergedFrame& m) {
  const DevCfg& dc = h->dc;
  const Xform& T = m.T;
  cudaStream_t s = m.s;
  const int B = 256;
  ++h->n_launches;
  k_tile_heads<<<grid_for(m.n_records, B), B, 0, s>>>(dc, h->d_cnt, h->map, h->rec_b, m.n_records, h->frame_stamp, h->tile_begin,
                                                      h->tile_cap);
  if (h->profiling) cudaEventRecord(h->ev[5], s);
  const int ctas_per_sm = std::max(1, std::min(8, (int)(220 * 1024 / std::max(1, h->apply_smem + 1024))));
  const int grid = h->sm_count * ctas_per_sm;
  if (h->hot_enabled) { const int rch = hot_voxel_prepass(h, s, T, m.n_records, &m.src, &m.n_hot); if (rch) return rch; }
  const ApplySrc& src = m.src;
  ++h->n_launches;
  if (m.n_hot > 0) {   // C <= 32, TMA staging (checked when hot_enabled was set)
    k_tile_apply<true, 1, true><<<grid, 256, h->apply_smem, s>>>(dc, T, h->d_cnt, h->map, h->d_luts, h->rec_b, m.n_records,
                                                                 h->tile_begin, h->tile_cap, src, h->tile_debug);
  } else {
    with_tma(h->use_tma, [&](auto tma) {
      with_nch(h->apply_nch, [&](auto nch) {
        k_tile_apply<decltype(tma)::value, decltype(nch)::value><<<grid, 256, h->apply_smem, s>>>(
            dc, T, h->d_cnt, h->map, h->d_luts, h->rec_b, m.n_records, h->tile_begin, h->tile_cap, src, h->tile_debug);
      });
    });
  }
  return KSG_OK;
}

// Update log (ksg_log.cuh), behind every apply kernel.  The unsorted record buffer (and the short queue in it) is free again:
// [head record indices : n_records ints][flags : n_records bytes], later [head record indices][the same, block-index order].
// The sort keys go to the log's own entry buffer, which the entries overwrite only after the sort (32 bytes per entry >= 16).
int merged_update_log(ksg_integrator* h, MergedFrame& m) {
  const DevCfg& dc = h->dc;
  cudaStream_t s = m.s;
  const int B = 256;
  const long long n_records = m.n_records;
  int* heads = (int*)h->rec_a;
  int* heads_alt = heads + n_records;
  uint8_t* flags = (uint8_t*)heads_alt;
  ++h->n_launches;
  k_merged_log_heads<<<grid_for(n_records, B), B, 0, s>>>(dc, h->map, h->rec_b, n_records, flags);
  size_t tb = h->cub_temp_bytes;
  ++h->n_libcalls;
  KSG_CUDA(cub::DeviceSelect::Flagged(h->cub_temp, tb, cub::CountingInputIterator<int>(0), flags, heads, &h->d_cnt->pad0, (int)n_records, s));
  int n_heads = 0;
  KSG_CUDA(cudaMemcpyAsync(&n_heads, &h->d_cnt->pad0, sizeof(int), cudaMemcpyDeviceToHost, s));
  KSG_CUDA(cudaStreamSynchronize(s));
  if (n_heads > 0 && n_heads <= h->log_cap) {
    uint64_t* keys = (uint64_t*)h->d_log_head;
    ++h->n_launches;
    k_merged_log_keys<<<grid_for(n_heads, B), B, 0, s>>>(dc, h->map, h->rec_b, heads, n_heads, keys);
    cub::DoubleBuffer<uint64_t> kb(keys, keys + n_heads);
    cub::DoubleBuffer<int> vb(heads, heads_alt);
    tb = h->cub_temp_bytes;
    ++h->n_libcalls;
    KSG_CUDA(cub::DeviceRadixSort::SortPairs(h->cub_temp, tb, kb, vb, n_heads, 0, 63, s));   // pack_key: 3 x 21 bits
    ++h->n_launches;
    k_merged_log_write<<<h->sm_count * 8, 256, 0, s>>>(dc, h->map, h->rec_b, vb.Current(), n_heads, h->d_log_head, h->d_log_prior);
  }
  return KSG_OK;
}

// Completion: the frame's counters on the host, its phase times, statistics and device-side error.  `applied`: the records were
// sorted and applied (no device-side error in the bundling, at least one record).
int merged_complete(ksg_integrator* h, const MergedFrame& m, bool applied, ksg_frame_stats* stats) {
  cudaStream_t s = m.s;
  if (h->profiling) { if (!applied) { cudaEventRecord(h->ev[4], s); cudaEventRecord(h->ev[5], s); } cudaEventRecord(h->ev[6], s); }
  ++h->n_launches;
  k_frame_finish<<<1, 1, 0, s>>>(h->d_cnt, h->map);
  KSG_CUDA(cudaGetLastError());
  const int rc = fetch_counters(h, s);
  if (rc) return rc;
  if (h->profiling) {
    cudaEventRecord(h->ev[7], s);
    cudaEventSynchronize(h->ev[7]);
    for (int p = 0; p < 6; ++p) { float ms = 0; if (cudaEventElapsedTime(&ms, h->ev[p], h->ev[p + 1]) == cudaSuccess) h->phase_ms[p] += ms; }
    { float ms = 0; if (cudaEventElapsedTime(&ms, h->ev[0], h->ev[7]) == cudaSuccess) h->phase_ms[6] += ms; }
    h->prof_frames += 1;
  }
  mirror_counters(h);
  h->last_hot_segments = m.n_hot;
  if (applied && h->d_log_head) h->merged_log_count = h->h_cnt->pad0;
  h->last_frame_queued = applied && h->voxel_apply;
  if (stats) {
    fill_stats(h, stats);
    stats->voxel_updates = m.n_records - (int64_t)h->h_cnt->n_skipped;   // this frame's records: none after a bundling error
    stats->hot_voxels = m.n_hot;
    if (h->hot_enabled && m.n_hot > 0) {
      int fb = 0;
      if (cudaMemcpyAsync(&fb, h->d_hot_counts + 1, sizeof(int), cudaMemcpyDeviceToHost, s) == cudaSuccess && cudaStreamSynchronize(s) == cudaSuccess)
        stats->hot_fallback_chunks = fb;
    }
  }
  return device_error(h);
}

// `merged` frame driver: the host reads the counters back after the bundling and at completion.
int integrate_merged(ksg_integrator* h, const InputDesc& in, const FrameIn& fin, const Xform& T, int cap, cudaStream_t s,
                     ksg_frame_stats* stats) {
  MergedFrame m{in, fin, T, cap, s};
  h->merged_log_count = 0;
  if (h->profiling) cudaEventRecord(h->ev[0], s);
  { const int rc = merged_bundles(h, m); if (rc) return rc; }
  if (h->profiling) cudaEventRecord(h->ev[2], s);
  if (!h->h_cnt->err) merged_emit(h, m);
  m.src.param = h->ray_param; m.src.label = nullptr; m.src.color = nullptr; m.src.tmp = h->tmp; m.src.tmp4 = h->tmp4;
  if (h->profiling) cudaEventRecord(h->ev[3], s);
  const bool applied = !h->h_cnt->err && m.n_records > 0;
  if (applied) {
    int rc = merged_sort_records(h, m);
    if (!rc) rc = h->voxel_apply ? merged_apply_voxels(h, m) : merged_apply_tiles(h, m);
    if (!rc && h->d_log_head) rc = merged_update_log(h, m);
    if (rc) return rc;
  }
  return merged_complete(h, m, applied, stats);
}

int integrate(ksg_integrator* h, const InputDesc& in, const float* T_host, cudaStream_t s, ksg_frame_stats* stats) {
  if (h->deferred_status) return h->fail(h->deferred_status, err_text(h->deferred_status));
  if (in.n == 0 && h->n_pend > 0) { const int rcp = finish_frame(h, nullptr); if (rcp) return rcp; }
  KSG_CUDA(cudaSetDevice(h->device));
  const bool fast = h->cfg.integrator_type == KSG_INTEGRATOR_FAST;
  const int cap = (int)in.n;  // host upper bound of the point count
  Xform T{T_host[0], T_host[1], T_host[2], T_host[3], T_host[4], T_host[5], T_host[6]};
  h->frame_stamp += 1;

  if (cap == 0) {
    if (stats) { std::memset(stats, 0, sizeof(*stats)); stats->blocks_allocated = h->num_blocks; }
    if (fast) { const int rcs = advance_sets(h, s); if (rcs) return rcs; }   // the sets are reset even for an empty frame
    else h->merged_log_count = 0;
    h->last_blocks_touched = 0;
    return KSG_OK;
  }

  FrameIn fin{};
  fin.xyz = in.d_xyz; fin.rgba = in.d_rgba; fin.labels = in.d_labels;
  fin.depth = in.d_depth; fin.label_img = in.d_label_img; fin.pix_list = h->pix_list;
  fin.point_of_seq = nullptr;
  fin.width = in.width;
  fin.cx = (float)in.K[2]; fin.cy = (float)in.K[3];   // depth_map_to_pointcloud.h:222-223 float center = model_.cx()
  if (in.d_depth) {  // depth_map_to_pointcloud.h:228-230: float constant = unit_scaling / f  (double division)
    fin.constant_x = (float)(in.unit_scaling / in.K[0]);
    fin.constant_y = (float)(in.unit_scaling / in.K[1]);
  }
  fin.z_scale = in.z_scale;
  fin.color_img = in.d_color_img;
  fin.freespace = in.freespace;
  if (fast) return integrate_fast(h, in, fin, T, cap, s, stats);
  return integrate_merged(h, in, fin, T, cap, s, stats);
}

bool is_pinned_host(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return a.type == cudaMemoryTypeHost;
}

// The argument check of every frame entry, made before anything is staged: at most max_points points, and not merged in ColorMode::kColor
// with both point colours and explicit labels (merged.h:82-86 blends the colours, merged.cpp:262-274; see ksg.h).
int check_frame(ksg_integrator* h, int64_t n, bool colors_and_labels) {
  if (n > h->cap_points) return h->fail(KSG_ERR_INVALID_ARGUMENT, "cloud / frame larger than ksg_config.max_points");
  if (colors_and_labels && h->cfg.integrator_type == KSG_INTEGRATOR_MERGED && h->cfg.color_mode == KSG_COLOR_MODE_COLOR)
    return h->fail(KSG_ERR_INVALID_ARGUMENT, "merged, ColorMode::kColor: explicit labels together with point colours are not supported - pass "
                                             "the colours alone (labels by colour) or choose another colour mode");
  return KSG_OK;
}

// A frame's input arrays of bytes[0 .. N) laid out one after another in a staging buffer, each at a 256-byte boundary: their offsets go
// to `off`, and the layout's total size is returned.
template <size_t N> size_t frame_slices(const size_t (&bytes)[N], size_t (&off)[N]) {
  size_t total = 0;
  for (size_t k = 0; k < N; ++k) { off[k] = total; total += (bytes[k] + 255) / 256 * 256; }
  return total;
}

int ensure_input(ksg_integrator* h, size_t bytes) {
  if (bytes > h->h_stage_bytes) KSG_CUDA(h->res.regrow_pinned(&h->h_stage, &h->h_stage_bytes, bytes));
  if (bytes > h->d_in_bytes) KSG_CUDA(h->res.regrow(&h->d_in, &h->d_in_bytes, bytes));
  return KSG_OK;
}

// A device copy of `v` in `tmp`, enqueued on `s`.
template <typename T> cudaError_t upload(Resources& tmp, const std::vector<T>& v, cudaStream_t s, T** d) {
  const cudaError_t e = tmp.device(d, v.size());
  return e != cudaSuccess ? e : cudaMemcpyAsync(*d, v.data(), sizeof(T) * v.size(), cudaMemcpyHostToDevice, s);
}

// The device side of a host-buffer entry's host arrays: one temporary allocation per call, one 256-byte aligned slice per array.  The
// caller declares the slices, each with the device pointer it sets, then run() makes them, uploads the inputs, launches, copies every
// output slice to its host array on the call's stream and synchronises once.
class HostStaging {
 public:
  // a slice for the host output `host` (NULL: not wanted, no slice and *dev = NULL, unless the kernel needs the slice anyway)
  template <typename T> void out(T** dev, T* host, size_t count, bool kernel_needs = false) {
    *dev = nullptr;
    if (host || kernel_needs) add(dev, host, nullptr, count);
  }
  // a slice holding a copy of the host input `host`
  template <typename T> void in(const T** dev, const T* host, size_t count) { add(dev, nullptr, host, count); }
  // launch() enqueues the work on `s` once the device pointers are set, and returns a status
  template <typename F> int run(ksg_integrator* h, cudaStream_t s, F&& launch) {
    size_t total = 0;
    for (const Slice& sl : slices_) total += aligned(sl.bytes);
    uint8_t* d = nullptr;
    KSG_CUDA(tmp_.device(&d, total));
    for (Slice& sl : slices_) {
      sl.at = d;
      sl.bind(sl.dev, d);
      if (sl.in) KSG_CUDA(cudaMemcpyAsync(d, sl.in, sl.bytes, cudaMemcpyHostToDevice, s));
      d += aligned(sl.bytes);
    }
    { const int rcl = launch(); if (rcl) return rcl; }
    KSG_CUDA(cudaGetLastError());
    for (const Slice& sl : slices_)
      if (sl.host) KSG_CUDA(cudaMemcpyAsync(sl.host, sl.at, sl.bytes, cudaMemcpyDeviceToHost, s));
    KSG_CUDA(cudaStreamSynchronize(s));
    return KSG_OK;
  }

 private:
  struct Slice {
    void* dev;                             // the T* that bind() points at the slice
    void (*bind)(void* dev, uint8_t* at);
    void* host;                            // an output's host array
    const void* in;                        // an input's host array
    size_t bytes;
    uint8_t* at = nullptr;
  };
  template <typename T> void add(T** dev, void* host, const void* in, size_t count) {
    slices_.push_back(Slice{dev, [](void* p, uint8_t* at) { *static_cast<T**>(p) = reinterpret_cast<T*>(at); }, host, in, count * sizeof(T)});
  }
  static size_t aligned(size_t bytes) { return (bytes + 255) / 256 * 256; }
  std::vector<Slice> slices_;
  Resources tmp_;
};

}  // namespace

extern "C" {

void ksg_default_config(ksg_config* c, int32_t integrator_type, float voxel_size, int32_t voxels_per_side, int32_t num_labels) {
  std::memset(c, 0, sizeof(*c));
  c->abi_version = KSG_ABI_VERSION;
  c->integrator_type = integrator_type;
  c->voxel_size = voxel_size;
  c->voxels_per_side = voxels_per_side;
  c->default_truncation_distance = 4.0f * voxel_size;  // voxblox_ros: truncation_distance = 4 * voxel_size
  c->max_weight = 10000.0f;
  c->voxel_carving_enabled = 1;
  c->min_ray_length_m = 0.1f;
  c->max_ray_length_m = 5.0f;
  c->use_const_weight = 0;
  c->allow_clear = 1;
  c->use_weight_dropoff = 1;
  c->use_sparsity_compensation_factor = 0;
  c->sparsity_compensation_factor = 1.0f;
  c->integration_order_mode = KSG_ORDER_MIXED;
  c->enable_anti_grazing = 0;
  c->start_voxel_subsampling_factor = 2.0f;
  c->max_consecutive_ray_collisions = 2;
  c->clear_checks_every_n_frames = 1;
  c->integrator_threads = 1;
  c->num_labels = num_labels;
  c->semantic_measurement_probability = 0.9f;  // base.h:77
  c->color_mode = KSG_COLOR_MODE_SEMANTIC;     // base.h:80
  for (int l = 0; l < 256; ++l) {
    c->label_color[l][0] = 127; c->label_color[l][1] = 127; c->label_color[l][2] = 127; c->label_color[l][3] = 255;
    c->label_color_known[l] = 1;
    c->dynamic_label[l] = 0;
  }
  c->device = 0;
  c->max_blocks = 8192;
  c->max_points = 640 * 480;
  c->max_ray_steps = 0;
  c->max_updates = 0;
  c->apply_mode = 0;
  c->shard_rank = 0;
  c->shard_count = 1;
  c->merged_bundle_order = KSG_BUNDLE_ORDER_LIBSTDCXX;   // the reference's unordered_map iteration order (merged.cpp:210-231)
  c->hot_voxel_mode = 0;   // opt-in (slower than the per-voxel kernels alone on merged2)
}

#define KSG_STR_(x) #x
#define KSG_STR(x) KSG_STR_(x)
const char* ksg_build_info(void) { return "ksg abi " KSG_STR(KSG_ABI_VERSION) " sm_90a nvcc " KSG_STR(__CUDACC_VER_MAJOR__) "." KSG_STR(__CUDACC_VER_MINOR__) " built " __DATE__; }

const char* ksg_last_error(const ksg_integrator* h) { return h ? h->err.c_str() : g_last_error.c_str(); }

int32_t ksg_create(const ksg_config* cfg, ksg_integrator** out) {
  if (!out) return KSG_ERR_INVALID_ARGUMENT;
  *out = nullptr;
  std::string why;
  int rc = validate(cfg, why);
  if (rc) { g_last_error = why; return rc; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || cfg->device >= ndev) {
    g_last_error = "no CUDA device (the integrator has no CPU fallback)";
    cudaGetLastError();
    return KSG_ERR_NO_DEVICE;
  }
  const Knobs knobs = read_knobs();
  std::unique_ptr<ksg_integrator> owner(new ksg_integrator());   // every early return below releases what was made so far
  ksg_integrator* h = owner.get();
  Resources& res = h->res;
  h->cfg = *cfg;
  h->device = cfg->device;
  KSG_CUDA(cudaSetDevice(h->device));
  cudaDeviceProp prop;
  KSG_CUDA(cudaGetDeviceProperties(&prop, h->device));
  h->sm_count = prop.multiProcessorCount;
  KSG_CUDA(res.stream(&h->own_stream));

  // ---- geometry (voxblox Layer: inverses are 1.0 / x in double, stored as float; A.1, base.cpp:84-89)
  DevCfg& dc = h->dc;
  dc.voxel_size = cfg->voxel_size;
  dc.vsi = (float)(1.0 / cfg->voxel_size);
  dc.vps = cfg->voxels_per_side;
  dc.vps_inv = (float)(1.0f / (float)cfg->voxels_per_side);
  dc.tile_side = std::min(cfg->voxels_per_side, kTileSideMax);
  dc.tile_side_log2 = ilog2(dc.tile_side);
  dc.tiles_per_side = dc.vps / dc.tile_side;
  dc.tiles_per_block = dc.tiles_per_side * dc.tiles_per_side * dc.tiles_per_side;
  dc.tile_voxels = dc.tile_side * dc.tile_side * dc.tile_side;
  dc.plane_f32 = round_up(4u * dc.tile_voxels, 16);
  dc.plane_u8 = round_up((uint32_t)dc.tile_voxels, 16);
  dc.head_bytes = 4 * dc.plane_f32 + dc.plane_u8;
  dc.C = cfg->num_labels;
  dc.prior_bytes = round_up(4u * (uint32_t)dc.tile_voxels * (uint32_t)dc.C, 16);
  dc.tile_stride = round_up(dc.head_bytes + dc.prior_bytes, 128);
  dc.full_stage = (dc.head_bytes + dc.prior_bytes + 8u * dc.tile_voxels + 64u) <= 72u * 1024u ? 1 : 0;
  dc.block_stride = (uint64_t)dc.tile_stride * dc.tiles_per_block;
  dc.tp.voxel_size = cfg->voxel_size;
  dc.tp.trunc = cfg->default_truncation_distance;
  dc.tp.max_weight = cfg->max_weight;
  dc.tp.sparsity_factor = cfg->sparsity_compensation_factor;
  dc.tp.use_weight_dropoff = cfg->use_weight_dropoff;
  dc.tp.use_sparsity = cfg->use_sparsity_compensation_factor;
  dc.min_ray = cfg->min_ray_length_m;
  dc.max_ray = cfg->max_ray_length_m;
  dc.start_inv = cfg->start_voxel_subsampling_factor * dc.vsi;  // fast.cpp:89
  dc.carving = cfg->voxel_carving_enabled;
  dc.const_weight = cfg->use_const_weight;
  // voxblox TsdfIntegratorBase ctor: clearing rays have no use without carving, so allow_clear is forced off there
  // (explicit freespace clouds still clear, isPointValid tests allow_clear || freespace_points)
  dc.allow_clear = (cfg->allow_clear && cfg->voxel_carving_enabled) ? 1 : 0;
  dc.maxc = cfg->max_consecutive_ray_collisions;
  dc.anti_grazing = cfg->enable_anti_grazing;
  // setSemanticProbabilities (base.cpp:93-128): std::log on float, on the host (same libm as the reference)
  dc.lm = std::log(cfg->semantic_measurement_probability);
  dc.ln = std::log(1.0f - cfg->semantic_measurement_probability);
  dc.color_mode = cfg->color_mode;
  dc.type = cfg->integrator_type;
  dc.shard_rank = cfg->shard_rank;
  dc.shard_count = cfg->shard_count > 1 ? cfg->shard_count : 1;

  // ---- look-up tables
  for (int l = 0; l < 256; ++l) {
    const uint8_t* c = cfg->label_color[l];
    h->h_luts.label_rgba[l] = cfg->label_color_known[l] ? ((uint32_t)c[0] | ((uint32_t)c[1] << 8) | ((uint32_t)c[2] << 16) | ((uint32_t)c[3] << 24)) : 0u;
    h->h_luts.dynamic_label[l] = cfg->dynamic_label[l];
  }
  for (int i = 0; i < 1024; ++i) { h->h_luts.c2l_keys[i] = 0xFFFFFFFFu; h->h_luts.c2l_vals[i] = 0; }
  KSG_CUDA(res.device(&h->d_luts, 1));
  KSG_CUDA(cudaMemcpy(h->d_luts, &h->h_luts, sizeof(Luts), cudaMemcpyHostToDevice));

  // ---- map
  h->ht_cap = 1024;
  while (h->ht_cap < 2u * (uint32_t)cfg->max_blocks) h->ht_cap <<= 1;
  if ((unsigned long long)h->ht_cap * dc.tiles_per_block >= (1ull << 32)) return h->fail(KSG_ERR_INVALID_ARGUMENT, "max_blocks too large");
  h->map.ht_mask = h->ht_cap - 1;
  h->map.max_blocks = cfg->max_blocks;
  h->map.new_cap = cfg->max_blocks;
  KSG_CUDA(res.device(&h->map.ht_keys, h->ht_cap));
  KSG_CUDA(res.device(&h->map.ht_slot, h->ht_cap));
  KSG_CUDA(res.device(&h->map.touched_stamp, h->ht_cap));
  KSG_CUDA(res.device(&h->map.touched_list, h->ht_cap));
  KSG_CUDA(res.device(&h->map.new_list, (size_t)cfg->max_blocks));
  KSG_CUDA(res.device(&h->map.slot_key, (size_t)cfg->max_blocks));
  KSG_CUDA(res.device(&h->map.pool, (size_t)dc.block_stride * (size_t)cfg->max_blocks));
  KSG_CUDA(res.device(&h->d_cnt, 1));
  KSG_CUDA(res.pinned(&h->h_cnt_base, 2));
  std::memset(h->h_cnt_base, 0, 2 * sizeof(Counters));
  h->h_cnt = h->h_cnt_base;
  for (int i = 0; i < 2; ++i) {
    KSG_CUDA(res.event(&h->ev_frame_s[i], cudaEventDisableTiming));
    KSG_CUDA(res.event(&h->ev_copy[i], cudaEventDisableTiming));
    KSG_CUDA(res.event(&h->ev_free[i], cudaEventDisableTiming));
  }
  KSG_CUDA(res.stream(&h->copy_stream));

  // ---- frame scratch
  const size_t N = (size_t)cfg->max_points;
  h->cap_points = cfg->max_points;
  const bool fast = cfg->integrator_type == KSG_INTEGRATOR_FAST;
  if (!fast) {   // merged's per-point state (fast keeps only the start-set key and the pixel per input index)
    KSG_CUDA(res.device(&h->pt_pC, N)); KSG_CUDA(res.device(&h->pt_pG, N));
    KSG_CUDA(res.device(&h->pt_label, N)); KSG_CUDA(res.device(&h->pt_flags, N));
    KSG_CUDA(res.device(&h->pt_color, N));
  }
  KSG_CUDA(res.device(&h->pt_key, N));
  KSG_CUDA(res.device(&h->flags8, 2 * N));
  KSG_CUDA(res.device(&h->pix_list, N));
  KSG_CUDA(res.device(&h->iota, N));
  k_iota<<<grid_for((long long)N, 256), 256>>>(h->iota, (int)N);
  if (cfg->integration_order_mode == KSG_ORDER_SORTED) {
    KSG_CUDA(res.device(&h->point_of_seq, N)); KSG_CUDA(res.device(&h->sq_keys, N)); KSG_CUDA(res.device(&h->sq_keys_out, N));
  }
  KSG_CUDA(res.device(&h->ray_param, N)); KSG_CUDA(res.device(&h->ray_flags, N)); KSG_CUDA(res.device(&h->nsteps, N));
  long long rec_cap = cfg->max_updates > 0 ? cfg->max_updates : (fast ? std::max<long long>(4ll << 20, 64ll * (long long)N) : (64ll << 20));
  if (fast) {
    KSG_CUDA(res.device(&h->start_rec, kSetSize)); KSG_CUDA(res.device(&h->start_table, kSetSize));
    KSG_CUDA(res.device(&h->start_touched, N));
    KSG_CUDA(res.device(&h->o3.head, kSetSize)); KSG_CUDA(res.device(&h->o3.slot_cnt, kSetSize));   // cleared per frame
    KSG_CUDA(res.device(&h->cast_seq, N));
    KSG_CUDA(res.device(&h->ray_label, N)); KSG_CUDA(res.device(&h->ray_color, N));
    KSG_CUDA(res.device(&h->ray_state, N)); KSG_CUDA(res.device(&h->ext_off, N * kExtSegs));
    long long ext = cfg->max_ray_steps > 0 ? cfg->max_ray_steps : std::max<long long>(16ll << 20, 64ll * (long long)N);
    Obs3& o3 = h->o3;
    o3.ext_base = (long long)N * kH0;
    o3.cand_cap = o3.ext_base + ext;
    if (o3.cand_cap >= 0x7FFFFFFFll) { o3.cand_cap = 0x7FFFFFFEll; }
    KSG_CUDA(res.device(&o3.cand, (size_t)o3.cand_cap));
    o3.ovf_cap = (int)std::min<long long>(std::max<long long>(1ll << 20, 4ll * (long long)N), 1ll << 28);
    KSG_CUDA(res.device(&o3.ovf, (size_t)o3.ovf_cap));
    KSG_CUDA(res.device(&o3.bkt, (size_t)kSetSize * kBkt3));
    KSG_CUDA(res.device(&o3.stamp_max, 2 * (size_t)kSetSize)); o3.stamp_min = o3.stamp_max + kSetSize;
    KSG_CUDA(res.device(&o3.table, kSetSize));
    KSG_CUDA(res.device(&h->rayrec, N));
    KSG_CUDA(res.device(&h->wl, 3 * N));
    KSG_CUDA(res.device(&h->mixed_list, N)); KSG_CUDA(res.device(&h->m_list, N));
    KSG_CUDA(res.device(&h->blk_run, (size_t)(o3.cand_cap / 16 + 16)));
  } else {
    KSG_CUDA(res.device(&h->ks_sorted, N)); KSG_CUDA(res.device(&h->seq_sorted, N));
    KSG_CUDA(res.device(&h->bstart, 2 * N)); KSG_CUDA(res.device(&h->bundle_f, N));
    KSG_CUDA(res.device(&h->hist, N * dc.C)); KSG_CUDA(res.device(&h->tmp, (N + 1) * dc.C));  // + the all-zero row
    KSG_CUDA(res.device(&h->b_key, N)); KSG_CUDA(res.device(&h->b_base, N));
    KSG_CUDA(res.device(&h->d_scan_tot, 16));
    // per-voxel apply kernels (default); the tile kernel stays for apply_mode 1 and KSG_MERGED_TILE_APPLY=1
    h->voxel_apply = cfg->apply_mode == 0 && !knobs.tile_apply;
    if (h->voxel_apply) {
      h->vq.long_cap = 4 * (rec_cap / kLongLen) + 64;
      h->vq.long_len = kLongLen;
      if (dc.C <= 32) {   // one thread per short voxel (ksg_voxel.cuh)
        KSG_CUDA(res.device(&h->tmp4, (N + 1) * (size_t)((dc.C + 3) & ~3)));
        h->vq.long_len = knobs.long_len ? knobs.long_len : kLongLenThread;
      }
      h->vq.short_cap = rec_cap;
      KSG_CUDA(res.device(&h->vq.long_items, (size_t)h->vq.long_cap));
      KSG_CUDA(res.device(&h->vq.counters, 8));
      {   // the long-segment kernel must get its CTAs placed before the short-segment kernel fills the register files: its stream has priority
        int lo_p = 0, hi_p = 0;
        KSG_CUDA(cudaDeviceGetStreamPriorityRange(&lo_p, &hi_p));
        KSG_CUDA(res.stream(&h->aux_stream, hi_p));
      }
      KSG_CUDA(res.event(&h->ev_fork, cudaEventDisableTiming));
      KSG_CUDA(res.event(&h->ev_join, cudaEventDisableTiming));
      h->long_threads = knobs.long_threads;
      h->long_grid = knobs.long_grid ? knobs.long_grid : h->sm_count;
      h->deep_threads = knobs.deep_threads;
      h->short_t_ctas = knobs.short_t_ctas;
      h->short_ctas = knobs.short_ctas;
      if (h->short_ctas < 6) {
        h->short_smem = std::min(200 * 1024, (220 * 1024) / h->short_ctas - 2048);
        rc = for_each_nch([&](auto nch) -> int {
          KSG_CUDA(cudaFuncSetAttribute(k_voxel_apply_short<decltype(nch)::value>, cudaFuncAttributeMaxDynamicSharedMemorySize, h->short_smem));
          return KSG_OK;
        });
        if (rc) return rc;
      }
    }
    if (cfg->hot_voxel_mode >= 1 && dc.C <= 32 && cfg->apply_mode == 0) {
      h->hot_enabled = true;
      h->hot_chunk_cap = rec_cap / kHotChunk + kHotMaxSegs;
      KSG_CUDA(res.device(&h->d_hot_segs, kHotMaxSegs)); KSG_CUDA(res.device(&h->d_hot_counts, 2));
      KSG_CUDA(cudaMemset(h->d_hot_counts, 0, 2 * sizeof(int)));
      KSG_CUDA(res.pinned(&h->h_hot_segs, kHotMaxSegs));
      KSG_CUDA(res.pinned(&h->h_hot_chunk_seg, (size_t)h->hot_chunk_cap));
      KSG_CUDA(res.device(&h->d_hot_chunk_seg, (size_t)h->hot_chunk_cap)); KSG_CUDA(res.device(&h->d_hot_guess, (size_t)h->hot_chunk_cap * 32));
      KSG_CUDA(res.device(&h->d_hot_sums, (size_t)h->hot_chunk_cap * 32)); KSG_CUDA(res.device(&h->d_hot_tables, (size_t)h->hot_chunk_cap * 32));
      KSG_CUDA(res.device(&h->d_hot_prior, (size_t)kHotMaxSegs * 32)); KSG_CUDA(res.device(&h->d_hot_same, (size_t)kHotMaxSegs));
      KSG_CUDA(cudaFuncSetAttribute(k_hot_chunk_tables, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(float) * 32 * kHotColStride)));
    }
    if (cfg->merged_bundle_order == KSG_BUNDLE_ORDER_LIBSTDCXX) {
      // rehash schedule of the platform's libstdc++ (depends on the size only): probe a real container once
      std::unordered_map<uint64_t, char> probe;
      size_t last = 0;
      for (size_t i = 0; i < N; ++i) {
        probe.emplace((uint64_t)i, 0);
        if (probe.bucket_count() != last) { last = probe.bucket_count(); h->bord_phases.push_back(std::make_pair((int)i, (uint32_t)last)); }
      }
      if (last >= 0x7fffffffull) return h->fail(KSG_ERR_INVALID_ARGUMENT, "max_points too large for merged_bundle_order");
      KSG_CUDA(res.device(&h->bord_hash, N)); KSG_CUDA(res.device(&h->bundle_f2, N));
      {   // scratch of k_bundle_order: [ord_a | ord_b | next | size_at | rank : N each][first | head : 2 * last each][cta_tot][phase tables]
        const size_t np = h->bord_phases.size();
        const size_t ints = 5 * N + 4 * last + 2 * kBordCluster + 2 * np + 64;
        KSG_CUDA(res.device(&h->bord_scratch, ints));
        int* p = h->bord_scratch;
        BordBuf& bb = h->bord;
        bb.hash = h->bord_hash;
        bb.ord_a = p; p += N; bb.ord_b = p; p += N; bb.next = p; p += N; bb.size_at = p; p += N; bb.rank = p; p += N;
        bb.first = p; p += 2 * last; bb.head = p; p += 2 * last; bb.cta_tot = p; p += 2 * kBordCluster;
        bb.bucket_cap = (uint32_t)last;
        bb.n_phases = (int)np;
        std::vector<int> ps(np); std::vector<uint32_t> pb(np);
        for (size_t i = 0; i < np; ++i) { ps[i] = h->bord_phases[i].first; pb[i] = h->bord_phases[i].second; }
        KSG_CUDA(cudaMemcpy(p, ps.data(), sizeof(int) * np, cudaMemcpyHostToDevice)); bb.phase_start = p; p += np;
        KSG_CUDA(cudaMemcpy(p, pb.data(), sizeof(uint32_t) * np, cudaMemcpyHostToDevice)); bb.phase_buckets = (const uint32_t*)p;
      }
    }
  }
  h->rec_cap = rec_cap;
  if (!fast) {     // merged's 64-bit records (fast keeps 32-bit keys in per-tile segments and its work items instead)
    KSG_CUDA(res.device(&h->rec_a, (size_t)rec_cap)); KSG_CUDA(res.device(&h->rec_b, (size_t)rec_cap));
    h->vq.short_items = (unsigned long long*)h->rec_a;   // the unsorted record buffer is free once the sort has run
  }
  h->tile_cap = (long long)std::min<unsigned long long>((unsigned long long)cfg->max_blocks * dc.tiles_per_block, (unsigned long long)rec_cap);
  KSG_CUDA(res.device(&h->tile_begin, (size_t)h->tile_cap));

  // ---- CUB temp storage: the largest of every call made per frame
  {
    size_t need = 0, t = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, t, h->rec_a, h->rec_b, rec_cap, 0, 64); need = std::max(need, t);
    cub::DeviceRadixSort::SortPairs(nullptr, t, h->pt_key, h->pt_key, h->iota, h->iota, (int)N, 0, 64); need = std::max(need, t);
    cub::DeviceRadixSort::SortPairs(nullptr, t, h->iota, h->iota, h->iota, h->iota, (int)N, 0, 32); need = std::max(need, t);
    cub::DeviceSelect::Flagged(nullptr, t, cub::CountingInputIterator<int>(0), h->flags8, h->pix_list, (int*)nullptr, (int)(2 * N));
    need = std::max(need, t);
    KSG_CUDA(res.regrow(&h->cub_temp, &h->cub_temp_bytes, need + 256));
  }

  // ---- tile-apply launch configuration
  {
    const int V = dc.tile_voxels;
    const size_t stage = dc.head_bytes + (dc.full_stage ? dc.prior_bytes : 0u);
    h->apply_smem = (int)(stage + (size_t)V * 8 + 64);
    h->apply_nch = dc.C <= 32 ? 1 : (dc.C <= 64 ? 2 : (dc.C <= 128 ? 4 : 8));
    h->use_tma = cfg->apply_mode == 0;
    KSG_CUDA(cudaFuncSetAttribute(k_tile_apply<true, 1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, h->apply_smem));
    rc = for_each_tma_nch([&](auto tma, auto nch) -> int {
      KSG_CUDA(cudaFuncSetAttribute(k_tile_apply<decltype(tma)::value, decltype(nch)::value>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    h->apply_smem));
      return KSG_OK;
    });
    if (rc) return rc;
  }
  if (fast) {
    // frame driver (ksg_fast.cuh)
    KSG_CUDA(res.device(&h->d_fc, 1));
    KSG_CUDA(cudaMemset(h->d_fc, 0, sizeof(FastCounters)));
    KSG_CUDA(res.pinned(&h->h_fc_base, 2));
    std::memset(h->h_fc_base, 0, 2 * sizeof(FastCounters));
    h->h_fc = h->h_fc_base;
    KSG_CUDA(res.device(&h->blk_cnt, N / kCountBlock + 2)); KSG_CUDA(res.device(&h->blk_off, N / kCountBlock + 2));
    KSG_CUDA(res.device(&h->cast_bits, N / 32 + 64)); KSG_CUDA(res.device(&h->warp_off, N / 32 + 64));
    if (cfg->integration_order_mode == KSG_ORDER_SORTED) KSG_CUDA(res.device(&h->seq_of_i, N));
    KSG_CUDA(res.device(&h->keys32, (size_t)rec_cap));
    const size_t n_tk = (size_t)h->ht_cap * dc.tiles_per_block;
    KSG_CUDA(res.device(&h->tile_cnt, n_tk)); KSG_CUDA(res.device(&h->tile_slot, n_tk));
    KSG_CUDA(cudaMemset(h->tile_cnt, 0, sizeof(int) * n_tk));
    KSG_CUDA(res.device(&h->tile_list, (size_t)h->tile_cap));
    {
      int per_sm = 0;
      h->solve_threads = knobs.solve_threads;
      h->solve_smem = (int)(sizeof(int) * kSortPerWarp * (h->solve_threads / 32));
      KSG_CUDA(cudaFuncSetAttribute(k_fast_solve3, cudaFuncAttributeMaxDynamicSharedMemorySize, h->solve_smem));
      KSG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_fast_solve3, h->solve_threads, (size_t)h->solve_smem));
      int coop = 0;
      cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, h->device);
      // k_fast_solve3 is a cooperative launch with every CTA resident (grid barriers between its phases)
      if (!coop || per_sm <= 0) return h->fail(KSG_ERR_NO_DEVICE, "this device cannot run the fast integrator's observed-set solver "
                                                                   "(k_fast_solve3 needs a cooperative launch with at least one CTA per SM)");
      h->solve_grid = h->sm_count * std::max(1, std::min(per_sm, knobs.solve_ctas_per_sm));
      h->profile_marks_only = knobs.profile_marks_only;
      int khz = 0;
      if (cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, h->device) == cudaSuccess && khz > 0) h->clock_khz = khz;
    }
    {
      // voxel update: k_fast_group sorts each touched tile's keys and lists its voxels as work items, k_fast_apply takes them a warp
      // each.  A frame's items number at most its records and at most 512 per tile.
      KSG_CUDA(res.device(&h->fast_tiles, (size_t)h->tile_cap));
      h->item_cap = (int)std::min<long long>({rec_cap, h->tile_cap * dc.tile_voxels, (long long)INT_MAX});
      KSG_CUDA(res.device(&h->fast_items, (size_t)h->item_cap));
      int per_sm = 0;
      KSG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_fast_group, kGroupThreads, 0));
      h->group_grid = h->sm_count * std::max(1, per_sm);
      rc = with_nch(h->apply_nch, [&](auto nch) -> int {
        KSG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_fast_apply<decltype(nch)::value>, kFastApplyThreads, 0));
        return KSG_OK;
      });
      if (rc) return rc;
      h->fast_apply_grid = h->sm_count * std::max(1, per_sm);
    }
  }
  KSG_CUDA(cudaDeviceSynchronize());
  rc = reset_map(h, h->own_stream);
  if (rc) return rc;
  *out = owner.release();
  return KSG_OK;
}

void ksg_destroy(ksg_integrator* h) { delete h; }

int32_t ksg_set_color_to_label(ksg_integrator* h, const uint8_t* rgb, const uint8_t* labels, int32_t n) {
  if (!h || n < 0 || n > 512 || (n > 0 && (!rgb || !labels))) return KSG_ERR_INVALID_ARGUMENT;
  for (int i = 0; i < 1024; ++i) { h->h_luts.c2l_keys[i] = 0xFFFFFFFFu; h->h_luts.c2l_vals[i] = 0; }
  for (int i = 0; i < n; ++i) {
    const uint32_t key = (uint32_t)rgb[3 * i] | ((uint32_t)rgb[3 * i + 1] << 8) | ((uint32_t)rgb[3 * i + 2] << 16);
    uint32_t p = color_home_slot(key);
    while (h->h_luts.c2l_keys[p] != 0xFFFFFFFFu && h->h_luts.c2l_keys[p] != key) p = (p + 1) & 1023;
    h->h_luts.c2l_keys[p] = key;
    h->h_luts.c2l_vals[p] = labels[i];  // later rows overwrite earlier ones (color.cpp:58-59)
  }
  KSG_CUDA(cudaSetDevice(h->device));
  KSG_CUDA(cudaMemcpy(h->d_luts, &h->h_luts, sizeof(Luts), cudaMemcpyHostToDevice));
  return KSG_OK;
}

int32_t ksg_integrate_points_device(ksg_integrator* h, const float* T, const float* d_xyz, const uint8_t* d_rgba,
                                    const uint8_t* d_labels, int64_t n, int32_t freespace, void* stream, ksg_frame_stats* stats) {
  if (!h || !T || n < 0 || (n > 0 && !d_xyz)) return KSG_ERR_INVALID_ARGUMENT;
  { const int rc = check_frame(h, n, d_rgba && d_labels); if (rc) return rc; }
  InputDesc in; in.d_xyz = d_xyz; in.d_rgba = d_rgba; in.d_labels = d_labels; in.n = n; in.freespace = freespace;
  return integrate(h, in, T, stream ? (cudaStream_t)stream : h->own_stream, stats);
}

int32_t ksg_integrate_depth_device_k64(ksg_integrator* h, const float* T, const float* d_depth, const uint8_t* d_label, int32_t width,
                                       int32_t height, const double* K, void* stream, ksg_frame_stats* stats) {
  if (!h || !T || !K || width <= 0 || height <= 0 || !d_depth || !d_label) return KSG_ERR_INVALID_ARGUMENT;
  { const int rc = check_frame(h, (int64_t)width * height, false); if (rc) return rc; }
  InputDesc in; in.d_depth = d_depth; in.d_label_img = d_label; in.width = width; in.height = height;
  in.n = (int64_t)width * height; std::memcpy(in.K, K, sizeof(in.K));
  return integrate(h, in, T, stream ? (cudaStream_t)stream : h->own_stream, stats);
}
int32_t ksg_integrate_depth_device(ksg_integrator* h, const float* T, const float* d_depth, const uint8_t* d_label, int32_t width,
                                   int32_t height, const float* K, void* stream, ksg_frame_stats* stats) {
  if (!K) return KSG_ERR_INVALID_ARGUMENT;
  const double K64[4] = {K[0], K[1], K[2], K[3]};   // exact widening: same results as before for float intrinsics
  return ksg_integrate_depth_device_k64(h, T, d_depth, d_label, width, height, K64, stream, stats);
}

int32_t ksg_integrate_points(ksg_integrator* h, const float* T, const float* xyz, const uint8_t* rgba, const uint8_t* labels,
                             int64_t n, int32_t freespace, ksg_frame_stats* stats) {
  if (!h || !T || n < 0 || (n > 0 && !xyz)) return KSG_ERR_INVALID_ARGUMENT;
  int rc = check_frame(h, n, rgba && labels);
  if (rc) return rc;
  KSG_CUDA(cudaSetDevice(h->device));
  const size_t b[3] = {(size_t)n * 12, rgba ? (size_t)n * 4 : 0, labels ? (size_t)n : 0};   // xyz | rgba | labels
  size_t o[3];
  const size_t total = frame_slices(b, o);
  rc = ensure_input(h, total);
  if (rc) return rc;
  if (n > 0) {
    std::memcpy(h->h_stage, xyz, b[0]);
    if (rgba) std::memcpy(h->h_stage + o[1], rgba, b[1]);
    if (labels) std::memcpy(h->h_stage + o[2], labels, b[2]);
    KSG_CUDA(cudaMemcpyAsync(h->d_in, h->h_stage, total, cudaMemcpyHostToDevice, h->own_stream));
  }
  InputDesc in; in.d_xyz = (const float*)h->d_in; in.d_rgba = rgba ? h->d_in + o[1] : nullptr;
  in.d_labels = labels ? h->d_in + o[2] : nullptr; in.n = n; in.freespace = freespace;
  ksg_frame_stats local;
  return integrate(h, in, T, h->own_stream, stats ? stats : &local);
}

int32_t ksg_integrate_depth_k64(ksg_integrator* h, const float* T, const float* depth, const uint8_t* label, int32_t width,
                                int32_t height, const double* K, ksg_frame_stats* stats) {
  if (!h || !T || !K || width <= 0 || height <= 0 || !depth || !label) return KSG_ERR_INVALID_ARGUMENT;
  const size_t P = (size_t)width * height;
  int rc = check_frame(h, (int64_t)P, false);
  if (rc) return rc;
  KSG_CUDA(cudaSetDevice(h->device));
  const size_t b[2] = {P * 4, P};   // depth | labels
  size_t o[2];
  const size_t total = frame_slices(b, o);
  rc = ensure_input(h, total);
  if (rc) return rc;
  if (is_pinned_host(depth) && is_pinned_host(label)) {   // caller's buffers are page-locked: copy straight from them
    KSG_CUDA(cudaMemcpyAsync(h->d_in, depth, b[0], cudaMemcpyHostToDevice, h->own_stream));
    KSG_CUDA(cudaMemcpyAsync(h->d_in + o[1], label, b[1], cudaMemcpyHostToDevice, h->own_stream));
  } else {
    std::memcpy(h->h_stage, depth, b[0]);
    std::memcpy(h->h_stage + o[1], label, b[1]);
    KSG_CUDA(cudaMemcpyAsync(h->d_in, h->h_stage, total, cudaMemcpyHostToDevice, h->own_stream));
  }
  InputDesc in; in.d_depth = (const float*)h->d_in; in.d_label_img = h->d_in + o[1]; in.width = width; in.height = height;
  in.n = (int64_t)P; std::memcpy(in.K, K, sizeof(in.K));
  ksg_frame_stats local;
  return integrate(h, in, T, h->own_stream, stats ? stats : &local);
}

int32_t ksg_integrate_image(ksg_integrator* h, const float* T, const void* depth, int32_t depth_type, const void* semantic, int32_t semantic_type,
                            int32_t width, int32_t height, const double* K, ksg_frame_stats* stats) {
  if (!h || !T || !K || width <= 0 || height <= 0 || !depth || !semantic) return KSG_ERR_INVALID_ARGUMENT;
  if (depth_type != KSG_DEPTH_F32_METRES && depth_type != KSG_DEPTH_U16_MILLIMETRES) return KSG_ERR_INVALID_ARGUMENT;
  if (semantic_type != KSG_SEMANTIC_LABEL_U8 && semantic_type != KSG_SEMANTIC_RGB8) return KSG_ERR_INVALID_ARGUMENT;
  const size_t P = (size_t)width * height;
  int rc = check_frame(h, (int64_t)P, false);
  if (rc) return rc;
  KSG_CUDA(cudaSetDevice(h->device));
  const size_t b[5] = {P * (depth_type == KSG_DEPTH_U16_MILLIMETRES ? 2 : 4), P * (semantic_type == KSG_SEMANTIC_RGB8 ? 3 : 1), P * 4, P, P * 4};
  size_t o[5];   // raw depth | raw semantic | float depth | label | colour
  rc = ensure_input(h, frame_slices(b, o));
  if (rc) return rc;
  std::memcpy(h->h_stage, depth, b[0]);
  std::memcpy(h->h_stage + o[1], semantic, b[1]);
  cudaStream_t s = h->own_stream;
  KSG_CUDA(cudaMemcpyAsync(h->d_in, h->h_stage, o[1] + b[1], cudaMemcpyHostToDevice, s));
  InputDesc in;
  in.width = width; in.height = height; in.n = (int64_t)P;
  std::memcpy(in.K, K, sizeof(in.K));
  if (depth_type == KSG_DEPTH_U16_MILLIMETRES) {
    ++h->n_launches;
    k_u16_to_f32<<<grid_for((long long)P, 256), 256, 0, s>>>((const uint16_t*)h->d_in, (int)P, (float*)(h->d_in + o[2]));
    in.d_depth = (const float*)(h->d_in + o[2]);
    in.unit_scaling = (double)0.001f;          // double unit_scaling = DepthTraits<uint16_t>::toMeters(1) = 1 * 0.001f
    in.z_scale = 0.001f;
  } else in.d_depth = (const float*)h->d_in;
  if (semantic_type == KSG_SEMANTIC_RGB8) {
    ++h->n_launches;
    k_rgb_to_label<<<grid_for((long long)P, 256), 256, 0, s>>>(h->d_in + o[1], (int)P, h->d_luts, h->d_in + o[3], (uint32_t*)(h->d_in + o[4]));
    in.d_label_img = h->d_in + o[3];
    in.d_color_img = (const uint32_t*)(h->d_in + o[4]);
  } else in.d_label_img = h->d_in + o[1];
  ksg_frame_stats local;
  return integrate(h, in, T, s, stats ? stats : &local);
}

int32_t ksg_integrate_depth(ksg_integrator* h, const float* T, const float* depth, const uint8_t* label, int32_t width,
                            int32_t height, const float* K, ksg_frame_stats* stats) {
  if (!K) return KSG_ERR_INVALID_ARGUMENT;
  const double K64[4] = {K[0], K[1], K[2], K[3]};
  return ksg_integrate_depth_k64(h, T, depth, label, width, height, K64, stats);
}

// Pipelined host-buffer entry: the H2D copy of this frame runs on a copy stream into one of two device staging buffers, so it
// overlaps the kernels of the previous frame; the frame's kernels wait for the copy with an event.  Returns without waiting.
int32_t ksg_integrate_depth_async(ksg_integrator* h, const float* T, const float* depth, const uint8_t* label, int32_t width,
                                  int32_t height, const float* K) {
  if (!h || !T || !K || width <= 0 || height <= 0 || !depth || !label) return KSG_ERR_INVALID_ARGUMENT;
  const size_t P = (size_t)width * height;
  { const int rc = check_frame(h, (int64_t)P, false); if (rc) return rc; }
  KSG_CUDA(cudaSetDevice(h->device));
  const size_t b[2] = {P * 4, P};   // depth | labels
  size_t o[2];
  const size_t total = frame_slices(b, o);
  const int slot = h->in_slot;
  h->in_slot ^= 1;
  if (total > h->in2_bytes[slot]) {
    if (h->in2_used[slot]) KSG_CUDA(cudaEventSynchronize(h->ev_free[slot]));
    h->res.release(h->h_stage2[slot]);   // both buffers of the slot go before either is replaced
    h->h_stage2[slot] = nullptr;
    KSG_CUDA(h->res.regrow(&h->d_in2[slot], &h->in2_bytes[slot], total));
    KSG_CUDA(h->res.regrow_pinned(&h->h_stage2[slot], &h->in2_bytes[slot], total));
  }
  // the slot's previous frame must have consumed the device buffer before it is overwritten
  if (h->in2_used[slot]) KSG_CUDA(cudaStreamWaitEvent(h->copy_stream, h->ev_free[slot], 0));
  if (is_pinned_host(depth) && is_pinned_host(label)) {   // page-locked caller buffers: read asynchronously (keep them unchanged until ksg_wait_frame)
    KSG_CUDA(cudaMemcpyAsync(h->d_in2[slot], depth, b[0], cudaMemcpyHostToDevice, h->copy_stream));
    KSG_CUDA(cudaMemcpyAsync(h->d_in2[slot] + o[1], label, b[1], cudaMemcpyHostToDevice, h->copy_stream));
  } else {
    if (h->in2_used[slot]) KSG_CUDA(cudaEventSynchronize(h->ev_copy[slot]));   // the staging buffer's previous copy has left the host
    std::memcpy(h->h_stage2[slot], depth, b[0]);
    std::memcpy(h->h_stage2[slot] + o[1], label, b[1]);
    KSG_CUDA(cudaMemcpyAsync(h->d_in2[slot], h->h_stage2[slot], total, cudaMemcpyHostToDevice, h->copy_stream));
  }
  KSG_CUDA(cudaEventRecord(h->ev_copy[slot], h->copy_stream));
  KSG_CUDA(cudaStreamWaitEvent(h->own_stream, h->ev_copy[slot], 0));
  InputDesc in; in.d_depth = (const float*)h->d_in2[slot]; in.d_label_img = h->d_in2[slot] + o[1]; in.width = width; in.height = height;
  in.n = (int64_t)P;
  in.K[0] = K[0]; in.K[1] = K[1]; in.K[2] = K[2]; in.K[3] = K[3];
  const bool deferred = h->cfg.integrator_type == KSG_INTEGRATOR_FAST;
  ksg_frame_stats st;
  const int rc = integrate(h, in, T, h->own_stream, deferred ? nullptr : &st);
  KSG_CUDA(cudaEventRecord(h->ev_free[slot], h->own_stream));
  h->in2_used[slot] = true;
  if (!deferred && h->n_stash < 4) h->stash[h->n_stash++] = st;   // drivers that complete inside the call: statistics are ready
  return rc;
}

// Completes the oldest frame submitted with ksg_integrate_depth_async and returns its statistics.
int32_t ksg_wait_frame(ksg_integrator* h, ksg_frame_stats* stats) {
  if (!h) return KSG_ERR_INVALID_ARGUMENT;
  cudaSetDevice(h->device);
  if (h->n_stash > 0) {
    if (stats) *stats = h->stash[0];
    for (int i = 1; i < h->n_stash; ++i) h->stash[i - 1] = h->stash[i];
    --h->n_stash;
    if (h->deferred_status) return h->fail(h->deferred_status, err_text(h->deferred_status));
    return KSG_OK;
  }
  if (h->n_pend > 0) return finish_oldest(h, stats);
  if (stats) fill_stats(h, stats);
  return h->deferred_status ? h->fail(h->deferred_status, err_text(h->deferred_status)) : KSG_OK;
}

namespace {
// entries of the last frame's update log: `fast` counts them in its frame counters, `merged` keeps the count of its last integrate call
int64_t update_log_count(const ksg_integrator* h) {
  if (h->cfg.integrator_type == KSG_INTEGRATOR_MERGED) return h->merged_log_count;
  return h->h_fc ? h->h_fc->log_count : 0;
}
}  // namespace

int32_t ksg_set_update_log(ksg_integrator* h, int64_t capacity_voxels) {
  if (!h || capacity_voxels < 0 || capacity_voxels > (1ll << 30)) return KSG_ERR_INVALID_ARGUMENT;
  { const int rcp = complete_frames(h); if (rcp) return rcp; }
  for (void* p : {(void*)h->d_log_head, (void*)h->d_log_prior, (void*)h->h_log_head, (void*)h->h_log_prior}) h->res.release(p);
  h->d_log_head = nullptr; h->d_log_prior = nullptr; h->h_log_head = nullptr; h->h_log_prior = nullptr; h->log_cap = 0;
  h->merged_log_count = 0;
  if (capacity_voxels == 0) return KSG_OK;
  if (h->cfg.integrator_type == KSG_INTEGRATOR_MERGED) {
    // the merged log pass compacts the segment heads of up to rec_cap records in the unsorted record buffer (ksg_log.cuh)
    if (h->rec_cap > 0x7fffffffll) return h->fail(KSG_ERR_INVALID_ARGUMENT, "update log: max_updates must be below 2^31 for the merged integrator");
    size_t t = 0, t2 = 0;
    KSG_CUDA(cub::DeviceSelect::Flagged(nullptr, t, cub::CountingInputIterator<int>(0), (uint8_t*)nullptr, (int*)nullptr, (int*)nullptr,
                                        (int)h->rec_cap));
    cub::DoubleBuffer<uint64_t> kb(nullptr, nullptr);
    cub::DoubleBuffer<int> vb(nullptr, nullptr);
    KSG_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t2, kb, vb, (int)std::min<int64_t>(capacity_voxels, h->rec_cap), 0, 63));
    t = std::max(t, t2);
    if (t > h->cub_temp_bytes) KSG_CUDA(h->res.regrow(&h->cub_temp, &h->cub_temp_bytes, t + 256));
  }
  const size_t n = (size_t)capacity_voxels;
  KSG_CUDA(h->res.device(&h->d_log_head, n));
  KSG_CUDA(h->res.device(&h->d_log_prior, n * h->dc.C));
  KSG_CUDA(h->res.pinned(&h->h_log_head, n));
  KSG_CUDA(h->res.pinned(&h->h_log_prior, n * h->dc.C));
  h->log_cap = (int)capacity_voxels;
  return KSG_OK;
}

int32_t ksg_fetch_update_log(ksg_integrator* h, int64_t* n_out, const ksg_voxel_update** heads, const float** priors) {
  if (!h || !n_out) return KSG_ERR_INVALID_ARGUMENT;
  *n_out = 0;
  if (!h->d_log_head) return h->fail(KSG_ERR_INVALID_ARGUMENT, "update log is off (ksg_set_update_log)");
  KSG_CUDA(cudaSetDevice(h->device));
  { const int rcp = finish_frame(h, nullptr); if (rcp) return rcp; }
  const int64_t n = update_log_count(h);
  if (n > h->log_cap) { *n_out = -1; return h->fail(KSG_ERR_SCRATCH_FULL, "update log too small for this frame: fall back to ksg_last_updated_blocks / ksg_export_blocks_by_index"); }
  if (n > 0) {
    KSG_CUDA(cudaMemcpyAsync(h->h_log_head, h->d_log_head, (size_t)n * sizeof(VoxelUpdate), cudaMemcpyDeviceToHost, h->own_stream));
    KSG_CUDA(cudaMemcpyAsync(h->h_log_prior, h->d_log_prior, (size_t)n * sizeof(float) * h->dc.C, cudaMemcpyDeviceToHost, h->own_stream));
    KSG_CUDA(cudaStreamSynchronize(h->own_stream));
  }
  *n_out = n;
  if (heads) *heads = reinterpret_cast<const ksg_voxel_update*>(h->h_log_head);
  if (priors) *priors = h->h_log_prior;
  return KSG_OK;
}

int32_t ksg_evaluate_labels(ksg_integrator* h, const ksg_world_object* objects, int32_t n_objects, float max_dist, float band, float checker_size,
                            float checker_margin, int64_t* evaluated, int64_t* correct, int64_t* observed) {
  if (!h || n_objects < 0 || (n_objects > 0 && !objects) || n_objects > 4096) return KSG_ERR_INVALID_ARGUMENT;
  static_assert(sizeof(ksg_world_object) == sizeof(WorldObject), "ksg_world_object layout");
  { const int rcp = complete_frames(h); if (rcp) return rcp; }
  unsigned long long res[3] = {0, 0, 0};
  if (h->num_blocks > 0 && n_objects > 0) {
    Resources tmp;
    WorldObject* d_objs = nullptr;
    unsigned long long* d_out = nullptr;
    KSG_CUDA(tmp.device(&d_objs, (size_t)n_objects));
    KSG_CUDA(tmp.device(&d_out, 3));
    KSG_CUDA(cudaMemcpy(d_objs, objects, sizeof(WorldObject) * (size_t)n_objects, cudaMemcpyHostToDevice));
    KSG_CUDA(cudaMemset(d_out, 0, sizeof(res)));
    ++h->n_launches;
    k_eval_labels<<<h->sm_count * 4, 256, 0, h->own_stream>>>(h->dc, h->map, (int)h->num_blocks, d_objs, n_objects, max_dist, band, checker_size,
                                                              checker_margin, d_out);
    KSG_CUDA(cudaMemcpyAsync(res, d_out, sizeof(res), cudaMemcpyDeviceToHost, h->own_stream));
    KSG_CUDA(cudaStreamSynchronize(h->own_stream));
  }
  if (evaluated) *evaluated = (int64_t)res[0];
  if (correct) *correct = (int64_t)res[1];
  if (observed) *observed = (int64_t)res[2];
  return KSG_OK;
}

namespace {
// Host copy of the block hash table (ht_keys / ht_slot), probed exactly as the device probes it: linear probing from mix64(key).
struct HostBlockTable {
  std::vector<uint64_t> keys;
  std::vector<int> slot_of;
  uint32_t mask = 0;

  int load(ksg_integrator* h) {
    mask = h->map.ht_mask;
    keys.resize((size_t)h->ht_cap);
    slot_of.resize((size_t)h->ht_cap);
    KSG_CUDA(cudaMemcpy(keys.data(), h->map.ht_keys, sizeof(uint64_t) * h->ht_cap, cudaMemcpyDeviceToHost));
    KSG_CUDA(cudaMemcpy(slot_of.data(), h->map.ht_slot, sizeof(int) * h->ht_cap, cudaMemcpyDeviceToHost));
    return KSG_OK;
  }
  int store(ksg_integrator* h) const {
    KSG_CUDA(cudaMemcpy(h->map.ht_keys, keys.data(), sizeof(uint64_t) * h->ht_cap, cudaMemcpyHostToDevice));
    KSG_CUDA(cudaMemcpy(h->map.ht_slot, slot_of.data(), sizeof(int) * h->ht_cap, cudaMemcpyHostToDevice));
    return KSG_OK;
  }
  // The slot of `key`, or -1.
  int find(uint64_t key) const {
    const uint32_t pos = probe(key);
    return (pos != kNone && keys[pos] == key) ? slot_of[pos] : -1;
  }
  // The slot of `key`; an absent key takes slot *n_blocks, which then grows by one.  -1: the table or the pool is full.
  int find_or_insert(uint64_t key, int64_t* n_blocks, int64_t max_blocks) {
    const uint32_t pos = probe(key);
    if (pos == kNone) return -1;
    if (keys[pos] == key) return slot_of[pos];
    if (*n_blocks >= max_blocks) return -1;
    keys[pos] = key; slot_of[pos] = (int)*n_blocks;
    return (int)(*n_blocks)++;
  }

 private:
  static constexpr uint32_t kNone = 0xFFFFFFFFu;
  // where `key` is, or the empty entry that ends its probe sequence; kNone: every entry probed
  uint32_t probe(uint64_t key) const {
    uint32_t pos = mix64(key) & mask;
    for (uint32_t n = 0; n <= mask; ++n) {
      if (keys[pos] == key || keys[pos] == kEmptyKey) return pos;
      pos = (pos + 1) & mask;
    }
    return kNone;
  }
};

void put_block_index(int32_t* block_index, int64_t i, uint64_t key) {
  const I3 b = unpack_key(key);
  block_index[3 * i] = b.x; block_index[3 * i + 1] = b.y; block_index[3 * i + 2] = b.z;
}

// The indices of `keys` in (z, y, x) order of their blocks (keys are packed as z:y:x, biased: numeric order = (z, y, x)).
std::vector<int> zyx_order(const std::vector<uint64_t>& keys) {
  std::vector<int> order(keys.size());
  std::iota(order.begin(), order.end(), 0);
  std::sort(order.begin(), order.end(), [&](int a, int b) { return keys[a] < keys[b]; });
  return order;
}

// The pool slots of the map's blocks in (z, y, x) order, and, where block_index is given, the blocks' indices in that order.
int slots_zyx(ksg_integrator* h, std::vector<int>* order, int32_t* block_index) {
  const int64_t nb = h->num_blocks;
  std::vector<uint64_t> keys((size_t)nb);
  KSG_CUDA(cudaMemcpy(keys.data(), h->map.slot_key, sizeof(uint64_t) * nb, cudaMemcpyDeviceToHost));
  *order = zyx_order(keys);
  if (block_index) for (int64_t i = 0; i < nb; ++i) put_block_index(block_index, i, keys[(*order)[i]]);
  return KSG_OK;
}

// Staging of ksg_export_blocks / ksg_import_blocks in d_exp, per batch of `cnt` blocks:
// [distance | weight | rgba | semantic rgba | priors | labels | (import) fresh-block flags], batches of at most 256 MiB.
struct BlockStaging {
  size_t VB, C, per_block;
  int64_t batch;
  BlockStaging(const DevCfg& dc, int64_t n)
      : VB((size_t)dc.vps * dc.vps * dc.vps), C((size_t)dc.C), per_block(VB * (4 + 4 + 4 + 1 + 4 + 4 * C) + 64),
        batch(std::max<int64_t>(1, std::min<int64_t>(n, (int64_t)((256ull << 20) / per_block)))) {}
  struct Parts { float* dist; float* wgt; uint32_t* rgba; uint32_t* srgba; float* prior; uint8_t* label; uint8_t* fresh; };
  Parts at(uint8_t* p, int64_t cnt) const {
    Parts q;
    q.dist = (float*)p; p += cnt * VB * 4;
    q.wgt = (float*)p; p += cnt * VB * 4;
    q.rgba = (uint32_t*)p; p += cnt * VB * 4;
    q.srgba = (uint32_t*)p; p += cnt * VB * 4;
    q.prior = (float*)p; p += cnt * VB * 4 * C;
    q.label = p; p += cnt * VB;
    q.fresh = p;
    return q;
  }
  // the slot list and the staging buffer for one batch; `bytes` is batch * per_block, plus the flags for an import
  int ensure(ksg_integrator* h, size_t bytes) const {
    if (h->exp_slots_cap < batch) KSG_CUDA(h->res.regrow(&h->d_exp_slots, &h->exp_slots_cap, (size_t)batch));
    if (h->d_exp_bytes < bytes) KSG_CUDA(h->res.regrow(&h->d_exp, &h->d_exp_bytes, bytes));
    return KSG_OK;
  }
};
}  // namespace

int32_t ksg_extract_mesh(ksg_integrator* h, float min_weight, int64_t vertex_capacity, float* vertices, uint8_t* rgba, uint8_t* labels,
                         int64_t block_capacity, int32_t* block_index, int64_t* block_first_vertex, int64_t* n_vertices, int64_t* n_blocks) {
  if (!h || vertex_capacity < 0 || block_capacity < 0) return KSG_ERR_INVALID_ARGUMENT;
  { const int rcp = complete_frames(h); if (rcp) return rcp; }
  const int64_t nb = h->num_blocks;
  if (n_blocks) *n_blocks = nb;
  if (n_vertices) *n_vertices = 0;
  if (nb == 0) { if (block_first_vertex && block_capacity >= 0) block_first_vertex[0] = 0; return KSG_OK; }
  if ((block_index || block_first_vertex) && nb > block_capacity) return h->fail(KSG_ERR_INVALID_ARGUMENT, "mesh: block capacity too small");
  // blocks in (z, y, x) order, as ksg_export_blocks lists them
  std::vector<int> order;
  { const int rco = slots_zyx(h, &order, block_index); if (rco) return rco; }
  Resources tmp;
  int* d_slots = nullptr; int* d_count = nullptr; long long* d_first = nullptr;
  KSG_CUDA(tmp.device(&d_slots, nb));
  KSG_CUDA(tmp.device(&d_count, nb));
  KSG_CUDA(tmp.device(&d_first, nb));
  KSG_CUDA(cudaMemcpy(d_slots, order.data(), sizeof(int) * nb, cudaMemcpyHostToDevice));
  cudaStream_t s = h->own_stream;
  const int grid = (int)std::min<int64_t>(nb, (int64_t)h->sm_count * 8);
  MeshBuf none{nullptr, nullptr, nullptr};
  ++h->n_launches;
  k_mesh_blocks<false><<<grid, kMeshThreads, 0, s>>>(h->dc, h->map, d_slots, (int)nb, min_weight, nullptr, d_count, none);
  std::vector<int> count((size_t)nb);
  KSG_CUDA(cudaMemcpyAsync(count.data(), d_count, sizeof(int) * nb, cudaMemcpyDeviceToHost, s));
  KSG_CUDA(cudaStreamSynchronize(s));
  std::vector<long long> first((size_t)nb + 1);
  first[0] = 0;
  for (int64_t i = 0; i < nb; ++i) first[i + 1] = first[i] + count[i];
  const int64_t total = first[nb];
  if (n_vertices) *n_vertices = total;
  if (block_first_vertex) for (int64_t i = 0; i <= nb && i <= block_capacity; ++i) block_first_vertex[i] = first[i];
  if (!vertices && !rgba && !labels) return KSG_OK;                 // counting call
  if (total > vertex_capacity) return h->fail(KSG_ERR_INVALID_ARGUMENT, "mesh: vertex capacity too small (n_vertices holds the need)");
  if (total == 0) return KSG_OK;
  KSG_CUDA(cudaMemcpyAsync(d_first, first.data(), sizeof(long long) * nb, cudaMemcpyHostToDevice, s));
  HostStaging st;
  MeshBuf mb{};
  st.out(&mb.vtx, vertices, 3 * (size_t)total, true);   // the kernel writes all three
  st.out(&mb.rgba, reinterpret_cast<uint32_t*>(rgba), (size_t)total, true);
  st.out(&mb.label, labels, (size_t)total, true);
  return st.run(h, s, [&] {
    ++h->n_launches;
    k_mesh_blocks<true><<<grid, kMeshThreads, 0, s>>>(h->dc, h->map, d_slots, (int)nb, min_weight, d_first, nullptr, mb);
    return KSG_OK;
  });
}

int32_t ksg_update_mesh(ksg_integrator* h, float min_weight, ksg_mesh_stats* stats) {
  if (!h) return KSG_ERR_INVALID_ARGUMENT;
  if (!(min_weight >= 0.0f)) return h->fail(KSG_ERR_INVALID_ARGUMENT, "mesh update: NaN or negative min_weight");
  if (h->dc.shard_count > 1) return h->fail(KSG_ERR_INVALID_ARGUMENT, "mesh update: a sharded integrator holds only its own tiles");
  { const int rcp = complete_frames(h); if (rcp) return rcp; }
  const int64_t nb = h->num_blocks;
  const bool full = h->mesh_full || h->mesh_far || min_weight != h->mesh_min_weight;
  ksg_mesh_stats st{};
  st.blocks = nb;
  st.full = full ? 1 : 0;
  if (!full && h->frame_stamp == h->mesh_stamp && nb == h->mesh_blocks) {   // nothing stamped, nothing allocated: no launch
    st.vertices = h->mesh_vertices;
    h->mesh_remeshed = 0;
    if (stats) *stats = st;
    return KSG_OK;
  }
  // Until this call succeeds the layer is not trusted: the marks and the arenas are rewritten in place.
  h->mesh_full = true;
  h->mesh_valid = false;
  const int64_t prev = full ? 0 : h->mesh_blocks;   // slots below prev hold the meshes of the last update
  const size_t rows = (size_t)h->map.max_blocks;
  Resources& res = h->res;
  if (!h->mesh_mark) {
    KSG_CUDA(res.device(&h->mesh_mark, rows));
    KSG_CUDA(res.device(&h->mesh_rpos, rows));
    KSG_CUDA(res.device(&h->mesh_list, rows));
    KSG_CUDA(res.device(&h->mesh_count, rows));
    KSG_CUDA(res.device(&h->mesh_lfirst, rows));
    KSG_CUDA(res.device(&h->mesh_first[0], rows + 1));
    KSG_CUDA(res.device(&h->mesh_first[1], rows + 1));
    KSG_CUDA(res.device(&h->d_mesh_ctr, 1));
    KSG_CUDA(res.pinned(&h->h_mesh_ctr, 1));
  }
  cudaStream_t s = h->own_stream;
  if (full) KSG_CUDA(cudaMemsetAsync(h->mesh_mark, 0, sizeof(unsigned) * rows, s));   // new, or left marked by a failed update
  MeshCounters& ctr = *h->h_mesh_ctr;
  std::memset(&ctr, 0, sizeof(ctr));
  const int src = h->mesh_cur, dst = 1 - src;
  if (nb > 0) {
    KSG_CUDA(cudaMemsetAsync(h->d_mesh_ctr, 0, sizeof(MeshCounters), s));
    const int64_t positions = (int64_t)h->ht_cap;
    ++h->n_launches;
    k_mesh_dirty<<<(int)std::min<int64_t>((positions + 255) / 256, (int64_t)h->sm_count * 8), 256, 0, s>>>(
        h->map, (int)nb, (int)prev, h->mesh_stamp, h->dc.vps, h->mesh_mark, h->mesh_rpos, h->mesh_list, h->d_mesh_ctr);
    KSG_CUDA(cudaMemcpyAsync(&ctr, h->d_mesh_ctr, sizeof(MeshCounters), cudaMemcpyDeviceToHost, s));
    KSG_CUDA(cudaStreamSynchronize(s));
    KSG_CUDA(cudaGetLastError());
  }
  const int nr = ctr.remeshed;
  const int grid = (int)std::min<int64_t>(std::max(nr, 1), (int64_t)h->sm_count * 8);
  if (nr > 0) {
    const MeshBuf none{nullptr, nullptr, nullptr};
    h->n_launches += 2;
    k_mesh_blocks<false><<<grid, kMeshThreads, 0, s>>>(h->dc, h->map, h->mesh_list, nr, min_weight, nullptr, h->mesh_count, none);
    k_mesh_scan<<<1, kMeshScanThreads, 0, s>>>((int)nb, h->mesh_mark, h->mesh_rpos, h->mesh_count, h->mesh_first[src], h->mesh_first[dst],
                                               h->mesh_lfirst, h->d_mesh_ctr);
    KSG_CUDA(cudaMemcpyAsync(&ctr.vertices, &h->d_mesh_ctr->vertices, 2 * sizeof(long long), cudaMemcpyDeviceToHost, s));
    KSG_CUDA(cudaStreamSynchronize(s));
    KSG_CUDA(cudaGetLastError());
    const int64_t total = ctr.vertices;
    if (total > h->mesh_cap[dst]) {
      MeshBuf& a = h->mesh_arena[dst];
      const size_t want = (size_t)total + (size_t)total / 4;   // room to grow without a reallocation every update
      int64_t c0 = 0, c1 = 0, c2 = 0;
      h->mesh_cap[dst] = 0;
      KSG_CUDA(res.regrow(&a.vtx, &c0, 3 * want));
      KSG_CUDA(res.regrow(&a.rgba, &c1, want));
      KSG_CUDA(res.regrow(&a.label, &c2, want));
      h->mesh_cap[dst] = (int64_t)want;
    }
    h->n_launches += 2;
    k_mesh_move<<<(int)std::min<int64_t>((nb + 7) / 8, (int64_t)h->sm_count * 16), 256, 0, s>>>(
        (int)nb, nullptr, h->mesh_first[src], h->mesh_first[dst], 1, h->mesh_mark, h->mesh_arena[src], h->mesh_arena[dst]);
    k_mesh_blocks<true><<<grid, kMeshThreads, 0, s>>>(h->dc, h->map, h->mesh_list, nr, min_weight, h->mesh_lfirst, nullptr, h->mesh_arena[dst]);
    KSG_CUDA(cudaStreamSynchronize(s));
    KSG_CUDA(cudaGetLastError());
    h->mesh_cur = dst;
  } else if (nb == 0) {
    KSG_CUDA(cudaMemsetAsync(h->mesh_first[src], 0, sizeof(long long), s));   // first[0] = the total = 0
    KSG_CUDA(cudaStreamSynchronize(s));
  }
  h->mesh_far = ctr.far != 0 || (!full && h->mesh_far);
  h->mesh_full = false;
  h->mesh_valid = true;
  h->mesh_min_weight = min_weight;
  h->mesh_stamp = h->frame_stamp;
  h->mesh_blocks = nb;
  h->mesh_vertices = nr > 0 ? ctr.vertices : h->mesh_vertices;
  if (nb == 0) h->mesh_vertices = 0;
  h->mesh_remeshed = nr;
  st.changed_blocks = ctr.changed;
  st.remeshed_blocks = nr;
  st.vertices = h->mesh_vertices;
  st.remeshed_vertices = nr > 0 ? ctr.remeshed_vertices : 0;
  if (stats) *stats = st;
  return KSG_OK;
}

int32_t ksg_export_mesh(ksg_integrator* h, int32_t changed_only, int64_t vertex_capacity, float* vertices, uint8_t* rgba, uint8_t* labels,
                        int64_t block_capacity, int32_t* block_index, int64_t* block_first_vertex, int64_t* n_vertices, int64_t* n_blocks) {
  if (!h || vertex_capacity < 0 || block_capacity < 0) return KSG_ERR_INVALID_ARGUMENT;
  if (!h->mesh_valid) return h->fail(KSG_ERR_INVALID_ARGUMENT, "mesh export: no ksg_update_mesh since the handle was created, cleared or reset");
  KSG_CUDA(cudaSetDevice(h->device));
  const int64_t nb = h->mesh_blocks;
  // the blocks to list (slots), in (z, y, x) order, and the layer's per-slot first vertices
  std::vector<uint64_t> keys((size_t)nb);
  std::vector<long long> first((size_t)nb + 1, 0);
  if (nb > 0) {
    KSG_CUDA(cudaMemcpy(keys.data(), h->map.slot_key, sizeof(uint64_t) * nb, cudaMemcpyDeviceToHost));
    KSG_CUDA(cudaMemcpy(first.data(), h->mesh_first[h->mesh_cur], sizeof(long long) * (nb + 1), cudaMemcpyDeviceToHost));
  }
  std::vector<int> list;
  if (changed_only) {
    list.resize((size_t)h->mesh_remeshed);
    if (!list.empty()) KSG_CUDA(cudaMemcpy(list.data(), h->mesh_list, sizeof(int) * list.size(), cudaMemcpyDeviceToHost));
    std::sort(list.begin(), list.end(), [&](int a, int b) { return keys[a] < keys[b]; });
  } else {
    list = zyx_order(keys);
  }
  const int64_t n = (int64_t)list.size();
  std::vector<long long> out_first((size_t)n + 1);
  out_first[0] = 0;
  for (int64_t i = 0; i < n; ++i) out_first[i + 1] = out_first[i] + (first[list[i] + 1] - first[list[i]]);
  const int64_t total = out_first[n];
  if (n_blocks) *n_blocks = n;
  if (n_vertices) *n_vertices = total;
  if ((block_index || block_first_vertex) && n > block_capacity)
    return h->fail(KSG_ERR_INVALID_ARGUMENT, "mesh export: block capacity too small (n_blocks holds the need)");
  if (block_index) for (int64_t i = 0; i < n; ++i) put_block_index(block_index, i, keys[list[i]]);
  if (block_first_vertex) for (int64_t i = 0; i <= n; ++i) block_first_vertex[i] = out_first[i];
  if (!vertices && !rgba && !labels) return KSG_OK;                 // counting call
  if (total > vertex_capacity) return h->fail(KSG_ERR_INVALID_ARGUMENT, "mesh export: vertex capacity too small (n_vertices holds the need)");
  if (total == 0) return KSG_OK;
  HostStaging st;
  const int* d_list = nullptr;
  const long long* d_out_first = nullptr;
  MeshBuf mb{};
  st.in(&d_list, list.data(), (size_t)n);
  st.in(&d_out_first, out_first.data(), (size_t)n);
  st.out(&mb.vtx, vertices, 3 * (size_t)total, true);   // the kernel writes all three
  st.out(&mb.rgba, reinterpret_cast<uint32_t*>(rgba), (size_t)total, true);
  st.out(&mb.label, labels, (size_t)total, true);
  cudaStream_t s = h->own_stream;
  return st.run(h, s, [&] {
    ++h->n_launches;
    k_mesh_move<<<(int)std::min<int64_t>((n + 7) / 8, (int64_t)h->sm_count * 16), 256, 0, s>>>(
        (int)n, d_list, h->mesh_first[h->mesh_cur], d_out_first, 0, nullptr, h->mesh_arena[h->mesh_cur], mb);
    return KSG_OK;
  });
}

int32_t ksg_mesh_view_device(ksg_integrator* h, int64_t* n_blocks, int64_t* n_vertices, const void** d_block_keys, const int64_t** d_block_first,
                             const float** d_vertices, const uint32_t** d_rgba, const uint8_t** d_labels) {
  if (!h) return KSG_ERR_INVALID_ARGUMENT;
  if (!h->mesh_valid) return h->fail(KSG_ERR_INVALID_ARGUMENT, "mesh view: no ksg_update_mesh since the handle was created, cleared or reset");
  static_assert(sizeof(long long) == sizeof(int64_t), "block_first layout");
  const MeshBuf& a = h->mesh_arena[h->mesh_cur];
  if (n_blocks) *n_blocks = h->mesh_blocks;
  if (n_vertices) *n_vertices = h->mesh_vertices;
  if (d_block_keys) *d_block_keys = h->map.slot_key;
  if (d_block_first) *d_block_first = reinterpret_cast<const int64_t*>(h->mesh_first[h->mesh_cur]);
  if (d_vertices) *d_vertices = a.vtx;
  if (d_rgba) *d_rgba = a.rgba;
  if (d_labels) *d_labels = a.label;
  return KSG_OK;
}

namespace {
bool query_wanted(const ksg_query_out& o) {
  return o.flags || o.tsdf_distance || o.tsdf_weight || o.tsdf_rgba || o.sem_label || o.sem_priors || o.sem_rgba || o.distance || o.gradient;
}
// *work = false: the call has nothing to compute (n = 0 or no output wanted) and launches nothing
int query_args(ksg_integrator* h, int64_t n, const float* xyz, float min_weight, const ksg_query_out* o, bool* work) {
  if (!h) return KSG_ERR_INVALID_ARGUMENT;
  if (!o || n < 0 || !(min_weight >= 0.0f)) return h->fail(KSG_ERR_INVALID_ARGUMENT, "query: NULL out, n < 0 or a NaN / negative min_weight");
  if (n > 0 && !xyz) return h->fail(KSG_ERR_INVALID_ARGUMENT, "query: NULL points");
  if (h->dc.shard_count > 1) return h->fail(KSG_ERR_INVALID_ARGUMENT, "query: a sharded integrator holds only its own tiles");
  *work = n > 0 && query_wanted(*o);
  return KSG_OK;
}
// the slices of the wanted host outputs `o` of a point query at n points; *d receives their device pointers
void stage_query_out(HostStaging* st, const ksg_query_out& o, size_t n, size_t C, ksg_query_out* d) {
  st->out(&d->flags, o.flags, n);
  st->out(&d->tsdf_distance, o.tsdf_distance, n);
  st->out(&d->tsdf_weight, o.tsdf_weight, n);
  st->out(&d->tsdf_rgba, o.tsdf_rgba, 4 * n);
  st->out(&d->sem_label, o.sem_label, n);
  st->out(&d->sem_priors, o.sem_priors, n * C);
  st->out(&d->sem_rgba, o.sem_rgba, 4 * n);
  st->out(&d->distance, o.distance, n);
  st->out(&d->gradient, o.gradient, 3 * n);
}
void launch_query(ksg_integrator* h, int64_t n, const float* d_xyz, float min_weight, const ksg_query_out& o, cudaStream_t s) {
  static_assert(sizeof(ksg_query_out) == sizeof(QueryOut), "ksg_query_out layout");
  QueryOut q{o.flags, o.tsdf_distance, o.tsdf_weight, o.tsdf_rgba, o.sem_label, o.sem_priors, o.sem_rgba, o.distance, o.gradient};
  const int grid = (int)std::min<int64_t>((n + kQueryThreads - 1) / kQueryThreads, (int64_t)h->sm_count * 8);
  ++h->n_launches;
  k_query_points<<<grid, kQueryThreads, 0, s>>>(h->dc, h->map, d_xyz, (long long)n, min_weight, q, (o.flags || o.distance) ? 1 : 0,
                                                (o.flags || o.gradient) ? 1 : 0);
}
}  // namespace

int32_t ksg_query_points(ksg_integrator* h, int64_t n, const float* xyz_G, float min_weight, const ksg_query_out* out) {
  bool work = false;
  { const int rca = query_args(h, n, xyz_G, min_weight, out, &work); if (rca) return rca; }
  { const int rcp = complete_frames(h); if (rcp) return rcp; }
  if (!work) return KSG_OK;
  HostStaging st;
  const float* d_xyz = nullptr;
  ksg_query_out dq{};
  st.in(&d_xyz, xyz_G, 3 * (size_t)n);
  stage_query_out(&st, *out, (size_t)n, (size_t)h->dc.C, &dq);
  cudaStream_t s = h->own_stream;
  return st.run(h, s, [&] { launch_query(h, n, d_xyz, min_weight, dq, s); return KSG_OK; });
}

int32_t ksg_query_points_device(ksg_integrator* h, int64_t n, const float* d_xyz_G, float min_weight, const ksg_query_out* d_out,
                                void* cuda_stream) {
  bool work = false;
  { const int rca = query_args(h, n, d_xyz_G, min_weight, d_out, &work); if (rca) return rca; }
  if (h->deferred_status) return h->fail(h->deferred_status, err_text(h->deferred_status));
  if (!work) return KSG_OK;
  KSG_CUDA(cudaSetDevice(h->device));
  launch_query(h, n, d_xyz_G, min_weight, *d_out, cuda_stream ? (cudaStream_t)cuda_stream : h->own_stream);
  KSG_CUDA(cudaGetLastError());
  return KSG_OK;
}

namespace {
// the checks both render entries share; fills the kernel's camera
int render_args(ksg_integrator* h, const float* T, const double* K, int32_t width, int32_t height, float min_depth, float max_depth,
                float min_weight, const ksg_render_out* o, RenderCam* c) {
  if (!h) return KSG_ERR_INVALID_ARGUMENT;
  if (!T || !K || !o) return h->fail(KSG_ERR_INVALID_ARGUMENT, "render: NULL pose, K or out");
  for (int k = 0; k < 7; ++k)
    if (!std::isfinite(T[k])) return h->fail(KSG_ERR_INVALID_ARGUMENT, "render: non-finite pose");
  for (int k = 0; k < 4; ++k)
    if (!std::isfinite(K[k])) return h->fail(KSG_ERR_INVALID_ARGUMENT, "render: non-finite K");
  if (!(K[0] > 0.0) || !(K[1] > 0.0)) return h->fail(KSG_ERR_INVALID_ARGUMENT, "render: fx or fy <= 0");
  if (width <= 0 || height <= 0) return h->fail(KSG_ERR_INVALID_ARGUMENT, "render: width or height <= 0");
  if (!std::isfinite(min_depth) || !(min_depth > 0.0f) || !std::isfinite(max_depth) || !(max_depth > min_depth))
    return h->fail(KSG_ERR_INVALID_ARGUMENT, "render: needs 0 < min_depth < max_depth, both finite");
  if (!(min_weight >= 0.0f)) return h->fail(KSG_ERR_INVALID_ARGUMENT, "render: NaN or negative min_weight");
  // the smallest z step, (kRenderPush * vs) / r at the corner pixel with the largest r, must be >= max_depth * 2^-20 (ksg_render.cuh)
  const double au = std::max(std::fabs(0.0 - K[2]), std::fabs((double)(width - 1) - K[2])) / K[0];
  const double av = std::max(std::fabs(0.0 - K[3]), std::fabs((double)(height - 1) - K[3])) / K[1];
  const double r_max = std::sqrt(au * au + av * av + 1.0);
  if (!((double)kRenderPush * (double)h->dc.voxel_size / r_max >= (double)max_depth * 0x1p-20))
    return h->fail(KSG_ERR_INVALID_ARGUMENT, "render: max_depth too large for the voxel size and field of view (a step would round away)");
  if (h->dc.shard_count > 1) return h->fail(KSG_ERR_INVALID_ARGUMENT, "render: a sharded integrator holds only its own tiles");
  c->T = Xform{T[0], T[1], T[2], T[3], T[4], T[5], T[6]};
  c->cx = (float)K[2];
  c->cy = (float)K[3];
  c->constant_x = (float)(1.0 / K[0]);
  c->constant_y = (float)(1.0 / K[1]);
  c->width = width;
  c->height = height;
  c->min_depth = min_depth;
  c->max_depth = max_depth;
  c->min_weight = min_weight;
  return KSG_OK;
}
// the march (writes depth and / or points), then the point query at the points when an at_hit output is wanted
void launch_render(ksg_integrator* h, const RenderCam& c, float* d_depth, float* d_points, const ksg_query_out& at_hit, cudaStream_t s) {
  const int64_t tiles = (int64_t)((c.width + kRenderTileW - 1) / kRenderTileW) * ((c.height + kRenderTileH - 1) / kRenderTileH);
  const int grid = (int)((tiles * 32 + kRenderThreads - 1) / kRenderThreads);
  ++h->n_launches;
  k_render_view<<<grid, kRenderThreads, 0, s>>>(h->dc, h->map, c, d_depth, d_points);
  if (query_wanted(at_hit)) launch_query(h, (int64_t)c.width * c.height, d_points, c.min_weight, at_hit, s);
}
}  // namespace

int32_t ksg_render_view(ksg_integrator* h, const float* T_G_C, const double* K, int32_t width, int32_t height, float min_depth,
                        float max_depth, float min_weight, const ksg_render_out* out) {
  RenderCam c{};
  { const int rca = render_args(h, T_G_C, K, width, height, min_depth, max_depth, min_weight, out, &c); if (rca) return rca; }
  { const int rcp = complete_frames(h); if (rcp) return rcp; }
  const bool at_hit = query_wanted(out->at_hit);
  if (!out->depth && !out->points_G && !at_hit) return KSG_OK;
  const size_t N = (size_t)width * (size_t)height;
  HostStaging st;
  float *d_depth = nullptr, *d_points = nullptr;
  ksg_query_out dq{};
  st.out(&d_depth, out->depth, N);
  st.out(&d_points, out->points_G, 3 * N, at_hit);   // the query at the hits reads the points
  stage_query_out(&st, out->at_hit, N, (size_t)h->dc.C, &dq);
  cudaStream_t s = h->own_stream;
  return st.run(h, s, [&] { launch_render(h, c, d_depth, d_points, dq, s); return KSG_OK; });
}

int32_t ksg_render_view_device(ksg_integrator* h, const float* T_G_C_host, const double* K_host, int32_t width, int32_t height,
                               float min_depth, float max_depth, float min_weight, const ksg_render_out* d_out, void* cuda_stream) {
  RenderCam c{};
  { const int rca = render_args(h, T_G_C_host, K_host, width, height, min_depth, max_depth, min_weight, d_out, &c); if (rca) return rca; }
  const bool at_hit = query_wanted(d_out->at_hit);
  if (at_hit && !d_out->points_G) return h->fail(KSG_ERR_INVALID_ARGUMENT, "render: an at_hit output needs points_G (the query reads it)");
  if (h->deferred_status) return h->fail(h->deferred_status, err_text(h->deferred_status));
  if (!d_out->depth && !d_out->points_G) return KSG_OK;
  KSG_CUDA(cudaSetDevice(h->device));
  launch_render(h, c, d_out->depth, d_out->points_G, d_out->at_hit, cuda_stream ? (cudaStream_t)cuda_stream : h->own_stream);
  KSG_CUDA(cudaGetLastError());
  return KSG_OK;
}

namespace {
// The work sets of the x and y passes and the neighbour tables of the three passes (ksg_esdf.cuh), from the keys of the allocated blocks
// (the site rows: the x pass table holds indices into alloc), which of them hold a site, and the z work set `out` (indices into alloc;
// NULL: every allocated block, in alloc order).  Blocks outside the key range hold no site, and neither does any block sharing their
// out-of-range coordinate, so their pass results are "none" and they are left out.
struct EsdfWork {
  int64_t n_x = 0, n_y = 0;
  std::vector<int> tx, ty, tz;   // per block of the x / y / z pass: 2 Rb + 1 indices into the previous stage, -1 = none

  void build(const std::vector<I3>& alloc, const std::vector<uint8_t>& has_site, int Rb, const std::vector<int>* out = nullptr) {
    const int span = 2 * Rb + 1;
    auto moved = [](I3 b, int axis, int k) { if (axis == 0) b.x += k; else if (axis == 1) b.y += k; else b.z += k; return b; };
    std::unordered_map<uint64_t, int> site_at;      // site block -> its index in alloc
    std::unordered_map<uint64_t, char> near_x;      // within Rb along x of a site block
    for (size_t a = 0; a < alloc.size(); ++a) {
      if (!has_site[a]) continue;
      site_at[pack_key(alloc[a])] = (int)a;
      for (int k = -Rb; k <= Rb; ++k) {
        const I3 b = moved(alloc[a], 0, k);
        if (key_in_range(b)) near_x[pack_key(b)] = 1;
      }
    }
    std::vector<I3> zs;
    if (out)
      for (int a : *out) zs.push_back(alloc[a]);
    const std::vector<I3>& z_blocks = out ? zs : alloc;
    // Y: within Rb along z of a z block, with a near_x block within Rb along y
    std::unordered_map<uint64_t, int> y_at;         // -1: looked at and left out
    std::vector<I3> ys;
    for (const I3& a : z_blocks)
      for (int k = -Rb; k <= Rb; ++k) {
        const I3 b = moved(a, 2, k);
        if (!key_in_range(b) || y_at.count(pack_key(b))) continue;
        bool keep = false;
        for (int j = -Rb; j <= Rb && !keep; ++j) {
          const I3 c = moved(b, 1, j);
          keep = key_in_range(c) && near_x.count(pack_key(c));
        }
        y_at[pack_key(b)] = keep ? (int)ys.size() : -1;
        if (keep) ys.push_back(b);
      }
    // X: within Rb along y of a Y block, and near_x
    std::unordered_map<uint64_t, int> x_at;
    std::vector<I3> xs;
    for (const I3& y : ys)
      for (int j = -Rb; j <= Rb; ++j) {
        const I3 b = moved(y, 1, j);
        if (!key_in_range(b) || !near_x.count(pack_key(b)) || x_at.count(pack_key(b))) continue;
        x_at[pack_key(b)] = (int)xs.size();
        xs.push_back(b);
      }
    n_x = (int64_t)xs.size();
    n_y = (int64_t)ys.size();
    auto table = [&](const std::vector<I3>& blocks, int axis, const std::unordered_map<uint64_t, int>& prev, std::vector<int>* t) {
      t->assign(blocks.size() * span, -1);
      for (size_t i = 0; i < blocks.size(); ++i)
        for (int k = -Rb; k <= Rb; ++k) {
          const I3 b = moved(blocks[i], axis, k);
          if (!key_in_range(b)) continue;
          const auto it = prev.find(pack_key(b));
          if (it != prev.end()) (*t)[i * span + Rb + k] = it->second;
        }
    };
    table(xs, 0, site_at, &tx);
    table(ys, 1, x_at, &ty);
    table(z_blocks, 2, y_at, &tz);
  }
};

int esdf_grid(ksg_integrator* h, int64_t blocks) {
  const int64_t items = blocks * (int64_t)h->dc.vps * h->dc.vps * h->dc.vps;
  return (int)std::max<int64_t>(1, std::min<int64_t>((items + kEsdfThreads - 1) / kEsdfThreads, (int64_t)h->sm_count * 16));
}

// the checks of ksg_compute_esdf and ksg_update_esdf; *W = the window
int esdf_args(ksg_integrator* h, float min_weight, float max_distance, int* W) {
  if (!h) return KSG_ERR_INVALID_ARGUMENT;
  if (!(min_weight >= 0.0f)) return h->fail(KSG_ERR_INVALID_ARGUMENT, "esdf: NaN or negative min_weight");
  if (!std::isfinite(max_distance) || !(max_distance > 0.0f)) return h->fail(KSG_ERR_INVALID_ARGUMENT, "esdf: max_distance must be finite and > 0");
  const double Wd = std::ceil((double)max_distance / (double)h->dc.voxel_size) + 1.0;
  if (!(Wd <= (double)kEsdfMaxWindow)) return h->fail(KSG_ERR_INVALID_ARGUMENT, "esdf: ceil(max_distance / voxel_size) + 1 > 512");
  if (h->dc.shard_count > 1) return h->fail(KSG_ERR_INVALID_ARGUMENT, "esdf: a sharded integrator holds only its own tiles");
  *W = (int)Wd;
  return KSG_OK;
}

// The sites step of ksg_compute_esdf and ksg_update_esdf: k_esdf_sites over the blocks at pool slots `slots`, whose site bytes go to
// `site` in row = the slot (slot_rows, the device layer) or the position in `slots` (the batch entry).  *d_slots: the uploaded list (in
// `tmp`); *has: each block's has-site byte, then, with `changed`, each block's changed byte.
int esdf_sites(ksg_integrator* h, Resources& tmp, const std::vector<int>& slots, float min_weight, int slot_rows, uint8_t* site, bool changed,
               int** d_slots, std::vector<uint8_t>* has) {
  const int64_t n = (int64_t)slots.size(), n_out = changed ? 2 * n : n;
  cudaStream_t s = h->own_stream;
  uint8_t* d_has = nullptr;
  KSG_CUDA(upload(tmp, slots, s, d_slots));
  KSG_CUDA(tmp.device(&d_has, n_out));
  ++h->n_launches;
  k_esdf_sites<<<(int)std::min<int64_t>(n, (int64_t)h->sm_count * 8), kEsdfThreads, 0, s>>>(h->dc, h->map, *d_slots, (int)n, min_weight,
                                                                                             slot_rows, site, d_has, changed ? d_has + n : nullptr);
  has->resize((size_t)n_out);
  KSG_CUDA(cudaMemcpyAsync(has->data(), d_has, n_out, cudaMemcpyDeviceToHost, s));
  KSG_CUDA(cudaStreamSynchronize(s));
  KSG_CUDA(cudaGetLastError());
  return KSG_OK;
}

// The passes step of both entries: the three windowed passes, enqueued.  blocks[i] is the block of site row i of `site`, has[i] whether
// it holds a site; the z work set is z_rows (row indices; NULL: every row, in row order), and eo.slots lists its pool slots on the
// device.  The z pass writes eo in work set order or, with slot_rows, in the rows of the pool slots.  *st (NULL: not wanted) receives
// the sizes of the three work sets.
int esdf_passes(ksg_integrator* h, Resources& tmp, int W, int Rb, const std::vector<I3>& blocks, const std::vector<uint8_t>& has,
                const std::vector<int>* z_rows, const uint8_t* site, const EsdfOut& eo, bool slot_rows, ksg_esdf_stats* st) {
  const size_t V = (size_t)h->dc.vps * h->dc.vps * h->dc.vps;
  const int64_t nz = z_rows ? (int64_t)z_rows->size() : (int64_t)blocks.size();
  cudaStream_t s = h->own_stream;
  EsdfWork wk;
  wk.build(blocks, has, Rb, z_rows);
  int *d_tx = nullptr, *d_ty = nullptr, *d_tz = nullptr, *d_a = nullptr, *d_b = nullptr;
  KSG_CUDA(upload(tmp, wk.tx, s, &d_tx));
  KSG_CUDA(upload(tmp, wk.ty, s, &d_ty));
  KSG_CUDA(upload(tmp, wk.tz, s, &d_tz));
  KSG_CUDA(tmp.device(&d_a, wk.n_x * V));
  KSG_CUDA(tmp.device(&d_b, wk.n_y * V));
  const EsdfOut none{nullptr, nullptr, nullptr, 0.0f, 0.0f};
  h->n_launches += 3;
  k_esdf_pass<0><<<esdf_grid(h, wk.n_x), kEsdfThreads, 0, s>>>(h->dc, h->map, (int)wk.n_x, W, Rb, d_tx, site, nullptr, d_a, nullptr, none);
  k_esdf_pass<1><<<esdf_grid(h, wk.n_y), kEsdfThreads, 0, s>>>(h->dc, h->map, (int)wk.n_y, W, Rb, d_ty, nullptr, d_a, d_b, nullptr, none);
  auto* const z_pass = slot_rows ? k_esdf_pass<2, true> : k_esdf_pass<2>;
  z_pass<<<esdf_grid(h, nz), kEsdfThreads, 0, s>>>(h->dc, h->map, (int)nz, W, Rb, d_tz, nullptr, d_b, nullptr, site, eo);
  KSG_CUDA(cudaGetLastError());
  if (st) { st->x_blocks = wk.n_x; st->y_blocks = wk.n_y; st->z_blocks = nz; }
  return KSG_OK;
}
}  // namespace

int32_t ksg_compute_esdf(ksg_integrator* h, float min_weight, float max_distance, int64_t capacity_blocks, int32_t* block_index,
                         float* distance, uint8_t* flags) {
  int W = 0;
  { const int rca = esdf_args(h, min_weight, max_distance, &W); if (rca) return rca; }
  { const int rcp = complete_frames(h); if (rcp) return rcp; }
  const int64_t nb = h->num_blocks;
  if (nb > capacity_blocks) return h->fail(KSG_ERR_INVALID_ARGUMENT, "esdf: block capacity too small");
  if (nb == 0) return KSG_OK;
  std::vector<int> order;
  std::vector<int32_t> index((size_t)(3 * nb));
  { const int rco = slots_zyx(h, &order, index.data()); if (rco) return rco; }
  if (block_index) std::memcpy(block_index, index.data(), sizeof(int32_t) * 3 * nb);
  if (!distance && !flags) return KSG_OK;
  const int vps = h->dc.vps, Rb = (W + vps - 1) / vps;
  const size_t V = (size_t)vps * vps * vps;
  cudaStream_t s = h->own_stream;
  // site rows of its own, in (z, y, x) position order: the device layer is not touched
  Resources tmp;
  uint8_t* d_site = nullptr;
  int* d_slots = nullptr;
  std::vector<uint8_t> has;
  KSG_CUDA(tmp.device(&d_site, nb * V));
  { const int rcs = esdf_sites(h, tmp, order, min_weight, 0, d_site, false, &d_slots, &has); if (rcs) return rcs; }
  std::vector<I3> blocks((size_t)nb);
  for (int64_t i = 0; i < nb; ++i) blocks[i] = I3{index[3 * i], index[3 * i + 1], index[3 * i + 2]};
  HostStaging st;
  EsdfOut eo{nullptr, nullptr, d_slots, min_weight, max_distance};
  st.out(&eo.distance, distance, nb * V);
  st.out(&eo.flags, flags, nb * V);
  return st.run(h, s, [&] { return esdf_passes(h, tmp, W, Rb, blocks, has, nullptr, d_site, eo, false, nullptr); });
}

int32_t ksg_update_esdf(ksg_integrator* h, float min_weight, float max_distance, ksg_esdf_stats* stats) {
  int W = 0;
  { const int rca = esdf_args(h, min_weight, max_distance, &W); if (rca) return rca; }
  { const int rcp = complete_frames(h); if (rcp) return rcp; }
  const int vps = h->dc.vps, Rb = (W + vps - 1) / vps;
  const size_t V = (size_t)vps * vps * vps;
  const int64_t nb = h->num_blocks;
  const bool full = h->esdf_full || min_weight != h->esdf_min_weight || max_distance != h->esdf_max_distance;
  // Until this call succeeds the layer is not trusted: the site bytes are rewritten in place before the passes run, so a call that
  // fails part-way would leave bytes that no longer differ from the map while their outputs are stale.  The next call is then full,
  // and export and query are refused until it succeeds.
  h->esdf_full = true;
  h->esdf_valid = false;
  const size_t rows = (size_t)h->map.max_blocks;
  if (!h->esdf_dist) KSG_CUDA(h->res.device(&h->esdf_dist, rows * V));
  if (!h->esdf_flags) KSG_CUDA(h->res.device(&h->esdf_flags, rows * V));
  if (!h->esdf_site) KSG_CUDA(h->res.device(&h->esdf_site, rows * V));
  if (h->esdf_has_site.size() != rows) h->esdf_has_site.assign(rows, 0);
  const int64_t prev = full ? 0 : h->esdf_blocks;   // rows below prev hold the sites and outputs of the last update
  cudaStream_t s = h->own_stream;
  std::vector<uint64_t> keys((size_t)nb);
  if (nb > 0) KSG_CUDA(cudaMemcpy(keys.data(), h->map.slot_key, sizeof(uint64_t) * nb, cudaMemcpyDeviceToHost));
  // C: the slots stamped after the last update, and the slots allocated since
  std::vector<uint8_t> in_c((size_t)nb, 0);
  for (int64_t i = prev; i < nb; ++i) in_c[i] = 1;
  if (prev > 0) {
    std::vector<int> pos_slot(h->ht_cap), pos_stamp(h->ht_cap);
    KSG_CUDA(cudaMemcpy(pos_slot.data(), h->map.ht_slot, sizeof(int) * h->ht_cap, cudaMemcpyDeviceToHost));
    KSG_CUDA(cudaMemcpy(pos_stamp.data(), h->map.touched_stamp, sizeof(int) * h->ht_cap, cudaMemcpyDeviceToHost));
    for (uint32_t p = 0; p < h->ht_cap; ++p)
      if (pos_slot[p] >= 0 && pos_slot[p] < nb && pos_stamp[p] > h->esdf_stamp) in_c[pos_slot[p]] = 1;
  }
  std::unordered_map<uint64_t, int> slot_of;
  slot_of.reserve((size_t)nb);
  for (int64_t i = 0; i < nb; ++i) slot_of[keys[i]] = (int)i;
  auto find = [&](I3 b) { if (!key_in_range(b)) return -1; const auto it = slot_of.find(pack_key(b)); return it == slot_of.end() ? -1 : it->second; };
  // R: C and its allocated face neighbours, whose site bytes are recomputed
  std::vector<uint8_t> in_r(in_c);
  int64_t n_c = 0;
  for (int64_t i = 0; i < nb; ++i) {
    if (!in_c[i]) continue;
    ++n_c;
    const I3 b = unpack_key(keys[i]);
    for (int k = 0; k < 6; ++k) {
      I3 nbk = b;
      const int d = (k & 1) ? 1 : -1;
      if (k < 2) nbk.x += d; else if (k < 4) nbk.y += d; else nbk.z += d;
      const int j = find(nbk);
      if (j >= 0) in_r[j] = 1;
    }
  }
  std::vector<int> r_slots;
  for (int64_t i = 0; i < nb; ++i) if (in_r[i]) r_slots.push_back((int)i);
  ksg_esdf_stats st{};
  st.blocks = nb;
  st.full = full ? 1 : 0;
  st.changed_blocks = n_c;
  st.site_blocks = (int64_t)r_slots.size();
  std::vector<int> d_list;
  if (!r_slots.empty()) {
    const int64_t nr = (int64_t)r_slots.size();
    Resources tmp;
    // rows new to the layer held no site before
    if (nb > prev) KSG_CUDA(cudaMemsetAsync(h->esdf_site + (size_t)prev * V, 0, (size_t)(nb - prev) * V, s));
    int* d_r = nullptr;
    std::vector<uint8_t> has;   // has_site, then changed
    { const int rcs = esdf_sites(h, tmp, r_slots, min_weight, 1, h->esdf_site, true, &d_r, &has); if (rcs) return rcs; }
    // S: the recomputed blocks whose site bytes changed; D = C + the allocated blocks within Rb (Chebyshev) of S, by a separable dilation
    // clamped to the allocated blocks' bounding box (an intermediate key takes the x, then the y coordinate of the allocated block it
    // reaches, so nothing outside the box is needed): the sets stay within |S| (2Rb + 1)^2 and the box, whatever the window
    I3 lo = unpack_key(keys[0]), hi = lo;
    for (int64_t i = 1; i < nb; ++i) {
      const I3 b = unpack_key(keys[i]);
      lo.x = std::min(lo.x, b.x); lo.y = std::min(lo.y, b.y); lo.z = std::min(lo.z, b.z);
      hi.x = std::max(hi.x, b.x); hi.y = std::max(hi.y, b.y); hi.z = std::max(hi.z, b.z);
    }
    std::unordered_set<uint64_t> sx, sxy;
    for (int64_t r = 0; r < nr; ++r) {
      h->esdf_has_site[r_slots[r]] = has[r];
      if (!has[nr + r]) continue;
      ++st.site_changed;
      const I3 b = unpack_key(keys[r_slots[r]]);
      for (int x = std::max(lo.x, b.x - Rb); x <= std::min(hi.x, b.x + Rb); ++x) { I3 c = b; c.x = x; sx.insert(pack_key(c)); }
    }
    for (uint64_t kx : sx) {
      const I3 b = unpack_key(kx);
      for (int y = std::max(lo.y, b.y - Rb); y <= std::min(hi.y, b.y + Rb); ++y) { I3 c = b; c.y = y; sxy.insert(pack_key(c)); }
    }
    for (int64_t i = 0; i < nb; ++i) {
      bool dirty = in_c[i];
      const I3 b = unpack_key(keys[i]);
      for (int z = std::max(lo.z, b.z - Rb); z <= std::min(hi.z, b.z + Rb) && !dirty && !sxy.empty(); ++z) {
        I3 c = b; c.z = z; dirty = sxy.count(pack_key(c)) > 0;
      }
      if (dirty) d_list.push_back((int)i);
    }
    std::sort(d_list.begin(), d_list.end(), [&](int a, int b) { return keys[a] < keys[b]; });
    // the passes over D, reading the stored site bytes of the whole map
    std::vector<I3> blocks((size_t)nb);
    for (int64_t i = 0; i < nb; ++i) blocks[i] = unpack_key(keys[i]);
    int* d_d = nullptr;
    KSG_CUDA(upload(tmp, d_list, s, &d_d));
    const EsdfOut eo{h->esdf_dist, h->esdf_flags, d_d, min_weight, max_distance};
    { const int rcp = esdf_passes(h, tmp, W, Rb, blocks, h->esdf_has_site, &d_list, h->esdf_site, eo, true, &st); if (rcp) return rcp; }
    KSG_CUDA(cudaStreamSynchronize(s));
  }
  h->esdf_full = false;
  h->esdf_valid = true;
  h->esdf_min_weight = min_weight;
  h->esdf_max_distance = max_distance;
  h->esdf_stamp = h->frame_stamp;
  h->esdf_blocks = nb;
  h->esdf_keys = std::move(keys);
  h->esdf_rewritten = std::move(d_list);
  if (stats) *stats = st;
  return KSG_OK;
}

int32_t ksg_export_esdf(ksg_integrator* h, int32_t changed_only, int64_t capacity_blocks, int64_t* n_blocks, int32_t* block_index,
                        float* distance, uint8_t* flags) {
  if (!h) return KSG_ERR_INVALID_ARGUMENT;
  if (!h->esdf_valid) return h->fail(KSG_ERR_INVALID_ARGUMENT, "esdf export: no ksg_update_esdf since the handle was created, cleared or reset");
  const std::vector<int> all = changed_only ? std::vector<int>() : zyx_order(h->esdf_keys);
  const std::vector<int>& list = changed_only ? h->esdf_rewritten : all;
  const int64_t n = (int64_t)list.size();
  if (n_blocks) *n_blocks = n;
  if (!block_index && !distance && !flags) return KSG_OK;
  if (n > capacity_blocks) return h->fail(KSG_ERR_INVALID_ARGUMENT, "esdf export: block capacity too small (n_blocks holds the need)");
  if (block_index) for (int64_t i = 0; i < n; ++i) put_block_index(block_index, i, h->esdf_keys[list[i]]);
  if ((!distance && !flags) || n == 0) return KSG_OK;
  KSG_CUDA(cudaSetDevice(h->device));
  const size_t V = (size_t)h->dc.vps * h->dc.vps * h->dc.vps;
  HostStaging st;
  const int* d_slots = nullptr; float* d_dist = nullptr; uint8_t* d_flags = nullptr;
  st.in(&d_slots, list.data(), (size_t)n);
  st.out(&d_dist, distance, n * V);
  st.out(&d_flags, flags, n * V);
  cudaStream_t s = h->own_stream;
  return st.run(h, s, [&] {
    ++h->n_launches;
    k_esdf_gather<<<esdf_grid(h, n), kEsdfThreads, 0, s>>>((int)V, d_slots, (int)n, h->esdf_dist, h->esdf_flags, d_dist, d_flags);
    return KSG_OK;
  });
}

namespace {
// *work = false: nothing to compute (n = 0 or no output wanted)
int esdf_query_args(ksg_integrator* h, int64_t n, const float* xyz, const ksg_esdf_query_out* o, bool* work) {
  if (!h) return KSG_ERR_INVALID_ARGUMENT;
  if (!o || n < 0) return h->fail(KSG_ERR_INVALID_ARGUMENT, "esdf query: NULL out or n < 0");
  if (n > 0 && !xyz) return h->fail(KSG_ERR_INVALID_ARGUMENT, "esdf query: NULL points");
  if (h->dc.shard_count > 1) return h->fail(KSG_ERR_INVALID_ARGUMENT, "esdf query: a sharded integrator holds only its own tiles");
  if (!h->esdf_valid) return h->fail(KSG_ERR_INVALID_ARGUMENT, "esdf query: no ksg_update_esdf since the handle was created, cleared or reset");
  *work = n > 0 && (o->flags || o->voxel_flags || o->voxel_distance || o->distance || o->gradient);
  return KSG_OK;
}
void launch_esdf_query(ksg_integrator* h, int64_t n, const float* d_xyz, const ksg_esdf_query_out& o, cudaStream_t s) {
  static_assert(sizeof(ksg_esdf_query_out) == sizeof(EsdfQueryOut), "ksg_esdf_query_out layout");
  const EsdfQueryOut q{o.flags, o.voxel_flags, o.voxel_distance, o.distance, o.gradient};
  const EsdfLayer layer{h->esdf_dist, h->esdf_flags, (int)h->esdf_blocks};
  const int grid = (int)std::min<int64_t>((n + kQueryThreads - 1) / kQueryThreads, (int64_t)h->sm_count * 8);
  ++h->n_launches;
  k_query_esdf<<<grid, kQueryThreads, 0, s>>>(h->dc, h->map, layer, d_xyz, (long long)n, q, (o.flags || o.distance) ? 1 : 0,
                                              (o.flags || o.gradient) ? 1 : 0);
}
}  // namespace

int32_t ksg_query_esdf(ksg_integrator* h, int64_t n, const float* xyz_G, const ksg_esdf_query_out* out) {
  bool work = false;
  { const int rca = esdf_query_args(h, n, xyz_G, out, &work); if (rca) return rca; }
  { const int rcp = complete_frames(h); if (rcp) return rcp; }
  if (!work) return KSG_OK;
  const size_t N = (size_t)n;
  HostStaging st;
  const float* d_xyz = nullptr;
  ksg_esdf_query_out dq{};
  st.in(&d_xyz, xyz_G, 3 * N);
  st.out(&dq.flags, out->flags, N);
  st.out(&dq.voxel_flags, out->voxel_flags, N);
  st.out(&dq.voxel_distance, out->voxel_distance, N);
  st.out(&dq.distance, out->distance, N);
  st.out(&dq.gradient, out->gradient, 3 * N);
  cudaStream_t s = h->own_stream;
  return st.run(h, s, [&] { launch_esdf_query(h, n, d_xyz, dq, s); return KSG_OK; });
}

int32_t ksg_query_esdf_device(ksg_integrator* h, int64_t n, const float* d_xyz_G, const ksg_esdf_query_out* d_out, void* cuda_stream) {
  bool work = false;
  { const int rca = esdf_query_args(h, n, d_xyz_G, d_out, &work); if (rca) return rca; }
  if (h->deferred_status) return h->fail(h->deferred_status, err_text(h->deferred_status));
  if (!work) return KSG_OK;
  KSG_CUDA(cudaSetDevice(h->device));
  launch_esdf_query(h, n, d_xyz_G, *d_out, cuda_stream ? (cudaStream_t)cuda_stream : h->own_stream);
  KSG_CUDA(cudaGetLastError());
  return KSG_OK;
}

int32_t ksg_sync(ksg_integrator* h) {
  if (!h) return KSG_ERR_INVALID_ARGUMENT;
  { const int rcp = complete_frames(h); if (rcp) return rcp; }
  if (h->deferred_status) return h->fail(h->deferred_status, err_text(h->deferred_status));
  return KSG_OK;
}

int64_t ksg_num_blocks(ksg_integrator* h) {
  if (!h) return 0;
  if (h->n_pend > 0) { cudaSetDevice(h->device); finish_frame(h, nullptr); }
  return h->num_blocks;
}

static int export_slots(ksg_integrator* h, const std::vector<int>& slots, float* tsdf_distance, float* tsdf_weight,
                        uint8_t* tsdf_rgba, uint8_t* sem_label, float* sem_priors, uint8_t* sem_rgba) {
  const int64_t nb = (int64_t)slots.size();
  if (nb == 0) return KSG_OK;
  const DevCfg& dc = h->dc;
  const BlockStaging st(dc, nb);
  const size_t VB = st.VB;
  { const int rcs = st.ensure(h, (size_t)st.batch * st.per_block); if (rcs) return rcs; }
  for (int64_t b0 = 0; b0 < nb; b0 += st.batch) {
    const int64_t cnt = std::min(st.batch, nb - b0);
    KSG_CUDA(cudaMemcpy(h->d_exp_slots, slots.data() + b0, sizeof(int) * cnt, cudaMemcpyHostToDevice));
    const BlockStaging::Parts o = st.at(h->d_exp, cnt);
    k_export<<<h->sm_count * 4, 256, 0, h->own_stream>>>(dc, h->map, h->d_exp_slots, (int)cnt, tsdf_distance ? o.dist : nullptr,
                                                         tsdf_weight ? o.wgt : nullptr, tsdf_rgba ? o.rgba : nullptr,
                                                         sem_label ? o.label : nullptr, sem_priors ? o.prior : nullptr,
                                                         sem_rgba ? o.srgba : nullptr);
    KSG_CUDA(cudaStreamSynchronize(h->own_stream));
    if (tsdf_distance) KSG_CUDA(cudaMemcpy(tsdf_distance + b0 * VB, o.dist, cnt * VB * 4, cudaMemcpyDeviceToHost));
    if (tsdf_weight) KSG_CUDA(cudaMemcpy(tsdf_weight + b0 * VB, o.wgt, cnt * VB * 4, cudaMemcpyDeviceToHost));
    if (tsdf_rgba) KSG_CUDA(cudaMemcpy(tsdf_rgba + b0 * VB * 4, o.rgba, cnt * VB * 4, cudaMemcpyDeviceToHost));
    if (sem_rgba) KSG_CUDA(cudaMemcpy(sem_rgba + b0 * VB * 4, o.srgba, cnt * VB * 4, cudaMemcpyDeviceToHost));
    if (sem_label) KSG_CUDA(cudaMemcpy(sem_label + b0 * VB, o.label, cnt * VB, cudaMemcpyDeviceToHost));
    if (sem_priors) KSG_CUDA(cudaMemcpy(sem_priors + b0 * VB * dc.C, o.prior, cnt * VB * 4 * dc.C, cudaMemcpyDeviceToHost));
  }
  return KSG_OK;
}

int32_t ksg_export_blocks(ksg_integrator* h, int64_t capacity_blocks, int32_t* block_index, float* tsdf_distance,
                          float* tsdf_weight, uint8_t* tsdf_rgba, uint8_t* sem_label, float* sem_priors, uint8_t* sem_rgba) {
  if (!h) return KSG_ERR_INVALID_ARGUMENT;
  KSG_CUDA(cudaSetDevice(h->device));
  KSG_CUDA(cudaDeviceSynchronize());
  finish_frame(h, nullptr);
  const int64_t nb = h->num_blocks;
  if (nb > capacity_blocks) return h->fail(KSG_ERR_INVALID_ARGUMENT, "export capacity too small");
  if (nb == 0) return KSG_OK;
  std::vector<int> order;
  { const int rco = slots_zyx(h, &order, block_index); if (rco) return rco; }
  if (!tsdf_distance && !tsdf_weight && !tsdf_rgba && !sem_label && !sem_priors && !sem_rgba) return KSG_OK;
  return export_slots(h, order, tsdf_distance, tsdf_weight, tsdf_rgba, sem_label, sem_priors, sem_rgba);
}

int32_t ksg_export_blocks_by_index(ksg_integrator* h, int64_t n, const int32_t* block_index, uint8_t* found, float* tsdf_distance,
                                   float* tsdf_weight, uint8_t* tsdf_rgba, uint8_t* sem_label, float* sem_priors, uint8_t* sem_rgba) {
  if (!h || n < 0 || (n > 0 && !block_index)) return KSG_ERR_INVALID_ARGUMENT;
  if (n == 0) return KSG_OK;
  KSG_CUDA(cudaSetDevice(h->device));
  KSG_CUDA(cudaDeviceSynchronize());
  finish_frame(h, nullptr);
  HostBlockTable table;
  { const int rct = table.load(h); if (rct) return rct; }
  std::vector<int> slots;
  std::vector<int64_t> where;
  for (int64_t i = 0; i < n; ++i) {
    I3 b; b.x = block_index[3 * i]; b.y = block_index[3 * i + 1]; b.z = block_index[3 * i + 2];
    const int slot = key_in_range(b) ? table.find(pack_key(b)) : -1;
    if (found) found[i] = slot >= 0 ? 1 : 0;
    if (slot >= 0) { slots.push_back(slot); where.push_back(i); }
  }
  if (slots.empty()) return KSG_OK;
  const size_t VB = (size_t)h->dc.vps * h->dc.vps * h->dc.vps;
  const size_t C = (size_t)h->dc.C;
  const bool dense = (int64_t)slots.size() == n;
  if (dense) return export_slots(h, slots, tsdf_distance, tsdf_weight, tsdf_rgba, sem_label, sem_priors, sem_rgba);
  // sparse hit list: export compactly, then scatter to the callers positions
  const size_t m = slots.size();
  std::vector<float> d(tsdf_distance ? m * VB : 0), w(tsdf_weight ? m * VB : 0), pr(sem_priors ? m * VB * C : 0);
  std::vector<uint8_t> c1(tsdf_rgba ? m * VB * 4 : 0), c2(sem_rgba ? m * VB * 4 : 0), lb(sem_label ? m * VB : 0);
  int rc = export_slots(h, slots, tsdf_distance ? d.data() : nullptr, tsdf_weight ? w.data() : nullptr, tsdf_rgba ? c1.data() : nullptr,
                        sem_label ? lb.data() : nullptr, sem_priors ? pr.data() : nullptr, sem_rgba ? c2.data() : nullptr);
  if (rc) return rc;
  for (size_t k = 0; k < m; ++k) {
    const size_t i = (size_t)where[k];
    if (tsdf_distance) std::memcpy(tsdf_distance + i * VB, d.data() + k * VB, VB * 4);
    if (tsdf_weight) std::memcpy(tsdf_weight + i * VB, w.data() + k * VB, VB * 4);
    if (tsdf_rgba) std::memcpy(tsdf_rgba + i * VB * 4, c1.data() + k * VB * 4, VB * 4);
    if (sem_rgba) std::memcpy(sem_rgba + i * VB * 4, c2.data() + k * VB * 4, VB * 4);
    if (sem_label) std::memcpy(sem_label + i * VB, lb.data() + k * VB, VB);
    if (sem_priors) std::memcpy(sem_priors + i * VB * C, pr.data() + k * VB * C, VB * C * 4);
  }
  return KSG_OK;
}

int32_t ksg_import_blocks(ksg_integrator* h, int64_t n, const int32_t* block_index, const float* tsdf_distance, const float* tsdf_weight,
                          const uint8_t* tsdf_rgba, const uint8_t* sem_label, const float* sem_priors, const uint8_t* sem_rgba) {
  if (!h || n < 0 || (n > 0 && !block_index)) return KSG_ERR_INVALID_ARGUMENT;
  if (h->deferred_status) return h->fail(h->deferred_status, err_text(h->deferred_status));
  if (n == 0) return KSG_OK;
  { const int rcp = complete_frames(h); if (rcp) return rcp; }
  h->esdf_full = true;     // the import writes blocks without stamping them
  h->mesh_full = true;
  const DevCfg& dc = h->dc;
  HostBlockTable table;
  { const int rct = table.load(h); if (rct) return rct; }
  std::vector<int> slots((size_t)n);
  std::vector<uint8_t> fresh((size_t)n, 0);
  std::vector<uint64_t> new_keys;
  int64_t nb = h->num_blocks;
  for (int64_t i = 0; i < n; ++i) {
    I3 b; b.x = block_index[3 * i]; b.y = block_index[3 * i + 1]; b.z = block_index[3 * i + 2];
    if (!key_in_range(b)) return h->fail(KSG_ERR_INDEX_RANGE, err_text(5));
    const uint64_t key = pack_key(b);
    const int64_t before = nb;
    slots[i] = table.find_or_insert(key, &nb, h->map.max_blocks);
    if (slots[i] < 0) return h->fail(KSG_ERR_POOL_FULL, err_text(3));
    if (nb != before) { fresh[i] = 1; new_keys.push_back(key); }
  }
  if (!new_keys.empty()) {
    { const int rct = table.store(h); if (rct) return rct; }
    KSG_CUDA(cudaMemcpy(h->map.slot_key + h->num_blocks, new_keys.data(), sizeof(uint64_t) * new_keys.size(), cudaMemcpyHostToDevice));
    const int pc = (int)nb;
    KSG_CUDA(cudaMemcpy(&h->d_cnt->pool_count, &pc, sizeof(int), cudaMemcpyHostToDevice));
    h->num_blocks = nb;
  }
  const BlockStaging st(dc, n);
  const size_t VB = st.VB;
  { const int rcs = st.ensure(h, (size_t)st.batch * st.per_block + (size_t)st.batch); if (rcs) return rcs; }
  for (int64_t b0 = 0; b0 < n; b0 += st.batch) {
    const int64_t cnt = std::min(st.batch, n - b0);
    KSG_CUDA(cudaMemcpy(h->d_exp_slots, slots.data() + b0, sizeof(int) * cnt, cudaMemcpyHostToDevice));
    const BlockStaging::Parts i = st.at(h->d_exp, cnt);
    if (tsdf_distance) KSG_CUDA(cudaMemcpy(i.dist, tsdf_distance + b0 * VB, cnt * VB * 4, cudaMemcpyHostToDevice));
    if (tsdf_weight) KSG_CUDA(cudaMemcpy(i.wgt, tsdf_weight + b0 * VB, cnt * VB * 4, cudaMemcpyHostToDevice));
    if (tsdf_rgba) KSG_CUDA(cudaMemcpy(i.rgba, tsdf_rgba + b0 * VB * 4, cnt * VB * 4, cudaMemcpyHostToDevice));
    if (sem_rgba) KSG_CUDA(cudaMemcpy(i.srgba, sem_rgba + b0 * VB * 4, cnt * VB * 4, cudaMemcpyHostToDevice));
    if (sem_label) KSG_CUDA(cudaMemcpy(i.label, sem_label + b0 * VB, cnt * VB, cudaMemcpyHostToDevice));
    if (sem_priors) KSG_CUDA(cudaMemcpy(i.prior, sem_priors + b0 * VB * dc.C, cnt * VB * 4 * dc.C, cudaMemcpyHostToDevice));
    KSG_CUDA(cudaMemcpy(i.fresh, fresh.data() + b0, cnt, cudaMemcpyHostToDevice));
    k_import<<<h->sm_count * 4, 256, 0, h->own_stream>>>(dc, h->map, h->d_exp_slots, i.fresh, (int)cnt, tsdf_distance ? i.dist : nullptr,
                                                         tsdf_weight ? i.wgt : nullptr, tsdf_rgba ? i.rgba : nullptr,
                                                         sem_label ? i.label : nullptr, sem_priors ? i.prior : nullptr,
                                                         sem_rgba ? i.srgba : nullptr);
    KSG_CUDA(cudaStreamSynchronize(h->own_stream));
  }
  return KSG_OK;
}

int32_t ksg_device_map_view(ksg_integrator* h, int64_t* n_blocks, int64_t* block_stride_bytes, void** d_pool, void** d_block_keys) {
  if (!h) return KSG_ERR_INVALID_ARGUMENT;
  { const int rcp = complete_frames(h); if (rcp) return rcp; }
  if (n_blocks) *n_blocks = h->num_blocks;
  if (block_stride_bytes) *block_stride_bytes = (int64_t)h->dc.block_stride;
  if (d_pool) *d_pool = h->map.pool;
  if (d_block_keys) *d_block_keys = h->map.slot_key;
  return KSG_OK;
}

int32_t ksg_copy_map_device(ksg_integrator* h, void* d_dst_pool, void* d_dst_keys, void* stream) {
  if (!h || !d_dst_pool || !d_dst_keys) return KSG_ERR_INVALID_ARGUMENT;
  KSG_CUDA(cudaSetDevice(h->device));
  { const int rcp = finish_frame(h, nullptr); if (rcp) return rcp; }
  cudaStream_t s = stream ? (cudaStream_t)stream : h->own_stream;
  if (h->num_blocks > 0) {
    KSG_CUDA(cudaMemcpyAsync(d_dst_pool, h->map.pool, (size_t)h->num_blocks * (size_t)h->dc.block_stride, cudaMemcpyDeviceToDevice, s));
    KSG_CUDA(cudaMemcpyAsync(d_dst_keys, h->map.slot_key, (size_t)h->num_blocks * sizeof(uint64_t), cudaMemcpyDeviceToDevice, s));
  }
  return KSG_OK;
}

int32_t ksg_merge_blocks_device(ksg_integrator* h, int64_t n_blocks, const void* d_block_keys, const void* d_pool_src, void* stream) {
  if (!h || n_blocks < 0 || (n_blocks > 0 && (!d_block_keys || !d_pool_src))) return KSG_ERR_INVALID_ARGUMENT;
  if (h->deferred_status) return h->fail(h->deferred_status, err_text(h->deferred_status));
  if (n_blocks == 0) return KSG_OK;
  KSG_CUDA(cudaSetDevice(h->device));
  { const int rcp = finish_frame(h, nullptr); if (rcp) return rcp; }
  cudaStream_t s = stream ? (cudaStream_t)stream : h->own_stream;
  if (h->exp_slots_cap < n_blocks) {
    KSG_CUDA(cudaStreamSynchronize(s));
    KSG_CUDA(h->res.regrow(&h->d_exp_slots, &h->exp_slots_cap, (size_t)n_blocks));
  }
  h->frame_stamp += 1;
  h->n_launches += 5;
  k_frame_reset<<<1, 1, 0, s>>>(h->d_cnt, 0);
  k_merge_insert<<<grid_for(n_blocks, 256), 256, 0, s>>>(h->d_cnt, h->map, (const uint64_t*)d_block_keys, (int)n_blocks, h->d_exp_slots, h->frame_stamp);
  k_block_init<<<h->sm_count * 4, 256, 0, s>>>(h->dc, h->d_cnt, h->map);
  k_frame_finish<<<1, 1, 0, s>>>(h->d_cnt, h->map);
  k_merge_tiles<<<h->sm_count * 8, 256, 0, s>>>(h->dc, h->d_cnt, h->map, h->d_luts, h->d_exp_slots, (const uint8_t*)d_pool_src, (int)n_blocks);
  return finish_sync(h, s);
}

int32_t ksg_copy_update_log_device(ksg_integrator* h, int64_t* n_out, void* d_dst_updates, void* d_dst_priors, int64_t capacity, void* stream) {
  if (!h || !n_out) return KSG_ERR_INVALID_ARGUMENT;
  *n_out = 0;
  if (!h->d_log_head) return h->fail(KSG_ERR_INVALID_ARGUMENT, "update log is off (ksg_set_update_log)");
  KSG_CUDA(cudaSetDevice(h->device));
  { const int rcp = finish_frame(h, nullptr); if (rcp) return rcp; }
  const int64_t n = update_log_count(h);
  if (n > h->log_cap) { *n_out = -1; return h->fail(KSG_ERR_SCRATCH_FULL, "update log too small for this frame"); }
  *n_out = n;
  if (!d_dst_updates && !d_dst_priors) return KSG_OK;                 // size query
  if (n > capacity) return h->fail(KSG_ERR_INVALID_ARGUMENT, "update log copy: capacity too small");
  cudaStream_t s = stream ? (cudaStream_t)stream : h->own_stream;
  if (n > 0) {
    if (d_dst_updates) KSG_CUDA(cudaMemcpyAsync(d_dst_updates, h->d_log_head, (size_t)n * sizeof(VoxelUpdate), cudaMemcpyDeviceToDevice, s));
    if (d_dst_priors) KSG_CUDA(cudaMemcpyAsync(d_dst_priors, h->d_log_prior, (size_t)n * sizeof(float) * h->dc.C, cudaMemcpyDeviceToDevice, s));
  }
  return KSG_OK;
}

int32_t ksg_merge_voxels_device(ksg_integrator* h, int32_t n_deltas, const int64_t* counts, int64_t stride, const void* d_updates, const void* d_priors,
                                void* stream) {
  if (!h || n_deltas < 0 || n_deltas > 16 || stride < 0 || (n_deltas > 0 && (!counts || !d_updates || !d_priors))) return KSG_ERR_INVALID_ARGUMENT;
  if (h->deferred_status) return h->fail(h->deferred_status, err_text(h->deferred_status));
  MergeCounts mc{};
  int64_t any = 0;
  for (int g = 0; g < n_deltas; ++g) {
    if (counts[g] < 0 || counts[g] > stride || counts[g] > 0x7fffffff) return KSG_ERR_INVALID_ARGUMENT;
    mc.n[g] = (int)counts[g];
    any += counts[g];
  }
  if (any == 0) return KSG_OK;
  KSG_CUDA(cudaSetDevice(h->device));
  { const int rcp = finish_frame(h, nullptr); if (rcp) return rcp; }
  cudaStream_t s = stream ? (cudaStream_t)stream : h->own_stream;
  const int64_t total = (int64_t)n_deltas * stride;
  if (total > 0x7fffffff) return h->fail(KSG_ERR_INVALID_ARGUMENT, "merge: n_deltas * stride_entries exceeds 2^31 - 1");
  if (h->exp_slots_cap < total) {
    KSG_CUDA(cudaStreamSynchronize(s));
    KSG_CUDA(h->res.regrow(&h->d_exp_slots, &h->exp_slots_cap, (size_t)total));
  }
  h->frame_stamp += 1;
  h->n_launches += 4 + n_deltas;
  const VoxelUpdate* upd = (const VoxelUpdate*)d_updates;
  const float* pri = (const float*)d_priors;
  k_frame_reset<<<1, 1, 0, s>>>(h->d_cnt, 0);
  k_mergev_insert<<<grid_for(total, 256), 256, 0, s>>>(h->d_cnt, h->map, upd, mc, n_deltas, (long long)stride, h->d_exp_slots, h->frame_stamp);
  k_block_init<<<h->sm_count * 4, 256, 0, s>>>(h->dc, h->d_cnt, h->map);
  k_frame_finish<<<1, 1, 0, s>>>(h->d_cnt, h->map);
  for (int g = 0; g < n_deltas; ++g) {      // frame order: a voxel that several deltas touched is merged delta by delta
    if (mc.n[g] == 0) continue;
    const int grid = (int)std::min<int64_t>((int64_t)h->sm_count * 16, (mc.n[g] + 7) / 8);
    k_mergev_apply<<<std::max(1, grid), 256, 0, s>>>(h->dc, h->map, h->d_luts, upd + (size_t)g * stride, pri + (size_t)g * stride * h->dc.C,
                                                    h->d_exp_slots + (size_t)g * stride, mc.n[g]);
  }
  return finish_sync(h, s);
}

int64_t ksg_last_updated_blocks(ksg_integrator* h, int64_t capacity_blocks, int32_t* block_index) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  if (h->n_pend > 0) finish_frame(h, nullptr);
  const int64_t n = h->last_blocks_touched;
  if (!block_index || capacity_blocks < n || n == 0) return n;
  cudaDeviceSynchronize();
  std::vector<int> pos((size_t)n);
  if (cudaMemcpy(pos.data(), h->map.touched_list, sizeof(int) * n, cudaMemcpyDeviceToHost) != cudaSuccess) return 0;
  std::vector<uint64_t> all((size_t)h->ht_cap);
  if (cudaMemcpy(all.data(), h->map.ht_keys, sizeof(uint64_t) * h->ht_cap, cudaMemcpyDeviceToHost) != cudaSuccess) return 0;
  std::vector<uint64_t> keys((size_t)n);
  for (int64_t i = 0; i < n; ++i) keys[i] = all[pos[i]];
  std::sort(keys.begin(), keys.end());   // (z, y, x) order
  for (int64_t i = 0; i < n; ++i) put_block_index(block_index, i, keys[i]);
  return n;
}

int64_t ksg_unordered_map_schedule(int64_t n, int64_t* bucket_count_after_insert) {
  if (n < 0 || (n > 0 && !bucket_count_after_insert)) return -1;
  std::unordered_map<uint64_t, char> probe;
  for (int64_t i = 0; i < n; ++i) {
    probe.emplace((uint64_t)i, 0);
    bucket_count_after_insert[i] = (int64_t)probe.bucket_count();
  }
  return n;
}

int32_t ksg_owner_mask(int32_t voxels_per_side, int32_t shard_rank, int32_t shard_count, int64_t n, const int32_t* block_index,
                       uint8_t* mask) {
  const int vps = voxels_per_side;
  if (vps <= 0 || (vps & (vps - 1)) || n < 0 || (n > 0 && (!block_index || !mask))) return KSG_ERR_INVALID_ARGUMENT;
  const int count = shard_count > 1 ? shard_count : 1;
  if (shard_rank < 0 || shard_rank >= count) return KSG_ERR_INVALID_ARGUMENT;
  const int T = std::min(vps, kTileSideMax), tps = vps / T;
  const size_t V = (size_t)vps * vps * vps;
  for (int64_t b = 0; b < n; ++b) {
    I3 bi; bi.x = block_index[3 * b]; bi.y = block_index[3 * b + 1]; bi.z = block_index[3 * b + 2];
    const uint64_t key = pack_key(bi);
    for (int z = 0; z < vps; ++z)
      for (int y = 0; y < vps; ++y)
        for (int x = 0; x < vps; ++x) {
          const int tile = (x / T) + tps * ((y / T) + tps * (z / T));
          mask[b * V + (size_t)x + (size_t)vps * ((size_t)y + (size_t)vps * z)] = tile_owner(key, tile, count) == shard_rank ? 1 : 0;
        }
  }
  return KSG_OK;
}

int32_t ksg_set_profiling(ksg_integrator* h, int32_t enable) {
  if (!h) return KSG_ERR_INVALID_ARGUMENT;
  cudaSetDevice(h->device);
  if (enable && !h->ev[0]) for (auto& e : h->ev) h->res.event(&e, cudaEventDefault);
  h->profiling = enable != 0;
  for (double& m : h->phase_ms) m = 0.0;
  h->prof_frames = 0; h->n_launches = 0; h->n_libcalls = 0;
  return KSG_OK;
}
int32_t ksg_get_profile(ksg_integrator* h, double* phase_ms, int64_t* frames, int64_t* kernel_launches, int64_t* library_calls) {
  if (!h) return KSG_ERR_INVALID_ARGUMENT;
  if (phase_ms) for (int p = 0; p < KSG_NUM_PHASES; ++p) phase_ms[p] = h->phase_ms[p];
  if (frames) *frames = h->prof_frames;
  if (kernel_launches) *kernel_launches = h->n_launches;
  if (library_calls) *library_calls = h->n_libcalls;
  return KSG_OK;
}

namespace {
__global__ void k_chain_debug(const float* __restrict__ terms, long long n, float s0, float* __restrict__ out) {
  const float s = chain_sum_warp(s0, terms, n);
  if ((threadIdx.x & 31) == 0) *out = s;
}
}  // namespace

int32_t ksg_debug_chain_sum(const float* terms, int64_t n, float s0, float* result) {
  if (n < 0 || (n > 0 && !terms) || !result || !(s0 < 0.0f)) return KSG_ERR_INVALID_ARGUMENT;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { cudaGetLastError(); return KSG_ERR_NO_DEVICE; }
  Resources tmp;
  float *d_terms = nullptr, *d_out = nullptr;
  int32_t rc = KSG_ERR_CUDA;
  if (tmp.device(&d_terms, (size_t)n) == cudaSuccess && tmp.device(&d_out, 1) == cudaSuccess &&
      (n == 0 || cudaMemcpy(d_terms, terms, sizeof(float) * (size_t)n, cudaMemcpyHostToDevice) == cudaSuccess)) {
    k_chain_debug<<<1, 32>>>(d_terms, (long long)n, s0, d_out);
    if (cudaMemcpy(result, d_out, sizeof(float), cudaMemcpyDeviceToHost) == cudaSuccess) rc = KSG_OK;
  }
  return rc;
}

namespace {
// one warp, the batch loop of k_voxel_apply_long's TSDF role with the measurements (sdf, uw, colour) given instead of computed
__global__ void k_tsdf_batch_debug(TsdfParams tp, int wide, long long n, const float* __restrict__ sdf, const float* __restrict__ uw,
                                   const uint32_t* __restrict__ col, int keep_blend, float* dist_io, float* wgt_io, uint32_t* rgba_io) {
  const int lane = threadIdx.x & 31;
  float dist = *dist_io, wgt = *wgt_io;
  uint32_t rgba = *rgba_io;
  __syncwarp();
  for (long long base = 0; base < n; base += 32) {
    const int nb = (n - base) < 32 ? (int)(n - base) : 32;
    const float s = (lane < nb) ? sdf[base + lane] : 0.0f;
    const float u = (lane < nb) ? uw[base + lane] : 0.0f;
    const uint32_t c = (col && lane < nb) ? col[base + lane] : 0u;
    if (wide) tsdf_batch<true>(tp, lane, nb, s, u, c, keep_blend != 0, dist, wgt, rgba);
    else tsdf_batch<false>(tp, lane, nb, s, u, c, keep_blend != 0, dist, wgt, rgba);
  }
  if (lane == 0) { *dist_io = dist; *wgt_io = wgt; *rgba_io = rgba; }
}
}  // namespace

int32_t ksg_debug_tsdf_batch(const ksg_config* cfg, int32_t wide, int64_t n, const float* sdf, const float* uw, const uint32_t* rgba_in,
                             int32_t keep_blend, float* dist, float* wgt, uint32_t* rgba) {
  if (!cfg || n < 0 || (n > 0 && (!sdf || !uw)) || !dist || !wgt || !rgba) return KSG_ERR_INVALID_ARGUMENT;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { cudaGetLastError(); return KSG_ERR_NO_DEVICE; }
  TsdfParams tp{};
  tp.voxel_size = cfg->voxel_size; tp.trunc = cfg->default_truncation_distance; tp.max_weight = cfg->max_weight;
  tp.sparsity_factor = cfg->sparsity_compensation_factor;
  tp.use_weight_dropoff = cfg->use_weight_dropoff; tp.use_sparsity = cfg->use_sparsity_compensation_factor;
  // one buffer: [sdf n][uw n][colour n][dist, weight, rgba]
  const size_t m = (size_t)std::max<int64_t>(n, 1);
  Resources tmp;
  uint32_t* d = nullptr;
  int32_t rc = KSG_ERR_CUDA;
  if (tmp.device(&d, 3 * m + 3) == cudaSuccess) {
    float* d_sdf = (float*)d; float* d_uw = (float*)(d + m); uint32_t* d_col = d + 2 * m; uint32_t* d_state = d + 3 * m;
    uint32_t state[3];
    std::memcpy(&state[0], dist, 4); std::memcpy(&state[1], wgt, 4); state[2] = *rgba;
    bool ok = cudaMemcpy(d_state, state, sizeof(state), cudaMemcpyHostToDevice) == cudaSuccess;
    if (n > 0) {
      ok = ok && cudaMemcpy(d_sdf, sdf, sizeof(float) * (size_t)n, cudaMemcpyHostToDevice) == cudaSuccess &&
           cudaMemcpy(d_uw, uw, sizeof(float) * (size_t)n, cudaMemcpyHostToDevice) == cudaSuccess &&
           (!rgba_in || cudaMemcpy(d_col, rgba_in, sizeof(uint32_t) * (size_t)n, cudaMemcpyHostToDevice) == cudaSuccess);
    }
    if (ok) {
      k_tsdf_batch_debug<<<1, 32>>>(tp, wide, (long long)n, d_sdf, d_uw, rgba_in ? d_col : nullptr, keep_blend, (float*)d_state,
                                    (float*)(d_state + 1), d_state + 2);
      if (cudaMemcpy(state, d_state, sizeof(state), cudaMemcpyDeviceToHost) == cudaSuccess) {
        std::memcpy(dist, &state[0], 4); std::memcpy(wgt, &state[1], 4); *rgba = state[2];
        rc = KSG_OK;
      }
    }
  }
  return rc;
}

int32_t ksg_debug_apply_routes(ksg_integrator* h, int64_t* out4) {
  if (!h || !out4) return KSG_ERR_INVALID_ARGUMENT;
  KSG_CUDA(cudaSetDevice(h->device));
  KSG_CUDA(cudaDeviceSynchronize());
  for (int i = 0; i < 4; ++i) out4[i] = 0;
  if (h->last_frame_queued) {
    int c[3] = {0, 0, 0};
    KSG_CUDA(cudaMemcpy(c, h->vq.counters, sizeof(c), cudaMemcpyDeviceToHost));
    out4[0] = c[0] / 2; out4[1] = c[1] / 2; out4[2] = c[2];   // a long voxel is two items, one per role
  }
  if (h->hot_enabled && h->cfg.hot_voxel_mode == 2 && h->last_hot_segments > 0) {
    std::vector<int> same((size_t)h->last_hot_segments);
    KSG_CUDA(cudaMemcpy(same.data(), h->d_hot_same, sizeof(int) * same.size(), cudaMemcpyDeviceToHost));
    for (int v : same) out4[3] += v != 0;
  }
  return KSG_OK;
}

int64_t ksg_debug_tile_times(ksg_integrator* h, int32_t enable, int64_t capacity, int64_t* records_and_cycles) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  if (enable && !h->tile_debug) {
    if (h->res.device(&h->tile_debug, 2 * (size_t)h->tile_cap) != cudaSuccess) { h->tile_debug = nullptr; return 0; }
  }
  const int64_t n = std::min<int64_t>(h->h_cnt->n_tiles, h->tile_cap);
  if (h->tile_debug && records_and_cycles && capacity >= n && n > 0)
    cudaMemcpy(records_and_cycles, h->tile_debug, sizeof(long long) * 2 * n, cudaMemcpyDeviceToHost);
  if (!enable && h->tile_debug) { h->res.release(h->tile_debug); h->tile_debug = nullptr; }
  return n;
}

int64_t ksg_debug_fast_timeline(ksg_integrator* h, int64_t* out64, int64_t* sweeps, double* clock_khz) {
  if (!h || !out64 || !h->h_fc) return 0;
  cudaSetDevice(h->device);
  if (h->n_pend > 0) finish_frame(h, nullptr);
  for (int i = 0; i < kTimelineSlots; ++i) out64[i] = (int64_t)h->h_fc->timeline[i];
  for (int i = 0; i < 16; ++i) out64[kTimelineSlots + i] = (int64_t)h->h_fc->dbg[i];
  if (sweeps) *sweeps = h->h_fc->sweeps_last;
  if (clock_khz) *clock_khz = h->clock_khz;
  return kTimelineSlots + 16;
}

int32_t ksg_clear_map(ksg_integrator* h) {
  if (!h) return KSG_ERR_INVALID_ARGUMENT;
  { const int rcp = complete_frames(h); if (rcp) return rcp; }
  cudaStream_t s = h->own_stream;
  KSG_CUDA(cudaMemsetAsync(h->map.ht_keys, 0xFF, sizeof(uint64_t) * h->ht_cap, s));
  KSG_CUDA(cudaMemsetAsync(h->map.ht_slot, 0xFF, sizeof(int) * h->ht_cap, s));
  KSG_CUDA(cudaMemsetAsync(h->map.touched_stamp, 0, sizeof(int) * h->ht_cap, s));
  if (h->tile_cnt) KSG_CUDA(cudaMemsetAsync(h->tile_cnt, 0, sizeof(int) * (size_t)h->ht_cap * h->dc.tiles_per_block, s));
  // the block pool restarts at slot 0; everything else in the counter block is per frame (rewritten by the next frame's first kernel)
  // or belongs to the integrator (sweep ids of the observed-set solver, which the slot stamps refer to) and stays
  KSG_CUDA(cudaMemsetAsync(&h->d_cnt->pool_count, 0, sizeof(int), s));
  KSG_CUDA(cudaMemsetAsync(&h->d_cnt->n_blocks_touched, 0, sizeof(int), s));
  KSG_CUDA(cudaMemsetAsync(&h->d_cnt->n_new_blocks, 0, sizeof(int), s));
  h->num_blocks = 0;
  h->last_blocks_touched = 0;
  h->esdf_full = true;     // the stamps restart at 0 while frame_stamp does not, and the slots are reused
  h->esdf_valid = false;
  h->mesh_full = true;
  h->mesh_valid = false;
  KSG_CUDA(cudaStreamSynchronize(s));
  return KSG_OK;
}

int32_t ksg_reset(ksg_integrator* h) {
  if (!h) return KSG_ERR_INVALID_ARGUMENT;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  h->n_pend = 0;
  return reset_map(h, h->own_stream);
}

}  // extern "C"
