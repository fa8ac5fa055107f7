// ksg_fast3.cuh — the `fast` integrator's observed-set solver, k_fast_solve3.
//
// voxel_observed_approx_set_ (fast.cpp:110-122, A.4) solved as a fixpoint:
//   candidates  = ray steps materialised so far (the first kH0 of every cast ray, further steps of a ray once it is found to
//                 survive that far),
//   U[r]        = number of voxels ray r updates (= index of the step at which it breaks),
//   a candidate (r,s) "collides" iff the latest PERFORMED candidate (s' < U[r']) that precedes it in (rank, step) order on the
//   same slot carries the same value (none: the persistent table decides).
// The dependency is triangular in rank order, so the fixpoint is unique (DESIGN.md section 4); sweeps re-evaluate rays until no
// U changes, and in-place / asynchronous updates only accelerate convergence.  None of the following alters the fixpoint:
//   1. WORKLIST.  Sweeps 1 to 3 scan every ray; a later sweep k+1 scans only the rays evaluated in sweep k and the rays that
//      examined a slot another ray toggled in sweep k (the slot's highest-ranked toggler of the sweep walks its bucket and
//      overflow chain and lists them).  Every examined step is in its slot's bucket: performed steps as usual, the break step as
//      a perf-0 entry.  Warps claim the rays of a sweep one at a time from a shared cursor, so a sweep ends with its last ray,
//      not with the unluckiest warp.
//   2. one 16-byte record per candidate {packed voxel index, bucket position, block of the voxel (see Cand)} and one per ray
//      {materialised steps, updates, length, last evaluation}: one load each; the set value (hash + offset) is recomputed from the
//      voxel index; flipping a candidate's "performed" bit is a plain store (the owner knows the whole entry).
//   3. per-slot toggle stamps (stamp_toggle): a ray is NOT dirty when the only toggle of the slot in its last sweep was its own.
//   4. no record buffer: after convergence the performed candidates are walked twice, fully parallel (8 lanes per ray):
//      pass 1 commits the persistent table, allocates blocks and counts records per tile; pass 2 writes the (voxel, rank) keys
//      straight into the tile's segment.  The voxel index kept per candidate replaces a second ray walk, and the block's hash
//      position that pass 1 leaves in the candidate's tog word replaces a second probe of the block table.
#pragma once
#include <cuda/atomic>
#include "ksg_fast.cuh"

namespace ksg {

// pos: >= 0 bucket entry, -2 not inserted, <= -3 overflow entry -3-pos.  tog: 0 until the sweeps end; pass 1 of fast3_walk_performed
// then stores the hash position of a performed candidate's block there (< 0: none), which pass 2 reads back.
struct __align__(16) Cand { uint64_t vkey; int pos; int tog; };
struct __align__(16) OvfEnt { uint64_t order_perf; uint32_t hi; int next; };
struct __align__(16) RayRec { int H, L, nsteps, eval_sweep; };
static constexpr int kBkt3 = 32;              // bucket entries per approximate-set slot (256 B): systematic aliases of the index hash stack 2-3 voxels per slot
static constexpr int kOvfPending = -2;        // overflow entry published, link not yet written
static constexpr int kSortPerWarp = 1024;     // visitors of a shared start-set slot sorted in shared memory (more: in place in global memory)

__device__ __forceinline__ Cand ld_cand(const Cand* p) {
  const int4 v = __ldcg((const int4*)p);
  Cand c; c.vkey = ((uint64_t)(uint32_t)v.y << 32) | (uint32_t)v.x; c.pos = v.z; c.tog = v.w;
  return c;
}
__device__ __forceinline__ void st_cand(Cand* p, uint64_t vkey, int pos, int tog) {
  __stcg((int4*)p, make_int4((int)(uint32_t)vkey, (int)(uint32_t)(vkey >> 32), pos, tog));
}
__device__ __forceinline__ void st_cand_state(Cand* p, int pos, int tog) { __stcg((int2*)p + 1, make_int2(pos, tog)); }
__device__ __forceinline__ uint64_t cand_value(uint64_t vkey, uint64_t offset) { return (uint64_t)index_hash(unpack_key(vkey)) + offset; }
__device__ __forceinline__ uint64_t make_entry(bool on, uint64_t order, uint64_t v) { return (on ? kEntPerf : 0ull) | (order << 13) | (v >> kSetBits); }
__device__ __forceinline__ long long cand_index3(const Obs3& o, const long long* ext_off, int r, int s) {
  if (s < kH0) return (long long)r * kH0 + s;
  const int k = 31 - __clz(s >> 4);
  return o.ext_base + __ldcg(&ext_off[(size_t)r * kExtSegs + k]) + (s - (kH0 << k));
}

// A toggle of `slot` by ray r in sweep k leaves (k, r) in two monotonic words: smax = max (k << 32 | r), smin = min ((~k) << 32 | r).
// Both are fire-and-forget reductions.  A ray evaluated last in sweep `last` is dirty iff the slot was toggled in a later sweep, or in
// sweep `last` by a ray other than itself (smallest and largest toggler of that sweep are not both the ray).
static constexpr uint32_t kSweepCap = 0x7FFFFFFFu;
__device__ __forceinline__ void stamp_toggle(const Obs3& o, uint32_t slot, int sweep, int r) {
  atomicMax((unsigned long long*)&o.stamp_max[slot], ((unsigned long long)(uint32_t)sweep << 32) | (uint32_t)r);
  atomicMin((unsigned long long*)&o.stamp_min[slot], ((unsigned long long)(kSweepCap - (uint32_t)sweep) << 32) | (uint32_t)r);
}
__device__ __forceinline__ bool stamp_dirty(const Obs3& o, uint32_t slot, int last, int r) {
  const unsigned long long a = __ldcg((const unsigned long long*)&o.stamp_max[slot]);
  const unsigned long long b = __ldcg((const unsigned long long*)&o.stamp_min[slot]);
  const int sk = (int)(a >> 32);
  if (sk > last) return true;
  if (sk < last) return false;
  return !((uint32_t)(b >> 32) == kSweepCap - (uint32_t)sk && (uint32_t)a == (uint32_t)r && (uint32_t)b == (uint32_t)r);
}

// first time a candidate turns performed: it enters the slot's bucket (or the overflow pool); returns its position code.
// The overflow push is one exchange, no retry loop.  The exchange releases the entry's fields and its pending link, and the link
// is then stored with release: a reader that acquires the head and every link (ovf_next_acquire) sees every entry it reaches
// complete, and the chain below it whole once the link resolves.  The chain walk of list_slot_visitors relies on that; the
// collision readers of the same sweep need not wait, because the inserter stamps the slot, which marks them dirty.
__device__ __forceinline__ int atom_exch_acq_rel(int* p, int v) {
  return cuda::atomic_ref<int, cuda::thread_scope_device>(*p).exchange(v, cuda::memory_order_acq_rel);
}
__device__ __forceinline__ void st_release(int* p, int v) { cuda::atomic_ref<int, cuda::thread_scope_device>(*p).store(v, cuda::memory_order_release); }
__device__ __forceinline__ int ld_acquire(const int* p) {
  return cuda::atomic_ref<int, cuda::thread_scope_device>(*const_cast<int*>(p)).load(cuda::memory_order_acquire);
}
__device__ __forceinline__ int cand_insert_raw(int* slot_cnt, uint64_t* bkt, int* head, OvfEnt* ovf, int ovf_cap, int* ovf_count, Counters* cnt,
                                            uint32_t slot, uint64_t entry) {
  const int idx = atomicAdd(&slot_cnt[slot], 1);
  if (idx < kBkt3) { const int pos = (int)slot * kBkt3 + idx; __stcg(&bkt[pos], entry); return pos; }
  const int id = atomicAdd(ovf_count, 1);
  if (id >= ovf_cap) { set_err(cnt, 4); return -2; }
  OvfEnt* e = &ovf[id];
  __stcg(&e->next, kOvfPending);
  __stcg(&e->order_perf, (entry & kEntPerf) | ((entry >> 13) & ((1ull << kEntOrderBits) - 1)));
  __stcg(&e->hi, (uint32_t)(entry & 0x1FFFull));
  const int old = atom_exch_acq_rel(&head[slot], id);
  st_release(&e->next, old);
  return -3 - id;
}
__device__ __forceinline__ int cand_insert3(const FastFrame& f, uint32_t slot, uint64_t entry) {
  return cand_insert_raw(f.o3.slot_cnt, f.o3.bkt, f.o3.head, f.o3.ovf, f.o3.ovf_cap, &f.fc->ovf_count, f.cnt, slot, entry);
}

// two bucket entries of one 16-byte load: keeps the latest performed entry that precedes `my_order`
__device__ __forceinline__ void scan_entries(const ulonglong2 v, int base, int n, uint64_t my_order, long long& best, int& best_hi) {
  const uint64_t e2[2] = {v.x, v.y};
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const uint64_t e = e2[k];
    const uint64_t eo = (e >> 13) & ((1ull << kEntOrderBits) - 1);
    if (base + k < n && (e & kEntPerf) && eo < my_order && (long long)eo > best) { best = (long long)eo; best_hi = (int)(e & 0x1FFF); }
  }
}
// latest performed visit of `slot` that precedes `my_order`: its (value >> 20), or -1.  (A non-inlined variant of these helpers made the
// whole frame slower, so they stay inline; the loops past the first 8 entries are rolled.)
// The slot's counter and the first 8 bucket entries are independent loads (one L2 round trip).  __ldcg: the structures change
// while the sweep runs, L1 must not serve stale lines.
__device__ __forceinline__ int latest_performed_before_raw(const uint64_t* bkt, const int* slot_cnt, const int* head, const OvfEnt* ovf, int ovf_cap,
                                                        uint32_t slot, uint64_t my_order) {
  const ulonglong2* b = (const ulonglong2*)(bkt + (size_t)slot * kBkt3);
  const int total = __ldcg(&slot_cnt[slot]);
  ulonglong2 v[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) v[q] = __ldcg(b + q);      // independent of the count: one round trip for the usual <= 8 entries
  const int n = total < kBkt3 ? total : kBkt3;
  long long best = -1;
  int best_hi = -1;
#pragma unroll
  for (int q = 0; q < 4; ++q) scan_entries(v[q], 2 * q, n, my_order, best, best_hi);
#pragma unroll 1
  for (int q0 = 4; 2 * q0 < n; q0 += 4) {
#pragma unroll
    for (int q = 0; q < 4; ++q) v[q] = __ldcg(b + q0 + q);
#pragma unroll
    for (int q = 0; q < 4; ++q) scan_entries(v[q], 2 * (q0 + q), n, my_order, best, best_hi);
  }
  if (total > kBkt3) {
    int guard = total - kBkt3 + 8;
#pragma unroll 1
    for (int id = __ldcg(&head[slot]); id >= 0 && id < ovf_cap && guard-- > 0; id = __ldcg(&ovf[id].next)) {
      const uint64_t op = __ldcg(&ovf[id].order_perf);
      const uint64_t eo = op & ~kEntPerf;
      if ((op & kEntPerf) && eo < my_order && (long long)eo > best) { best = (long long)eo; best_hi = (int)__ldcg(&ovf[id].hi); }
    }
  }
  return best_hi;
}
__device__ __forceinline__ int latest_performed_before3(const Obs3& o, uint32_t slot, uint64_t my_order) {
  return latest_performed_before_raw(o.bkt, o.slot_cnt, o.head, o.ovf, o.ovf_cap, slot, my_order);
}
__device__ __forceinline__ bool later_performed_exists_raw(const uint64_t* bkt, const int* slot_cnt, const int* head, const OvfEnt* ovf, int ovf_cap,
                                                        uint32_t slot, uint64_t my_order) {
  const ulonglong2* b = (const ulonglong2*)(bkt + (size_t)slot * kBkt3);
  const int total = __ldcg(&slot_cnt[slot]);
  const int n = total < kBkt3 ? total : kBkt3;
  bool later = false;
#pragma unroll 1
  for (int q0 = 0; 2 * q0 < n && !later; q0 += 4) {       // 8 entries per round trip, as latest_performed_before_raw
    ulonglong2 v[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) v[q] = __ldcg(b + q0 + q);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint64_t e2[2] = {v[q].x, v[q].y};
#pragma unroll
      for (int k = 0; k < 2; ++k)
        if (2 * (q0 + q) + k < n && (e2[k] & kEntPerf) && ((e2[k] >> 13) & ((1ull << kEntOrderBits) - 1)) > my_order) later = true;
    }
  }
  if (total > kBkt3) {
    int guard = total - kBkt3 + 8;
#pragma unroll 1
    for (int id = __ldcg(&head[slot]); id >= 0 && id < ovf_cap && !later && guard-- > 0; id = __ldcg(&ovf[id].next)) {
      const uint64_t op = __ldcg(&ovf[id].order_perf);
      if ((op & kEntPerf) && (op & ~kEntPerf) > my_order) later = true;
    }
  }
  return later;
}
__device__ __forceinline__ bool later_performed_exists3(const Obs3& o, uint32_t slot, uint64_t my_order) {
  return later_performed_exists_raw(o.bkt, o.slot_cnt, o.head, o.ovf, o.ovf_cap, slot, my_order);
}

// ray r goes on the scan list of sweep `next`, at most once
__device__ __forceinline__ void list_ray(const FastFrame& f, int r, int next) {
  if (atomicMax(&f.wl_listed[r], next) < next) __stcg(&((next & 1) ? f.wl_list[1] : f.wl_list[0])[atomicAdd(&f.fc->wl_count[next & 3], 1)], r);
}
// Ray r toggled `slot` in sweep next-1 (>= 3): every other ray with an entry in the slot goes on the next scan list.  The rays that
// need it were not evaluated in this sweep, so their entries date from earlier sweeps: their bucket words are visible after the
// grid barrier, and their overflow entries lie below every entry pushed in this sweep.  A push of this sweep may be under way
// while the walk runs; its link is acquired and waited for while it is still pending (cand_insert_raw), so the walk always
// reaches the older part of the chain.  An entry written concurrently belongs to a ray evaluated in this sweep (listed anyway),
// and a stale bucket word read in its place lists a ray for nothing (rank checked against n_cast).
__device__ __forceinline__ int ovf_next_acquire(const FastFrame& f, int id) {
  int nx = ld_acquire(&f.o3.ovf[id].next);
  for (int spin = 0; nx == kOvfPending; ++spin) {   // the pusher stores the link right after its exchange
    if (spin > (1 << 24)) { set_err(f.cnt, 2); return -1; }
    nx = ld_acquire(&f.o3.ovf[id].next);
  }
  return nx;
}
__device__ __forceinline__ void list_slot_visitors(const FastFrame& f, uint32_t slot, int r, int next) {
  const Obs3& o = f.o3;
  const int n_cast = __ldcg(&f.cnt->n_cast);
  const ulonglong2* b = (const ulonglong2*)(o.bkt + (size_t)slot * kBkt3);
  const int total = __ldcg(&o.slot_cnt[slot]);
  const int n = total < kBkt3 ? total : kBkt3;
#pragma unroll 1
  for (int q0 = 0; 2 * q0 < n; q0 += 2) {
    ulonglong2 v[2];
#pragma unroll
    for (int q = 0; q < 2; ++q) v[q] = __ldcg(b + q0 + q);
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const uint64_t e2[2] = {v[q].x, v[q].y};
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int r2 = (int)(((e2[k] >> 13) & ((1ull << kEntOrderBits) - 1)) >> kOrderStepBits);
        if (2 * (q0 + q) + k < n && r2 != r && r2 < n_cast) list_ray(f, r2, next);
      }
    }
  }
  if (total > kBkt3) {   // every entry reached was pushed this frame (the head starts at -1), so the chain ends at -1
#pragma unroll 1
    for (int id = ld_acquire(&o.head[slot]); id >= 0 && id < o.ovf_cap; id = ovf_next_acquire(f, id)) {
      const int r2 = (int)((__ldcg(&o.ovf[id].order_perf) & ~kEntPerf) >> kOrderStepBits);
      if (r2 != r && r2 < n_cast) list_ray(f, r2, next);
    }
  }
}

// single writer per candidate: the warp that owns the ray.  c.pos is updated when the candidate enters a bucket.
// No fence between the entry and the stamp: a reader of the same sweep that misses the entry is flagged by the stamp (another
// ray toggled its slot in its own sweep), and every store is visible after the grid barrier that ends the sweep.
// `enter` (with on = false): the ray's break step, examined but not performed, enters the bucket as a perf-0 entry so that a later
// toggle of the slot finds the ray; it is stamped like a toggle because a reader may have caught the reserved entry unwritten.
__device__ __forceinline__ void set_performed3(const FastFrame& f, Cand& c, long long ci, uint32_t slot, uint64_t order, uint64_t v, bool on,
                                               bool enter, int sweep, int r) {
  const Obs3& o = f.o3;
  if (c.pos >= 0) __stcg(&o.bkt[c.pos], make_entry(on, order, v));
  else if (c.pos <= -3) __stcg(&o.ovf[-3 - c.pos].order_perf, (on ? kEntPerf : 0ull) | order);
  else if (on || enter) { c.pos = cand_insert3(f, slot, make_entry(on, order, v)); st_cand_state(&o.cand[ci], c.pos, 0); }
  else return;                       // never entered a bucket and stays unperformed: invisible to every other ray
  stamp_toggle(o, slot, sweep, r);
}

// ---------------------------------------------------------------------------------------------
// RayCaster steps (A.7) of ONE ray by a whole warp.  The serial walk picks, at every step, the axis with the smallest
// t_to_next_boundary_ (first minimum wins) and adds that axis' t_step_size_ to it: per axis the boundary times form the chain
// a(j+1) = fl(a(j) + ts), independent of the other axes, and the walk is the merge of the three non-decreasing chains ordered by
// (time, axis, index).  So: three lanes run the three chains (W dependent additions each instead of 3 W dependent steps), every
// element finds its rank with two binary searches, and the element of rank s carries the per-axis step counts before step s,
// i.e. the voxel emitted at step s.  Bit-identical to dda_next as long as every time and step is finite and every step positive
// (else the caller walks serially: NaN / zero components follow the comparison semantics of the serial code).
// ---------------------------------------------------------------------------------------------
static constexpr int kWin = 64;               // steps per window (= the evaluation block)
struct WarpDdaScratch { float a[3][kWin + 1]; int endc[4]; uint64_t out[kWin]; int n_scanned; };   // n_scanned: profiling

__device__ __forceinline__ bool ray_state_parallel_ok(const RayState& st) {
  const bool fin = isfinite(st.tn0) && isfinite(st.tn1) && isfinite(st.tn2) && isfinite(st.ts0) && isfinite(st.ts1) && isfinite(st.ts2);
  return fin && st.ts0 > 0.0f && st.ts1 > 0.0f && st.ts2 > 0.0f;
}
// W <= kWin steps from `st`; sc->out[0..W) = packed voxel indices, st advanced by W steps.  Returns false if an index left the packed range.
__device__ __forceinline__ bool warp_dda_window(RayState& st, int W, WarpDdaScratch* sc, int lane) {
  if (lane < 3) {
    float a = lane == 0 ? st.tn0 : (lane == 1 ? st.tn1 : st.tn2);
    const float ts = lane == 0 ? st.ts0 : (lane == 1 ? st.ts1 : st.ts2);
    sc->a[lane][0] = a;
    for (int j = 1; j <= W; ++j) { a = a + ts; sc->a[lane][j] = a; }
  }
  __syncwarp();
  const int sg0 = (st.sg & 3) - 1, sg1 = ((st.sg >> 2) & 3) - 1, sg2 = ((st.sg >> 4) & 3) - 1;
  bool ok = true;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    for (int j = lane; j <= W; j += 32) {
      const float v = sc->a[k][j];
      int cnt[3];
      cnt[k] = j;
#pragma unroll
      for (int d = 1; d < 3; ++d) {
        const int k2 = (k + d) % 3;
        const float* b = sc->a[k2];
        // elements of axis k2 that precede (v, k): value < v, or value == v when k2 < k
        int lo = 0, hi = W + 1;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          const float x = b[mid];
          const bool before = (k2 < k) ? (x <= v) : (x < v);
          if (before) lo = mid + 1; else hi = mid;
        }
        cnt[k2] = lo;
      }
      const int rank = cnt[0] + cnt[1] + cnt[2];
      if (rank <= W) {
        I3 g; g.x = st.cx + sg0 * cnt[0]; g.y = st.cy + sg1 * cnt[1]; g.z = st.cz + sg2 * cnt[2];
        if (rank < W) { if (key_in_range(g)) sc->out[rank] = pack_key(g); else ok = false; }
        else { sc->endc[0] = cnt[0]; sc->endc[1] = cnt[1]; sc->endc[2] = cnt[2]; }
      }
    }
  }
  __syncwarp();
  const int e0 = sc->endc[0], e1 = sc->endc[1], e2 = sc->endc[2];
  st.cx += sg0 * e0; st.cy += sg1 * e1; st.cz += sg2 * e2;
  st.tn0 = sc->a[0][e0]; st.tn1 = sc->a[1][e1]; st.tn2 = sc->a[2][e2];
  return __all_sync(0xffffffffu, ok);
}

// evaluation blocks: [0,16), [16,32), [32,64), then 64 steps at a time; a block never straddles a storage segment
__device__ __forceinline__ void block_of_step(int s, int& s0, int& blen) {
  if (s < kH0) { s0 = 0; blen = kH0; return; }
  const int k = 31 - __clz(s >> 4);
  const int seg = kH0 << k;
  if (seg <= kWin) { s0 = seg; blen = seg; }
  else { s0 = seg + ((s - seg) & ~(kWin - 1)); blen = kWin; }
}

__device__ __forceinline__ void fast3_ray_setup(const FastFrame& f, int r, int n_cast) {
  const DevCfg& cfg = f.cfg;
  const Obs3& o = f.o3;
  int h = 0;
  const long long t_begin = f.profile ? clock64() : 0;
  long long t_ins = 0;
  if (r < n_cast) {
    // the cast point again from its input (fast_point, as k_fast_classify computed it)
    const int seq = f.cast_seq[r];
    const int i = f.sb.i_of_seq ? f.sb.i_of_seq[seq] : mixed_index(seq, __ldcg(&f.cnt->n_points));
    const int pix = f.in.depth ? f.pt_pix[i] : i;
    const FastPoint q = fast_point(f, pix, f.in.depth ? __ldg(f.in.depth + pix) : 0.0f);
    const float4 p = make_float4(q.pG.x, q.pG.y, q.pG.z, q.w);
    const uint8_t fl = (q.valid ? 1 : 0) | (q.clearing ? 2 : 0);
    f.ray_param[r] = p;
    f.ray_label[r] = q.label;
    f.ray_flags[r] = fl;
    f.ray_color[r] = q.color;
    if (f.profile) dbg_max(f, 12, clock64() - t_begin);
    Dda d;
    raycaster_init(d, f3(f.T.tx, f.T.ty, f.T.tz), f3(p.x, p.y, p.z), (fl & 2) != 0, cfg.carving != 0, cfg.max_ray, cfg.vsi, cfg.tp.trunc,
                   /*cast_from_origin=*/false);
    int n = d.length_in_steps + 1;
    if (!d.in_range || n >= (1 << kOrderStepBits)) { set_err(f.cnt, 5); n = 0; }
    if (f.profile) dbg_max(f, 13, clock64() - t_begin);
    h = n < kH0 ? n : kH0;
    const int l0 = h < cfg.maxc ? h : cfg.maxc;   // a ray cannot break before `maxc` consecutive collisions
    for (int s = 0; s < h; ++s) {
      const I3 g = dda_next(d);
      if (!key_in_range(g)) { set_err(f.cnt, 5); h = s; break; }
      const uint64_t vkey = pack_key(g);
      const long long ci = (long long)r * kH0 + s;
      int pos = -2;
      if (s < l0) {
        const long long t0 = f.profile ? clock64() : 0;
        const uint64_t v = (uint64_t)index_hash(g) + f.set_offset;
        pos = cand_insert3(f, (uint32_t)v & kSetMask, make_entry(true, ((uint64_t)r << kOrderStepBits) | (uint64_t)s, v));
        if (f.profile) t_ins += clock64() - t0;
      }
      st_cand(&o.cand[ci], vkey, pos, 0);
    }
    if (f.profile) dbg_max(f, 14, clock64() - t_begin);
    RayState st; save_state(st, d); f.ray_state[r] = st;
    RayRec rr; rr.H = h; rr.L = (h < l0) ? h : l0; rr.nsteps = (h < kH0 && h < n) ? h : n; rr.eval_sweep = 0;
    *(int4*)&f.rayrec[r] = make_int4(rr.H, rr.L, rr.nsteps, rr.eval_sweep);
  }
  warp_add(&f.cnt->ray_steps, (unsigned long long)h);
  if (f.profile) { dbg_max(f, 0, clock64() - t_begin); dbg_max(f, 1, t_ins); }
}

// Ray r in one sweep, by one warp.  A ray is re-evaluated only from the first block that holds a dirty step (the
// consecutive-collision count at every block start is kept), in blocks of up to 64 steps = two steps per lane; steps that do not
// exist yet are produced by the warp-parallel ray walk.  Returns (-1, -1) for a clean ray; for an evaluated one the steps it
// toggled, [x, y] (empty when y < x, x >= 0).
__device__ __forceinline__ int2 fast3_ray(const FastFrame& f, int r, int sweep, WarpDdaScratch* sc) {
  const Obs3& o = f.o3;
  const DevCfg& cfg = f.cfg;
  Counters* cnt = f.cnt;
  const int lane = threadIdx.x & 31;
  {
    const int4 rr = __ldcg((const int4*)&f.rayrec[r]);
    int h = rr.x;
    const int old = rr.y, n = rr.z, last = rr.w;
    int fd = 0x7fffffff;                                        // first dirty step
    if (last == 0) fd = 0;
    else {
      const int upto = (old < h - 1) ? old : h - 1;             // steps 0..upto were examined last time
      for (int s = lane; s <= upto; s += 32) {
        const Cand c = ld_cand(&o.cand[cand_index3(o, f.ext_off, r, s)]);
        const uint32_t slot = (uint32_t)cand_value(c.vkey, f.set_offset) & kSetMask;
        if (stamp_dirty(o, slot, last, r)) { fd = s; break; }
      }
      for (int d = 16; d > 0; d >>= 1) { const int t = __shfl_xor_sync(0xffffffffu, fd, d); fd = t < fd ? t : fd; }
    }
    if (fd == 0x7fffffff) return make_int2(-1, -1);
    const long long t_eval = f.profile ? clock64() : 0;
    int n_blocks_eval = 0, n_blocks_mat = 0;
    int s0, blen;
    block_of_step(fd, s0, blen);
    long long base_ci = cand_index3(o, f.ext_off, r, s0);
    int run = (s0 == 0) ? 0 : __ldcg(&f.blk_run[base_ci >> 4]);
    int U = -1;
    while (s0 < n && U < 0) {
      const int cend = (s0 + blen < n) ? s0 + blen : n;
      ++n_blocks_eval;
      bool fresh = false;   // the block's voxel keys are in sc->out, its candidates in no bucket
      if (s0 >= h) {   // materialise the block: continue the ray walk (A.7) from the saved state
        ++n_blocks_mat;
        int ok = 1;
        if (lane == 0 && s0 >= kH0 && (s0 & (s0 - 1)) == 0) {   // s0 = 16 << k: first block of storage segment k (steps [16<<k, 32<<k))
          const int k = 31 - __clz(s0 >> 4);
          const long long need_c = s0;
          const long long off = (long long)atomicAdd(&cnt->n_cand_ext, (unsigned long long)need_c);
          if (o.ext_base + off + need_c > o.cand_cap) { set_err(cnt, 4); ok = 0; }
          else f.ext_off[(size_t)r * kExtSegs + k] = off;
        }
        ok = __shfl_sync(0xffffffffu, ok, 0);
        if (ok) {
          __syncwarp();
          base_ci = cand_index3(o, f.ext_off, r, s0);
          RayState st = f.ray_state[r];
          const int W = cend - s0;
          if (ray_state_parallel_ok(st)) {
            if (!warp_dda_window(st, W, sc, lane)) { set_err(cnt, 5); ok = 0; }
            else {
              for (int t = lane; t < W; t += 32) st_cand(&o.cand[base_ci + t], sc->out[t], -2, 0);
              if (lane == 0) f.ray_state[r] = st;
              fresh = true;
            }
            __syncwarp();
          } else {
            if (lane == 0) {
              Dda d; load_state(d, st);
              for (int t = 0; t < W; ++t) {
                const I3 g = dda_next(d);
                if (!key_in_range(g)) { set_err(cnt, 5); ok = 0; break; }
                st_cand(&o.cand[base_ci + t], pack_key(g), -2, 0);
              }
              if (ok) { save_state(st, d); f.ray_state[r] = st; }
            }
            ok = __shfl_sync(0xffffffffu, ok, 0);
            __syncwarp();
          }
          if (ok && lane == 0) { f.rayrec[r].H = cend; atomicAdd(&cnt->ray_steps, (unsigned long long)W); }
        }
        if (!ok) { U = s0; break; }   // scratch exhausted / index range (flagged): stop here
        h = cend;
      }
      if (lane == 0 && s0 > 0) f.blk_run[base_ci >> 4] = run;
      // ---- collisions of the block's steps: two per lane
      Cand c[2];
      uint64_t v[2];
      bool coll[2];
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int s = s0 + q * 32 + lane;
        c[q].vkey = 0; c[q].pos = -2; c[q].tog = 0; v[q] = 0; coll[q] = false;
        if (s < cend) {
          if (fresh) c[q].vkey = sc->out[q * 32 + lane];
          else c[q] = ld_cand(&o.cand[base_ci + q * 32 + lane]);
          v[q] = cand_value(c[q].vkey, f.set_offset);
        }
      }
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int s = s0 + q * 32 + lane;
        if (s < cend) {
          const uint32_t slot = (uint32_t)v[q] & kSetMask;
          const uint32_t stale = o.table[slot];   // issued together with the bucket loads
          const int hi = latest_performed_before3(o, slot, ((uint64_t)r << kOrderStepBits) | (uint64_t)s);
          coll[q] = (hi >= 0) ? ((uint32_t)hi == (uint32_t)(v[q] >> kSetBits)) : (stale == (uint32_t)(v[q] >> kSetBits));
        }
      }
      const unsigned bits0 = __ballot_sync(0xffffffffu, coll[0]), bits1 = __ballot_sync(0xffffffffu, coll[1]);
      if (f.profile && lane == 0 && n_blocks_eval == 1) dbg_max(f, 15, clock64() - t_eval);
      int brk = -1;
      for (int jj = 0; s0 + jj < cend; ++jj) {
        const unsigned bit = (jj < 32) ? ((bits0 >> jj) & 1u) : ((bits1 >> (jj - 32)) & 1u);
        if (bit) ++run; else run = 0;                          // fast.cpp:115-119
        if (run > cfg.maxc) { brk = s0 + jj; break; }          // fast.cpp:120-122
      }
      const int perf_end = (brk >= 0) ? brk : cend;
#pragma unroll
      for (int q = 0; q < 2; ++q) {                            // newly performed steps of this block, the break step
        const int s = s0 + q * 32 + lane;
        const bool perf = s < perf_end && s >= old;
        if (perf || (s == brk && c[q].pos == -2))
          set_performed3(f, c[q], base_ci + q * 32 + lane, (uint32_t)v[q] & kSetMask, ((uint64_t)r << kOrderStepBits) | (uint64_t)s, v[q],
                         perf, true, sweep, r);
      }
      __syncwarp();
      if (brk >= 0) { U = brk; break; }
      s0 = cend;
      if (s0 < n) { int nb; block_of_step(s0, s0, nb); blen = nb; if (s0 < h) base_ci = cand_index3(o, f.ext_off, r, s0); }
    }
    if (U < 0) U = n;   // the ray ran its full length
    if (U < old) {      // steps [U, old) are no longer performed
      for (int s = U + lane; s < old; s += 32) {
        const long long ci = cand_index3(o, f.ext_off, r, s);
        Cand c = ld_cand(&o.cand[ci]);
        const uint64_t v = cand_value(c.vkey, f.set_offset);
        set_performed3(f, c, ci, (uint32_t)v & kSetMask, ((uint64_t)r << kOrderStepBits) | (uint64_t)s, v, false, false, sweep, r);
      }
    }
    if (lane == 0) {
      if (U != old) { f.rayrec[r].L = U; cnt->changed[sweep & 3] = 1; }
      f.rayrec[r].eval_sweep = sweep;
      if (f.profile) { dbg_max(f, 3, clock64() - t_eval); dbg_add(f, 4, 1); dbg_add(f, 5, n_blocks_eval); dbg_add(f, 6, n_blocks_mat); if (U != old) dbg_add(f, 7, 1); }
    }
    if (U != old) {   // every step this evaluation toggled lies in [lo, hi]
      const int hi = U < old ? old : U;
      return make_int2(U < old ? U : old, hi < h - 1 ? hi : h - 1);
    }
  }
  return make_int2(0, -1);
}

// After ray r's evaluation in sweep >= 3: lists the other visitors of every slot the evaluation toggled (steps [lo, hi]).  A slot
// is walked when stamp_max (a max over sweep << 32 | rank) still names r, i.e. when r is the highest-ranked toggler of the slot
// seen so far in this sweep; the highest-ranked toggler of the whole sweep therefore always walks it, after its own toggle.
__device__ __forceinline__ void fast3_list_toggled(const FastFrame& f, int r, int sweep, int2 steps, int lane) {
  const Obs3& o = f.o3;
  const unsigned long long me = ((unsigned long long)(uint32_t)sweep << 32) | (uint32_t)r;
  for (int s = steps.x + lane; s <= steps.y; s += 32) {
    const Cand c = ld_cand(&o.cand[cand_index3(o, f.ext_off, r, s)]);
    const uint32_t slot = (uint32_t)cand_value(c.vkey, f.set_offset) & kSetMask;
    if (__ldcg((const unsigned long long*)&o.stamp_max[slot]) == me) list_slot_visitors(f, slot, r, sweep + 1);
  }
}

// One sweep.  Sweeps 1 to 3 scan every ray in rank order (sweep 1 evaluates every ray); a later sweep scans the list the previous
// sweep built.  Lists are built from sweep 3 on: sweep 2 takes back most of sweep 1's toggles, and listing them (the self-listing
// of ~30 K evaluated rays on one counter, a bucket walk per toggled slot) cost more than the full scan of sweep 3 it saved.  The
// first item of a warp is its warp index (consecutive items to different CTAs); the rest are claimed one at a time from a shared
// cursor, so the sweep ends with its last ray.  (A claim is issued after the ray: one in flight during the evaluation would cost a
// register, and spills.)
// `it`: 1 for the frame's first sweep.
__device__ __forceinline__ void fast3_sweep(const FastFrame& f, int sweep, int it, WarpDdaScratch* sc) {
  const int lane = threadIdx.x & 31;
  const bool all = it <= 3;
  const bool track = it >= 3;
  const int n_items = all ? __ldcg(&f.cnt->n_cast) : ((volatile int*)f.fc->wl_count)[sweep & 3];
  if (blockIdx.x == 0 && threadIdx.x == 0) {   // the counters of sweep+2 are idle until then: slot (sweep+2) & 3 was sweep-2's
    f.cnt->changed[(sweep + 1) & 3] = 0;
    f.fc->wl_claim[(sweep + 2) & 3] = 0;
    f.fc->wl_count[(sweep + 2) & 3] = 0;
  }
  if (lane == 0) sc->n_scanned = 0;
  __syncwarp();
  const int warps_total = (gridDim.x * blockDim.x) >> 5;
  int i = (threadIdx.x >> 5) * gridDim.x + blockIdx.x;
  while (i < n_items) {
    const int r = all ? i : __ldcg(&((sweep & 1) ? f.wl_list[1] : f.wl_list[0])[i]);   // (a select: an indexed parameter array goes to the stack)
    const int2 toggled = fast3_ray(f, r, sweep, sc);
    if (track && toggled.x >= 0) {   // evaluated: listed for the next sweep, and so are the other visitors of what it toggled
      if (lane == 0) list_ray(f, r, sweep + 1);
      fast3_list_toggled(f, r, sweep, toggled, lane);
    }
    if (f.profile && lane == 0) ++sc->n_scanned;
    int next = 0;
    if (lane == 0) next = warps_total + atomicAdd(&f.fc->wl_claim[sweep & 3], 1);
    i = __shfl_sync(0xffffffffu, next, 0);
  }
  if (f.profile && lane == 0 && sc->n_scanned) dbg_add(f, 2, sc->n_scanned);   // rays scanned, one add per warp and sweep
}

// The performed candidates of every ray.  A warp takes four rays at a time and spreads their performed steps over its 32 lanes
// (lane q of the flattened list: ray j with U[0] + .. + U[j-1] <= q, step q minus that sum), so a ray that updates many voxels
// does not hold the phase while three lanes in four idle.  PASS 1: persistent table commit (the last performed visit of a slot
// survives the frame), block allocation (base.cpp:205-254), records per tile.  PASS 2: (voxel, rank) key into the tile's segment,
// from the block's hash position that pass 1 left in the candidate (no second probe).
// The kernel's thread index (consecutive 32-item chunks on different CTAs), read afresh from the special registers: after the
// sweeps it is recomputed, not carried (or spilled) through them.
__device__ __forceinline__ int solve_gtid_fresh() {
  unsigned t, b;
  asm volatile("mov.u32 %0, %%tid.x;" : "=r"(t));
  asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(b));
  return (int)((((t >> 5) * gridDim.x + b) << 5) | (t & 31));
}

template <int PASS>
__device__ __forceinline__ void fast3_walk_performed(const FastFrame& f, int n_cast, int n_tiles, int gt) {
  const Obs3& o = f.o3;
  const DevCfg& cfg = f.cfg;
  const int rays_total = (gridDim.x * blockDim.x) >> 3;   // four rays per warp and round
  const int lane = gt & 31;
  for (int rb = (gt >> 5) << 2; rb < n_cast; rb += rays_total) {
    const int u = (lane < 4 && rb + lane < n_cast) ? __ldcg(&f.rayrec[rb + lane].L) : 0;
    const int p1 = __shfl_sync(0xffffffffu, u, 0);
    const int p2 = p1 + __shfl_sync(0xffffffffu, u, 1);
    const int p3 = p2 + __shfl_sync(0xffffffffu, u, 2);
    const int total = p3 + __shfl_sync(0xffffffffu, u, 3);
    for (int q = lane; q < total; q += 32) {
      const int j = (q >= p1) + (q >= p2) + (q >= p3);
      const int r = rb + j;
      const int s = q - (j == 0 ? 0 : (j == 1 ? p1 : (j == 2 ? p2 : p3)));
      const long long ci = cand_index3(o, f.ext_off, r, s);
      const Cand c = ld_cand(&o.cand[ci]);
      const I3 g = unpack_key(c.vkey);
      int htpos = c.tog;   // pass 2: the block's hash position, left by pass 1
      if (PASS == 1) {
        const uint64_t v = (uint64_t)index_hash(g) + f.set_offset;
        const uint32_t slot = (uint32_t)v & kSetMask;
        if (!later_performed_exists3(o, slot, ((uint64_t)r << kOrderStepBits) | (uint64_t)s)) o.table[slot] = (uint32_t)(v >> kSetBits);
        const I3 b = block_of_voxel(g, cfg.vps_inv);
        if (!key_in_range(b)) { set_err(f.cnt, 5); htpos = -1; }
        else htpos = ht_find_or_insert(f.map, pack_key(b), f.cnt);
        __stcg(&o.cand[ci].tog, htpos);   // the lane that owns the candidate is the word's one writer
      }
      if (htpos < 0) continue;
      const uint64_t rec = make_record(cfg, htpos, g, (uint32_t)r);
      const uint32_t tk = (uint32_t)(rec >> 32);
      if (PASS == 1) {
        if (atomicAdd(&f.tile_cnt[tk], 1) == 0) {
          const int idx = atomicAdd(&f.fc->n_tile_list, 1);
          if (idx < f.tile_cap) { f.tile_list[idx].tk = tk; f.tile_slot[tk] = idx; } else set_err(f.cnt, 4);
        }
      } else {
        const int at = atomicSub(&f.tile_cnt[tk], 1) - 1;
        const int idx = __ldcg(&f.tile_slot[tk]);
        if (idx >= 0 && idx < n_tiles && at >= 0) f.keys[__ldcg(&f.tile_list[idx].off) + at] = (uint32_t)rec;
      }
    }
  }
}

__global__ void __launch_bounds__(kSolveThreads, 1) k_fast_solve3(FastFrame f, int max_sweeps) {
  unsigned int epoch = 0;
  unsigned int* bar = &f.fc->gridbar;
  const int lane = threadIdx.x & 31;
  const int gtid0 = (((threadIdx.x >> 5) * gridDim.x + blockIdx.x) << 5) | lane;   // consecutive 32-item chunks go to different CTAs
  const int gthreads = gridDim.x * blockDim.x;
  Counters* cnt = f.cnt;
  const int n_points = cnt->n_points;
  int tl = 0;
  timeline_mark(f, tl++);
  extern __shared__ int s_sort[];            // kSortPerWarp ints per warp
  // ---- phase 0a: start-set slots shared by several cells: every visitor files its sequence position in the slot's list (the
  // records of the other slots were emptied by k_fast_start_slots: no visits)
  const int n_mixed = ((volatile int*)&f.fc->n_mixed)[0];
  if (n_mixed > 0) {
    if (gtid0 == 0) f.fc->wl_claim[0] = 0;
    for (int i = gtid0; i < n_points; i += gthreads) {
      const uint64_t v = __ldcg(&f.pt_key[i]);
      if (v == ~0ull) continue;
      StartRec* r = &f.sb.rec[(uint32_t)v & kSetMask];
      if (__ldcg(&r->visits) != 0) f.m_list[atomicAdd(&r->first, 1u)] = f.seq_of_i ? f.seq_of_i[i] : inv_mixed_index(i, n_points);
    }
    solve_barrier(bar, epoch);
    timeline_mark(f, 57);
    // ---- phase 0b: one warp per such slot: visitors in sequence order; the first is cast iff the table holds another value, a later
    // one iff its predecessor carried another value; the table takes the last visitor's value and the record is emptied.
    // Visitor counts vary by two or three orders of magnitude: a warp's first slot is its warp index, the next ones are claimed
    // from a cursor (wl_claim[0], zeroed in phase 0a; the sweeps zero it again before they use it), so no warp draws several
    // large slots while others idle.
    const int warps_total = gthreads >> 5;
    int* scratch = s_sort + (threadIdx.x >> 5) * kSortPerWarp;
    auto key_of_seq = [&](int seq) { return __ldcg(&f.pt_key[f.sb.i_of_seq ? f.sb.i_of_seq[seq] : mixed_index(seq, n_points)]); };
    for (int mi = (threadIdx.x >> 5) * gridDim.x + blockIdx.x; mi < n_mixed;) {
      const int slot = f.mixed_list[mi];
      StartRec* rec = &f.sb.rec[slot];
      const int n = (int)__ldcg(&rec->visits);
      int* seg = f.m_list + ((int)__ldcg(&rec->first) - n);   // phase 0a left the cursor at the end of the list
      int* a = seg;
      if (n <= kSortPerWarp) { for (int i = lane; i < n; i += 32) scratch[i] = __ldcg(&seg[i]); a = scratch; }
      __syncwarp();
      warp_sort_i32(a, n, lane);
      for (int i = lane; i < n; i += 32) {
        const int sb = a[i];
        const uint64_t kb = key_of_seq(sb);
        const bool cast = i == 0 ? f.sb.table[slot] != (uint32_t)(kb >> kSetBits) : key_of_seq(a[i - 1]) != kb;
        if (cast) atomicOr(&f.cast_bits[sb >> 5], 1u << (sb & 31));
      }
      __syncwarp();
      if (lane == 0) {
        f.sb.table[slot] = (uint32_t)(key_of_seq(a[n - 1]) >> kSetBits);
        *(uint4*)rec = start_rec_empty();
      }
      if (f.profile && lane == 0) { dbg_max(f, 8, n); dbg_add(f, 9, n); }
      int next = 0;
      if (lane == 0) next = warps_total + atomicAdd(&f.fc->wl_claim[0], 1);
      mi = __shfl_sync(0xffffffffu, next, 0);
    }
    solve_barrier(bar, epoch);
    timeline_mark(f, 58);
  }
  // ---- phase 0c: offsets of the cast points (block 0), then compaction in sequence order (= ray rank order); every word of the
  // cast bits is cleared once read
  const int n_words = (f.capacity + 31) >> 5;
  if (blockIdx.x == 0) {
    const int total = block_scan_array<true>((const int*)f.cast_bits, f.warp_off, n_words);
    if (threadIdx.x == 0) cnt->n_cast = total;
  }
  solve_barrier(bar, epoch);
  timeline_mark(f, 59);
  const int n_cast = ((volatile int*)&cnt->n_cast)[0];
  for (int w = gtid0; w < n_words; w += gthreads) {
    uint32_t m = __ldcg(&f.cast_bits[w]);
    if (m == 0u) continue;
    f.cast_bits[w] = 0u;
    for (int at = __ldcg(&f.warp_off[w]); m; m &= m - 1u) f.cast_seq[at++] = (w << 5) | (__ffs(m) - 1);
  }
  const int sweep_base0 = ((volatile int*)&f.fc->sweep_base)[0];   // sweep ids are monotonic across frames (31 bits: never wraps in practice)
  if (gtid0 == 0) for (int k = 0; k < 4; ++k) { f.fc->wl_claim[k] = 0; f.fc->wl_count[k] = 0; }
  solve_barrier(bar, epoch);
  timeline_mark(f, tl++);
  // ---- phase 1: ray set-up (first kH0 steps of every ray)
  for (int r0 = (gtid0 & ~31); r0 < n_cast; r0 += gthreads) fast3_ray_setup(f, r0 + lane, n_cast);
  solve_barrier(bar, epoch);
  timeline_mark(f, tl++);
  // ---- phase 2: observed-set fixpoint
  // (n_cast and the frame's first sweep are not carried through the loop: registers there are the solver's)
  int sweep = (sweep_base0 + 4) & ~3;   // counter slot (sweep + 1) & 3 of the first sweep was zeroed by the frame reset
  bool converged = n_cast == 0;
  int it = 0;
  while (!converged && it < max_sweeps) {
    ++it;
    ++sweep;
    fast3_sweep(f, sweep, it, (WarpDdaScratch*)(s_sort + (threadIdx.x >> 5) * kSortPerWarp));
    solve_barrier(bar, epoch);
    if (tl < kTimelineSlots - 12) timeline_mark(f, tl++);
    const int changed = ((volatile int*)cnt->changed)[sweep & 3];
    const int err = ((volatile int*)&cnt->err)[0];
    if (err) break;
    converged = !changed;
  }
  const bool failed = !converged;
  const int gtid = solve_gtid_fresh();
  if (gtid == 0) {
    cnt->last_sweep = sweep;
    f.fc->sweep_base = sweep;
    f.fc->sweeps_last = it;
    if (failed && !((volatile int*)&cnt->err)[0]) set_err(cnt, 2 /*KSG_ERR_CUDA: the solver did not converge*/);
    if (f.prof_marks) f.fc->timeline[kTimelineSlots - 1] = tl;
  }
  tl = kTimelineSlots - 12;
  timeline_mark(f, tl++);
  // ---- phase 3: table commit + block allocation + records per tile
  if (!failed) fast3_walk_performed<1>(f, ((volatile int*)&cnt->n_cast)[0], 0, gtid);
  solve_barrier(bar, epoch);
  timeline_mark(f, tl++);
  timeline_mark(f, tl++);     // (an empty phase: the host reads the records -> tile segments span as marks tb+1 .. tb+4)
  const bool ok = ((volatile int*)&cnt->err)[0] == 0 && !failed;
  const int n_new_all = ((volatile int*)&cnt->n_new_blocks)[0];
  const int n_new = n_new_all < f.map.new_cap ? n_new_all : f.map.new_cap;
  const int pool_base = ((volatile int*)&cnt->pool_count)[0];
  // ---- phase 4: key segment per tile, updated() bookkeeping, ownership (spatial sharding), new blocks
  const int n_tiles = (int)min((long long)((volatile int*)&f.fc->n_tile_list)[0], f.tile_cap);
  for (int base = (gtid & ~31); base < n_tiles; base += gthreads) {
    const int idx = base + lane;
    int n = 0;
    uint32_t tk = 0;
    if (idx < n_tiles) { tk = f.tile_list[idx].tk; n = __ldcg(&f.tile_cnt[tk]); }
    const long long off = (long long)warp_alloc(&f.fc->rec_cursor, (unsigned long long)n);
    if (idx < n_tiles) {
      const int pos = (int)(tk / (uint32_t)f.cfg.tiles_per_block);
      const int old = atomicExch(&f.map.touched_stamp[pos], f.frame_stamp);
      if (old != f.frame_stamp) f.map.touched_list[atomicAdd(&cnt->n_blocks_touched, 1)] = pos;
      const bool owned = f.cfg.shard_count <= 1 ||
                         tile_owner(f.map.ht_keys[pos], (int)(tk % (uint32_t)f.cfg.tiles_per_block), f.cfg.shard_count) == f.cfg.shard_rank;
      if (off + n > f.rec_cap) { set_err(cnt, 4); n = 0; }
      f.tile_list[idx].n = owned ? n : -n;
      f.tile_list[idx].off = off;
    }
  }
  if (ok) fast_block_init(f, n_new, pool_base);
  solve_barrier(bar, epoch);
  timeline_mark(f, tl++);
  // ---- phase 5: keys into the tile segments (the per-tile counters run back to zero: nothing to clear for the next frame)
  const bool ok2 = ((volatile int*)&cnt->err)[0] == 0 && !failed;
  if (!failed) fast3_walk_performed<2>(f, ((volatile int*)&cnt->n_cast)[0], ok2 ? n_tiles : 0, gtid);
  if (gtid == 0) {
    int add = n_new;
    if (pool_base + add > f.map.max_blocks) add = f.map.max_blocks - pool_base;
    if (ok) cnt->pool_count = pool_base + (add > 0 ? add : 0);
    cnt->n_tiles = ok2 ? n_tiles : 0;
    cnt->n_records = ((volatile unsigned long long*)&f.fc->rec_cursor)[0];
    f.fc->tile_cursor = 0;
    f.fc->n_tile_list = 0;
    f.fc->rec_cursor = 0;
    f.fc->ovf_count = 0;
    if (f.profile) { f.fc->dbg[10] = ((volatile int*)&f.fc->n_mixed)[0]; f.fc->dbg[11] = ((volatile int*)&cnt->n_cast)[0]; }
    f.fc->n_mixed = 0;
    f.fc->m_cursor = 0;
    f.fc->n_touched = 0;
    f.fc->log_count = 0;
  }
  timeline_mark(f, tl++);
}

}  // namespace ksg
