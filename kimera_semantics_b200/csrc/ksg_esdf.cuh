// ksg_esdf.cuh — batch Euclidean signed distance field of the device map (ksg_compute_esdf): an exact separable distance transform of
// the map's surface voxels.
//
// What voxblox offers here is EsdfIntegrator::updateFromTsdfLayerBatch (voxblox/integrator/esdf_integrator.h), a queue propagation whose
// result depends on the order it visits voxels.  It is not part of the reference tree, and this file does not restate it: the field is
// a closed-form minimum, the same whatever the launch shape or the order of computation ("parity unpinned").
//
// Inputs: min_weight >= 0 (the mesher's and the queries' rule) and max_distance m, finite and > 0.  vs = voxel_size and
// W = ceil(m / vs) + 1, computed in double on the host: the half-width of the window the passes search.
//   * OBSERVED: a voxel of an allocated block with weight > min_weight.  Voxels of unallocated blocks are not observed.
//   * SURFACE voxel (site): an observed voxel v with at least one observed face neighbour n (also in another block) such that
//     (d_v > 0) != (d_n > 0) (zero is on the non-positive side, as in ksg_render.cuh) and |d_v| <= |d_n| (the nearer voxel of each
//     crossing edge; on a tie, both).  In an exact (1-Lipschitz) distance field |d_v| + |d_n| = |d_v - d_n| <= vs, so every site has
//     |d| <= vs / 2; an integrated projective TSDF need not be Lipschitz, so this is not a rule for integrated maps.
//   * Q(v) = min over all sites s of dx^2 + dy^2 + dz^2, in integer voxel offsets.
//   * Output, for every voxel of every allocated block (ksg_export_blocks order, voxblox linear voxel order):
//       unobserved:  distance NaN (bits 0x7FC00000), flags 0;
//       site:        distance d_v (the TSDF value), flags OBSERVED | SURFACE;
//       otherwise:   mag = fl(sqrtf((float)Q) * vs) if Q exists and mag < m, else mag = m and flag CAPPED; distance +mag if d_v > 0,
//                    else -mag; flags OBSERVED (| CAPPED).
//
// Why three windowed passes give the output exactly.  A site outside the cube max(|dx|, |dy|, |dz|) <= W is at Q >= (W + 1)^2 < 2^24;
// both roundings are monotone and W + 1 is exact, so sqrtf((float)Q) >= W + 1 and mag >= fl((W + 1) vs) >= (m + 2 vs)(1 - 2^-24) > m
// (W + 1 >= m / vs + 2, and m <= 512 vs): it is capped whether it is the nearest site or not.  So the passes only search the window,
// in int32, over x, then y, then z:
//   A(p) = min over |i| <= W of (site(p + i e_x) ? i^2 : none),  B(p) = min over |j| <= W of A(p + j e_y) + j^2,
//   Q(p) = min over |k| <= W of B(p + k e_z) + k^2,  none + anything = none;
// each is the exact minimum over the sites of the window (the squared distance separates by axis).  "none" after the z pass makes the
// voxel CAPPED.  Inside the window Q <= 3 W^2 <= 786432 < 2^24, so (float)Q is exact and the only rounding is sqrtf and the product,
// each correctly rounded (no fast math), so the output does not depend on how the work is split.
//
// Error against the true distance D of an exact SDF (non-site, not capped, v observed).  The site s nearest v has |d_s| <= vs / 2, so
// D <= |v - s| + |d_s| gives out >= D - vs / 2.  If the zero set, where it is nearest v, passes through a cell of 2x2x2 voxel centres
// whose corners have both signs (always so for a plane: a plane through the interior of a cube separates its corners), one of the
// cell's edges crosses and its nearer end is a site within sqrt(3) vs of that point, so out <= D + sqrt(3) vs.  With the two roundings:
//   -vs / 2 - 2^-22 m <= out - D <= sqrt(3) vs + 2^-22 m,
// and a capped voxel has D >= m - sqrt(3) vs.  This is a bound from the rules, not a measured spread (tests/test_esdf_ref_cpu.py writes
// the measured one beside it).
//
// W <= 512 (rejected otherwise) bounds the work per voxel, 3 (2W + 1) candidates, and the block dilation of the work sets.
//
// Kernels, all launched once per call (4 launches when distance or flags is wanted, none otherwise):
//   k_esdf_sites     one CTA per allocated block: the site byte of each voxel (face neighbours in other blocks through
//                    ht_lookup_slot), and whether the block holds a site;
//   k_esdf_pass<0>   x pass over the X work set, reading the site bytes;
//   k_esdf_pass<1>   y pass over the Y work set, reading the x pass;
//   k_esdf_pass<2>   z pass over the allocated blocks, reading the y pass, writing the distance and the flags.
// With Rb = ceil(W / vps): the Y work set is every block within Rb along z of an allocated block that has a site block within Rb along x
// and y; the X work set is every block within Rb along y of a Y block and within Rb along x of a site block.  Outside these sets the pass
// result is "none" everywhere, so they are exact; the host builds them from the block keys, and memory scales with their block counts.
// Each pass takes, per work block, a table of the 2 Rb + 1 blocks along its axis in the previous stage (-1: none there).  One thread per
// output voxel, threads in linear voxel order (x fastest): for every axis, the 32 lanes of a warp read consecutive x at the same offset,
// so the loads coalesce without staging in shared memory, and each thread visits only the table blocks that exist.  Brute force over the
// window: simple and exact; a lower-envelope transform is the option if the measured time asks for it.
// The numpy twin is tests/esdf_ref.py; tests/test_gpu_esdf.py compares bit for bit.
//
// The device layer (ksg_update_esdf): the same output, kept per pool slot (distance, flags and the site byte of every voxel, max_blocks
// rows) and brought up to date from what changed.  The host keeps the frame stamp of the last update; MapRef::touched_stamp holds per
// hash position the stamp of the block's last touch, and every path that writes voxels sets it (fast's solve kernel, merged's heads
// kernels, k_merge_insert, k_mergev_insert).  Pool slots are handed out in order, so the blocks allocated since the last update are the
// slots from its block count on.  The rule:
//   C = the blocks whose stamp is newer than the last update's, and the slots allocated since;
//   R = C and its allocated face neighbours: k_esdf_sites recomputes their site bytes in place and flags each block whose bytes changed
//       against the stored ones (a new slot's row is zeroed first): that gives S;
//   D = C and every allocated block within Chebyshev distance Rb of a block of S (a separable dilation of S on the host);
//   the z pass runs over D, the y pass over the blocks within Rb along z of D that have a near-x block within Rb along y, the x pass
//   over those within Rb along y of a y block and near-x (EsdfWork::build with D as the z work set); all read the stored site bytes of
//   the whole map, and the z pass writes D's rows.  R empty: no launch.
// Why it is exact.  A site byte depends only on its voxel and the voxel's 6 face neighbours; a voxel outside C kept its TSDF value and
// weight, so a byte can differ from the stored one only in a block of C or in a face neighbour of one - R recomputes all of those, and
// every other stored byte is still right.  A voxel's output depends on its own voxel and on the site bytes within its window, which lie
// in blocks within Rb = ceil(W / vps) of its block (Chebyshev).  So an output can change only if its block is in C or a block within Rb
// holds a changed byte (S): that is D, and every other stored output is still right.  The passes then compute D's outputs from site
// bytes that are all right, by the batch definition, so the layer equals ksg_compute_esdf bit for bit.  (An output moves only for
// sqrt(Q) < m / vs <= W - 1, so Rb is conservative by up to one block; tests/test_esdf_incremental_cpu.py shows which windows reach it.)
// A change of (min_weight, max_distance), and any ksg_clear_map (stamps zeroed, slots reused, frame_stamp kept), ksg_reset (frame_stamp
// back to 0) or ksg_import_blocks (writes without stamping) since the last update make the next update full: C = every block, stored
// bytes taken as zero.  So does a call that fails after its argument checks: the site bytes are rewritten in place before the passes,
// and a retry would find them unchanged while their outputs are stale.  The numpy model is tests/esdf_incremental_ref.py; tests/test_gpu_esdf_incremental.py compares bit for bit.
//
// Point queries on the layer (k_query_esdf): ksg_query.cuh's rules and its arithmetic (query_stencil with the EsdfCorner fetch); a
// corner is valid when its block is in the layer (slot < the layer's block count) and its voxel is OBSERVED.  For an exact SDF whose
// zero set is a plane, the trilinear form of the exact distance is exact, so each value keeps the voxel bound above,
// -vs / 2 - 2^-22 m <= D_esdf(p) - D(p) <= sqrt(3) vs + 2^-22 m where the surface point nearest p lies inside the map, and a gradient
// component is off by at most (sqrt(3) + 1 / 2) / 2 (tests/test_esdf_incremental_cpu.py prints the measured spread).
#pragma once
#include "ksg_kernels.cuh"
#include "ksg_query.cuh"

namespace ksg {

static constexpr int kEsdfThreads = 256;
static constexpr int kEsdfMaxWindow = 512;
static constexpr int kEsdfNone = 0x7FFFFFFF;
static constexpr uint32_t kEsdfNaNBits = 0x7FC00000u;
enum : int { kEsdfObserved = 1, kEsdfSurface = 2, kEsdfCapped = 4 };

// slots[blk]: pool slot of work block blk; site[row * V + v]: 1 for a site, row = the slot (slot_rows, the device layer) or blk (the
// batch entry); has_site[blk]: 1 when the block holds one; changed[blk] (NULL: not wanted): 1 when a site byte differs from the one the
// row held before
__global__ void __launch_bounds__(kEsdfThreads) k_esdf_sites(DevCfg cfg, MapRef map, const int* __restrict__ slots, int n_blocks,
                                                             float min_weight, int slot_rows, uint8_t* __restrict__ site,
                                                             uint8_t* __restrict__ has_site, uint8_t* __restrict__ changed) {
  __shared__ int s_nb[7];   // this block, then -x, +x, -y, +y, -z, +z
  const int tid = threadIdx.x;
  const int vps = cfg.vps, vm = vps - 1, nvox = vps * vps * vps;
  for (int blk = blockIdx.x; blk < n_blocks; blk += gridDim.x) {
    const int slot = slots[blk];
    __syncthreads();
    if (tid < 7) {
      I3 nb = unpack_key(map.slot_key[slot]);
      const int a = (tid - 1) >> 1, sgn = (tid & 1) ? -1 : 1;
      if (tid > 0) { if (a == 0) nb.x += sgn; else if (a == 1) nb.y += sgn; else nb.z += sgn; }
      s_nb[tid] = (tid == 0) ? slot : (key_in_range(nb) ? ht_lookup_slot(map, pack_key(nb)) : -1);
    }
    __syncthreads();
    uint8_t* const row = site + (size_t)(slot_rows ? slot : blk) * nvox;
    int any = 0, diff = 0;
    for (int v = tid; v < nvox; v += kEsdfThreads) {
      const int l[3] = {v & vm, (v / vps) & vm, v / (vps * vps)};
      int vox;
      const uint8_t* chunk = mesh_voxel_chunk(cfg, map, slot, l[0], l[1], l[2], vox);
      const float d = __ldg((const float*)chunk + vox);
      int is_site = 0;
      if (__ldg((const float*)(chunk + cfg.plane_f32) + vox) > min_weight) {
#pragma unroll 1
        for (int k = 1; k < 7; ++k) {
          const int a = (k - 1) >> 1, sgn = (k & 1) ? -1 : 1;
          int n[3] = {l[0], l[1], l[2]};
          n[a] += sgn;
          const int s = ((unsigned)n[a] < (unsigned)vps) ? slot : s_nb[k];
          if (s < 0) continue;
          int nv;
          const uint8_t* nc = mesh_voxel_chunk(cfg, map, s, n[0] & vm, n[1] & vm, n[2] & vm, nv);
          if (!(__ldg((const float*)(nc + cfg.plane_f32) + nv) > min_weight)) continue;
          const float dn = __ldg((const float*)nc + nv);
          if (((d > 0.0f) != (dn > 0.0f)) && fabsf(d) <= fabsf(dn)) { is_site = 1; break; }
        }
      }
      if (changed) diff |= row[v] != is_site;
      row[v] = (uint8_t)is_site;
      any |= is_site;
    }
    any = __syncthreads_or(any);
    if (changed) diff = __syncthreads_or(diff);
    if (tid == 0) {
      has_site[blk] = (uint8_t)(any ? 1 : 0);
      if (changed) changed[blk] = (uint8_t)(diff ? 1 : 0);
    }
  }
}

struct EsdfOut {   // z pass only: NULL = not wanted
  float* distance;
  uint8_t* flags;
  const int* slots;   // pool slot of each z work block
  float min_weight, max_distance;
};

// One windowed pass along AXIS over n_blocks work blocks; nbr[blk * (2 Rb + 1) + Rb + k] is the previous stage's index of the block
// k blocks along AXIS (-1: none).  AXIS 0 reads the site bytes (in8); 1 and 2 read the previous pass (in32).  AXIS 0 and 1 write
// out32; AXIS 2 writes the final distance and flags (eo), in row blk (the batch entry) or, with SLOT_ROWS, in the row of the block's pool
// slot (the device layer; the site bytes are read from the same row).
template <int AXIS, bool SLOT_ROWS = false>
__global__ void __launch_bounds__(kEsdfThreads) k_esdf_pass(DevCfg cfg, MapRef map, int n_blocks, int W, int Rb, const int* __restrict__ nbr,
                                                            const uint8_t* __restrict__ in8, const int* __restrict__ in32,
                                                            int* __restrict__ out32, const uint8_t* __restrict__ site, EsdfOut eo) {
  const int vps = cfg.vps, vm = vps - 1, nvox = vps * vps * vps;
  const int stride = AXIS == 0 ? 1 : AXIS == 1 ? vps : vps * vps;
  const long long n = (long long)n_blocks * nvox;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int blk = (int)(i / nvox), v = (int)(i - (long long)blk * nvox);
    const int la = AXIS == 0 ? (v & vm) : AXIS == 1 ? ((v / vps) & vm) : v / (vps * vps);
    const int base = v - la * stride;
    const int* row = nbr + (size_t)blk * (2 * Rb + 1) + Rb;
    const int k_lo = (la - W + Rb * vps) / vps - Rb, k_hi = (la + W) / vps;   // blocks the window [la - W, la + W] touches
    int best = kEsdfNone;
    for (int k = k_lo; k <= k_hi; ++k) {
      const int src = __ldg(row + k);
      if (src < 0) continue;
      const int c_lo = max(k * vps, la - W), c_hi = min(k * vps + vm, la + W);
      const size_t at = (size_t)src * nvox + base;
      for (int c = c_lo; c <= c_hi; ++c) {
        const int t = c - la;
        const int e = (c - k * vps) * stride;
        if (AXIS == 0) {
          if (__ldg(in8 + at + e)) best = min(best, t * t);
        } else {
          const int q = __ldg(in32 + at + e);
          if (q != kEsdfNone) best = min(best, q + t * t);
        }
      }
    }
    if (AXIS != 2) { out32[i] = best; continue; }
    const int slot = eo.slots[blk];
    const size_t o = SLOT_ROWS ? (size_t)slot * nvox + v : (size_t)i;
    int vox;
    const uint8_t* chunk = mesh_voxel_chunk(cfg, map, slot, v & vm, (v / vps) & vm, v / (vps * vps), vox);
    const float d = __ldg((const float*)chunk + vox);
    float dist = __int_as_float((int)kEsdfNaNBits);
    int flags = 0;
    if (__ldg((const float*)(chunk + cfg.plane_f32) + vox) > eo.min_weight) {
      flags = kEsdfObserved;
      if (__ldg(site + o)) {
        flags |= kEsdfSurface;
        dist = d;
      } else {
        float mag = best == kEsdfNone ? eo.max_distance : sqrtf((float)best) * cfg.voxel_size;
        if (!(best != kEsdfNone && mag < eo.max_distance)) { mag = eo.max_distance; flags |= kEsdfCapped; }
        dist = d > 0.0f ? mag : -mag;
      }
    }
    if (eo.distance) eo.distance[o] = dist;
    if (eo.flags) eo.flags[o] = (uint8_t)flags;
  }
}

// ksg_export_esdf: rows slots[b] of the device layer, one after the other
__global__ void __launch_bounds__(kEsdfThreads) k_esdf_gather(int nvox, const int* __restrict__ slots, int n_blocks, const float* __restrict__ src_d,
                                                              const uint8_t* __restrict__ src_f, float* __restrict__ dst_d, uint8_t* __restrict__ dst_f) {
  const long long n = (long long)n_blocks * nvox;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int blk = (int)(i / nvox);
    const size_t at = (size_t)__ldg(slots + blk) * nvox + (size_t)(i - (long long)blk * nvox);
    if (dst_d) dst_d[i] = __ldg(src_d + at);
    if (dst_f) dst_f[i] = __ldg(src_f + at);
  }
}

struct EsdfLayer {   // the device layer as of the last ksg_update_esdf: rows by pool slot, slots [0, n_blocks)
  const float* distance;
  const uint8_t* flags;
  int n_blocks;
};

// Corner fetch of the ESDF query (query_stencil, ksg_query.cuh): the ESDF distance of voxel g when its block is in the layer and the
// voxel is OBSERVED there
struct EsdfCorner {
  const DevCfg& cfg;
  const MapRef& map;
  QueryBlocks& w;
  EsdfLayer layer;
  __device__ __forceinline__ bool operator()(I3 g, float& d) const {
    const int s = query_block_slot(map, w, block_of_voxel(g, cfg.vps_inv));
    if (s < 0 || s >= layer.n_blocks) return false;
    const int vps = cfg.vps, vm = vps - 1;
    const size_t i = (size_t)s * vps * vps * vps + (size_t)((g.x & vm) + vps * ((g.y & vm) + vps * (g.z & vm)));
    if (!(__ldg(layer.flags + i) & kEsdfObserved)) return false;
    d = __ldg(layer.distance + i);
    return true;
  }
};

struct EsdfQueryOut {   // mirror of ksg_esdf_query_out (include/ksg.h); NULL = not wanted
  uint8_t* flags;
  uint8_t* voxel_flags;
  float* voxel_distance;
  float* distance;
  float* gradient;
};

// ksg_query_esdf: ksg_query_points' rules (ksg_query.cuh) on the ESDF layer.  ALLOCATED: the block is in the layer; OBSERVED: the voxel's
// ESDF flags hold KSG_ESDF_OBSERVED; the corners of D(p) are the layer's OBSERVED voxels.  One thread per query.
__global__ void __launch_bounds__(kQueryThreads) k_query_esdf(DevCfg cfg, MapRef map, EsdfLayer layer, const float* __restrict__ xyz,
                                                              long long n, EsdfQueryOut out, int need_interp, int need_grad) {
  const float nan = __int_as_float((int)kQueryNaNBits);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int flags = 0, vflags = 0;
    float vdist = nan, interp = nan, gx = nan, gy = nan, gz = nan;
    const F3 p = f3(__ldg(xyz + 3 * i), __ldg(xyz + 3 * i + 1), __ldg(xyz + 3 * i + 2));
    if (index_in_range(f3(p.x * cfg.vsi, p.y * cfg.vsi, p.z * cfg.vsi))) {
      const I3 g = grid_index(p, cfg.vsi);
      const I3 b = block_of_voxel(g, cfg.vps_inv);
      if (key_in_range(b)) {
        QueryBlocks w;
        I3 lo = g;
        lo.x -= 2; lo.y -= 2; lo.z -= 2;
        w.base = block_of_voxel(lo, cfg.vps_inv);
#pragma unroll
        for (int j = 0; j < 8; ++j) w.slot[j] = -2;
        const int s = query_block_slot(map, w, b);
        if (s >= 0 && s < layer.n_blocks) {
          const int vps = cfg.vps, vm = vps - 1;
          const size_t at = (size_t)s * vps * vps * vps + (size_t)((g.x & vm) + vps * ((g.y & vm) + vps * (g.z & vm)));
          vflags = __ldg(layer.flags + at);
          vdist = __ldg(layer.distance + at);
          flags = kQueryAllocated | ((vflags & kEsdfObserved) ? kQueryObserved : 0);
        }
        query_stencil(cfg, EsdfCorner{cfg, map, w, layer}, p, need_interp && (flags & kQueryObserved), need_grad, flags, interp, gx, gy, gz);
      }
    }
    if (out.flags) out.flags[i] = (uint8_t)flags;
    if (out.voxel_flags) out.voxel_flags[i] = (uint8_t)vflags;
    if (out.voxel_distance) out.voxel_distance[i] = vdist;
    if (out.distance) out.distance[i] = interp;
    if (out.gradient) { out.gradient[3 * i] = gx; out.gradient[3 * i + 1] = gy; out.gradient[3 * i + 2] = gz; }
  }
}

}  // namespace ksg
