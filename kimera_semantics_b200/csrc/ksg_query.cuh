// ksg_query.cuh — point queries on the device map (ksg_query_points / ksg_query_points_device): the containing voxel of each point with
// its semantic row, and voxblox's trilinear distance and its gradient.
//
// What a host caller of voxblox asks a map about a point is Layer::getVoxelPtrByCoordinates and Interpolator<TsdfVoxel>::getDistance /
// getGradient with interpolate = true (voxblox/interpolator/interpolator_inl.h).  That code is not part of the reference tree: "parity
// unpinned" - this file restates it from knowledge of that code:
//   * containing voxel: g = grid_index(p, 1/vs) = floor(p * (1/vs) + 1e-6) (A.2), block b = block_of_voxel(g, 1/vps), local index
//     g & (vps - 1) - exactly how k_mesh_blocks maps a vertex to its voxel.  A point failing index_in_range(p / vs) (also every
//     non-finite point) or key_in_range(b) gets flags 0.  ALLOCATED: b is in the hash.  OBSERVED: ALLOCATED and weight > min_weight
//     (the mesher's rule).  The voxel's fields (distance, weight, colour, label, log-probability row, semantic colour) are written
//     whenever ALLOCATED is set, also for an unobserved default voxel;
//   * trilinear distance D(p) (Interpolator::getInterpDistance, the matrix form of PM159): lower corner g0 = g, minus one on every axis a
//     where p_a < (g_a + 0.5) * vs; q_a = (p_a - (g0_a + 0.5) * vs) * (1/vs); corner i = g0 + (i >> 2, (i >> 1) & 1, i & 1) with distance
//     d_i.  Valid (INTERPOLATED) only when all 8 corners are allocated and observed.  With x, y, z = q, in exactly this order:
//       b0 = d0, b1 = -d0 + d4, b2 = -d0 + d2, b3 = -d0 + d1, b4 = ((d0 - d2) - d4) + d6, b5 = ((d0 - d1) - d2) + d3,
//       b6 = ((d0 - d1) - d4) + d5, b7 = ((((((-d0 + d1) + d2) - d3) + d4) - d5) - d6) + d7,
//       D = ((((((b0 + x*b1) + y*b2) + z*b3) + (x*y)*b4) + (y*z)*b5) + (z*x)*b6) + ((x*y)*z)*b7;
//   * gradient (getGradient, interpolate = true): grad_a = (D(p + vs e_a) - D(p - vs e_a)) / (2 vs), the offsets one float add on one
//     axis; valid (GRADIENT) only when all six evaluations are;
//   * what is not valid is NaN (bits 0x7FC00000) for floats and 0 for bytes.
// The containing voxel is always one of the 8 corners of D(p), so INTERPOLATED implies OBSERVED.  One thread per query; the blocks of
// its stencil are probed once each (QueryBlocks); the log-probability rows are copied by the whole warp, lanes = classes.  Every result
// is a function of the point and the map alone, whatever the launch shape.  The numpy twin is tests/query_ref.py;
// tests/test_gpu_query.py compares bit for bit.
#pragma once
#include "ksg_kernels.cuh"

namespace ksg {

struct QueryOut {   // mirror of ksg_query_out (include/ksg.h); NULL = not wanted
  uint8_t* flags;
  float *tsdf_distance, *tsdf_weight;
  uint8_t* tsdf_rgba;
  uint8_t* sem_label;
  float* sem_priors;
  uint8_t* sem_rgba;
  float* distance;
  float* gradient;
};

static constexpr int kQueryThreads = 256;
static constexpr uint32_t kQueryNaNBits = 0x7FC00000u;
enum : int { kQueryAllocated = 1, kQueryObserved = 2, kQueryInterpolated = 4, kQueryGradient = 8 };

// Pool slots of the 2x2x2 blocks from `base`, probed on first use (-2: not probed yet, -1: not allocated).  base = the block of
// g - (2, 2, 2): from voxels_per_side 4 upward every corner of the gradient stencil (voxels g - 2 .. g + 2) lies in the window; with 1
// and 2 the corners outside it are probed one by one.
// The probes go through the mesher's ht_lookup_slot, whose plain loads are kept as they are: the voxel planes and rows (the bulk of the
// bytes) are read through the read-only path (__ldg) below, while a query probes at most 8 blocks (voxels_per_side >= 4), and on sm_90
// plain global loads are cached in L1 as well.  The table is not written while either kernel runs, so the result is the same on either path.
struct QueryBlocks {
  I3 base;
  int slot[8];
};

__device__ __forceinline__ int query_block_slot(const MapRef& map, QueryBlocks& w, I3 b) {
  const int dx = b.x - w.base.x, dy = b.y - w.base.y, dz = b.z - w.base.z;
  if ((unsigned)dx < 2u && (unsigned)dy < 2u && (unsigned)dz < 2u) {
    const int k = dx | (dy << 1) | (dz << 2);
    int s = -2;
#pragma unroll
    for (int j = 0; j < 8; ++j) if (j == k) s = w.slot[j];   // selects, not a local-memory array
    if (s == -2) {
      s = key_in_range(b) ? ht_lookup_slot(map, pack_key(b)) : -1;
#pragma unroll
      for (int j = 0; j < 8; ++j) if (j == k) w.slot[j] = s;
    }
    return s;
  }
  return key_in_range(b) ? ht_lookup_slot(map, pack_key(b)) : -1;
}

// distance of voxel g if it is allocated and observed
__device__ __forceinline__ bool query_corner(const DevCfg& cfg, const MapRef& map, QueryBlocks& w, I3 g, float min_weight, float& d) {
  const int s = query_block_slot(map, w, block_of_voxel(g, cfg.vps_inv));
  if (s < 0) return false;
  const int vm = cfg.vps - 1;
  int vox;
  const uint8_t* chunk = mesh_voxel_chunk(cfg, map, s, g.x & vm, g.y & vm, g.z & vm, vox);
  if (!(__ldg((const float*)(chunk + cfg.plane_f32) + vox) > min_weight)) return false;
  d = __ldg((const float*)chunk + vox);
  return true;
}

// trilinear distance D(p); false when p is out of range or a corner is missing / unobserved
__device__ __forceinline__ bool query_interp(const DevCfg& cfg, const MapRef& map, QueryBlocks& w, F3 p, float min_weight, float& out) {
  if (!index_in_range(f3(p.x * cfg.vsi, p.y * cfg.vsi, p.z * cfg.vsi))) return false;
  const float vs = cfg.voxel_size;
  I3 g0 = grid_index(p, cfg.vsi);
  if (p.x < ((float)g0.x + 0.5f) * vs) g0.x -= 1;
  if (p.y < ((float)g0.y + 0.5f) * vs) g0.y -= 1;
  if (p.z < ((float)g0.z + 0.5f) * vs) g0.z -= 1;
  const float x = (p.x - ((float)g0.x + 0.5f) * vs) * cfg.vsi;
  const float y = (p.y - ((float)g0.y + 0.5f) * vs) * cfg.vsi;
  const float z = (p.z - ((float)g0.z + 0.5f) * vs) * cfg.vsi;
  float d[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    I3 c = g0;
    c.x += i >> 2; c.y += (i >> 1) & 1; c.z += i & 1;
    if (!query_corner(cfg, map, w, c, min_weight, d[i])) return false;
  }
  const float b0 = d[0];
  const float b1 = -d[0] + d[4];
  const float b2 = -d[0] + d[2];
  const float b3 = -d[0] + d[1];
  const float b4 = ((d[0] - d[2]) - d[4]) + d[6];
  const float b5 = ((d[0] - d[1]) - d[2]) + d[3];
  const float b6 = ((d[0] - d[1]) - d[4]) + d[5];
  const float b7 = ((((((-d[0] + d[1]) + d[2]) - d[3]) + d[4]) - d[5]) - d[6]) + d[7];
  out = ((((((b0 + x * b1) + y * b2) + z * b3) + (x * y) * b4) + (y * z) * b5) + (z * x) * b6) + ((x * y) * z) * b7;
  return true;
}

// need_interp / need_grad: evaluate D(p) / the gradient (for the flags or the outputs that carry them)
__global__ void __launch_bounds__(kQueryThreads) k_query_points(DevCfg cfg, MapRef map, const float* __restrict__ xyz, long long n, float min_weight,
                                                                QueryOut out, int need_interp, int need_grad) {
  const int lane = threadIdx.x & 31;
  const float nan = __int_as_float((int)kQueryNaNBits);
  const long long stride = (long long)gridDim.x * blockDim.x;
  // warp-uniform loop: the row copy below needs every lane
  for (long long i0 = (long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31); i0 < n; i0 += stride) {
    const long long i = i0 + lane;
    const float* row = nullptr;   // log-probability row of the containing voxel
    if (i < n) {
      int flags = 0;
      float dist = nan, wgt = nan, interp = nan, gx = nan, gy = nan, gz = nan;
      uint32_t rgba = 0, srgba = 0;
      int label = 0;
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
          if (s >= 0) {
            const int vm = cfg.vps - 1;
            int vox;
            const uint8_t* chunk = mesh_voxel_chunk(cfg, map, s, g.x & vm, g.y & vm, g.z & vm, vox);
            dist = __ldg((const float*)chunk + vox);
            wgt = __ldg((const float*)(chunk + cfg.plane_f32) + vox);
            rgba = __ldg((const unsigned int*)(chunk + 2 * cfg.plane_f32) + vox);
            srgba = __ldg((const unsigned int*)(chunk + 3 * cfg.plane_f32) + vox);
            label = __ldg(chunk + 4 * cfg.plane_f32 + vox);
            row = (const float*)(chunk + cfg.head_bytes) + (size_t)vox * cfg.C;
            flags = kQueryAllocated | (wgt > min_weight ? kQueryObserved : 0);
          }
          // evaluation 0: D(p); 2a + 1 / 2a + 2: D(p + vs e_a) / D(p - vs e_a).  One loop (not unrolled): the probe code is emitted once.
          const float vs = cfg.voxel_size;
          float dplus = 0.0f, ga[3] = {0.0f, 0.0f, 0.0f};
          const int e_first = (need_interp && (flags & kQueryObserved)) ? 0 : 1;   // the containing voxel is a corner of D(p)
          const int e_end = need_grad ? 7 : 1;
#pragma unroll 1
          for (int e = e_first; e < e_end; ++e) {
            const int a = (e - 1) >> 1;
            const float off = (e & 1) ? vs : -vs;
            const F3 pe = f3(a == 0 ? p.x + off : p.x, a == 1 ? p.y + off : p.y, a == 2 ? p.z + off : p.z);
            float v;
            const bool ok = query_interp(cfg, map, w, pe, min_weight, v);
            if (e == 0) {
              if (ok) { flags |= kQueryInterpolated; interp = v; }
              continue;
            }
            if (!ok) break;
            if (e & 1) { dplus = v; continue; }
            const float gv = (dplus - v) / (2.0f * vs);
            if (a == 0) ga[0] = gv; else if (a == 1) ga[1] = gv; else ga[2] = gv;
            if (e == 6) { flags |= kQueryGradient; gx = ga[0]; gy = ga[1]; gz = ga[2]; }
          }
        }
      }
      if (out.flags) out.flags[i] = (uint8_t)flags;
      if (out.tsdf_distance) out.tsdf_distance[i] = dist;
      if (out.tsdf_weight) out.tsdf_weight[i] = wgt;
      if (out.tsdf_rgba) for (int k = 0; k < 4; ++k) out.tsdf_rgba[4 * i + k] = (uint8_t)(rgba >> (8 * k));
      if (out.sem_label) out.sem_label[i] = (uint8_t)label;
      if (out.sem_rgba) for (int k = 0; k < 4; ++k) out.sem_rgba[4 * i + k] = (uint8_t)(srgba >> (8 * k));
      if (out.distance) out.distance[i] = interp;
      if (out.gradient) { out.gradient[3 * i] = gx; out.gradient[3 * i + 1] = gy; out.gradient[3 * i + 2] = gz; }
    }
    if (out.sem_priors) {
      // rows one after the other, lanes = classes: the voxel-major row is read and the output row written in whole segments
      unsigned act = __ballot_sync(0xffffffffu, i < n);
      while (act) {
        const int j = __ffs(act) - 1;
        act &= act - 1;
        const float* r = (const float*)__shfl_sync(0xffffffffu, (unsigned long long)row, j);
        float* o = out.sem_priors + (i0 + j) * (long long)cfg.C;
        for (int c = lane; c < cfg.C; c += 32) o[c] = r ? __ldg(r + c) : nan;
      }
    }
  }
}

}  // namespace ksg
