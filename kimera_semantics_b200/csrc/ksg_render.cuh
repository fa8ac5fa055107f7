// ksg_render.cuh — depth and semantic images of the device map from a camera pose (ksg_render_view / ksg_render_view_device): one ray
// march per pixel to the first zero crossing of voxblox's trilinear distance, then the point query (ksg_query.cuh) at the hit.
//
// A new capability, not part of the reference tree: "parity unpinned".  Every rule and constant is stated here; the numpy twin
// (tests/render_ref.py) follows them in float32 with the same operation order (the library is built with -fmad=false, IEEE div / sqrt):
//   * pixel (u, v) has index v * W + u.  K = fx fy cx cy (float64); cx = float(K[2]), cy = float(K[3]), constant_x = float(1.0 / fx),
//     constant_y = float(1.0 / fy), as ksg_integrate_depth_k64 computes them.  The sample at camera depth z is
//       p_G(z) = xform_apply(T_G_C, (((u - cx) * z) * constant_x, ((v - cy) * z) * constant_y, z))
//     - the float expressions of the depth entry, so a render at an integration pose walks exactly the rays its pixels integrated.
//     a = (u - cx) * constant_x, b = (v - cy) * constant_y, r = norm3((a, b, 1)) = sqrt((a*a + b*b) + 1) turns a Euclidean length along
//     the ray into a z length; dir_G = xform_apply(T_G_C with t = 0, (a, b, 1)) is the world direction per unit z (slab test only);
//   * the march starts at z = min_depth and samples while z <= max_depth.  At each sample p = p_G(z), with g = grid_index(p, 1/vs) and
//     the block bc = block_of_voxel(g) (the point query's containing voxel):
//       (a) p fails index_in_range(p / vs) or bc fails key_in_range: the pixel is a miss;
//       (b) bc is not allocated: z = (z + t) + (kRenderPush * vs) / r, t = max(0, min over the axes with dir_a != 0 of
//           (face_a - p_a) / dir_a), face_a = float(bc_a + 1) * bs for dir_a > 0, float(bc_a) * bs for dir_a < 0, bs = float(vps) * vs:
//           the ray's exit from bc's box plus a push of a quarter voxel, so the next sample lies in the next block;
//       (c) D(p) (query_interp: all 8 corners allocated and weight > min_weight) is not valid: z = z + vs / r;
//       (d) valid D > 0: remember (z0, D0) = (z, D), then z = z + max(kRenderKappa * D, 0.5 * vs) / r.  kRenderKappa < 1 because the
//           projective TSDF overestimates the distance at grazing angles;
//       (e) valid D, not > 0 (D <= 0): when the previous sample was a (d), it is the hit:
//             z_hit = z0 + (z - z0) * (D0 / (D0 - D));
//           otherwise the camera is inside or behind a surface: z = z + (0.5 * vs) / r and go on.
//     Only a (d) sample is a predecessor: (b), (c) and a non-hit (e) forget it.  Past max_depth the pixel is a miss;
//   * termination: every step adds at least (kRenderPush * vs) / r to z.  The entries reject a call unless that step is at least
//     max_depth * 2^-20 for r at the image corner farthest from (cx, cy) (include/ksg.h), i.e. 8 ulp of any z <= max_depth, so z grows
//     by a fixed fraction of that step per sample and the loop ends after a bounded number of samples; there is no iteration cap;
//   * outputs: depth = z_hit and points_G = p_G(z_hit), NaN (bits 0x7FC00000) on a miss.  Everything else is k_query_points, unchanged,
//     on points_G with the same min_weight (a miss is a NaN point: flags 0, NaN, 0 bytes).
// One thread per pixel; a warp takes an 8 x 4 pixel tile, so neighbouring rays read the same blocks through L1.  Each ray keeps one
// QueryBlocks window, placed so that it reaches ahead along the ray and moved only when the stencil of D(p) leaves it: a block is probed
// about once per ray.  The map is read through __ldg as in ksg_query.cuh.  tests/test_gpu_render.py compares with the twin bit for bit.
#pragma once
#include "ksg_query.cuh"

namespace ksg {

static constexpr int kRenderThreads = 128;
static constexpr float kRenderKappa = 0.9f;
static constexpr float kRenderPush = 0.25f;
static constexpr int kRenderTileW = 8, kRenderTileH = 4;   // pixels of one warp

struct RenderCam {
  Xform T;
  float cx, cy, constant_x, constant_y;
  int width, height;
  float min_depth, max_depth, min_weight;
};

__device__ __forceinline__ F3 render_point(const RenderCam& c, float fu, float fv, float z) {
  return xform_apply(c.T, f3((fu - c.cx) * z * c.constant_x, (fv - c.cy) * z * c.constant_y, z));
}

// camera depth of the first zero crossing along pixel (u, v), NaN on a miss
__device__ __forceinline__ float render_march(const DevCfg& cfg, const MapRef& map, const RenderCam& c, int u, int v) {
  const float nan = __int_as_float((int)kQueryNaNBits);
  const float fu = (float)u, fv = (float)v;
  const float a = (fu - c.cx) * c.constant_x, b = (fv - c.cy) * c.constant_y;
  const float r = norm3(f3(a, b, 1.0f));
  Xform R = c.T;
  R.tx = 0.0f; R.ty = 0.0f; R.tz = 0.0f;
  const F3 dir = xform_apply(R, f3(a, b, 1.0f));
  const float vs = cfg.voxel_size, bs = (float)cfg.vps * vs;
  const float step_vox = vs / r, step_half = (0.5f * vs) / r, step_push = (kRenderPush * vs) / r;
  QueryBlocks w;
  w.base.x = w.base.y = w.base.z = 1 << 30;   // no block key lies there: the first sample places the window
  float z = c.min_depth, z0 = 0.0f, d0 = 0.0f;
  bool pos = false;
  while (z <= c.max_depth) {
    const F3 p = render_point(c, fu, fv, z);
    if (!index_in_range(f3(p.x * cfg.vsi, p.y * cfg.vsi, p.z * cfg.vsi))) return nan;
    const I3 g = grid_index(p, cfg.vsi);
    const I3 bc = block_of_voxel(g, cfg.vps_inv);
    if (!key_in_range(bc)) return nan;
    // the stencil of D(p): voxels g0 .. g0 + 1 (query_interp's corners), blocks lo .. hi on each axis
    I3 g0 = g;
    if (p.x < ((float)g0.x + 0.5f) * vs) g0.x -= 1;
    if (p.y < ((float)g0.y + 0.5f) * vs) g0.y -= 1;
    if (p.z < ((float)g0.z + 0.5f) * vs) g0.z -= 1;
    I3 g1 = g0;
    g1.x += 1; g1.y += 1; g1.z += 1;
    const I3 lo = block_of_voxel(g0, cfg.vps_inv), hi = block_of_voxel(g1, cfg.vps_inv);
    if ((unsigned)(lo.x - w.base.x) >= 2u || (unsigned)(lo.y - w.base.y) >= 2u || (unsigned)(lo.z - w.base.z) >= 2u ||
        (unsigned)(hi.x - w.base.x) >= 2u || (unsigned)(hi.y - w.base.y) >= 2u || (unsigned)(hi.z - w.base.z) >= 2u) {
      // reach ahead along the ray: the window's second layer lies on the side the ray moves to
      w.base.x = dir.x >= 0.0f ? lo.x : hi.x - 1;
      w.base.y = dir.y >= 0.0f ? lo.y : hi.y - 1;
      w.base.z = dir.z >= 0.0f ? lo.z : hi.z - 1;
#pragma unroll
      for (int j = 0; j < 8; ++j) w.slot[j] = -2;
    }
    if (query_block_slot(map, w, bc) < 0) {   // (b) skip the unallocated block
      float t = __int_as_float(0x7f800000);
      if (dir.x > 0.0f) t = fminf(t, ((float)(bc.x + 1) * bs - p.x) / dir.x);
      else if (dir.x < 0.0f) t = fminf(t, ((float)bc.x * bs - p.x) / dir.x);
      if (dir.y > 0.0f) t = fminf(t, ((float)(bc.y + 1) * bs - p.y) / dir.y);
      else if (dir.y < 0.0f) t = fminf(t, ((float)bc.y * bs - p.y) / dir.y);
      if (dir.z > 0.0f) t = fminf(t, ((float)(bc.z + 1) * bs - p.z) / dir.z);
      else if (dir.z < 0.0f) t = fminf(t, ((float)bc.z * bs - p.z) / dir.z);
      z = (z + fmaxf(t, 0.0f)) + step_push;
      pos = false;
      continue;
    }
    float d;
    if (!query_interp(cfg, map, w, p, c.min_weight, d)) {   // (c)
      z = z + step_vox;
      pos = false;
      continue;
    }
    if (d > 0.0f) {   // (d)
      z0 = z;
      d0 = d;
      pos = true;
      z = z + fmaxf(kRenderKappa * d, 0.5f * vs) / r;
      continue;
    }
    if (pos) return z0 + (z - z0) * (d0 / (d0 - d));   // (e)
    z = z + step_half;
  }
  return nan;
}

// one warp per 8 x 4 tile, tiles row-major over the image; depth / points_G may be NULL (not written)
__device__ __forceinline__ void render_tile(const DevCfg& cfg, const MapRef& map, const RenderCam& c, long long tile, int lane,
                                            float* __restrict__ depth, float* __restrict__ points_G) {
  const int tiles_x = (c.width + kRenderTileW - 1) / kRenderTileW;
  const int u = (int)(tile % tiles_x) * kRenderTileW + (lane % kRenderTileW);
  const int v = (int)(tile / tiles_x) * kRenderTileH + (lane / kRenderTileW);
  if (u >= c.width || v >= c.height) return;
  const float zh = render_march(cfg, map, c, u, v);
  const long long i = (long long)v * c.width + u;
  if (depth) depth[i] = zh;
  if (points_G) {
    const float nan = __int_as_float((int)kQueryNaNBits);
    const F3 p = zh == zh ? render_point(c, (float)u, (float)v, zh) : f3(nan, nan, nan);
    points_G[3 * i] = p.x;
    points_G[3 * i + 1] = p.y;
    points_G[3 * i + 2] = p.z;
  }
}

// A plain grid, one warp per tile.  Persistent warps claiming tiles from a counter (grid = 16 blocks per SM) computed the same bits and
// took 0.422 ms against 0.406 ms for a 640x480 depth render of the fast5 map (H100 80GB HBM3, 700 W): the grid stays.
__global__ void __launch_bounds__(kRenderThreads) k_render_view(DevCfg cfg, MapRef map, RenderCam c, float* __restrict__ depth,
                                                                float* __restrict__ points_G) {
  render_tile(cfg, map, c, ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, threadIdx.x & 31, depth, points_G);
}

}  // namespace ksg
