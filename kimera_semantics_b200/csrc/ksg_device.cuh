// ksg_device.cuh — device-side arithmetic of the semantic TSDF integrator (sm_90a).
//
// Every float expression here is written in the operation order of the reference path so that
// voxel / block indices come out bit-identical to the CPU integrator; the translation unit is
// compiled with -fmad=false (no FMA contraction), IEEE sqrt / division (no --use_fast_math).
// Reference citations: fast.cpp / merged.cpp / base.cpp = kimera_semantics/src/semantic_tsdf_integrator_fast.cpp,
// ..._merged.cpp, semantic_integrator_base.cpp; "A.n" = SURVEY.md Appendix A (voxblox behaviour).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ksg {

static constexpr float kEps = 1e-6f;           // voxblox kEpsilon / kFloatEpsilon / kCoordinateEpsilon
static constexpr int kSetBits = 20;            // ApproxHashSet<20, 10000, ...>  fast.h:98-107
static constexpr uint32_t kSetSize = 1u << kSetBits;
static constexpr uint32_t kSetMask = kSetSize - 1;
static constexpr uint32_t kSetNever = 0xFFFFFFFFu;  // compact table entry that matches no value
static constexpr int kTileSideMax = 8;         // device tiles are min(vps, 8)^3 voxels

struct F3 { float x, y, z; };
struct I3 { int x, y, z; };

__host__ __device__ __forceinline__ F3 f3(float x, float y, float z) { F3 r; r.x = x; r.y = y; r.z = z; return r; }
__host__ __device__ __forceinline__ F3 add(F3 a, F3 b) { return f3(a.x + b.x, a.y + b.y, a.z + b.z); }
__host__ __device__ __forceinline__ F3 sub(F3 a, F3 b) { return f3(a.x - b.x, a.y - b.y, a.z - b.z); }
__host__ __device__ __forceinline__ F3 mul(F3 a, float s) { return f3(a.x * s, a.y * s, a.z * s); }
__host__ __device__ __forceinline__ F3 divs(F3 a, float s) { return f3(a.x / s, a.y / s, a.z / s); }
// Eigen 3-vector reductions: (x*x + y*y) + z*z
__host__ __device__ __forceinline__ float dot3(F3 a, F3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
__host__ __device__ __forceinline__ float norm3(F3 a) { return sqrtf(dot3(a, a)); }
__host__ __device__ __forceinline__ F3 normalized3(F3 a) {
  const float n2 = dot3(a, a);
  if (n2 > 0.0f) return divs(a, sqrtf(n2));
  return a;
}
__host__ __device__ __forceinline__ F3 cross3(F3 a, F3 b) {
  return f3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}

// minkindr QuatTransformation<float> (A.8): T*p = (p + w*uv + qv x uv) + t with uv = 2*(qv x p)
struct Xform { float qw, qx, qy, qz, tx, ty, tz; };
__host__ __device__ __forceinline__ F3 xform_apply(const Xform& T, F3 p) {
  const F3 qv = f3(T.qx, T.qy, T.qz);
  F3 uv = cross3(qv, p);
  uv = add(uv, uv);
  const F3 r = add(add(p, mul(uv, T.qw)), cross3(qv, uv));
  return add(r, f3(T.tx, T.ty, T.tz));
}

// voxblox getGridIndexFromPoint (A.2). Indices are kept in int32 on the device; the caller range-checks.
__host__ __device__ __forceinline__ I3 grid_index(F3 p, float inv) {
  I3 r;
  r.x = (int)floorf(p.x * inv + kEps);
  r.y = (int)floorf(p.y * inv + kEps);
  r.z = (int)floorf(p.z * inv + kEps);
  return r;
}
__host__ __device__ __forceinline__ I3 grid_index_scaled(F3 s) {
  I3 r;
  r.x = (int)floorf(s.x + kEps);
  r.y = (int)floorf(s.y + kEps);
  r.z = (int)floorf(s.z + kEps);
  return r;
}
__host__ __device__ __forceinline__ bool index_in_range(F3 scaled) {
  const float lim = 1.0e9f;  // < 2^30: every later integer op stays inside int32
  return fabsf(scaled.x) < lim && fabsf(scaled.y) < lim && fabsf(scaled.z) < lim;
}
// LongIndexHash (A.2): 64-bit modular arithmetic truncated to 32 bits
__host__ __device__ __forceinline__ uint32_t index_hash(I3 g) {
  const uint64_t sl = 17191ull, sl2 = sl * sl;
  return (uint32_t)((uint64_t)(int64_t)g.x + (uint64_t)(int64_t)g.y * sl + (uint64_t)(int64_t)g.z * sl2);
}

// ---------------------------------------------------------------------------------------------
// RayCaster (A.7; voxblox integrator_utils)  — call sites fast.cpp:95-102,110  merged.cpp:288-294,305
// ---------------------------------------------------------------------------------------------
struct Dda {
  I3 cur;
  float tn[3];   // t_to_next_boundary_
  float ts[3];   // t_step_size_
  int sg[3];     // ray_step_signs_
  int length_in_steps;  // emits length_in_steps + 1 indices
  bool in_range;
};

__host__ __device__ __forceinline__ int signum_f(float x) { return (0.0f < x) - (x < 0.0f); }

__host__ __device__ __forceinline__ void dda_setup(Dda& d, F3 s, F3 e) {
  d.in_range = true;
  if (isnan(s.x) || isnan(s.y) || isnan(s.z) || isnan(e.x) || isnan(e.y) || isnan(e.z)) {
    // upstream: ray_length_in_steps_ = 0 and return with a default index; one (0,0,0) index is emitted
    d.cur.x = d.cur.y = d.cur.z = 0;
    d.length_in_steps = 0;
    d.sg[0] = d.sg[1] = d.sg[2] = 0;
    d.tn[0] = d.tn[1] = d.tn[2] = 0.0f;
    d.ts[0] = d.ts[1] = d.ts[2] = 0.0f;
    return;
  }
  if (!index_in_range(s) || !index_in_range(e)) { d.in_range = false; }
  d.cur = grid_index_scaled(s);
  const I3 endi = grid_index_scaled(e);
  d.length_in_steps = abs(endi.x - d.cur.x) + abs(endi.y - d.cur.y) + abs(endi.z - d.cur.z);
  const float r[3] = {e.x - s.x, e.y - s.y, e.z - s.z};
  const float shifted[3] = {s.x - (float)d.cur.x, s.y - (float)d.cur.y, s.z - (float)d.cur.z};
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    d.sg[k] = signum_f(r[k]);
    const float corr = (float)(d.sg[k] > 0 ? d.sg[k] : 0);
    d.tn[k] = (corr - shifted[k]) / r[k];
    d.ts[k] = (float)d.sg[k] / r[k];
  }
}

// RayCaster ctor. cast_from_origin = true for merged (default arg), false for fast (fast.cpp:94).
__host__ __device__ __forceinline__ void raycaster_init(Dda& d, F3 origin, F3 point_G, bool is_clearing, bool carving,
                                                        float max_len, float vsi, float trunc, bool cast_from_origin) {
  const F3 unit_ray = normalized3(sub(point_G, origin));
  F3 ray_start, ray_end;
  if (is_clearing) {
    float ray_length = norm3(sub(point_G, origin));
    ray_length = fminf(fmaxf(ray_length - trunc, 0.0f), max_len);
    ray_end = add(origin, mul(unit_ray, ray_length));
    ray_start = carving ? origin : ray_end;
  } else {
    ray_end = add(point_G, mul(unit_ray, trunc));
    ray_start = carving ? origin : sub(point_G, mul(unit_ray, trunc));
  }
  const F3 ss = mul(ray_start, vsi);
  const F3 es = mul(ray_end, vsi);
  if (cast_from_origin) dda_setup(d, ss, es); else dda_setup(d, es, ss);
}

// nextRayIndex: returns the current index, then advances along argmin(t_next) (first minimum wins)
__host__ __device__ __forceinline__ I3 dda_next(Dda& d) {
  const I3 out = d.cur;
  // argmin of t_to_next_boundary_, first minimum wins (written without a run-time array index: the state stays in registers)
  int k = 0;
  float m = d.tn[0];
  if (d.tn[1] < m) { k = 1; m = d.tn[1]; }
  if (d.tn[2] < m) k = 2;
  if (k == 0) { d.cur.x += d.sg[0]; d.tn[0] += d.ts[0]; }
  else if (k == 1) { d.cur.y += d.sg[1]; d.tn[1] += d.ts[1]; }
  else { d.cur.z += d.sg[2]; d.tn[2] += d.ts[2]; }
  return out;
}

// ---------------------------------------------------------------------------------------------
// TSDF update (A.6; voxblox TsdfIntegratorBase::updateTsdfVoxel / computeDistance / blendTwoColors)
// ---------------------------------------------------------------------------------------------
struct TsdfParams {
  float voxel_size, trunc, max_weight, sparsity_factor;
  int use_weight_dropoff, use_sparsity;
};

__host__ __device__ __forceinline__ uint32_t blend_two_colors(uint32_t c1, float w1, uint32_t c2, float w2) {
  const float total = w1 + w2;
  w1 /= total;
  w2 /= total;
  uint32_t out = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int a = (int)((c1 >> (8 * k)) & 0xFF), b = (int)((c2 >> (8 * k)) & 0xFF);
    const float v = roundf((float)a * w1 + (float)b * w2);
    out |= ((uint32_t)(uint8_t)v) << (8 * k);
  }
  return out;
}

// One updateTsdfVoxel call on (dist, weight, rgba) of the voxel whose centre is `center`.
__host__ __device__ __forceinline__ void tsdf_update(const TsdfParams& P, F3 origin, F3 point_G, F3 center, uint32_t color,
                                                     float w, float& dist, float& weight, uint32_t& rgba) {
  const F3 v_voxel_origin = sub(center, origin);
  const F3 v_point_origin = sub(point_G, origin);
  const float dist_G = norm3(v_point_origin);
  const float dist_G_V = dot3(v_voxel_origin, v_point_origin) / dist_G;
  const float sdf = dist_G - dist_G_V;
  float uw = w;
  const float dropoff_epsilon = P.voxel_size;
  if (P.use_weight_dropoff && sdf < -dropoff_epsilon) {
    uw = w * (P.trunc + sdf) / (P.trunc - dropoff_epsilon);
    uw = fmaxf(uw, 0.0f);
  }
  if (P.use_sparsity) {
    if (fabsf(sdf) < P.trunc) uw *= P.sparsity_factor;
  }
  const float new_weight = weight + uw;
  if (new_weight < kEps) return;
  const float new_sdf = (sdf * uw + dist * weight) / new_weight;
  if (fabsf(sdf) < P.trunc) rgba = blend_two_colors(rgba, weight, color, uw);
  dist = (new_sdf > 0.0f) ? fminf(P.trunc, new_sdf) : fmaxf(-P.trunc, new_sdf);
  weight = fminf(P.max_weight, new_weight);
}

// The two halves of updateTsdfVoxel, split so that the measurement part (independent of the voxel state) can be
// evaluated for many records in parallel while the state recurrence runs in the reference's order.
__host__ __device__ __forceinline__ void tsdf_measure(const TsdfParams& P, F3 origin, F3 point_G, F3 center, float w,
                                                      float& sdf, float& uw) {
  const F3 v_voxel_origin = sub(center, origin);
  const F3 v_point_origin = sub(point_G, origin);
  const float dist_G = norm3(v_point_origin);
  const float dist_G_V = dot3(v_voxel_origin, v_point_origin) / dist_G;
  sdf = dist_G - dist_G_V;
  uw = w;
  const float dropoff_epsilon = P.voxel_size;
  if (P.use_weight_dropoff && sdf < -dropoff_epsilon) {
    uw = w * (P.trunc + sdf) / (P.trunc - dropoff_epsilon);
    uw = fmaxf(uw, 0.0f);
  }
  if (P.use_sparsity) {
    if (fabsf(sdf) < P.trunc) uw *= P.sparsity_factor;
  }
}
__host__ __device__ __forceinline__ void tsdf_chain_step(const TsdfParams& P, float sdf, float uw, uint32_t color, bool blend,
                                                         float& dist, float& weight, uint32_t& rgba) {
  const float new_weight = weight + uw;
  if (new_weight < kEps) return;
  const float new_sdf = (sdf * uw + dist * weight) / new_weight;
  if (blend && fabsf(sdf) < P.trunc) rgba = blend_two_colors(rgba, weight, color, uw);
  dist = (new_sdf > 0.0f) ? fminf(P.trunc, new_sdf) : fmaxf(-P.trunc, new_sdf);
  weight = fminf(P.max_weight, new_weight);
}

__host__ __device__ __forceinline__ F3 voxel_center(I3 g, float voxel_size) {
  return f3(((float)g.x + 0.5f) * voxel_size, ((float)g.y + 0.5f) * voxel_size, ((float)g.z + 0.5f) * voxel_size);
}

// voxblox rainbowColorMap (double arithmetic), ColorMode::kSemanticProbability base.cpp:181-185
__host__ __device__ __forceinline__ uint32_t rainbow_color_map(double h) {
  const double s = 1.0, v = 1.0;
  h -= floor(h);
  h *= 6;
  const int i = (int)floor(h);
  double f = h - i;
  if (!(i & 1)) f = 1 - f;
  const double m = v * (1 - s);
  const double n = v * (1 - s * f);
  uint8_t r, g, b;
  switch (i) {
    case 6:
    case 0: r = (uint8_t)(255 * v); g = (uint8_t)(255 * n); b = (uint8_t)(255 * m); break;
    case 1: r = (uint8_t)(255 * n); g = (uint8_t)(255 * v); b = (uint8_t)(255 * m); break;
    case 2: r = (uint8_t)(255 * m); g = (uint8_t)(255 * v); b = (uint8_t)(255 * n); break;
    case 3: r = (uint8_t)(255 * m); g = (uint8_t)(255 * n); b = (uint8_t)(255 * v); break;
    case 4: r = (uint8_t)(255 * n); g = (uint8_t)(255 * m); b = (uint8_t)(255 * v); break;
    case 5: r = (uint8_t)(255 * v); g = (uint8_t)(255 * m); b = (uint8_t)(255 * n); break;
    default: r = 255; g = 127; b = 127; break;
  }
  return (uint32_t)r | ((uint32_t)g << 8) | ((uint32_t)b << 16) | (255u << 24);
}

// ---------------------------------------------------------------------------------------------
// block keys / spatial hash
// ---------------------------------------------------------------------------------------------
static constexpr uint64_t kEmptyKey = ~0ull;
static constexpr int kKeyBias = 1 << 20;  // block / voxel coordinates must lie in [-2^20, 2^20)

__host__ __device__ __forceinline__ bool key_in_range(I3 b) {
  return b.x >= -kKeyBias && b.x < kKeyBias && b.y >= -kKeyBias && b.y < kKeyBias && b.z >= -kKeyBias && b.z < kKeyBias;
}
__host__ __device__ __forceinline__ uint64_t pack_key(I3 b) {
  return ((uint64_t)(uint32_t)(b.z + kKeyBias) << 42) | ((uint64_t)(uint32_t)(b.y + kKeyBias) << 21) | (uint64_t)(uint32_t)(b.x + kKeyBias);
}
__host__ __device__ __forceinline__ I3 unpack_key(uint64_t k) {
  I3 b;
  b.x = (int)(k & 0x1FFFFF) - kKeyBias;
  b.y = (int)((k >> 21) & 0x1FFFFF) - kKeyBias;
  b.z = (int)((k >> 42) & 0x1FFFFF) - kKeyBias;
  return b;
}
__host__ __device__ __forceinline__ uint32_t mix64(uint64_t k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return (uint32_t)k;
}
// Spatial sharding (SURVEY.md 8e): every 8^3 tile of the map has exactly one owner among `count` ranks. The owner is a
// function of the block index and the tile position only, so every rank computes the same partition.
__host__ __device__ __forceinline__ int tile_owner(uint64_t block_key, int tile, int count) {
  if (count <= 1) return 0;
  return (int)(mix64(block_key * 0x9E3779B97F4A7C15ull + (uint64_t)tile + 1ull) % (uint32_t)count);
}
// voxblox getBlockIndexFromGlobalVoxelIndex: floor(float(g) * vps_inv) (A.2)
__host__ __device__ __forceinline__ I3 block_of_voxel(I3 g, float vps_inv) {
  I3 b;
  b.x = (int)floorf((float)g.x * vps_inv);
  b.y = (int)floorf((float)g.y * vps_inv);
  b.z = (int)floorf((float)g.z * vps_inv);
  return b;
}

}  // namespace ksg
