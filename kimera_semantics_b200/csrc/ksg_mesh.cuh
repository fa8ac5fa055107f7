// ksg_mesh.cuh — NEXT-4 (SURVEY.md 8f): semantic mesh extraction on the device.
//
// What the reference shows of its map is a voxblox mesh whose vertex colours are TsdfVoxel.color - the field the semantic integrators
// overwrite with the label colour (kimera_semantics/src/semantic_integrator_base.cpp:172-191, launch/kimera_semantics.launch:130-132).
// The mesher itself is voxblox's MeshIntegrator + MarchingCubes, which is NOT under /root/reference: "parity unpinned" - this file
// restates it from knowledge of that code (voxblox/mesh/mesh_integrator.h, marching_cubes.h, utils/meshing_utils.h):
//   * one cube per voxel, corners = the voxel and its +x / +y / +z neighbours (also across block borders; a cube with a corner in a
//     missing block or with weight <= min_weight produces nothing),
//   * corner coordinates = block origin + (local index + 0.5) * voxel_size (+ voxel_size per offset), vertex on a crossed edge =
//     v1 + sdf1 / (sdf1 - sdf2) * (v2 - v1)  (midpoint if |sdf1 - sdf2| < 1e-6),
//   * vertex colour (and, here, also the semantic label) = those of the voxel that contains the vertex, (0,0,0,0) / 0 if that voxel is
//     unobserved (weight <= min_weight) or missing.
// Deliberate differences: the triangle table is generated (tools/make_mc_table.py: watertight on ambiguous faces) and the cubes of a
// block are emitted in linear voxel order (voxblox: interior cubes first, then the three border planes) - a mesh is a set of triangles.
// The numpy twin is tests/mesh_ref.py; tests/test_gpu_mesh.py compares bit for bit.
//
// The device mesh layer (ksg_update_mesh / ksg_export_mesh / ksg_mesh_view_device) keeps every block's mesh, as k_mesh_blocks emits it,
// in a vertex arena laid out by pool slot, and re-meshes only the blocks a map change can reach.
//
// What block B's mesh reads.  k_mesh_blocks builds it from (a) the voxels of the blocks B + {0,1}^3 (the cube corners), (b) which of
// those blocks exist, and (c) the containing voxel of every vertex, for its colour and label.  (c) lies in B + {0,1}^3 as well, by the
// window bound below, for every block within it.
//
// The dirty set.  Per update:
//   C = the slots whose touched_stamp is newer than the last update, plus the slots allocated since it;
//   R = the allocated blocks b with b + e in C for some e in {0,1}^3, i.e. C and its allocated lower neighbours at the 7 offsets -e.
// The update re-meshes R and keeps every other block's mesh.  Why this is exact: voxel contents change only through the integrate calls
// and ksg_merge_blocks_device / ksg_merge_voxels_device, which all stamp the blocks they write, and through ksg_import_blocks,
// ksg_clear_map and ksg_reset, which all make the next update full (as for the ESDF layer).  Block existence changes only by allocation,
// and a block allocated since the last update is in C.  So a block outside R has, in B + {0,1}^3, no voxel that changed and no block that
// appeared, and its mesh is what it was.  A new min_weight changes what every cube reads, so it too makes the update full.
// This is deliberately stricter than voxblox's only_mesh_updated_blocks, which (as far as it can be restated here; voxblox is not in the
// reference tree, so this is unpinned) re-meshes only the updated blocks: the cubes of a lower neighbour that cross into an updated block
// keep stale triangles there.  tests/mesh_incremental_ref.py models C and R; tests/test_mesh_incremental_cpu.py shows that the rule is
// exact on random edits and that it catches its mutants (face neighbours only, upper instead of lower neighbours, new blocks ignored).
//
// The window bound.  The colour lookup falls back to ht_lookup_slot for a vertex whose containing voxel lies outside B + {0,1}^3; R does
// not cover that case, so it must not happen for a block the incremental rule keeps.  Per axis, let g = b * vps + l be the global index
// of the cube's lower corner voxel, K = (|b| + 1) * vps + 2, u = 2^-24.  Both edge ends are computed from B's origin, fl(b * (vps * vs))
// (vps * vs is exact: vps is a power of two), as base = fl(origin + fl((l + 0.5) * vs)), then + vs per offset; each of these roundings
// errs by at most u times a magnitude <= K * vs, so each end is off by <= 4 u K vs.  On the edge's axis t = fl(sa / (sa - sb)) lies in
// [0, 1] (the signs differ, and fl(|sa| + |sb|) >= |sa|), and p = fl(pa + fl(t * fl(pb - pa))) is within 13 u K vs of
// (g + 0.5 + t) * vs; on the other two axes p equals the corner's coordinate.  fl(p * vsi), vsi = fl(1 / vs), adds 2 u K more, and
// floor(. + 1e-6) stays in {g, g + 1} while 16 u K + 1e-6 < 0.5, i.e. K < 2^19.  The layer takes K <= 2^18 = kMeshNearVoxels (twice the
// margin; -fmad=false keeps every rounding above separate).  A block beyond it is "far": its vertices may read a voxel outside its
// window.  The dirty kernel flags a far block when it enters the layer; that update is still exact (the far block is new, hence in C and
// in R, and no far block was there before it), and from then on every update is full until a clear or reset.
// tests/test_mesh_incremental_cpu.py checks the bound numerically at K = 2^18 and shows the window failing far out.
//
// Device side of an update, in stream order (no per-block array is read back; the host reads 3 scalars, then 2):
//   k_mesh_dirty      over hash positions: marks C and, through ht_lookup_slot, its 7 lower neighbours; lists R (atomic order);
//   k_mesh_blocks<0>  vertex counts of R;
//   k_mesh_scan       one CTA: per-slot counts (R's new ones, the kept ones from the previous first[]), exclusive scan -> first[];
//   k_mesh_move       copies every kept block's range from the previous arena into the new one, and clears the marks;
//   k_mesh_blocks<1>  emits R's meshes in place.
// The arena is double-buffered: O(live mesh) device copies per update and at most twice the live mesh in memory.
#pragma once
#include "ksg_kernels.cuh"
#include "ksg_mc_table.h"

namespace ksg {

struct MeshBuf {
  float* vtx;        // 3 floats per vertex, 3 vertices per triangle
  uint32_t* rgba;    // TsdfVoxel.color of the voxel containing the vertex (r | g << 8 | b << 16 | a << 24)
  uint8_t* label;    // SemanticVoxel.semantic_label of that voxel
};

static constexpr int kMeshThreads = 256;

// EMIT == false: count[blk] = vertices of block slots[blk];  EMIT == true: write them at first[blk]
template <bool EMIT>
__global__ void __launch_bounds__(kMeshThreads) k_mesh_blocks(DevCfg cfg, MapRef map, const int* __restrict__ slots, int n_blocks, float min_weight,
                                                              const long long* __restrict__ first, int* __restrict__ count, MeshBuf out) {
  __shared__ int s_nb[8];
  __shared__ int s_wsum[kMeshThreads / 32];
  __shared__ int s_run;
  __shared__ float s_sdf[8][kMeshThreads];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int vps = cfg.vps, vm = vps - 1, nvox = vps * vps * vps;
  const float vs = cfg.voxel_size;
  const float block_size = (float)vps * vs;
  for (int blk = blockIdx.x; blk < n_blocks; blk += gridDim.x) {
    const int slot = slots[blk];
    const I3 bi = unpack_key(map.slot_key[slot]);
    __syncthreads();
    if (tid < 8) {
      I3 nb = bi;
      nb.x += tid & 1; nb.y += (tid >> 1) & 1; nb.z += tid >> 2;
      s_nb[tid] = (tid == 0) ? slot : (key_in_range(nb) ? ht_lookup_slot(map, pack_key(nb)) : -1);
    }
    if (tid == 0) s_run = 0;
    __syncthreads();
    const F3 origin = f3((float)bi.x * block_size, (float)bi.y * block_size, (float)bi.z * block_size);
    int my_total = 0;
    for (int v0 = 0; v0 < nvox; v0 += kMeshThreads) {
      const int v = v0 + tid;
      const int lx = v & vm, ly = (v / vps) & vm, lz = v / (vps * vps);
      int cfg_idx = 0;
      bool ok = v < nvox;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int ox = ((i + 1) >> 1) & 1, oy = (i >> 1) & 1, oz = i >> 2;   // (0,0,0) (1,0,0) (1,1,0) (0,1,0) (0,0,1) (1,0,1) (1,1,1) (0,1,1)
        if (ok) {
          const int cx = lx + ox, cy = ly + oy, cz = lz + oz;
          const int s = s_nb[(cx >= vps ? 1 : 0) | (cy >= vps ? 2 : 0) | (cz >= vps ? 4 : 0)];
          if (s < 0) ok = false;
          else {
            int vox;
            const uint8_t* chunk = mesh_voxel_chunk(cfg, map, s, cx & vm, cy & vm, cz & vm, vox);
            const float w = ((const float*)(chunk + cfg.plane_f32))[vox];
            const float d = ((const float*)chunk)[vox];
            if (w <= min_weight) ok = false;
            s_sdf[i][tid] = d;
            if (d < 0.0f) cfg_idx |= 1 << i;
          }
        }
      }
      const int ntri = ok ? (int)kMcTris[cfg_idx] : 0;
      if (!EMIT) { my_total += ntri; continue; }
      // exclusive scan of the triangle counts in voxel order
      int incl = ntri;
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
      if (lane == 31) s_wsum[wid] = incl;
      __syncthreads();
      int before = s_run + incl - ntri;
      for (int w = 0; w < wid; ++w) before += s_wsum[w];
      __syncthreads();
      if (tid == kMeshThreads - 1) s_run = before + ntri;
      if (ntri > 0) {
        const F3 base = f3(origin.x + ((float)lx + 0.5f) * vs, origin.y + ((float)ly + 0.5f) * vs, origin.z + ((float)lz + 0.5f) * vs);
        long long at = first[blk] + 3ll * before;
        for (int k = 0; k < 3 * ntri; ++k, ++at) {
          const int e = kMcTable[cfg_idx][k];
          // edge e joins corners a, b: (0,1) (1,2) (2,3) (3,0) (4,5) (5,6) (6,7) (7,4) (0,4) (1,5) (2,6) (3,7)
          const int a = (e < 8) ? e : e - 8;
          const int b = (e < 4) ? ((e + 1) & 3) : (e < 8) ? (4 + ((e + 1) & 3)) : e - 4;
          const float sa = s_sdf[a][tid], sb = s_sdf[b][tid];
          const F3 pa = f3(base.x + (float)(((a + 1) >> 1) & 1) * vs, base.y + (float)((a >> 1) & 1) * vs, base.z + (float)(a >> 2) * vs);
          const F3 pb = f3(base.x + (float)(((b + 1) >> 1) & 1) * vs, base.y + (float)((b >> 1) & 1) * vs, base.z + (float)(b >> 2) * vs);
          const float diff = sa - sb;
          F3 p;
          if (fabsf(diff) >= 1.0e-6f) {
            const float t = sa / diff;
            p = f3(pa.x + t * (pb.x - pa.x), pa.y + t * (pb.y - pa.y), pa.z + t * (pb.z - pa.z));
          } else {
            p = f3(0.5f * (pa.x + pb.x), 0.5f * (pa.y + pb.y), 0.5f * (pa.z + pb.z));
          }
          out.vtx[3 * at] = p.x; out.vtx[3 * at + 1] = p.y; out.vtx[3 * at + 2] = p.z;
          // colour / label of the voxel that contains the vertex
          uint32_t col = 0;
          uint8_t lab = 0;
          if (index_in_range(f3(p.x * cfg.vsi, p.y * cfg.vsi, p.z * cfg.vsi))) {
            const I3 g = grid_index(p, cfg.vsi);
            const I3 gb = block_of_voxel(g, cfg.vps_inv);
            const int dx = gb.x - bi.x, dy = gb.y - bi.y, dz = gb.z - bi.z;
            int s = -1;
            if ((unsigned)dx < 2u && (unsigned)dy < 2u && (unsigned)dz < 2u) s = s_nb[dx | (dy << 1) | (dz << 2)];
            else if (key_in_range(gb)) s = ht_lookup_slot(map, pack_key(gb));
            if (s >= 0) {
              int vox;
              const uint8_t* chunk = mesh_voxel_chunk(cfg, map, s, g.x & vm, g.y & vm, g.z & vm, vox);
              if (((const float*)(chunk + cfg.plane_f32))[vox] > min_weight) {
                col = ((const uint32_t*)(chunk + 2 * cfg.plane_f32))[vox];
                lab = (chunk + 4 * cfg.plane_f32)[vox];
              }
            }
          }
          out.rgba[at] = col;
          out.label[at] = lab;
        }
      }
    }
    if (!EMIT) {
      for (int o = 16; o > 0; o >>= 1) my_total += __shfl_down_sync(0xffffffffu, my_total, o);
      if (lane == 0) s_wsum[wid] = my_total;
      __syncthreads();
      if (tid == 0) { int t = 0; for (int w = 0; w < kMeshThreads / 32; ++w) t += s_wsum[w]; count[blk] = 3 * t; }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// device mesh layer (see the header)
// ---------------------------------------------------------------------------------------------
static constexpr int kMeshNearVoxels = 1 << 18;
static constexpr int kMeshScanThreads = 1024;

struct MeshCounters {
  int changed;              // |C|
  int remeshed;             // |R|
  int far;                  // a block the dirty kernel looked at lies beyond the window bound
  int pad;
  long long vertices;       // vertices of the layer after the update
  long long remeshed_vertices;
};

__device__ __forceinline__ bool mesh_block_far(I3 b, int vps) {
  const long long lim = kMeshNearVoxels - 2;
  return ((long long)abs(b.x) + 1) * vps > lim || ((long long)abs(b.y) + 1) * vps > lim || ((long long)abs(b.z) + 1) * vps > lim;
}

// mark[s] |= bit; the first mark of a slot lists it in R
__device__ __forceinline__ void mesh_mark(int s, unsigned bit, unsigned* mark, int* rpos, int* list, MeshCounters* ctr) {
  if (atomicOr(mark + s, bit) == 0u) {
    const int i = atomicAdd(&ctr->remeshed, 1);
    list[i] = s;
    rpos[s] = i;
  }
}

// Over hash positions: slot s in [0, nb) is in C when it was allocated since the last update (s >= prev; prev = 0: a full update) or
// its stamp is newer than `stamp`; C and the allocated blocks at the 7 offsets -e of a C block are marked and listed in R.  Marks are
// 0 on entry (k_mesh_move clears them).  Slots >= prev are also checked against the window bound.
__global__ void __launch_bounds__(256) k_mesh_dirty(MapRef map, int nb, int prev, int stamp, int vps, unsigned* __restrict__ mark,
                                                    int* __restrict__ rpos, int* __restrict__ list, MeshCounters* __restrict__ ctr) {
  const long long cap = (long long)map.ht_mask + 1;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long p0 = (long long)blockIdx.x * blockDim.x; p0 < cap; p0 += stride) {   // warp-uniform trip count (ballots below)
    const long long p = p0 + threadIdx.x;
    int s = -1;
    bool in_c = false, far = false;
    if (p < cap) {
      s = map.ht_slot[p];
      if (s >= 0 && s < nb) {
        in_c = s >= prev || map.touched_stamp[p] > stamp;
        if (s >= prev) far = mesh_block_far(unpack_key(map.slot_key[s]), vps);
      }
    }
    const unsigned c_ballot = __ballot_sync(0xffffffffu, in_c), f_ballot = __ballot_sync(0xffffffffu, far);
    if ((threadIdx.x & 31) == 0) {
      if (c_ballot) atomicAdd(&ctr->changed, __popc(c_ballot));
      if (f_ballot) atomicOr(&ctr->far, 1);
    }
    if (!in_c) continue;
    mesh_mark(s, 1u, mark, rpos, list, ctr);
    const I3 b = unpack_key(map.slot_key[s]);
    for (int e = 1; e < 8; ++e) {
      const I3 n{b.x - (e & 1), b.y - ((e >> 1) & 1), b.z - (e >> 2)};
      if (!key_in_range(n)) continue;
      const int t = ht_lookup_slot(map, pack_key(n));
      if (t >= 0 && t < nb) mesh_mark(t, 2u, mark, rpos, list, ctr);
    }
  }
}

// One CTA.  Per slot s < nb: its vertex count, count[rpos[s]] when marked (R), else old_first[s + 1] - old_first[s]; new_first = the
// exclusive scan, new_first[nb] = the total.  R's entries get lfirst[rpos[s]] = new_first[s] (where k_mesh_blocks<true> emits them).
__global__ void __launch_bounds__(kMeshScanThreads) k_mesh_scan(int nb, const unsigned* __restrict__ mark, const int* __restrict__ rpos,
                                                               const int* __restrict__ count, const long long* __restrict__ old_first,
                                                               long long* __restrict__ new_first, long long* __restrict__ lfirst,
                                                               MeshCounters* __restrict__ ctr) {
  constexpr int kItems = 4, kTile = kMeshScanThreads * kItems;
  __shared__ long long s_warp[kMeshScanThreads / 32];
  __shared__ long long s_carry;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) s_carry = 0;
  long long remeshed = 0;
  for (int base = 0; base < nb; base += kTile) {
    long long c[kItems], sum = 0;
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
      const int s = base + tid * kItems + k;
      c[k] = 0;
      if (s < nb) {
        if (mark[s]) { c[k] = count[rpos[s]]; remeshed += c[k]; }
        else c[k] = old_first[s + 1] - old_first[s];
      }
      sum += c[k];
    }
    long long incl = sum;
    for (int o = 1; o < 32; o <<= 1) { const long long t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    if (lane == 31) s_warp[wid] = incl;
    __syncthreads();
    long long at = s_carry + incl - sum;
    for (int w = 0; w < wid; ++w) at += s_warp[w];
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
      const int s = base + tid * kItems + k;
      if (s < nb) {
        new_first[s] = at;
        if (mark[s]) lfirst[rpos[s]] = at;
      }
      at += c[k];
    }
    __syncthreads();
    if (tid == kMeshScanThreads - 1) s_carry = at;
    __syncthreads();
  }
  for (int o = 16; o > 0; o >>= 1) remeshed += __shfl_down_sync(0xffffffffu, remeshed, o);
  if (lane == 0) s_warp[wid] = remeshed;
  __syncthreads();
  if (tid == 0) {
    long long r = 0;
    for (int w = 0; w < kMeshScanThreads / 32; ++w) r += s_warp[w];
    new_first[nb] = s_carry;
    ctr->vertices = s_carry;
    ctr->remeshed_vertices = r;
  }
}

// Vertex ranges from one arena to another, one warp per range: range j = slot slots[j] (slots NULL: j), from src_first[slot] to
// dst_first[slot] (dst_by_slot) or dst_first[j].  With `mark`, a marked slot is skipped and its mark cleared (the update's carry-over);
// without it every range is copied (the export's gather).
__global__ void __launch_bounds__(256) k_mesh_move(int n, const int* __restrict__ slots, const long long* __restrict__ src_first,
                                                   const long long* __restrict__ dst_first, int dst_by_slot, unsigned* __restrict__ mark,
                                                   MeshBuf src, MeshBuf dst) {
  const int lane = threadIdx.x & 31;
  const int warps = (gridDim.x * blockDim.x) >> 5;
  for (int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < n; j += warps) {
    const int slot = slots ? slots[j] : j;
    if (mark) {
      const unsigned m = mark[slot];
      __syncwarp();
      if (m) { if (lane == 0) mark[slot] = 0u; continue; }
    }
    const long long from = src_first[slot], cnt = src_first[slot + 1] - from, to = dst_first[dst_by_slot ? slot : j];
    for (long long i = lane; i < 3 * cnt; i += 32) dst.vtx[3 * to + i] = src.vtx[3 * from + i];
    for (long long i = lane; i < cnt; i += 32) {
      dst.rgba[to + i] = src.rgba[from + i];
      dst.label[to + i] = src.label[from + i];
    }
  }
}

}  // namespace ksg
