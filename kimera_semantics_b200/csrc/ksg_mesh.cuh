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

}  // namespace ksg
