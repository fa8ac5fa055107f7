// Checkpoint / resume of the two host layers (SURVEY.md 8f NEXT-3: "a simple binary for the semantic layer - the reference has
// none"; the reference saves only the TSDF layer, through voxblox's .vxblx writer, kimera_semantics_rosbag.cpp:148-166 - that
// format is in vxblx_io.h).  One self-describing little-endian file for BOTH layers:
//   "KSGM", u32 version = 1, f32 voxel_size, u32 voxels_per_side, u32 num_labels, u64 num_blocks, then per block (sorted z,y,x):
//   i32 index[3], f32 distance[V], f32 weight[V], u8 tsdf_rgba[4V], u8 label[V], f32 priors[V*C], u8 semantic_rgba[4V]
// Host-only code; SemanticTsdfServer::loadMap() pushes the loaded layers to the device map through ksg_import_blocks.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <fstream>
#include <string>
#include <vector>
#include "kimera_semantics/semantic_voxel.h"
#include "voxblox/core/layer.h"
#include "voxblox/core/voxel.h"

namespace kimera {
namespace map_io {

static const char kMagic[4] = {'K', 'S', 'G', 'M'};
static const uint32_t kVersion = 1u;

template <typename VoxelType>
inline std::vector<vxb::BlockIndex> sortedBlocks(const vxb::Layer<VoxelType>& layer) {
  vxb::BlockIndexList all;
  layer.getAllAllocatedBlocks(&all);
  std::vector<vxb::BlockIndex> v(all.begin(), all.end());
  std::sort(v.begin(), v.end(), [](const vxb::BlockIndex& a, const vxb::BlockIndex& b) {
    return a.z() != b.z() ? a.z() < b.z() : (a.y() != b.y() ? a.y() < b.y() : a.x() < b.x());
  });
  return v;
}

// Returns false (and leaves a partial file) on I/O errors or when a TSDF block has no semantic twin.
inline bool saveLayers(const std::string& path, const vxb::Layer<vxb::TsdfVoxel>& tsdf, const vxb::Layer<SemanticVoxel>& semantic) {
  std::ofstream o(path.c_str(), std::ios::binary);
  if (!o.good()) return false;
  const std::vector<vxb::BlockIndex> blocks = sortedBlocks(tsdf);
  const float voxel_size = tsdf.voxel_size();
  const uint32_t vps = (uint32_t)tsdf.voxels_per_side(), C = (uint32_t)kTotalNumberOfLabels;
  const uint64_t nb = blocks.size();
  o.write(kMagic, 4);
  o.write(reinterpret_cast<const char*>(&kVersion), 4);
  o.write(reinterpret_cast<const char*>(&voxel_size), 4);
  o.write(reinterpret_cast<const char*>(&vps), 4);
  o.write(reinterpret_cast<const char*>(&C), 4);
  o.write(reinterpret_cast<const char*>(&nb), 8);
  const size_t V = (size_t)vps * vps * vps;
  std::vector<float> dist(V), weight(V), priors(V * C);
  std::vector<uint8_t> rgba(4 * V), label(V), srgba(4 * V);
  for (const vxb::BlockIndex& bi : blocks) {
    const vxb::Block<vxb::TsdfVoxel>::ConstPtr tb = tsdf.getBlockPtrByIndex(bi);
    const vxb::Block<SemanticVoxel>::ConstPtr sb = semantic.getBlockPtrByIndex(bi);
    if (!tb || !sb) return false;
    for (size_t v = 0; v < V; ++v) {
      const vxb::TsdfVoxel& tv = tb->getVoxelByLinearIndex(v);
      const SemanticVoxel& sv = sb->getVoxelByLinearIndex(v);
      dist[v] = tv.distance;
      weight[v] = tv.weight;
      rgba[4 * v] = tv.color.r; rgba[4 * v + 1] = tv.color.g; rgba[4 * v + 2] = tv.color.b; rgba[4 * v + 3] = tv.color.a;
      label[v] = sv.semantic_label;
      for (size_t c = 0; c < C; ++c) priors[v * C + c] = sv.semantic_priors[c];
      srgba[4 * v] = sv.color.r; srgba[4 * v + 1] = sv.color.g; srgba[4 * v + 2] = sv.color.b; srgba[4 * v + 3] = sv.color.a;
    }
    const int32_t idx[3] = {bi.x(), bi.y(), bi.z()};
    o.write(reinterpret_cast<const char*>(idx), 12);
    o.write(reinterpret_cast<const char*>(dist.data()), 4 * V);
    o.write(reinterpret_cast<const char*>(weight.data()), 4 * V);
    o.write(reinterpret_cast<const char*>(rgba.data()), 4 * V);
    o.write(reinterpret_cast<const char*>(label.data()), V);
    o.write(reinterpret_cast<const char*>(priors.data()), 4 * V * C);
    o.write(reinterpret_cast<const char*>(srgba.data()), 4 * V);
  }
  o.flush();
  return o.good();
}

// Replaces the contents of both layers by the file's blocks.  Returns false - layers untouched - when the file is not a KSGM
// file of this version or its geometry / label count differs from the layers'; false with partially filled layers on a
// truncated file.
inline bool loadLayers(const std::string& path, vxb::Layer<vxb::TsdfVoxel>* tsdf, vxb::Layer<SemanticVoxel>* semantic) {
  if (!tsdf || !semantic) return false;
  std::ifstream f(path.c_str(), std::ios::binary);
  if (!f.good()) return false;
  char magic[4];
  uint32_t version = 0, vps = 0, C = 0;
  float voxel_size = 0.0f;
  uint64_t nb = 0;
  f.read(magic, 4);
  f.read(reinterpret_cast<char*>(&version), 4);
  f.read(reinterpret_cast<char*>(&voxel_size), 4);
  f.read(reinterpret_cast<char*>(&vps), 4);
  f.read(reinterpret_cast<char*>(&C), 4);
  f.read(reinterpret_cast<char*>(&nb), 8);
  if (!f.good() || std::memcmp(magic, kMagic, 4) != 0 || version != kVersion) return false;
  if (voxel_size != tsdf->voxel_size() || vps != tsdf->voxels_per_side() || C != kTotalNumberOfLabels ||
      voxel_size != semantic->voxel_size() || vps != semantic->voxels_per_side()) return false;
  const size_t V = (size_t)vps * vps * vps;
  {   // nothing is touched unless the file holds exactly the nb blocks its header announces (truncated / corrupt files leave the layers as they are)
    const std::streampos here = f.tellg();
    f.seekg(0, std::ios::end);
    const uint64_t file_bytes = (uint64_t)f.tellg();
    f.seekg(here);
    const uint64_t per_block = 12ull + (uint64_t)V * (4ull + 4ull + 4ull + 1ull + 4ull * C + 4ull);
    if (!f.good() || nb > (file_bytes / per_block) || (uint64_t)here + nb * per_block != file_bytes) return false;
  }
  tsdf->removeAllBlocks();
  semantic->removeAllBlocks();
  std::vector<float> dist(V), weight(V), priors(V * C);
  std::vector<uint8_t> rgba(4 * V), label(V), srgba(4 * V);
  for (uint64_t b = 0; b < nb; ++b) {
    int32_t idx[3];
    f.read(reinterpret_cast<char*>(idx), 12);
    f.read(reinterpret_cast<char*>(dist.data()), 4 * V);
    f.read(reinterpret_cast<char*>(weight.data()), 4 * V);
    f.read(reinterpret_cast<char*>(rgba.data()), 4 * V);
    f.read(reinterpret_cast<char*>(label.data()), V);
    f.read(reinterpret_cast<char*>(priors.data()), 4 * V * C);
    f.read(reinterpret_cast<char*>(srgba.data()), 4 * V);
    if (!f.good()) return false;
    const vxb::BlockIndex bi(idx[0], idx[1], idx[2]);
    vxb::Block<vxb::TsdfVoxel>::Ptr tb = tsdf->allocateBlockPtrByIndex(bi);
    vxb::Block<SemanticVoxel>::Ptr sb = semantic->allocateBlockPtrByIndex(bi);
    for (size_t v = 0; v < V; ++v) {
      vxb::TsdfVoxel& tv = tb->getVoxelByLinearIndex(v);
      tv.distance = dist[v];
      tv.weight = weight[v];
      tv.color = vxb::Color(rgba[4 * v], rgba[4 * v + 1], rgba[4 * v + 2], rgba[4 * v + 3]);
      SemanticVoxel& sv = sb->getVoxelByLinearIndex(v);
      sv.semantic_label = label[v];
      for (size_t c = 0; c < C; ++c) sv.semantic_priors[c] = priors[v * C + c];
      sv.color = HashableColor(srgba[4 * v], srgba[4 * v + 1], srgba[4 * v + 2], srgba[4 * v + 3]);
    }
    tb->has_data() = true;
    sb->has_data() = true;
  }
  return true;
}

}  // namespace map_io
}  // namespace kimera
