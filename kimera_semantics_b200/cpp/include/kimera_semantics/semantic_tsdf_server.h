// ROS-free counterpart of kimera::SemanticTsdfServer (reference kimera_semantics_ros/src/semantic_tsdf_server.cpp:58-79 and the
// part of voxblox_ros TsdfServer it relies on): owns Layer<TsdfVoxel> + Layer<SemanticVoxel>, builds the integrator through
// SemanticTsdfIntegratorFactory exactly as the reference constructor does, and feeds it clouds (integratePointCloud) or
// depth + label frames (the fused back-projection entry of the C-ABI).  SURVEY.md 8f NEXT-2.
#pragma once
#include <memory>
#include <string>
#include "kimera_semantics/map_io.h"
#include "kimera_semantics/ply_io.h"
#include "kimera_semantics/vxblx_io.h"
#include "kimera_semantics/semantic_tsdf_integrator_factory.h"
#include "kimera_semantics/semantic_tsdf_integrator_fast.h"
#include "kimera_semantics/semantic_tsdf_integrator_merged.h"

namespace kimera {

class SemanticTsdfServer {
 public:
  struct Params {                      // the rosparams the reference reads (ros_params.cpp:20-77, kimera_semantics.launch:98-122)
    vxb::FloatingPoint tsdf_voxel_size = 0.05f;
    size_t tsdf_voxels_per_side = 16u;
    std::string method = "fast";       // ros_params.cpp:24-28
    double min_time_between_msgs_sec = 0.0;   // kimera_semantics.launch:101 uses 0.2
    LayerSyncMode layer_sync = LayerSyncMode::kEager;
  };

  SemanticTsdfServer(const Params& params, const vxb::TsdfIntegratorBase::Config& integrator_config,
                     const SemanticIntegratorBase::SemanticConfig& semantic_config)
      : params_(params), semantic_config_(semantic_config) {
    tsdf_layer_.reset(new vxb::Layer<vxb::TsdfVoxel>(params.tsdf_voxel_size, params.tsdf_voxels_per_side));
    // semantic_tsdf_server.cpp:68-69: the semantic layer copies the TSDF layer's geometry
    semantic_layer_.reset(new vxb::Layer<SemanticVoxel>(params.tsdf_voxel_size, params.tsdf_voxels_per_side));
    // semantic_tsdf_server.cpp:71-77: replace the default integrator by the semantic one
    tsdf_integrator_ = SemanticTsdfIntegratorFactory::create(params.method, integrator_config, semantic_config_, tsdf_layer_.get(),
                                                             semantic_layer_.get());
    KSG_CHECK(tsdf_integrator_ != nullptr);
    gpu().setLayerSyncMode(params.layer_sync);
  }

  // TsdfServer::processPointCloudMessageAndInsert -> integratePointcloud (kimera_semantics_rosbag.cpp:134).
  // Returns false when the frame is dropped by the min_time_between_msgs_sec throttle.
  bool processPointCloud(const vxb::Transformation& T_G_C, const vxb::Pointcloud& points_C, const vxb::Colors& colors,
                         double stamp_sec, bool is_freespace_pointcloud = false) {
    if (have_last_ && stamp_sec - last_stamp_sec_ < params_.min_time_between_msgs_sec) return false;
    last_stamp_sec_ = stamp_sec;
    have_last_ = true;
    tsdf_integrator_->integratePointCloud(T_G_C, points_C, colors, is_freespace_pointcloud);
    return true;
  }

  // The same for a depth + label frame (what kimera_semantics_rosbag.cpp:112-134 turns into a coloured cloud first): the
  // back-projection runs on the device.  K = fx fy cx cy of the camera info message.
  bool processDepthFrame(const vxb::Transformation& T_G_C, const float* depth, const SemanticLabel* label, int width, int height,
                         const double K[4], double stamp_sec) {
    if (have_last_ && stamp_sec - last_stamp_sec_ < params_.min_time_between_msgs_sec) return false;
    last_stamp_sec_ = stamp_sec;
    have_last_ = true;
    gpu().integrateDepth(T_G_C, depth, label, width, height, K);
    return true;
  }

  GpuIntegratorCore& gpu() {
    if (auto* f = dynamic_cast<FastSemanticTsdfIntegrator*>(tsdf_integrator_.get())) return f->gpu();
    auto* m = dynamic_cast<MergedSemanticTsdfIntegrator*>(tsdf_integrator_.get());
    KSG_CHECK(m != nullptr);
    return m->gpu();
  }
  // bring the host layers up to date (needed before meshing / saving when layer_sync == kLazy)
  void updateLayers() { gpu().syncLayers(); }

  // Checkpoint / resume (the reference saves its TSDF layer with TsdfServer::saveMap, kimera_semantics_rosbag.cpp:150; here both
  // layers go into one file, see map_io.h).  saveMap brings the host layers up to date first; loadMap replaces the host layers
  // AND the device map by the file's contents, after which integration continues as if it had never stopped (the fast
  // integrator's per-scan approximate sets restart empty, exactly as after constructing a new reference integrator).
  bool saveMap(const std::string& path) {
    updateLayers();
    return map_io::saveLayers(path, *tsdf_layer_, *semantic_layer_);
  }
  bool loadMap(const std::string& path) {
    if (!map_io::loadLayers(path, tsdf_layer_.get(), semantic_layer_.get())) return false;
    gpu().uploadLayers();
    return true;
  }

  // The reference's own output file: the TSDF layer as a voxblox .vxblx (TsdfServer::saveMap -> voxblox::io::SaveLayer,
  // kimera_semantics_rosbag.cpp:148-166), readable by voxblox tools; see vxblx_io.h for the (restated, unpinned) format.
  bool saveTsdfVxblx(const std::string& path) {
    updateLayers();
    return vxblx_io::saveTsdfLayer(path, *tsdf_layer_);
  }

  // What the reference's server publishes for display: the voxblox mesh coloured by TsdfVoxel.color (launch/kimera_semantics.launch:130-132),
  // here extracted from the device map (ksg_extract_mesh, csrc/ksg_mesh.cuh): a triangle soup (3 consecutive vertices per triangle) with
  // the voxel colour and the semantic label per vertex; blocks in (z, y, x) order, block_first[i] = first vertex of block i.
  struct SemanticMesh {
    std::vector<float> vertices;          // 3 per vertex
    std::vector<uint8_t> rgba, labels;    // 4 / 1 per vertex
    std::vector<int32_t> block_index;     // 3 per block
    std::vector<int64_t> block_first;     // blocks + 1
  };
  bool extractMesh(SemanticMesh* mesh, float min_weight = 1e-4f) {
    return gpu().extractMesh(min_weight, &mesh->vertices, &mesh->rgba, &mesh->labels, &mesh->block_index, &mesh->block_first);
  }
  // voxblox's TsdfServer::updateMesh: brings the device mesh layer up to date with the map, re-meshing only the blocks a change since the
  // last call can reach (GpuIntegratorCore::updateMesh, csrc/ksg_mesh.cuh), and returns in *changed the meshes of the blocks to publish:
  // those re-meshed (a block whose mesh is now empty included: a viewer must drop its triangles), or after a full update every block
  // (*full, may be NULL, says which).  A viewer keeps one mesh per block and replaces the blocks it is given.  Needs no updateLayers().
  bool updateMesh(SemanticMesh* changed, float min_weight = 1e-4f, bool* full = nullptr) {
    return gpu().updateMesh(min_weight, &changed->vertices, &changed->rgba, &changed->labels, &changed->block_index, &changed->block_first, full);
  }
  // voxblox's TsdfServer::generateMesh: the whole mesh layer, brought up to date as updateMesh does (GpuIntegratorCore::meshLayer),
  // written to `ply_path` - the file the reference's `mesh_filename` parameter names - as the ASCII .ply of ply_io.h.  The next
  // updateMesh returns every block.
  bool generateMesh(const std::string& ply_path, float min_weight = 1e-4f) {
    SemanticMesh mesh;
    if (!gpu().meshLayer(min_weight, &mesh.vertices, &mesh.rgba, &mesh.labels, &mesh.block_index, &mesh.block_first)) return false;
    return kimera_semantics::writeMeshPly(ply_path, mesh.vertices, mesh.rgba, mesh.labels);
  }

  // What a planner / scene-graph builder asks the map about points (Layer::getVoxelPtrByCoordinates + Interpolator::getDistance /
  // getGradient on the host), answered on the device from the device map (ksg_query_points, csrc/ksg_query.cuh): needs no updateLayers().
  bool queryPoints(const vxb::Pointcloud& points_G, float min_weight, GpuIntegratorCore::QueryResult* result) {
    return gpu().queryPoints(points_G, min_weight, result);
  }

  // What a camera at T_G_C would see of the fused map - depth, hit points, labels, normals (gradient) - rendered on the device from the
  // device map (ksg_render_view, csrc/ksg_render.cuh): needs no updateLayers().
  bool renderView(const vxb::Transformation& T_G_C, const double K[4], int w, int h, float min_depth, float max_depth, float min_weight,
                  GpuIntegratorCore::RenderResult* result) {
    return gpu().renderView(T_G_C, K, w, h, min_depth, max_depth, min_weight, result);
  }

  // voxblox's EsdfServer::updateEsdfBatch(full_euclidean_distance = true), the last step of the reference's offline driver
  // (kimera_semantics_rosbag.cpp:160-166): the ESDF of the whole map, computed on the device from the device map
  // (GpuIntegratorCore::computeEsdf, csrc/ksg_esdf.cuh; not voxblox's queue algorithm): needs no updateLayers().
  bool updateEsdfBatch(vxb::Layer<vxb::EsdfVoxel>* esdf_layer, float max_distance, float min_weight = 1e-4f) {
    return gpu().computeEsdf(min_weight, max_distance, esdf_layer);
  }
  // voxblox's EsdfServer::updateEsdf: brings *esdf_layer up to date with the map, recomputing on the device only what the blocks changed
  // since the last call can have changed (GpuIntegratorCore::updateEsdf); the same field as updateEsdfBatch, and like it needs no
  // updateLayers().
  bool updateEsdf(vxb::Layer<vxb::EsdfVoxel>* esdf_layer, float max_distance, float min_weight = 1e-4f) {
    return gpu().updateEsdf(min_weight, max_distance, esdf_layer);
  }

  vxb::Layer<vxb::TsdfVoxel>* getTsdfLayerPtr() { return tsdf_layer_.get(); }
  vxb::Layer<SemanticVoxel>* getSemanticLayerPtr() { return semantic_layer_.get(); }
  vxb::TsdfIntegratorBase* getIntegratorPtr() { return tsdf_integrator_.get(); }

 private:
  Params params_;
  SemanticIntegratorBase::SemanticConfig semantic_config_;
  std::unique_ptr<vxb::Layer<vxb::TsdfVoxel>> tsdf_layer_;
  std::unique_ptr<vxb::Layer<SemanticVoxel>> semantic_layer_;
  std::unique_ptr<vxb::TsdfIntegratorBase> tsdf_integrator_;
  double last_stamp_sec_ = 0.0;
  bool have_last_ = false;
};

}  // namespace kimera
