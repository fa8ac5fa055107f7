// Shared implementation of the two drop-in integrators: owns the ksg handle (include/ksg.h) and keeps the host
// Layer<TsdfVoxel> / Layer<SemanticVoxel> in step with the device-resident map.
#pragma once
#include <vector>
#include "kimera_semantics/semantic_integrator_base.h"
struct ksg_integrator;
namespace kimera {
// How the host layers follow the device map after integratePointCloud returns (SURVEY.md 8b "Ownership"):
//  kEager (default, reference semantics): every block the call updated is copied back before the call returns;
//  kLazy : nothing is copied until syncLayers() is called (mesher / ESDF / save should call it first).
enum class LayerSyncMode : int { kEager = 0, kLazy = 1 };

class GpuIntegratorCore {
 public:
  GpuIntegratorCore(int integrator_type, const vxb::TsdfIntegratorBase::Config& config,
                    const SemanticIntegratorBase::SemanticConfig& semantic_config, vxb::Layer<vxb::TsdfVoxel>* tsdf_layer,
                    vxb::Layer<SemanticVoxel>* semantic_layer);
  ~GpuIntegratorCore();
  GpuIntegratorCore(const GpuIntegratorCore&) = delete;
  GpuIntegratorCore& operator=(const GpuIntegratorCore&) = delete;

  void integrate(const vxb::Transformation& T_G_C, const vxb::Pointcloud& points_C, const vxb::Color* colors,
                 const SemanticLabel* labels, bool freespace_points);
  // Depth + label frame entry (SURVEY.md 8f NEXT-1): the back-projection of PointCloudFromDepth::convert<float>
  // (kimera_semantics_ros/include/kimera_semantics_ros/depth_map_to_pointcloud.h:222-266) fused into the device path, so the caller
  // skips the point-cloud round trip.  depth: height*width float32 metres (non-finite = invalid), label: height*width uint8,
  // K = fx fy cx cy as the doubles of sensor_msgs/CameraInfo.
  void integrateDepth(const vxb::Transformation& T_G_C, const float* depth, const SemanticLabel* label, int width, int height,
                      const double K[4]);
  void setLayerSyncMode(LayerSyncMode m) { sync_mode_ = m; }
  void syncLayers();           // copy every device block into the host layers
  void syncUpdatedBlocks();    // copy the blocks of the last integrate call
  // The other direction: replace the device map by the contents of the host layers (ksg_reset + ksg_import_blocks), e.g. after
  // map_io::loadLayers.  The fast integrator's two approximate sets start empty, as in a freshly constructed reference integrator.
  void uploadLayers();
  // Semantic mesh of the device map (ksg_extract_mesh): triangle soup, per-vertex TsdfVoxel.color and semantic label, blocks in (z, y, x) order
  bool extractMesh(float min_weight, std::vector<float>* vertices, std::vector<uint8_t>* rgba, std::vector<uint8_t>* labels,
                   std::vector<int32_t>* block_index, std::vector<int64_t>* block_first);
  // The semantic mesh kept on the device (ksg_update_mesh): re-meshes the blocks a change since the last call can reach, then returns,
  // in extractMesh's layout, the meshes of the blocks that update re-meshed (ksg_export_mesh changed_only, blocks whose mesh is now
  // empty included) - after a full update (first call, new min_weight, after a clear / reset / import, or after a call that failed)
  // every block.  *full (may be NULL) tells which.  Works in kLazy mode without syncLayers().
  bool updateMesh(float min_weight, std::vector<float>* vertices, std::vector<uint8_t>* rgba, std::vector<uint8_t>* labels,
                  std::vector<int32_t>* block_index, std::vector<int64_t>* block_first, bool* full);
  // The whole device mesh layer after bringing it up to date (ksg_update_mesh, then ksg_export_mesh of every block); the next
  // updateMesh then returns every block.
  bool meshLayer(float min_weight, std::vector<float>* vertices, std::vector<uint8_t>* rgba, std::vector<uint8_t>* labels,
                 std::vector<int32_t>* block_index, std::vector<int64_t>* block_first);
  // Point queries on the device map (ksg_query_points), read-only and without a copy of the map: works in kLazy mode without
  // syncLayers().  Per point: flags (KSG_QUERY_*), the containing voxel (TsdfVoxel fields, SemanticVoxel label / log-probabilities /
  // colour; NaN / 0 when its block is not allocated), voxblox's trilinear distance and its gradient (NaN when not valid).
  struct QueryResult {
    std::vector<uint8_t> flags;                       // n
    std::vector<float> tsdf_distance, tsdf_weight;    // n, n
    std::vector<uint8_t> tsdf_rgba, sem_label;        // 4n, n
    std::vector<float> sem_priors;                    // n * kTotalNumberOfLabels
    std::vector<uint8_t> sem_rgba;                    // 4n
    std::vector<float> distance, gradient;            // n, 3n
  };
  bool queryPoints(const vxb::Pointcloud& points_G, float min_weight, QueryResult* result);
  // Depth and semantic images of the device map from pose T_G_C (ksg_render_view), read-only like queryPoints: works in kLazy mode
  // without syncLayers().  K = fx fy cx cy.  Per pixel (row-major, w * h): the camera depth and world point of the first surface hit
  // (NaN on a miss) and queryPoints' answer at that point.
  struct RenderResult {
    std::vector<float> depth;      // w * h
    std::vector<float> points_G;   // 3 * w * h
    QueryResult at_hit;            // w * h points
  };
  bool renderView(const vxb::Transformation& T_G_C, const double K[4], int w, int h, float min_depth, float max_depth, float min_weight,
                  RenderResult* result);
  // Batch Euclidean signed distance field of the device map (ksg_compute_esdf, csrc/ksg_esdf.cuh), read-only like queryPoints: works in
  // kLazy mode without syncLayers().  Replaces the contents of *esdf_layer (same voxel size and voxels_per_side as the map) with one
  // block per allocated map block: observed = OBSERVED, fixed = SURFACE, distance as computed; an unobserved voxel is voxblox's default
  // EsdfVoxel (distance 0, not observed).
  bool computeEsdf(float min_weight, float max_distance, vxb::Layer<vxb::EsdfVoxel>* esdf_layer);
  // The ESDF kept on the device (ksg_update_esdf): brings the device layer up to date from the blocks that changed since the last call,
  // then refreshes in *esdf_layer only the blocks that update rewrote (ksg_export_esdf changed_only), allocating new ones - after a full
  // update (first call, new parameters, after a clear / reset / import, or after a call that failed) the whole layer.  Afterwards
  // *esdf_layer holds what computeEsdf would give, provided only this call wrote it.  Works in kLazy mode without syncLayers().
  bool updateEsdf(float min_weight, float max_distance, vxb::Layer<vxb::EsdfVoxel>* esdf_layer);
  // ESDF point queries on the device layer as of the last updateEsdf (ksg_query_esdf): per point the KSG_QUERY_* flags, the containing
  // voxel's KSG_ESDF_* flags and distance, the trilinear ESDF distance and its gradient.
  struct EsdfQueryResult {
    std::vector<uint8_t> flags, voxel_flags;   // n, n
    std::vector<float> voxel_distance;         // n
    std::vector<float> distance;               // n
    std::vector<float> gradient;               // 3n
  };
  bool queryEsdf(const vxb::Pointcloud& points_G, EsdfQueryResult* result);
  int64_t lastVoxelUpdates() const { return last_voxel_updates_; }
  ksg_integrator* handle() { return handle_; }

 private:
  void copyBlocks(const std::vector<int32_t>& idx);
  bool exportMesh(int32_t changed_only, std::vector<float>* vertices, std::vector<uint8_t>* rgba, std::vector<uint8_t>* labels,
                  std::vector<int32_t>* block_index, std::vector<int64_t>* block_first);
  void syncAfterCall();        // eager mode: update log (fast) or updated blocks (merged)
  bool update_log_tried_ = false, update_log_on_ = false;
  bool esdf_resync_ = true;    // updateEsdf: the host layer must be refreshed whole (first call, or the last call failed)
  bool mesh_resync_ = true;    // updateMesh: the caller must be given every block (first call, or the last call failed)
  ksg_integrator* handle_ = nullptr;
  vxb::Layer<vxb::TsdfVoxel>* tsdf_layer_;
  vxb::Layer<SemanticVoxel>* semantic_layer_;
  LayerSyncMode sync_mode_ = LayerSyncMode::kEager;
  int64_t last_voxel_updates_ = 0;
};
}  // namespace kimera
