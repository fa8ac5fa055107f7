// semantic_tsdf_integrator_gpu.h -- the file a kimera_semantics maintainer adds next to semantic_tsdf_integrator_{fast,merged}.h
// to route both integrator types to the H100 library (INTEGRATION.md section B).  It is written against the REFERENCE's headers
// (kimera_semantics/semantic_integrator_base.h, voxblox/integrator/tsdf_integrator.h) and the C-ABI in include/ksg.h only; in this
// repository it is compile- and link-checked against the reference's real kimera_semantics headers with `make -C oracle ref`
// (oracle/_ref/gpu_binding_check; voxblox / Eigen / glog come from the stand-ins there, from the real packages in a catkin build).
//
// Semantics kept from the reference integrators: same constructor arguments, integratePointCloud() is synchronous and on return
// both host layers hold every block the call updated (what updateLayerWithStoredBlocks / updateSemanticLayerWithStoredBlocks
// guarantee, fast.cpp:194-197), contract violations abort through glog CHECKs.
#pragma once

#include <cstdint>
#include <vector>

#include <glog/logging.h>
#include <voxblox/integrator/tsdf_integrator.h>

#include "kimera_semantics/common.h"
#include "kimera_semantics/semantic_integrator_base.h"
#include "kimera_semantics/semantic_voxel.h"

#include "ksg.h"

namespace kimera {

class GpuSemanticTsdfIntegrator : public vxb::TsdfIntegratorBase, public SemanticIntegratorBase {
 public:
  EIGEN_MAKE_ALIGNED_OPERATOR_NEW

  /// ksg_type: KSG_INTEGRATOR_FAST or KSG_INTEGRATOR_MERGED (same numbering as SemanticTsdfIntegratorType).
  GpuSemanticTsdfIntegrator(int ksg_type, const Config& config, const SemanticConfig& semantic_config,
                            vxb::Layer<vxb::TsdfVoxel>* tsdf_layer, vxb::Layer<SemanticVoxel>* semantic_layer)
      : TsdfIntegratorBase(config, CHECK_NOTNULL(tsdf_layer)), SemanticIntegratorBase(semantic_config, CHECK_NOTNULL(semantic_layer)) {
    CHECK(semantic_config.semantic_label_to_color_);
    ksg_config c;
    ksg_default_config(&c, ksg_type, tsdf_layer->voxel_size(), static_cast<int32_t>(tsdf_layer->voxels_per_side()),
                       static_cast<int32_t>(kTotalNumberOfLabels));
    // vxb::TsdfIntegratorBase::Config, field by field (config_ already went through the base-class constructor's fix-ups)
    c.default_truncation_distance = config_.default_truncation_distance;
    c.max_weight = config_.max_weight;
    c.voxel_carving_enabled = config_.voxel_carving_enabled;
    c.min_ray_length_m = config_.min_ray_length_m;
    c.max_ray_length_m = config_.max_ray_length_m;
    c.use_const_weight = config_.use_const_weight;
    c.allow_clear = config_.allow_clear;
    c.use_weight_dropoff = config_.use_weight_dropoff;
    c.use_sparsity_compensation_factor = config_.use_sparsity_compensation_factor;
    c.sparsity_compensation_factor = config_.sparsity_compensation_factor;
    c.integration_order_mode = config_.integration_order_mode == "sorted" ? KSG_ORDER_SORTED : KSG_ORDER_MIXED;
    CHECK(config_.integration_order_mode == "sorted" || config_.integration_order_mode == "mixed")
        << "Unknown integration order mode: '" << config_.integration_order_mode << "'!";
    c.enable_anti_grazing = config_.enable_anti_grazing;
    c.start_voxel_subsampling_factor = config_.start_voxel_subsampling_factor;
    c.max_consecutive_ray_collisions = config_.max_consecutive_ray_collisions;
    c.clear_checks_every_n_frames = config_.clear_checks_every_n_frames;
    c.merged_bundle_order = KSG_BUNDLE_ORDER_LIBSTDCXX;   // the reference's unordered_map iteration order (merged.cpp:210-231)
    // SemanticConfig
    c.semantic_measurement_probability = semantic_config.semantic_measurement_probability_;
    c.color_mode = static_cast<int32_t>(semantic_config.color_mode);
    for (int l = 0; l < 256; ++l) c.label_color_known[l] = 0;   // an unknown label colours (0,0,0,0), color.cpp:89-93
    for (const auto& kv : semantic_config.semantic_label_to_color_->semantic_label_to_color_map_) {
      c.label_color_known[kv.first] = 1;
      c.label_color[kv.first][0] = kv.second.r;
      c.label_color[kv.first][1] = kv.second.g;
      c.label_color[kv.first][2] = kv.second.b;
      c.label_color[kv.first][3] = kv.second.a;
    }
    for (const SemanticLabel l : semantic_config.dynamic_labels_) c.dynamic_label[l] = 1;
    c.max_points = max_points_;
    CHECK_EQ(ksg_create(&c, &handle_), KSG_OK) << "ksg_create: " << ksg_last_error(nullptr);

    // colour -> label lookups are made with alpha forced to 255 (fast.cpp:157, merged.cpp:87): other alphas can never match
    std::vector<uint8_t> rgb, labels;
    for (const auto& kv : semantic_config.semantic_label_to_color_->color_to_semantic_label_) {
      if (kv.first.a != 255u) continue;
      rgb.push_back(kv.first.r);
      rgb.push_back(kv.first.g);
      rgb.push_back(kv.first.b);
      labels.push_back(kv.second);
    }
    CHECK_EQ(ksg_set_color_to_label(handle_, rgb.data(), labels.data(), static_cast<int32_t>(labels.size())), KSG_OK)
        << ksg_last_error(handle_);
  }

  ~GpuSemanticTsdfIntegrator() override { ksg_destroy(handle_); }
  GpuSemanticTsdfIntegrator(const GpuSemanticTsdfIntegrator&) = delete;
  GpuSemanticTsdfIntegrator& operator=(const GpuSemanticTsdfIntegrator&) = delete;

  void integratePointCloud(const vxb::Transformation& T_G_C, const vxb::Pointcloud& points_C, const vxb::Colors& colors,
                           const bool freespace_points = false) override {
    CHECK_EQ(points_C.size(), colors.size());
    CHECK_LE(points_C.size(), static_cast<size_t>(max_points_)) << "raise GpuSemanticTsdfIntegrator::max_points_";
    static_assert(sizeof(vxb::Point) == 3 * sizeof(float), "vxb::Point must be three packed floats");
    static_assert(sizeof(vxb::Color) == 4, "vxb::Color must be four bytes r,g,b,a");
    const auto q = T_G_C.getRotation().toImplementation();   // Eigen::Quaternionf in minkindr
    const vxb::Point& t = T_G_C.getPosition();
    const float T[7] = {q.w(), q.x(), q.y(), q.z(), t.x(), t.y(), t.z()};
    CHECK_EQ(ksg_integrate_points(handle_, T, points_C.empty() ? nullptr : points_C[0].data(),
                                  reinterpret_cast<const uint8_t*>(colors.data()), /*labels=*/nullptr,
                                  static_cast<int64_t>(points_C.size()), freespace_points ? 1 : 0, /*stats=*/nullptr),
             KSG_OK)
        << "ksg_integrate_points: " << ksg_last_error(handle_);
    refreshUpdatedBlocks();
  }

  ksg_integrator* handle() { return handle_; }

 private:
  // Copies the blocks the last call updated from the device map into the two host layers (linear voxel order
  // x + vps * (y + vps * z) on both sides) and marks them updated, like the reference's temp-block merge does.
  void refreshUpdatedBlocks() {
    const int64_t n = ksg_last_updated_blocks(handle_, 0, nullptr);
    if (n <= 0) return;
    const size_t V = voxels_per_side_ * voxels_per_side_ * voxels_per_side_, C = kTotalNumberOfLabels, N = static_cast<size_t>(n);
    idx_.resize(3 * N);
    CHECK_EQ(ksg_last_updated_blocks(handle_, n, idx_.data()), n);
    found_.resize(N);
    dist_.resize(N * V);
    weight_.resize(N * V);
    rgba_.resize(N * V * 4);
    label_.resize(N * V);
    priors_.resize(N * V * C);
    srgba_.resize(N * V * 4);
    CHECK_EQ(ksg_export_blocks_by_index(handle_, n, idx_.data(), found_.data(), dist_.data(), weight_.data(), rgba_.data(),
                                        label_.data(), priors_.data(), srgba_.data()), KSG_OK) << ksg_last_error(handle_);
    for (size_t b = 0; b < N; ++b) {
      if (!found_[b]) continue;
      const vxb::BlockIndex bi(idx_[3 * b], idx_[3 * b + 1], idx_[3 * b + 2]);
      vxb::Block<vxb::TsdfVoxel>::Ptr tsdf_block = layer_->allocateBlockPtrByIndex(bi);
      vxb::Block<SemanticVoxel>::Ptr semantic_block = semantic_layer_->allocateBlockPtrByIndex(bi);
      for (size_t v = 0; v < V; ++v) {
        const size_t i = b * V + v;
        vxb::TsdfVoxel& tv = tsdf_block->getVoxelByLinearIndex(v);
        tv.distance = dist_[i];
        tv.weight = weight_[i];
        tv.color = vxb::Color(rgba_[4 * i], rgba_[4 * i + 1], rgba_[4 * i + 2], rgba_[4 * i + 3]);
        SemanticVoxel& sv = semantic_block->getVoxelByLinearIndex(v);
        sv.semantic_label = label_[i];
        for (size_t c = 0; c < C; ++c) sv.semantic_priors[c] = priors_[i * C + c];
        sv.color = HashableColor(srgba_[4 * i], srgba_[4 * i + 1], srgba_[4 * i + 2], srgba_[4 * i + 3]);
      }
      tsdf_block->updated() = true;      // as base.cpp:248 does for the semantic block
      semantic_block->updated() = true;
    }
  }

  static constexpr int32_t max_points_ = 1 << 20;   // largest cloud per call; sizes the device scratch
  ksg_integrator* handle_ = nullptr;
  std::vector<int32_t> idx_;
  std::vector<uint8_t> found_, rgba_, label_, srgba_;
  std::vector<float> dist_, weight_, priors_;
};

}  // namespace kimera
