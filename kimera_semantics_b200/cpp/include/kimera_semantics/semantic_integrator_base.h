// Mirror of kimera_semantics/include/kimera_semantics/semantic_integrator_base.h (reference base.h:54-225) for the
// H100 build: same ColorMode / SemanticConfig / constructor contract / public data members.  The per-voxel update
// (base.cpp:136-194) does not run on the host any more: it lives in the CUDA tile kernel behind include/ksg.h.
#pragma once
#include <memory>
#include "kimera_semantics/color.h"
#include "kimera_semantics/common.h"
#include "kimera_semantics/semantic_voxel.h"
#include "voxblox/integrator/tsdf_integrator.h"
namespace kimera {
enum class ColorMode : int { kColor = 0, kSemantic = 1, kSemanticProbability = 2 };

class SemanticIntegratorBase {
 public:
  typedef std::shared_ptr<SemanticIntegratorBase> Ptr;
  struct SemanticConfig {
    SemanticProbability semantic_measurement_probability_ = 0.9f;
    ColorMode color_mode = ColorMode::kSemantic;
    std::shared_ptr<SemanticLabel2Color> semantic_label_to_color_ = nullptr;
    SemanticLabels dynamic_labels_ = SemanticLabels();
  };
  SemanticIntegratorBase(const SemanticConfig& semantic_config, vxb::Layer<SemanticVoxel>* semantic_layer);
  virtual ~SemanticIntegratorBase() = default;

  SemanticProbability computeMeasurementProbability(vxb::FloatingPoint ray_distance) { (void)ray_distance; return 1.0; }  // base.cpp:131-134
  // THREAD SAFE helpers that do not touch the map (base.cpp:283-380).  They are the reference's public per-vector utilities; the
  // integrators here never call them (the per-voxel update runs in the CUDA tile kernel) - they exist for callers that post-process
  // a voxel's probabilities on the host.
  // *prior += semantic_log_likelihood_ * measurement_frequencies   (base.cpp:283-314; columns accumulated in ascending order)
  void updateSemanticVoxelProbabilities(const SemanticProbabilities& measurement_frequencies,
                                        SemanticProbabilities* semantic_prior_probability) const;
  // L2-normalises the vector (sic, base.cpp:317-350); aborts like the reference when (*p)[0] >= 0
  void normalizeProbabilities(SemanticProbabilities* unnormalized_probs) const;
  void calculateMaximumLikelihoodLabel(const SemanticProbabilities& semantic_posterior, SemanticLabel* semantic_label) const;
  void updateSemanticVoxelColor(const SemanticLabel& semantic_label, HashableColor* semantic_voxel_color) const;

 protected:
  bool isSemanticLabelValid(const SemanticLabel& semantic_label) const;  // base.h:170-175

 private:
  void setSemanticLayer(vxb::Layer<SemanticVoxel>* semantic_layer);  // base.cpp:78-91
  void setSemanticProbabilities();                                    // base.cpp:93-128

 public:
  const SemanticConfig semantic_config_;
  vxb::Layer<SemanticVoxel>* semantic_layer_;
  SemanticProbability log_match_probability_;
  SemanticProbability log_non_match_probability_;
  SemanticLikelihoodFunction semantic_log_likelihood_;
  vxb::FloatingPoint semantic_voxel_size_;
  size_t semantic_voxels_per_side_;
  vxb::FloatingPoint semantic_block_size_;
  vxb::FloatingPoint semantic_voxel_size_inv_;
  vxb::FloatingPoint semantic_voxels_per_side_inv_;
  vxb::FloatingPoint semantic_block_size_inv_;
};
}  // namespace kimera
