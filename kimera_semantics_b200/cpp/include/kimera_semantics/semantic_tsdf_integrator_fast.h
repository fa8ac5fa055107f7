// Drop-in for kimera::FastSemanticTsdfIntegrator (reference fast.h:63-135): same base classes, constructor and
// virtual integratePointCloud; the work is done by the sm_90a kernels behind include/ksg.h.
#pragma once
#include "kimera_semantics/gpu_integrator_core.h"
namespace kimera {
class FastSemanticTsdfIntegrator : public vxb::TsdfIntegratorBase, public SemanticIntegratorBase {
 public:
  FastSemanticTsdfIntegrator(const Config& config, const SemanticConfig& semantic_config,
                             vxb::Layer<vxb::TsdfVoxel>* tsdf_layer, vxb::Layer<SemanticVoxel>* semantic_layer);
  virtual ~FastSemanticTsdfIntegrator() = default;
  virtual void integratePointCloud(const vxb::Transformation& T_G_C, const vxb::Pointcloud& points_C,
                                   const vxb::Colors& colors, const bool freespace_points = false) override;
  GpuIntegratorCore& gpu() { return core_; }
 private:
  GpuIntegratorCore core_;
};
}  // namespace kimera
