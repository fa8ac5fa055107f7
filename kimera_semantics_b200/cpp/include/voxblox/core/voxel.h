#pragma once
#include "voxblox/core/common.h"
namespace voxblox {
struct TsdfVoxel {
  float distance = 0.0f;
  float weight = 0.0f;
  Color color;
};
// voxblox's EsdfVoxel without the Eigen `parent` (only voxblox's incremental queue uses it)
struct EsdfVoxel {
  float distance = 0.0f;
  bool observed = false;
  bool hallucinated = false;
  bool in_queue = false;
  bool fixed = false;
};
}  // namespace voxblox
