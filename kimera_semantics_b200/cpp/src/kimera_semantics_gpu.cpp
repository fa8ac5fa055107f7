// Host shim: the reference's C++ integrator API (SemanticTsdfIntegratorFactory, Fast/MergedSemanticTsdfIntegrator,
// SemanticIntegratorBase, SemanticLabel2Color) implemented on top of the C-ABI of include/ksg.h.  No CUDA, Eigen, glog
// or ROS here; errors follow the reference's convention (abort with a message).  There is no CPU fallback: when the
// device library reports an error (including "no CUDA device") construction aborts.
#include <algorithm>
#include <cstring>
#include <fstream>

#include "../../../include/ksg.h"
#include "kimera_semantics/semantic_tsdf_integrator_factory.h"
#include "kimera_semantics/semantic_tsdf_integrator_fast.h"
#include "kimera_semantics/semantic_tsdf_integrator_merged.h"

namespace kimera {

// ------------------------------------------------------------------------------------------------
// SemanticLabel2Color (color.cpp:42-94)
// ------------------------------------------------------------------------------------------------
SemanticLabel2Color::SemanticLabel2Color(const std::string& filename) {
  std::ifstream file(filename.c_str());
  KSG_CHECK(file.good()) << "Couldn't open file: " << filename;
  std::string line;
  size_t row_number = 1;
  while (std::getline(file, line)) {  // CSVIterator: one row per line, comma separated (csv_iterator.cpp:22-38)
    if (!line.empty() && line.back() == '\r') line.pop_back();
    if (line.empty()) continue;
    std::vector<std::string> cells;
    std::stringstream ss(line);
    std::string cell;
    while (std::getline(ss, cell, ',')) cells.push_back(cell);
    if (!line.empty() && line.back() == ',') cells.push_back("");
    KSG_CHECK(cells.size() == 6u) << "Row " << row_number << " is invalid.";
    // the header row parses to (0,0,0,0) -> 0 exactly as std::atoi does in the reference (color.cpp:52-56)
    const uint8_t r = std::atoi(cells[1].c_str()), g = std::atoi(cells[2].c_str()), b = std::atoi(cells[3].c_str());
    const uint8_t a = std::atoi(cells[4].c_str()), id = std::atoi(cells[5].c_str());
    const HashableColor rgba(r, g, b, a);
    semantic_label_to_color_map_[id] = rgba;
    color_to_semantic_label_[rgba] = id;
    row_number++;
  }
  semantic_label_to_color_map_[kUnknownSemanticLabelId] = HashableColor(vxb::Color::White());  // color.cpp:64-66
  color_to_semantic_label_[HashableColor(vxb::Color::White())] = kUnknownSemanticLabelId;
}
SemanticLabel2Color::SemanticLabel2Color(const SemanticLabelToColorMap& label_to_color) : semantic_label_to_color_map_(label_to_color) {
  for (const auto& kv : label_to_color) color_to_semantic_label_[kv.second] = kv.first;
}
SemanticLabel SemanticLabel2Color::getSemanticLabelFromColor(const HashableColor& color) const {
  const auto it = color_to_semantic_label_.find(color);
  return it != color_to_semantic_label_.end() ? it->second : kUnknownSemanticLabelId;  // color.cpp:74-81 (LOG(ERROR) dropped)
}
HashableColor SemanticLabel2Color::getColorFromSemanticLabel(const SemanticLabel& semantic_label) const {
  const auto it = semantic_label_to_color_map_.find(semantic_label);
  return it != semantic_label_to_color_map_.end() ? it->second : HashableColor();  // color.cpp:88-93
}

// ------------------------------------------------------------------------------------------------
// SemanticIntegratorBase (base.cpp:57-128, 352-380)
// ------------------------------------------------------------------------------------------------
SemanticIntegratorBase::SemanticIntegratorBase(const SemanticConfig& semantic_config, vxb::Layer<SemanticVoxel>* semantic_layer)
    : semantic_config_(semantic_config), semantic_layer_(nullptr) {
  setSemanticLayer(semantic_layer);
  KSG_CHECK(semantic_layer_ != nullptr);
  setSemanticProbabilities();
}
void SemanticIntegratorBase::setSemanticLayer(vxb::Layer<SemanticVoxel>* semantic_layer) {
  KSG_CHECK(semantic_layer != nullptr);
  semantic_layer_ = semantic_layer;
  semantic_voxel_size_ = semantic_layer_->voxel_size();
  semantic_block_size_ = semantic_layer_->block_size();
  semantic_voxels_per_side_ = semantic_layer_->voxels_per_side();
  semantic_voxel_size_inv_ = 1.0 / semantic_voxel_size_;
  semantic_block_size_inv_ = 1.0 / semantic_block_size_;
  semantic_voxels_per_side_inv_ = 1.0 / semantic_voxels_per_side_;
}
void SemanticIntegratorBase::setSemanticProbabilities() {
  const SemanticProbability match_probability = semantic_config_.semantic_measurement_probability_;
  const SemanticProbability non_match_probability = 1.0f - semantic_config_.semantic_measurement_probability_;
  KSG_CHECK(match_probability > 0.0);
  KSG_CHECK(non_match_probability > 0.0);
  KSG_CHECK(match_probability < 1.0);
  KSG_CHECK(non_match_probability < 1.0);
  log_match_probability_ = std::log(match_probability);
  log_non_match_probability_ = std::log(non_match_probability);
  KSG_CHECK(log_match_probability_ > log_non_match_probability_) << "Your probabilities do not make sense...";
  for (size_t i = 0; i < kTotalNumberOfLabels; ++i)
    for (size_t j = 0; j < kTotalNumberOfLabels; ++j)
      semantic_log_likelihood_(i, j) = (i == j) ? log_match_probability_ : log_non_match_probability_;
  for (size_t i = 0; i < kTotalNumberOfLabels; ++i) semantic_log_likelihood_(i, kUnknownSemanticLabelId) = 0.0f;  // base.cpp:127
}
void SemanticIntegratorBase::updateSemanticVoxelProbabilities(const SemanticProbabilities& measurement_frequencies,
                                                              SemanticProbabilities* semantic_prior_probability) const {
  KSG_CHECK(semantic_prior_probability != nullptr);
  // dense product as in base.cpp:306-307, accumulated column by column (j ascending) before it is added to the prior
  SemanticProbabilities product;
  for (size_t i = 0; i < kTotalNumberOfLabels; ++i) product[i] = semantic_log_likelihood_(i, 0) * measurement_frequencies[0];
  for (size_t j = 1; j < kTotalNumberOfLabels; ++j)
    for (size_t i = 0; i < kTotalNumberOfLabels; ++i) product[i] += semantic_log_likelihood_(i, j) * measurement_frequencies[j];
  for (size_t i = 0; i < kTotalNumberOfLabels; ++i) (*semantic_prior_probability)[i] += product[i];
}
void SemanticIntegratorBase::normalizeProbabilities(SemanticProbabilities* unnormalized_probs) const {
  KSG_CHECK(unnormalized_probs != nullptr);
  KSG_CHECK((*unnormalized_probs)[0] < 0.0) << "Are you sure you are usinglog odds?";   // base.cpp:322-323 (text as upstream)
  const SemanticProbability normalization_factor = unnormalized_probs->norm();
  KSG_CHECK(normalization_factor >= 0.0);
  if (normalization_factor != 0.0) {
    unnormalized_probs->normalize();
  } else {
    // base.cpp:335-341: std::log(1 / kTotalNumberOfLabels) with INTEGER division, i.e. log(0) = -inf; unreachable after the
    // CHECK_LT above (a vector whose first entry is negative has a positive norm), kept for fidelity
    unnormalized_probs->setConstant(std::log(static_cast<SemanticProbability>(1 / kTotalNumberOfLabels)));
  }
  KSG_CHECK(std::abs(unnormalized_probs->norm() - 1.0f) <= vxb::kFloatEpsilon);           // the reference's kDebug CHECK_NEAR
}
void SemanticIntegratorBase::calculateMaximumLikelihoodLabel(const SemanticProbabilities& semantic_posterior,
                                                             SemanticLabel* semantic_label) const {
  KSG_CHECK(semantic_label != nullptr);
  semantic_posterior.maxCoeff(semantic_label);
}
void SemanticIntegratorBase::updateSemanticVoxelColor(const SemanticLabel& semantic_label, HashableColor* semantic_voxel_color) const {
  KSG_CHECK(semantic_voxel_color != nullptr);
  *semantic_voxel_color = semantic_config_.semantic_label_to_color_->getColorFromSemanticLabel(semantic_label);
}
bool SemanticIntegratorBase::isSemanticLabelValid(const SemanticLabel& semantic_label) const {
  return std::find(semantic_config_.dynamic_labels_.begin(), semantic_config_.dynamic_labels_.end(), semantic_label) ==
         semantic_config_.dynamic_labels_.end();
}

// ------------------------------------------------------------------------------------------------
// GpuIntegratorCore
// ------------------------------------------------------------------------------------------------
GpuIntegratorCore::GpuIntegratorCore(int integrator_type, const vxb::TsdfIntegratorBase::Config& config,
                                     const SemanticIntegratorBase::SemanticConfig& sc, vxb::Layer<vxb::TsdfVoxel>* tsdf_layer,
                                     vxb::Layer<SemanticVoxel>* semantic_layer)
    : tsdf_layer_(tsdf_layer), semantic_layer_(semantic_layer) {
  KSG_CHECK(tsdf_layer != nullptr);
  KSG_CHECK(semantic_layer != nullptr);
  KSG_CHECK(tsdf_layer->voxels_per_side() == semantic_layer->voxels_per_side());
  KSG_CHECK(tsdf_layer->voxel_size() == semantic_layer->voxel_size());
  KSG_CHECK(sc.semantic_label_to_color_ != nullptr);  // CHECK(semantic_config_.semantic_label_to_color_) fast.cpp:154
  ksg_config c;
  ksg_default_config(&c, integrator_type, tsdf_layer->voxel_size(), (int)tsdf_layer->voxels_per_side(), (int)kTotalNumberOfLabels);
  c.default_truncation_distance = config.default_truncation_distance;
  c.max_weight = config.max_weight;
  c.voxel_carving_enabled = config.voxel_carving_enabled;
  c.min_ray_length_m = config.min_ray_length_m;
  c.max_ray_length_m = config.max_ray_length_m;
  c.use_const_weight = config.use_const_weight;
  c.allow_clear = config.allow_clear;
  c.use_weight_dropoff = config.use_weight_dropoff;
  c.use_sparsity_compensation_factor = config.use_sparsity_compensation_factor;
  c.sparsity_compensation_factor = config.sparsity_compensation_factor;
  if (config.integration_order_mode == "mixed") c.integration_order_mode = KSG_ORDER_MIXED;
  else if (config.integration_order_mode == "sorted") c.integration_order_mode = KSG_ORDER_SORTED;
  else KSG_LOG_FATAL << "Unknown integration order mode: '" << config.integration_order_mode << "'!";  // ThreadSafeIndexFactory
  c.enable_anti_grazing = config.enable_anti_grazing;
  c.start_voxel_subsampling_factor = config.start_voxel_subsampling_factor;
  c.max_consecutive_ray_collisions = config.max_consecutive_ray_collisions;
  c.clear_checks_every_n_frames = config.clear_checks_every_n_frames;
  c.integrator_threads = (int)config.integrator_threads;
  c.semantic_measurement_probability = sc.semantic_measurement_probability_;
  c.color_mode = static_cast<int>(sc.color_mode);
  for (int l = 0; l < 256; ++l) {
    const auto it = sc.semantic_label_to_color_->semantic_label_to_color_map_.find((SemanticLabel)l);
    const bool known = it != sc.semantic_label_to_color_->semantic_label_to_color_map_.end();
    c.label_color_known[l] = known ? 1 : 0;
    c.label_color[l][0] = known ? it->second.r : 0; c.label_color[l][1] = known ? it->second.g : 0;
    c.label_color[l][2] = known ? it->second.b : 0; c.label_color[l][3] = known ? it->second.a : 0;
    c.dynamic_label[l] = 0;
  }
  for (const SemanticLabel l : sc.dynamic_labels_) c.dynamic_label[l] = 1;
  if (const char* e = std::getenv("KSG_MAX_POINTS")) c.max_points = std::atoi(e); else c.max_points = 1 << 20;
  if (const char* e = std::getenv("KSG_MAX_BLOCKS")) c.max_blocks = std::atoi(e);
  if (const char* e = std::getenv("KSG_MAX_UPDATES")) c.max_updates = std::atoll(e);
  if (const char* e = std::getenv("KSG_DEVICE")) c.device = std::atoi(e);
  // merged only: the default (ksg_default_config) is the reference's std::unordered_map iteration order (ksg.h KSG_BUNDLE_ORDER_LIBSTDCXX = 1);
  // KSG_MERGED_BUNDLE_ORDER=0 selects first-insertion order
  if (const char* e = std::getenv("KSG_MERGED_BUNDLE_ORDER")) c.merged_bundle_order = std::atoi(e);
  const int rc = ksg_create(&c, &handle_);
  KSG_CHECK(rc == KSG_OK) << "ksg_create failed (" << rc << "): " << ksg_last_error(nullptr);
  // eager layer sync goes through the device-side update log (one entry per updated voxel); it must be on before the first frame
  update_log_tried_ = true;
  update_log_on_ = std::getenv("KSG_NO_UPDATE_LOG") == nullptr && ksg_set_update_log(handle_, 1 << 21) == KSG_OK;
  // colour -> label table (color.cpp:69-82); alpha is forced to 255 by the callers
  std::vector<uint8_t> rgb, lab;
  for (const auto& kv : sc.semantic_label_to_color_->color_to_semantic_label_) {
    if (kv.first.a != 255) continue;  // can never match a lookup made with alpha 255
    rgb.push_back(kv.first.r); rgb.push_back(kv.first.g); rgb.push_back(kv.first.b);
    lab.push_back(kv.second);
  }
  KSG_CHECK(ksg_set_color_to_label(handle_, rgb.data(), lab.data(), (int)lab.size()) == KSG_OK) << ksg_last_error(handle_);
}
GpuIntegratorCore::~GpuIntegratorCore() { ksg_destroy(handle_); }

void GpuIntegratorCore::integrate(const vxb::Transformation& T_G_C, const vxb::Pointcloud& points_C, const vxb::Color* colors,
                                  const SemanticLabel* labels, bool freespace_points) {
  static_assert(sizeof(vxb::Point) == 12, "Point must be 3 packed floats");
  static_assert(sizeof(vxb::Color) == 4, "Color must be 4 packed bytes");
  const vxb::FloatingPoint* q = T_G_C.getRotationWxyz();
  const vxb::Point& t = T_G_C.getPosition();
  const float T[7] = {q[0], q[1], q[2], q[3], t.x(), t.y(), t.z()};
  ksg_frame_stats st;
  const int rc = ksg_integrate_points(handle_, T, points_C.empty() ? nullptr : &points_C[0].v[0], reinterpret_cast<const uint8_t*>(colors),
                                      labels, (int64_t)points_C.size(), freespace_points ? 1 : 0, &st);
  KSG_CHECK(rc == KSG_OK) << "ksg_integrate_points failed (" << rc << "): " << ksg_last_error(handle_);
  last_voxel_updates_ = st.voxel_updates;
  if (sync_mode_ == LayerSyncMode::kEager) syncAfterCall();
}

// Eager sync (the reference's contract: the host layers hold the frame's result when integratePointCloud returns).  Both integrators keep
// an update log on the device: one entry per updated voxel, fetched with two DMA transfers and written into the layers here; a frame that
// overflows the log (or KSG_NO_UPDATE_LOG) copies the updated blocks.
void GpuIntegratorCore::syncAfterCall() {
  if (!update_log_on_) { syncUpdatedBlocks(); return; }
  int64_t n = 0;
  const ksg_voxel_update* up = nullptr;
  const float* priors = nullptr;
  const int rc = ksg_fetch_update_log(handle_, &n, &up, &priors);
  if (rc != KSG_OK || n < 0) { syncUpdatedBlocks(); return; }
  const size_t C = kTotalNumberOfLabels;
  vxb::BlockIndex last_bi(0x7fffffff, 0x7fffffff, 0x7fffffff);
  vxb::Block<vxb::TsdfVoxel>::Ptr tb;
  vxb::Block<SemanticVoxel>::Ptr sb;
  for (int64_t i = 0; i < n; ++i) {
    const ksg_voxel_update& u = up[i];
    const vxb::BlockIndex bi(u.block_index[0], u.block_index[1], u.block_index[2]);
    if (!(bi == last_bi)) {           // entries come in runs of one tile (`merged`: block by block): the block changes rarely; any order is correct
      last_bi = bi;
      tb = tsdf_layer_->allocateBlockPtrByIndex(bi);        // base.cpp:257-265: new blocks appear in both layers
      sb = semantic_layer_->allocateBlockPtrByIndex(bi);
      tb->updated() = true; sb->updated() = true;           // base.cpp:248
      tb->has_data() = true; sb->has_data() = true;
    }
    const size_t lin = u.lin_label & 0xFFFFFFu;
    vxb::TsdfVoxel& tv = tb->getVoxelByLinearIndex(lin);
    tv.distance = u.tsdf_distance;
    tv.weight = u.tsdf_weight;
    tv.color = vxb::Color(u.tsdf_rgba[0], u.tsdf_rgba[1], u.tsdf_rgba[2], u.tsdf_rgba[3]);
    SemanticVoxel& sv = sb->getVoxelByLinearIndex(lin);
    sv.semantic_label = (SemanticLabel)(u.lin_label >> 24);
    std::memcpy(sv.semantic_priors.data(), priors + (size_t)i * C, C * sizeof(float));
    sv.color = HashableColor(u.sem_rgba[0], u.sem_rgba[1], u.sem_rgba[2], u.sem_rgba[3]);
  }
}

void GpuIntegratorCore::integrateDepth(const vxb::Transformation& T_G_C, const float* depth, const SemanticLabel* label, int width,
                                       int height, const double K[4]) {
  KSG_CHECK(depth != nullptr && label != nullptr && width > 0 && height > 0);
  const vxb::FloatingPoint* q = T_G_C.getRotationWxyz();
  const vxb::Point& t = T_G_C.getPosition();
  const float T[7] = {q[0], q[1], q[2], q[3], t.x(), t.y(), t.z()};
  ksg_frame_stats st;
  const int rc = ksg_integrate_depth_k64(handle_, T, depth, label, width, height, K, &st);
  KSG_CHECK(rc == KSG_OK) << "ksg_integrate_depth_k64 failed (" << rc << "): " << ksg_last_error(handle_);
  last_voxel_updates_ = st.voxel_updates;
  if (sync_mode_ == LayerSyncMode::kEager) syncAfterCall();
}

void GpuIntegratorCore::copyBlocks(const std::vector<int32_t>& idx) {
  const size_t nb = idx.size() / 3;
  if (nb == 0) return;
  const size_t vps = tsdf_layer_->voxels_per_side(), V = vps * vps * vps, C = kTotalNumberOfLabels;
  std::vector<float> dist(nb * V), wgt(nb * V), priors(nb * V * C);
  std::vector<uint8_t> rgba(nb * V * 4), srgba(nb * V * 4), label(nb * V), found(nb);
  const int rc = ksg_export_blocks_by_index(handle_, (int64_t)nb, idx.data(), found.data(), dist.data(), wgt.data(), rgba.data(),
                                            label.data(), priors.data(), srgba.data());
  KSG_CHECK(rc == KSG_OK) << "ksg_export_blocks_by_index failed: " << ksg_last_error(handle_);
  for (size_t b = 0; b < nb; ++b) {
    if (!found[b]) continue;
    const vxb::BlockIndex bi(idx[3 * b], idx[3 * b + 1], idx[3 * b + 2]);
    // base.cpp:257-265 / voxblox updateLayerWithStoredBlocks: blocks appear in both layers
    vxb::Block<vxb::TsdfVoxel>::Ptr tb = tsdf_layer_->allocateBlockPtrByIndex(bi);
    vxb::Block<SemanticVoxel>::Ptr sb = semantic_layer_->allocateBlockPtrByIndex(bi);
    for (size_t v = 0; v < V; ++v) {
      vxb::TsdfVoxel& tv = tb->getVoxelByLinearIndex(v);
      tv.distance = dist[b * V + v];
      tv.weight = wgt[b * V + v];
      const uint8_t* c = &rgba[(b * V + v) * 4];
      tv.color = vxb::Color(c[0], c[1], c[2], c[3]);
      SemanticVoxel& sv = sb->getVoxelByLinearIndex(v);
      sv.semantic_label = label[b * V + v];
      std::memcpy(sv.semantic_priors.data(), &priors[(b * V + v) * C], C * sizeof(float));
      const uint8_t* s = &srgba[(b * V + v) * 4];
      sv.color = HashableColor(s[0], s[1], s[2], s[3]);
    }
    tb->updated() = true;  // base.cpp:248
    sb->updated() = true;
    tb->has_data() = true;
    sb->has_data() = true;
  }
}
void GpuIntegratorCore::syncUpdatedBlocks() {
  const int64_t n = ksg_last_updated_blocks(handle_, 0, nullptr);
  std::vector<int32_t> idx((size_t)n * 3);
  if (n) ksg_last_updated_blocks(handle_, n, idx.data());
  copyBlocks(idx);
}
bool GpuIntegratorCore::extractMesh(float min_weight, std::vector<float>* vertices, std::vector<uint8_t>* rgba, std::vector<uint8_t>* labels,
                                    std::vector<int32_t>* block_index, std::vector<int64_t>* block_first) {
  int64_t nv = 0, nb = 0;
  if (ksg_extract_mesh(handle_, min_weight, 0, nullptr, nullptr, nullptr, 0, nullptr, nullptr, &nv, &nb) != KSG_OK) return false;
  vertices->assign((size_t)nv * 3, 0.0f);
  rgba->assign((size_t)nv * 4, 0);
  labels->assign((size_t)nv, 0);
  block_index->assign((size_t)nb * 3, 0);
  block_first->assign((size_t)nb + 1, 0);
  return ksg_extract_mesh(handle_, min_weight, nv, vertices->data(), rgba->data(), labels->data(), nb, block_index->data(), block_first->data(),
                          &nv, &nb) == KSG_OK;
}
bool GpuIntegratorCore::exportMesh(int32_t changed_only, std::vector<float>* vertices, std::vector<uint8_t>* rgba,
                                   std::vector<uint8_t>* labels, std::vector<int32_t>* block_index, std::vector<int64_t>* block_first) {
  int64_t nv = 0, nb = 0;
  if (ksg_export_mesh(handle_, changed_only, 0, nullptr, nullptr, nullptr, 0, nullptr, nullptr, &nv, &nb) != KSG_OK) return false;
  vertices->assign((size_t)nv * 3, 0.0f);
  rgba->assign((size_t)nv * 4, 0);
  labels->assign((size_t)nv, 0);
  block_index->assign((size_t)nb * 3, 0);
  block_first->assign((size_t)nb + 1, 0);
  return ksg_export_mesh(handle_, changed_only, nv, vertices->data(), rgba->data(), labels->data(), nb, block_index->data(),
                         block_first->data(), &nv, &nb) == KSG_OK;
}
bool GpuIntegratorCore::updateMesh(float min_weight, std::vector<float>* vertices, std::vector<uint8_t>* rgba, std::vector<uint8_t>* labels,
                                   std::vector<int32_t>* block_index, std::vector<int64_t>* block_first, bool* full) {
  const bool resync = mesh_resync_;
  mesh_resync_ = true;
  ksg_mesh_stats st;
  if (ksg_update_mesh(handle_, min_weight, &st) != KSG_OK) return false;
  const bool all = st.full || resync;
  if (!exportMesh(all ? 0 : 1, vertices, rgba, labels, block_index, block_first)) return false;
  if (full) *full = all;
  mesh_resync_ = false;
  return true;
}
bool GpuIntegratorCore::meshLayer(float min_weight, std::vector<float>* vertices, std::vector<uint8_t>* rgba, std::vector<uint8_t>* labels,
                                  std::vector<int32_t>* block_index, std::vector<int64_t>* block_first) {
  mesh_resync_ = true;   // this update's re-meshed blocks are not handed out: the next updateMesh returns every block
  return ksg_update_mesh(handle_, min_weight, nullptr) == KSG_OK && exportMesh(0, vertices, rgba, labels, block_index, block_first);
}

bool GpuIntegratorCore::queryPoints(const vxb::Pointcloud& points_G, float min_weight, QueryResult* r) {
  static_assert(sizeof(vxb::Point) == 3 * sizeof(float), "points are passed as packed xyz triples");
  const size_t n = points_G.size();
  r->flags.assign(n, 0);
  r->tsdf_distance.assign(n, 0.0f);
  r->tsdf_weight.assign(n, 0.0f);
  r->tsdf_rgba.assign(4 * n, 0);
  r->sem_label.assign(n, 0);
  r->sem_priors.assign(n * kTotalNumberOfLabels, 0.0f);
  r->sem_rgba.assign(4 * n, 0);
  r->distance.assign(n, 0.0f);
  r->gradient.assign(3 * n, 0.0f);
  ksg_query_out out = {r->flags.data(), r->tsdf_distance.data(), r->tsdf_weight.data(), r->tsdf_rgba.data(), r->sem_label.data(),
                       r->sem_priors.data(), r->sem_rgba.data(), r->distance.data(), r->gradient.data()};
  return ksg_query_points(handle_, (int64_t)n, n ? reinterpret_cast<const float*>(points_G.data()) : nullptr, min_weight, &out) == KSG_OK;
}

bool GpuIntegratorCore::renderView(const vxb::Transformation& T_G_C, const double K[4], int w, int h, float min_depth, float max_depth,
                                   float min_weight, RenderResult* r) {
  const vxb::FloatingPoint* q = T_G_C.getRotationWxyz();
  const vxb::Point& t = T_G_C.getPosition();
  const float T[7] = {q[0], q[1], q[2], q[3], t.x(), t.y(), t.z()};
  const size_t n = (w > 0 && h > 0) ? (size_t)w * (size_t)h : 0;
  QueryResult& a = r->at_hit;
  r->depth.assign(n, 0.0f);
  r->points_G.assign(3 * n, 0.0f);
  a.flags.assign(n, 0);
  a.tsdf_distance.assign(n, 0.0f);
  a.tsdf_weight.assign(n, 0.0f);
  a.tsdf_rgba.assign(4 * n, 0);
  a.sem_label.assign(n, 0);
  a.sem_priors.assign(n * kTotalNumberOfLabels, 0.0f);
  a.sem_rgba.assign(4 * n, 0);
  a.distance.assign(n, 0.0f);
  a.gradient.assign(3 * n, 0.0f);
  ksg_render_out out = {r->depth.data(), r->points_G.data(),
                        {a.flags.data(), a.tsdf_distance.data(), a.tsdf_weight.data(), a.tsdf_rgba.data(), a.sem_label.data(),
                         a.sem_priors.data(), a.sem_rgba.data(), a.distance.data(), a.gradient.data()}};
  return ksg_render_view(handle_, T, K, w, h, min_depth, max_depth, min_weight, &out) == KSG_OK;
}

namespace {
// one ESDF block from rows of ksg_compute_esdf / ksg_export_esdf: observed = OBSERVED, fixed = SURFACE; every other voxel is voxblox's
// default EsdfVoxel
void fillEsdfBlock(vxb::Block<vxb::EsdfVoxel>* blk, size_t V, const float* distance, const uint8_t* flags) {
  blk->has_data() = true;
  for (size_t v = 0; v < V; ++v) {
    vxb::EsdfVoxel& e = blk->getVoxelByLinearIndex(v);
    e = vxb::EsdfVoxel();
    if (!(flags[v] & KSG_ESDF_OBSERVED)) continue;
    e.distance = distance[v];
    e.observed = true;
    e.fixed = (flags[v] & KSG_ESDF_SURFACE) != 0;
  }
}
}  // namespace

bool GpuIntegratorCore::computeEsdf(float min_weight, float max_distance, vxb::Layer<vxb::EsdfVoxel>* esdf) {
  if (!esdf || esdf->voxels_per_side() != tsdf_layer_->voxels_per_side()) return false;
  const int64_t nb = ksg_num_blocks(handle_);
  const size_t V = esdf->voxels_per_side() * esdf->voxels_per_side() * esdf->voxels_per_side();
  std::vector<int32_t> index(3 * (size_t)nb);
  std::vector<float> distance((size_t)nb * V);
  std::vector<uint8_t> flags((size_t)nb * V);
  if (ksg_compute_esdf(handle_, min_weight, max_distance, nb, index.data(), distance.data(), flags.data()) != KSG_OK) return false;
  esdf->removeAllBlocks();
  for (int64_t b = 0; b < nb; ++b)
    fillEsdfBlock(esdf->allocateNewBlock(vxb::BlockIndex(index[3 * b], index[3 * b + 1], index[3 * b + 2])).get(), V,
                  distance.data() + b * V, flags.data() + b * V);
  return true;
}

bool GpuIntegratorCore::updateEsdf(float min_weight, float max_distance, vxb::Layer<vxb::EsdfVoxel>* esdf) {
  if (!esdf || esdf->voxels_per_side() != tsdf_layer_->voxels_per_side()) return false;
  // a call that fails leaves the host layer behind the device layer: the next one refreshes every block
  const bool whole = esdf_resync_;
  esdf_resync_ = true;
  ksg_esdf_stats st;
  if (ksg_update_esdf(handle_, min_weight, max_distance, &st) != KSG_OK) return false;
  const int32_t changed_only = (st.full || whole) ? 0 : 1;
  int64_t n = 0;
  if (ksg_export_esdf(handle_, changed_only, 0, &n, nullptr, nullptr, nullptr) != KSG_OK) return false;
  const size_t V = esdf->voxels_per_side() * esdf->voxels_per_side() * esdf->voxels_per_side();
  std::vector<int32_t> index(3 * (size_t)n);
  std::vector<float> distance((size_t)n * V);
  std::vector<uint8_t> flags((size_t)n * V);
  if (n > 0 && ksg_export_esdf(handle_, changed_only, n, &n, index.data(), distance.data(), flags.data()) != KSG_OK) return false;
  // a refresh of every block starts the host layer over, as computeEsdf's does (after a clear or reset blocks may have gone)
  if (!changed_only) esdf->removeAllBlocks();
  for (int64_t b = 0; b < n; ++b)
    fillEsdfBlock(esdf->allocateBlockPtrByIndex(vxb::BlockIndex(index[3 * b], index[3 * b + 1], index[3 * b + 2])).get(), V,
                  distance.data() + b * V, flags.data() + b * V);
  esdf_resync_ = false;
  return true;
}

bool GpuIntegratorCore::queryEsdf(const vxb::Pointcloud& points_G, EsdfQueryResult* r) {
  if (!r) return false;
  const size_t n = points_G.size();
  r->flags.assign(n, 0);
  r->voxel_flags.assign(n, 0);
  r->voxel_distance.assign(n, 0.0f);
  r->distance.assign(n, 0.0f);
  r->gradient.assign(3 * n, 0.0f);
  ksg_esdf_query_out out = {r->flags.data(), r->voxel_flags.data(), r->voxel_distance.data(), r->distance.data(), r->gradient.data()};
  return ksg_query_esdf(handle_, (int64_t)n, n ? reinterpret_cast<const float*>(points_G.data()) : nullptr, &out) == KSG_OK;
}

void GpuIntegratorCore::uploadLayers() {
  vxb::BlockIndexList blocks;
  tsdf_layer_->getAllAllocatedBlocks(&blocks);
  KSG_CHECK(ksg_reset(handle_) == KSG_OK) << "ksg_reset failed: " << ksg_last_error(handle_);
  const size_t nb = blocks.size();
  if (nb == 0) return;
  const size_t vps = tsdf_layer_->voxels_per_side(), V = vps * vps * vps, C = kTotalNumberOfLabels;
  std::vector<int32_t> idx(nb * 3);
  std::vector<float> dist(nb * V), wgt(nb * V), priors(nb * V * C);
  std::vector<uint8_t> rgba(nb * V * 4), srgba(nb * V * 4), label(nb * V);
  for (size_t b = 0; b < nb; ++b) {
    const vxb::BlockIndex& bi = blocks[b];
    idx[3 * b] = bi.x(); idx[3 * b + 1] = bi.y(); idx[3 * b + 2] = bi.z();
    vxb::Block<vxb::TsdfVoxel>::Ptr tb = tsdf_layer_->getBlockPtrByIndex(bi);
    vxb::Block<SemanticVoxel>::Ptr sb = semantic_layer_->allocateBlockPtrByIndex(bi);   // a TSDF-only block gets default semantics
    for (size_t v = 0; v < V; ++v) {
      const vxb::TsdfVoxel& tv = tb->getVoxelByLinearIndex(v);
      const SemanticVoxel& sv = sb->getVoxelByLinearIndex(v);
      dist[b * V + v] = tv.distance;
      wgt[b * V + v] = tv.weight;
      uint8_t* c = &rgba[(b * V + v) * 4];
      c[0] = tv.color.r; c[1] = tv.color.g; c[2] = tv.color.b; c[3] = tv.color.a;
      label[b * V + v] = sv.semantic_label;
      std::memcpy(&priors[(b * V + v) * C], sv.semantic_priors.data(), C * sizeof(float));
      uint8_t* s = &srgba[(b * V + v) * 4];
      s[0] = sv.color.r; s[1] = sv.color.g; s[2] = sv.color.b; s[3] = sv.color.a;
    }
  }
  const int rc = ksg_import_blocks(handle_, (int64_t)nb, idx.data(), dist.data(), wgt.data(), rgba.data(), label.data(), priors.data(),
                                   srgba.data());
  KSG_CHECK(rc == KSG_OK) << "ksg_import_blocks failed: " << ksg_last_error(handle_);
}
void GpuIntegratorCore::syncLayers() {
  const int64_t n = ksg_num_blocks(handle_);
  std::vector<int32_t> idx((size_t)n * 3);
  if (n) KSG_CHECK(ksg_export_blocks(handle_, n, idx.data(), nullptr, nullptr, nullptr, nullptr, nullptr, nullptr) == KSG_OK);
  copyBlocks(idx);
}

// ------------------------------------------------------------------------------------------------
// the two integrators + factory
// ------------------------------------------------------------------------------------------------
FastSemanticTsdfIntegrator::FastSemanticTsdfIntegrator(const Config& config, const SemanticConfig& semantic_config,
                                                       vxb::Layer<vxb::TsdfVoxel>* tsdf_layer, vxb::Layer<SemanticVoxel>* semantic_layer)
    : TsdfIntegratorBase(config, tsdf_layer), SemanticIntegratorBase(semantic_config, semantic_layer),
      core_(KSG_INTEGRATOR_FAST, config, semantic_config, tsdf_layer, semantic_layer) {}

void FastSemanticTsdfIntegrator::integratePointCloud(const vxb::Transformation& T_G_C, const vxb::Pointcloud& points_C,
                                                     const vxb::Colors& colors, const bool freespace_points) {
  KSG_CHECK(points_C.size() == colors.size());  // CHECK_EQ fast.cpp:161
  core_.integrate(T_G_C, points_C, colors.data(), nullptr, freespace_points);
}

MergedSemanticTsdfIntegrator::MergedSemanticTsdfIntegrator(const Config& config, const SemanticConfig& semantic_config,
                                                           vxb::Layer<vxb::TsdfVoxel>* tsdf_layer, vxb::Layer<SemanticVoxel>* semantic_layer)
    : MergedTsdfIntegrator(config, tsdf_layer), SemanticIntegratorBase(semantic_config, semantic_layer),
      core_(KSG_INTEGRATOR_MERGED, config, semantic_config, tsdf_layer, semantic_layer) {}

void MergedSemanticTsdfIntegrator::integratePointCloud(const vxb::Transformation& T_G_C, const vxb::Pointcloud& points_C,
                                                       const vxb::Colors& colors, const bool freespace_points) {
  KSG_CHECK(points_C.size() == colors.size());
  core_.integrate(T_G_C, points_C, colors.data(), nullptr, freespace_points);
}
void MergedSemanticTsdfIntegrator::integratePointCloud(const vxb::Transformation& T_G_C, const vxb::Pointcloud& points_C,
                                                       const HashableColors& colors, const SemanticLabels& semantic_labels,
                                                       const bool freespace_points) {
  KSG_CHECK(points_C.size() == colors.size());            // merged.cpp:103-105
  KSG_CHECK(points_C.size() == semantic_labels.size());
  for (const SemanticLabel l : semantic_labels) KSG_CHECK(l < kTotalNumberOfLabels);  // CHECK_LT merged.cpp:278
  // the reference blends the explicit colours into the TSDF colour (merged.cpp:262-274); the device path keeps them out of it, which is
  // exact for the colour modes that overwrite the TSDF colour with the semantic one
  KSG_CHECK(semantic_config_.color_mode != ColorMode::kColor)
      << "MergedSemanticTsdfIntegrator(GPU): the label-explicit overload is not supported in ColorMode::kColor";
  core_.integrate(T_G_C, points_C, nullptr, semantic_labels.data(), freespace_points);
}

std::unique_ptr<vxb::TsdfIntegratorBase> SemanticTsdfIntegratorFactory::create(
    const std::string& integrator_type_name, const vxb::TsdfIntegratorBase::Config& config,
    const SemanticIntegratorBase::SemanticConfig& semantic_config, vxb::Layer<vxb::TsdfVoxel>* tsdf_layer,
    vxb::Layer<SemanticVoxel>* semantic_layer) {
  KSG_CHECK(!integrator_type_name.empty());
  int integrator_type = 0;
  for (const std::string& valid : kSemanticTsdfIntegratorTypeNames) {
    if (integrator_type_name == valid)
      return create(static_cast<SemanticTsdfIntegratorType>(integrator_type), config, semantic_config, tsdf_layer, semantic_layer);
    ++integrator_type;
  }
  KSG_LOG_FATAL << "Unknown TSDF integrator type: " << integrator_type_name;  // factory.cpp:61
  return nullptr;
}
std::unique_ptr<vxb::TsdfIntegratorBase> SemanticTsdfIntegratorFactory::create(
    const SemanticTsdfIntegratorType& integrator_type, const vxb::TsdfIntegratorBase::Config& config,
    const SemanticIntegratorBase::SemanticConfig& semantic_config, vxb::Layer<vxb::TsdfVoxel>* tsdf_layer,
    vxb::Layer<SemanticVoxel>* semantic_layer) {
  KSG_CHECK(tsdf_layer != nullptr);
  switch (integrator_type) {
    case SemanticTsdfIntegratorType::kFast:
      return kimera::make_unique<FastSemanticTsdfIntegrator>(config, semantic_config, tsdf_layer, semantic_layer);
    case SemanticTsdfIntegratorType::kMerged:
      return kimera::make_unique<MergedSemanticTsdfIntegrator>(config, semantic_config, tsdf_layer, semantic_layer);
    default:
      KSG_LOG_FATAL << "Unknown Semantic/TSDF integrator type: " << static_cast<int>(integrator_type);  // factory.cpp:83
  }
  return nullptr;
}

}  // namespace kimera
