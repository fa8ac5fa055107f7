// Drives the drop-in C++ API exactly the way SemanticTsdfServer does (kimera_semantics_ros/src/semantic_tsdf_server.cpp:58-79):
// build both layers, SemanticTsdfIntegratorFactory::create(method, ...), then integratePointCloud per frame.
//   shim_demo <fast|merged|bogus> <frames.bin> <out.bin> [lazy] [--load ckpt] [--save ckpt] [--skip N] [--query in out] [--render in out]
//     --load: SemanticTsdfServer::loadMap before the first frame; --save: saveMap after the last; --skip: ignore the first N frames
//     --depth file: instead of the clouds of frames.bin (whose frame count must then be 0) feed depth + label frames:
//              int32 n, int32 width, int32 height, double K[4], then per frame float T[7], float depth[w*h], uint8 label[w*h]
//     --query in out: after the last frame (before any layer sync, also in lazy mode) SemanticTsdfServer::queryPoints on the points of
//              `in` (int32 n, float xyz[3n], world frame; min_weight 1e-4); `out` = the arrays of QueryResult one after the other:
//              flags[n] u8, tsdf_distance[n] f32, tsdf_weight[n] f32, tsdf_rgba[4n] u8, sem_label[n] u8, sem_priors[n*C] f32,
//              sem_rgba[4n] u8, distance[n] f32, gradient[3n] f32
//     --render in out: after the last frame (also before any layer sync) SemanticTsdfServer::renderView with `in` = float T_G_C[7],
//              double K[4], int32 w, int32 h, float min_depth, max_depth, min_weight; `out` = depth[n] f32, points_G[3n] f32, then the
//              arrays of --query's output for the n = w * h hit points
// frames.bin : int32 n_frames, float voxel_size, int32 vps, int32 n_palette, palette n*(r,g,b,a,id), int32 n_dynamic, ids...,
//              then per frame: int32 n, float T[7], float xyz[3n], uint8 rgba[4n]
// out.bin    : int32 n_blocks, then per block (sorted z,y,x): int32 idx[3], per voxel: float d, float w, u8 rgba[4], u8 label,
//              float priors[C], u8 sem_rgba[4]
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <vector>
#include "../../../include/ksg.h"
#include "kimera_semantics/semantic_tsdf_integrator_factory.h"
#include "kimera_semantics/semantic_tsdf_integrator_fast.h"
#include "kimera_semantics/semantic_tsdf_integrator_merged.h"
#include "kimera_semantics/semantic_tsdf_server.h"

using namespace kimera;
template <typename T> static T rd(std::ifstream& f) { T v; f.read(reinterpret_cast<char*>(&v), sizeof(T)); return v; }

int main(int argc, char** argv) {
  if (argc < 4) { std::fprintf(stderr, "usage: shim_demo <fast|merged> frames.bin out.bin [lazy]\n"); return 2; }
  std::ifstream f(argv[2], std::ios::binary);
  KSG_CHECK(f.good()) << "cannot open " << argv[2];
  const int n_frames = rd<int32_t>(f);
  const float voxel_size = rd<float>(f);
  const int vps = rd<int32_t>(f);
  SemanticLabelToColorMap pal;
  const int n_pal = rd<int32_t>(f);
  for (int i = 0; i < n_pal; ++i) { uint8_t e[5]; f.read(reinterpret_cast<char*>(e), 5); pal[e[4]] = HashableColor(e[0], e[1], e[2], e[3]); }
  SemanticIntegratorBase::SemanticConfig sc;
  sc.semantic_label_to_color_ = std::make_shared<SemanticLabel2Color>(pal);
  const int n_dyn = rd<int32_t>(f);
  for (int i = 0; i < n_dyn; ++i) sc.dynamic_labels_.push_back(rd<uint8_t>(f));
  vxb::TsdfIntegratorBase::Config config;
  config.default_truncation_distance = 4.0f * voxel_size;  // voxblox_ros
  bool lazy = false;
  const char *load_path = nullptr, *save_path = nullptr, *depth_path = nullptr, *query_in = nullptr, *query_out = nullptr;
  const char *render_in = nullptr, *render_out = nullptr;
  int skip = 0;
  for (int a = 4; a < argc; ++a) {
    if (std::strcmp(argv[a], "lazy") == 0) lazy = true;
    else if (std::strcmp(argv[a], "--load") == 0 && a + 1 < argc) load_path = argv[++a];
    else if (std::strcmp(argv[a], "--save") == 0 && a + 1 < argc) save_path = argv[++a];
    else if (std::strcmp(argv[a], "--skip") == 0 && a + 1 < argc) skip = std::atoi(argv[++a]);
    else if (std::strcmp(argv[a], "--depth") == 0 && a + 1 < argc) depth_path = argv[++a];
    else if (std::strcmp(argv[a], "--query") == 0 && a + 2 < argc) { query_in = argv[++a]; query_out = argv[++a]; }
    else if (std::strcmp(argv[a], "--render") == 0 && a + 2 < argc) { render_in = argv[++a]; render_out = argv[++a]; }
  }
  SemanticTsdfServer::Params params;
  params.tsdf_voxel_size = voxel_size;
  params.tsdf_voxels_per_side = vps;
  params.method = argv[1];
  params.layer_sync = lazy ? LayerSyncMode::kLazy : LayerSyncMode::kEager;
  SemanticTsdfServer server(params, config, sc);   // builds both layers + SemanticTsdfIntegratorFactory::create(method, ...)
  vxb::Layer<vxb::TsdfVoxel>& tsdf_layer = *server.getTsdfLayerPtr();
  vxb::Layer<SemanticVoxel>& semantic_layer = *server.getSemanticLayerPtr();
  GpuIntegratorCore* core = &server.gpu();
  if (load_path) KSG_CHECK(server.loadMap(load_path)) << "cannot load " << load_path;
  for (int fr = 0; fr < n_frames; ++fr) {
    const int n = rd<int32_t>(f);
    float T[7]; f.read(reinterpret_cast<char*>(T), sizeof(T));
    vxb::Pointcloud pts(n); vxb::Colors cols(n);
    f.read(reinterpret_cast<char*>(pts.data()), sizeof(float) * 3 * n);
    f.read(reinterpret_cast<char*>(cols.data()), 4 * (size_t)n);
    if (fr < skip) continue;
    server.processPointCloud(vxb::Transformation(T[0], T[1], T[2], T[3], vxb::Point(T[4], T[5], T[6])), pts, cols, /*stamp=*/0.2 * fr);
    std::printf("frame %d: %d points, %lld voxel updates, %zu blocks in the host layer\n", fr, n, (long long)core->lastVoxelUpdates(),
                tsdf_layer.getNumberOfAllocatedBlocks());
  }
  if (depth_path) {
    std::ifstream df(depth_path, std::ios::binary);
    KSG_CHECK(df.good()) << "cannot open " << depth_path;
    const int n = rd<int32_t>(df), w = rd<int32_t>(df), h = rd<int32_t>(df);
    double K[4];
    df.read(reinterpret_cast<char*>(K), sizeof(K));
    std::vector<float> depth((size_t)w * h);
    std::vector<uint8_t> label((size_t)w * h);
    for (int fr = 0; fr < n; ++fr) {
      float T[7];
      df.read(reinterpret_cast<char*>(T), sizeof(T));
      df.read(reinterpret_cast<char*>(depth.data()), 4 * depth.size());
      df.read(reinterpret_cast<char*>(label.data()), label.size());
      server.processDepthFrame(vxb::Transformation(T[0], T[1], T[2], T[3], vxb::Point(T[4], T[5], T[6])), depth.data(), label.data(), w, h, K,
                               /*stamp=*/0.2 * fr);
      std::printf("depth frame %d: %lld voxel updates\n", fr, (long long)core->lastVoxelUpdates());
    }
  }
  if (query_in) {
    std::ifstream qf(query_in, std::ios::binary);
    KSG_CHECK(qf.good()) << "cannot open " << query_in;
    const int n = rd<int32_t>(qf);
    vxb::Pointcloud pts(n);
    qf.read(reinterpret_cast<char*>(pts.data()), sizeof(float) * 3 * n);
    GpuIntegratorCore::QueryResult q;
    KSG_CHECK(server.queryPoints(pts, 1e-4f, &q)) << "point query failed";
    std::ofstream qo(query_out, std::ios::binary);
    auto put = [&qo](const void* p, size_t bytes) { qo.write(reinterpret_cast<const char*>(p), bytes); };
    put(q.flags.data(), q.flags.size());
    put(q.tsdf_distance.data(), 4 * q.tsdf_distance.size());
    put(q.tsdf_weight.data(), 4 * q.tsdf_weight.size());
    put(q.tsdf_rgba.data(), q.tsdf_rgba.size());
    put(q.sem_label.data(), q.sem_label.size());
    put(q.sem_priors.data(), 4 * q.sem_priors.size());
    put(q.sem_rgba.data(), q.sem_rgba.size());
    put(q.distance.data(), 4 * q.distance.size());
    put(q.gradient.data(), 4 * q.gradient.size());
    size_t hits = 0;
    for (uint8_t fl : q.flags) hits += (fl & KSG_QUERY_OBSERVED) ? 1 : 0;
    std::printf("point query: %d points, %zu in observed voxels%s\n", n, hits, lazy ? " (host layers not synchronised)" : "");
  }
  if (render_in) {
    std::ifstream rf(render_in, std::ios::binary);
    KSG_CHECK(rf.good()) << "cannot open " << render_in;
    float T[7];
    double K[4];
    rf.read(reinterpret_cast<char*>(T), sizeof(T));
    rf.read(reinterpret_cast<char*>(K), sizeof(K));
    const int w = rd<int32_t>(rf), h = rd<int32_t>(rf);
    float depth_range[3];
    rf.read(reinterpret_cast<char*>(depth_range), sizeof(depth_range));
    GpuIntegratorCore::RenderResult rr;
    KSG_CHECK(server.renderView(vxb::Transformation(T[0], T[1], T[2], T[3], vxb::Point(T[4], T[5], T[6])), K, w, h, depth_range[0],
                                depth_range[1], depth_range[2], &rr)) << "render failed";
    std::ofstream ro(render_out, std::ios::binary);
    auto put = [&ro](const void* p, size_t bytes) { ro.write(reinterpret_cast<const char*>(p), bytes); };
    const GpuIntegratorCore::QueryResult& q = rr.at_hit;
    put(rr.depth.data(), 4 * rr.depth.size());
    put(rr.points_G.data(), 4 * rr.points_G.size());
    put(q.flags.data(), q.flags.size());
    put(q.tsdf_distance.data(), 4 * q.tsdf_distance.size());
    put(q.tsdf_weight.data(), 4 * q.tsdf_weight.size());
    put(q.tsdf_rgba.data(), q.tsdf_rgba.size());
    put(q.sem_label.data(), q.sem_label.size());
    put(q.sem_priors.data(), 4 * q.sem_priors.size());
    put(q.sem_rgba.data(), q.sem_rgba.size());
    put(q.distance.data(), 4 * q.distance.size());
    put(q.gradient.data(), 4 * q.gradient.size());
    size_t hits = 0;
    for (float d : rr.depth) hits += (d == d) ? 1 : 0;
    std::printf("render: %dx%d pixels, %zu hits%s\n", w, h, hits, lazy ? " (host layers not synchronised)" : "");
  }
  if (lazy) server.updateLayers();
  {
    SemanticTsdfServer::SemanticMesh mesh;
    KSG_CHECK(server.extractMesh(&mesh)) << "mesh extraction failed";
    KSG_CHECK(mesh.vertices.size() % 9 == 0 && mesh.block_first.back() == (int64_t)mesh.labels.size());
    std::printf("semantic mesh: %zu triangles over %zu blocks\n", mesh.vertices.size() / 9, mesh.block_index.size() / 3);
  }
  if (save_path) KSG_CHECK(server.saveMap(save_path)) << "cannot save " << save_path;
  vxb::BlockIndexList blocks;
  tsdf_layer.getAllAllocatedBlocks(&blocks);
  std::sort(blocks.begin(), blocks.end(), [](const vxb::BlockIndex& a, const vxb::BlockIndex& b) {
    return a.z() != b.z() ? a.z() < b.z() : (a.y() != b.y() ? a.y() < b.y() : a.x() < b.x()); });
  std::ofstream o(argv[3], std::ios::binary);
  const int32_t nb = (int32_t)blocks.size();
  o.write(reinterpret_cast<const char*>(&nb), 4);
  for (const auto& bi : blocks) {
    const int32_t idx[3] = {bi.x(), bi.y(), bi.z()};
    o.write(reinterpret_cast<const char*>(idx), 12);
    auto tb = tsdf_layer.getBlockPtrByIndex(bi);
    auto sb = semantic_layer.getBlockPtrByIndex(bi);
    KSG_CHECK(sb != nullptr) << "semantic layer misses a block of the TSDF layer";
    for (size_t v = 0; v < tb->num_voxels(); ++v) {
      const vxb::TsdfVoxel& tv = tb->getVoxelByLinearIndex(v);
      const SemanticVoxel& sv = sb->getVoxelByLinearIndex(v);
      o.write(reinterpret_cast<const char*>(&tv.distance), 4);
      o.write(reinterpret_cast<const char*>(&tv.weight), 4);
      const uint8_t c[4] = {tv.color.r, tv.color.g, tv.color.b, tv.color.a};
      o.write(reinterpret_cast<const char*>(c), 4);
      o.write(reinterpret_cast<const char*>(&sv.semantic_label), 1);
      o.write(reinterpret_cast<const char*>(sv.semantic_priors.v.data()), 4 * kTotalNumberOfLabels);
      const uint8_t s[4] = {sv.color.r, sv.color.g, sv.color.b, sv.color.a};
      o.write(reinterpret_cast<const char*>(s), 4);
    }
  }
  std::printf("wrote %d blocks\n", nb);
  return 0;
}
