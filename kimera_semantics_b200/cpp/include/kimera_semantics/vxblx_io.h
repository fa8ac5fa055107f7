// voxblox ".vxblx" layer files for the TSDF layer (SURVEY.md 8f NEXT-3, second half): what the reference's rosbag tool writes at the end
// of a run (kimera_semantics_ros/src/kimera_semantics_rosbag.cpp:148-166 -> voxblox::io::SaveLayer) and what voxblox tools read.
//
// voxblox (voxblox/io/layer_io_inl.h, utils/protobuf_utils.cc, proto/voxblox/{Layer,Block}.proto) is NOT under /root/reference: the
// format is restated from knowledge of that code ("parity unpinned"), written directly in protobuf wire format (no protobuf dependency):
//   file      = varint32 N, then N length-delimited messages (varint32 size + bytes): one LayerProto, then N - 1 BlockProto
//   LayerProto: 1 double voxel_size, 2 uint32 voxels_per_side, 3 string type ("tsdf")
//   BlockProto: 1 int32 voxels_per_side, 2 double voxel_size, 3/4/5 double origin_x/y/z, 6 bool has_data, 7 repeated uint32 voxel_data
//               (packed); a TSDF voxel is 3 words: distance bits, weight bits, (r << 24 | g << 16 | b << 8 | a); an ESDF voxel
//               (saveEsdfLayer, LayerProto type "esdf") is 2 words: distance bits, observed | hallucinated << 8 | in_queue << 16 | fixed << 24
// tests/test_shim_cpu.py parses a file written here with google.protobuf against exactly this schema.  Host-only code.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#include <fstream>
#include <string>
#include <vector>
#include "kimera_semantics/map_io.h"

namespace kimera {
namespace vxblx_io {

namespace wire {
inline void varint(std::string* o, uint64_t v) {
  while (v >= 0x80u) { o->push_back((char)((v & 0x7Fu) | 0x80u)); v >>= 7; }
  o->push_back((char)v);
}
inline void f64(std::string* o, int field, double v) {
  varint(o, ((uint64_t)field << 3) | 1u);
  char b[8];
  std::memcpy(b, &v, 8);
  o->append(b, 8);
}
inline void u64(std::string* o, int field, uint64_t v) { varint(o, ((uint64_t)field << 3) | 0u); varint(o, v); }
inline void bytes(std::string* o, int field, const std::string& v) { varint(o, ((uint64_t)field << 3) | 2u); varint(o, v.size()); o->append(v); }

struct Reader {
  const uint8_t* p;
  const uint8_t* end;
  bool ok;
  Reader(const uint8_t* b, size_t n) : p(b), end(b + n), ok(true) {}
  bool done() const { return p >= end; }
  uint64_t varint() {
    uint64_t v = 0;
    for (int shift = 0; shift < 64; shift += 7) {
      if (p >= end) { ok = false; return 0; }
      const uint8_t c = *p++;
      v |= (uint64_t)(c & 0x7Fu) << shift;
      if (!(c & 0x80u)) return v;
    }
    ok = false;
    return 0;
  }
  double f64() {
    if (end - p < 8) { ok = false; return 0.0; }
    double v;
    std::memcpy(&v, p, 8);
    p += 8;
    return v;
  }
  Reader sub() {   // length-delimited payload
    const uint64_t n = varint();
    if (!ok || (uint64_t)(end - p) < n) { ok = false; return Reader(p, 0); }
    Reader r(p, (size_t)n);
    p += n;
    return r;
  }
  void skip(int wire_type) {
    if (wire_type == 0) varint();
    else if (wire_type == 1) { if (end - p < 8) ok = false; else p += 8; }
    else if (wire_type == 2) sub();
    else if (wire_type == 5) { if (end - p < 4) ok = false; else p += 4; }
    else ok = false;
  }
};
}  // namespace wire

// The file head and the blocks of voxblox::io::SaveLayer; `words(block, &data)` appends a block's packed voxel_data.
template <typename VoxelType, typename Words>
bool saveLayer(const std::string& path, const vxb::Layer<VoxelType>& layer, const char* type, Words words) {
  std::ofstream o(path.c_str(), std::ios::binary | std::ios::trunc);
  if (!o.good()) return false;
  const std::vector<vxb::BlockIndex> blocks = map_io::sortedBlocks(layer);
  std::string head, msg;
  wire::varint(&head, 1u + blocks.size());
  wire::f64(&msg, 1, (double)layer.voxel_size());
  wire::u64(&msg, 2, (uint64_t)layer.voxels_per_side());
  wire::bytes(&msg, 3, type);
  wire::varint(&head, msg.size());
  o.write(head.data(), (std::streamsize)head.size());
  o.write(msg.data(), (std::streamsize)msg.size());
  std::string data;
  for (const vxb::BlockIndex& bi : blocks) {
    const typename vxb::Block<VoxelType>::ConstPtr b = layer.getBlockPtrByIndex(bi);
    msg.clear();
    wire::u64(&msg, 1, (uint64_t)b->voxels_per_side());
    wire::f64(&msg, 2, (double)b->voxel_size());
    wire::f64(&msg, 3, (double)b->origin().x());
    wire::f64(&msg, 4, (double)b->origin().y());
    wire::f64(&msg, 5, (double)b->origin().z());
    wire::u64(&msg, 6, b->has_data() ? 1u : 0u);
    data.clear();
    words(*b, &data);
    wire::bytes(&msg, 7, data);
    head.clear();
    wire::varint(&head, msg.size());
    o.write(head.data(), (std::streamsize)head.size());
    o.write(msg.data(), (std::streamsize)msg.size());
  }
  return o.good();
}

// voxblox::io::SaveLayer for Layer<EsdfVoxel> (what EsdfServer::saveMap writes beside the TSDF): restated from knowledge of voxblox's
// Block<EsdfVoxel> serialisation, unpinned like saveTsdfLayer.  Two words per voxel: the distance bits, then
// observed | hallucinated << 8 | in_queue << 16 | fixed << 24.
inline bool saveEsdfLayer(const std::string& path, const vxb::Layer<vxb::EsdfVoxel>& layer) {
  return saveLayer(path, layer, "esdf", [](const vxb::Block<vxb::EsdfVoxel>& b, std::string* data) {
    for (size_t v = 0; v < b.num_voxels(); ++v) {
      const vxb::EsdfVoxel& e = b.getVoxelByLinearIndex(v);
      uint32_t d;
      std::memcpy(&d, &e.distance, 4);
      wire::varint(data, d);
      wire::varint(data, (uint32_t)e.observed | ((uint32_t)e.hallucinated << 8) | ((uint32_t)e.in_queue << 16) | ((uint32_t)e.fixed << 24));
    }
  });
}

// voxblox::io::SaveLayer for Layer<TsdfVoxel>: all allocated blocks, (z, y, x) order (voxblox: hash-map order; readers do not depend on it)
inline bool saveTsdfLayer(const std::string& path, const vxb::Layer<vxb::TsdfVoxel>& layer) {
  return saveLayer(path, layer, "tsdf", [](const vxb::Block<vxb::TsdfVoxel>& b, std::string* data) {
    for (size_t v = 0; v < b.num_voxels(); ++v) {
      const vxb::TsdfVoxel& t = b.getVoxelByLinearIndex(v);
      uint32_t d, w;
      std::memcpy(&d, &t.distance, 4);
      std::memcpy(&w, &t.weight, 4);
      wire::varint(data, d);
      wire::varint(data, w);
      wire::varint(data, ((uint32_t)t.color.r << 24) | ((uint32_t)t.color.g << 16) | ((uint32_t)t.color.b << 8) | (uint32_t)t.color.a);
    }
  });
}

// voxblox::io::LoadLayer / LoadBlocksFromFile (kReplace) for Layer<TsdfVoxel>: the layer must have the file's voxel size and voxels per
// side (and the file's type must be "tsdf"); returns false and leaves the layer unchanged otherwise or when the file is malformed.
inline bool loadTsdfLayer(const std::string& path, vxb::Layer<vxb::TsdfVoxel>* layer) {
  std::ifstream in(path.c_str(), std::ios::binary);
  if (!in.good() || !layer) return false;
  const std::string buf((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
  wire::Reader r(reinterpret_cast<const uint8_t*>(buf.data()), buf.size());
  const uint64_t n_msgs = r.varint();
  if (!r.ok || n_msgs < 1) return false;
  {
    wire::Reader m = r.sub();
    if (!r.ok) return false;
    double voxel_size = 0.0;
    uint64_t vps = 0;
    std::string type;
    while (m.ok && !m.done()) {
      const uint64_t tag = m.varint();
      const int field = (int)(tag >> 3), wt = (int)(tag & 7u);
      if (field == 1 && wt == 1) voxel_size = m.f64();
      else if (field == 2 && wt == 0) vps = m.varint();
      else if (field == 3 && wt == 2) { wire::Reader s = m.sub(); type.assign(reinterpret_cast<const char*>(s.p), (size_t)(s.end - s.p)); }
      else m.skip(wt);
    }
    if (!m.ok || type != "tsdf" || vps != layer->voxels_per_side() || std::fabs(voxel_size - (double)layer->voxel_size()) > 1e-6) return false;
  }
  struct Loaded { vxb::BlockIndex index; bool has_data; std::vector<uint32_t> words; };
  std::vector<Loaded> loaded;
  const size_t V = layer->voxels_per_side() * layer->voxels_per_side() * layer->voxels_per_side();
  for (uint64_t k = 1; k < n_msgs; ++k) {
    wire::Reader m = r.sub();
    if (!r.ok) return false;
    Loaded b;
    b.has_data = false;
    double origin[3] = {0.0, 0.0, 0.0}, voxel_size = 0.0;
    uint64_t vps = 0;
    while (m.ok && !m.done()) {
      const uint64_t tag = m.varint();
      const int field = (int)(tag >> 3), wt = (int)(tag & 7u);
      if (field == 1 && wt == 0) vps = m.varint();
      else if (field == 2 && wt == 1) voxel_size = m.f64();
      else if (field >= 3 && field <= 5 && wt == 1) origin[field - 3] = m.f64();
      else if (field == 6 && wt == 0) b.has_data = m.varint() != 0;
      else if (field == 7 && wt == 2) { wire::Reader d = m.sub(); while (d.ok && !d.done()) b.words.push_back((uint32_t)d.varint()); if (!d.ok) m.ok = false; }
      else if (field == 7 && wt == 0) b.words.push_back((uint32_t)m.varint());      // unpacked encoding of the same field
      else m.skip(wt);
    }
    if (!m.ok || vps != layer->voxels_per_side() || std::fabs(voxel_size - (double)layer->voxel_size()) > 1e-6 || b.words.size() != 3 * V) return false;
    const double bs = (double)layer->block_size();
    b.index = vxb::BlockIndex((int)std::lround(origin[0] / bs), (int)std::lround(origin[1] / bs), (int)std::lround(origin[2] / bs));
    loaded.push_back(std::move(b));
  }
  layer->removeAllBlocks();
  for (const Loaded& b : loaded) {
    vxb::Block<vxb::TsdfVoxel>::Ptr blk = layer->allocateBlockPtrByIndex(b.index);
    blk->has_data() = b.has_data;
    for (size_t v = 0; v < V; ++v) {
      vxb::TsdfVoxel& t = blk->getVoxelByLinearIndex(v);
      std::memcpy(&t.distance, &b.words[3 * v], 4);
      std::memcpy(&t.weight, &b.words[3 * v + 1], 4);
      const uint32_t c = b.words[3 * v + 2];
      t.color = vxb::Color((uint8_t)(c >> 24), (uint8_t)(c >> 16), (uint8_t)(c >> 8), (uint8_t)c);
    }
  }
  return true;
}

}  // namespace vxblx_io
}  // namespace kimera
