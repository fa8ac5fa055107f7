// Writes a host Layer<EsdfVoxel> with vxblx_io::saveEsdfLayer: 8 voxels per side, 5 cm, three blocks; voxel v of block b has
// distance (v - 100) * 0.01 * (b + 1) and the flags observed = v % 2, hallucinated = v % 3 == 0, in_queue = v % 5 == 0,
// fixed = v % 7 == 0.  tests/test_esdf_file_cpu.py parses the file against voxblox's schema.
//   esdf_io_test <out.vxblx>
#include <cstdio>
#include "kimera_semantics/vxblx_io.h"

using namespace kimera;

int main(int argc, char** argv) {
  if (argc != 2) { std::fprintf(stderr, "usage: esdf_io_test <out.vxblx>\n"); return 2; }
  vxb::Layer<vxb::EsdfVoxel> layer(0.05f, 8);
  const vxb::BlockIndex blocks[3] = {vxb::BlockIndex(0, 0, 0), vxb::BlockIndex(-1, 2, 3), vxb::BlockIndex(5, -7, 1)};
  for (int b = 0; b < 3; ++b) {
    vxb::Block<vxb::EsdfVoxel>::Ptr blk = layer.allocateNewBlock(blocks[b]);
    blk->has_data() = b != 2;
    for (size_t v = 0; v < blk->num_voxels(); ++v) {
      vxb::EsdfVoxel& e = blk->getVoxelByLinearIndex(v);
      e.distance = ((float)v - 100.0f) * 0.01f * (float)(b + 1);
      e.observed = v % 2 == 1;
      e.hallucinated = v % 3 == 0;
      e.in_queue = v % 5 == 0;
      e.fixed = v % 7 == 0;
    }
  }
  if (!vxblx_io::saveEsdfLayer(argv[1], layer)) { std::fprintf(stderr, "cannot write %s\n", argv[1]); return 1; }
  std::printf("esdf io ok\n");
  return 0;
}
