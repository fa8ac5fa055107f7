// ASCII .ply of a semantic mesh soup, the file SemanticTsdfServer::generateMesh writes to the path `mesh_filename` names.  The layout
// follows voxblox's outputMeshAsPly as far as it can be restated (voxblox is not in the reference tree, so this is unpinned): vertex
// x y z (float) and red green blue alpha (uchar), here with one more uchar property, the semantic label, then one face "3 i i+1 i+2"
// per triangle of the soup (3 consecutive vertices).  Coordinates are printed with 9 significant digits, so every float reads back
// exactly.
#pragma once
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

namespace kimera_semantics {

// vertices: 3 floats per vertex; rgba: 4 bytes per vertex; labels: 1 byte per vertex; the vertex count must be a multiple of 3
inline bool writeMeshPly(const std::string& path, const std::vector<float>& vertices, const std::vector<uint8_t>& rgba,
                         const std::vector<uint8_t>& labels) {
  const size_t n = labels.size();
  if (vertices.size() != 3 * n || rgba.size() != 4 * n || n % 3 != 0) return false;
  std::FILE* f = std::fopen(path.c_str(), "w");
  if (!f) return false;
  std::fprintf(f, "ply\nformat ascii 1.0\nelement vertex %zu\nproperty float x\nproperty float y\nproperty float z\n", n);
  std::fprintf(f, "property uchar red\nproperty uchar green\nproperty uchar blue\nproperty uchar alpha\nproperty uchar label\n");
  std::fprintf(f, "element face %zu\nproperty list uchar int vertex_indices\nend_header\n", n / 3);
  for (size_t i = 0; i < n; ++i)
    std::fprintf(f, "%.9g %.9g %.9g %u %u %u %u %u\n", (double)vertices[3 * i], (double)vertices[3 * i + 1], (double)vertices[3 * i + 2],
                 (unsigned)rgba[4 * i], (unsigned)rgba[4 * i + 1], (unsigned)rgba[4 * i + 2], (unsigned)rgba[4 * i + 3], (unsigned)labels[i]);
  for (size_t t = 0; t < n / 3; ++t) std::fprintf(f, "3 %zu %zu %zu\n", 3 * t, 3 * t + 1, 3 * t + 2);
  const bool ok = !std::ferror(f);
  return std::fclose(f) == 0 && ok;
}

}  // namespace kimera_semantics
