"""The shim's ASCII .ply writer (kimera_semantics_b200/cpp/include/kimera_semantics/ply_io.h, what SemanticTsdfServer::generateMesh
writes): compiled and run on a small fixed mesh, then parsed back here - vertex x y z (float), red green blue alpha and label (uchar),
and one face 3 i i+1 i+2 per triangle of the soup."""
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, "kimera_semantics_b200", "cpp", "include")


def parse_ply(path):
    """dict(vertices [n, 3] f32, rgba [n, 4] u8, labels [n] u8, faces [m, 3] i64) of an ASCII .ply in the writer's layout"""
    with open(path) as f:
        lines = f.read().split("\n")
    assert lines[0] == "ply" and lines[1] == "format ascii 1.0"
    end = lines.index("end_header")
    head = lines[:end]
    nv = int(next(l for l in head if l.startswith("element vertex")).split()[2])
    nf = int(next(l for l in head if l.startswith("element face")).split()[2])
    props = [l.split()[1:] for l in head if l.startswith("property")]
    assert props == [["float", "x"], ["float", "y"], ["float", "z"], ["uchar", "red"], ["uchar", "green"], ["uchar", "blue"],
                     ["uchar", "alpha"], ["uchar", "label"], ["list", "uchar", "int", "vertex_indices"]], props
    rows = [l.split() for l in lines[end + 1:end + 1 + nv]]
    vtx = np.array([[np.float32(r[k]) for k in range(3)] for r in rows], np.float32).reshape(-1, 3)
    rgba = np.array([[int(r[k]) for k in range(3, 7)] for r in rows], np.uint8).reshape(-1, 4)
    lab = np.array([int(r[7]) for r in rows], np.uint8)
    faces = np.array([[int(x) for x in l.split()] for l in lines[end + 1 + nv:end + 1 + nv + nf]], np.int64).reshape(-1, 4)
    assert (faces[:, 0] == 3).all()
    return {"vertices": vtx, "rgba": rgba, "labels": lab, "faces": faces[:, 1:]}


PROGRAM = r"""
#include <cstdio>
#include <vector>
#include "kimera_semantics/ply_io.h"
int main(int, char** argv) {
  std::vector<float> v = {0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f, 1.f, 0.f, 0.1f, -2.5e-3f, 123.456f, 1e-8f, -0.f, 3.4e38f, 0.3f, 0.7f, 1.f / 3.f};
  std::vector<unsigned char> rgba, labels;
  for (int i = 0; i < 6; ++i) { rgba.push_back(10 * i); rgba.push_back(255 - i); rgba.push_back(i); rgba.push_back(200 + i); labels.push_back(i * 40); }
  return kimera_semantics::writeMeshPly(argv[1], v, rgba, labels) ? 0 : 1;
}
"""


def test_ply_writer_round_trips(tmp_path):
    src, exe, out = tmp_path / "ply.cpp", tmp_path / "ply", tmp_path / "mesh.ply"
    src.write_text(PROGRAM)
    subprocess.check_call(["g++", "-O2", "-std=c++11", "-Wall", "-Wextra", "-Werror", "-I" + INCLUDE, "-o", str(exe), str(src)])
    subprocess.check_call([str(exe), str(out)])
    p = parse_ply(out)
    want = np.array([0, 0, 0, 1, 0, 0, 0, 1, 0, 0.1, -2.5e-3, 123.456, 1e-8, -0.0, 3.4e38, 0.3, 0.7, 1 / 3], np.float32).reshape(-1, 3)
    assert p["vertices"].tobytes() == want.tobytes()                  # %.9g: every float32 reads back exactly
    assert p["rgba"].tolist() == [[10 * i, 255 - i, i, 200 + i] for i in range(6)]
    assert p["labels"].tolist() == [40 * i for i in range(6)]
    assert p["faces"].tolist() == [[0, 1, 2], [3, 4, 5]]
