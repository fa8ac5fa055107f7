"""The .vxblx ESDF layer file (vxblx_io::saveEsdfLayer): a host Layer<EsdfVoxel> written by cpp/test/esdf_io_test.cpp parses with
google.protobuf against voxblox's schema (Layer.proto / Block.proto, restated in vxblx_io.h) in voxblox's framing, with type "esdf",
two words per voxel and the flags packed as observed | hallucinated << 8 | in_queue << 16 | fixed << 24."""
import os
import subprocess

import numpy as np

from test_shim_cpu import CPP, demo  # noqa: F401


def parse_vxblx(path):
    """(LayerProto, [BlockProto]) of a .vxblx file: varint32 message count, then length-delimited LayerProto + BlockProto messages"""
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    fd = descriptor_pb2.FileDescriptorProto(name="vxblx_esdf_restated.proto", package="voxblox", syntax="proto2")
    T = descriptor_pb2.FieldDescriptorProto
    lay = fd.message_type.add(name="LayerProto")
    for name, num, typ in (("voxel_size", 1, T.TYPE_DOUBLE), ("voxels_per_side", 2, T.TYPE_UINT32), ("type", 3, T.TYPE_STRING)):
        lay.field.add(name=name, number=num, type=typ, label=T.LABEL_OPTIONAL)
    blk = fd.message_type.add(name="BlockProto")
    for name, num, typ in (("voxels_per_side", 1, T.TYPE_INT32), ("voxel_size", 2, T.TYPE_DOUBLE), ("origin_x", 3, T.TYPE_DOUBLE),
                           ("origin_y", 4, T.TYPE_DOUBLE), ("origin_z", 5, T.TYPE_DOUBLE), ("has_data", 6, T.TYPE_BOOL)):
        blk.field.add(name=name, number=num, type=typ, label=T.LABEL_OPTIONAL)
    f = blk.field.add(name="voxel_data", number=7, type=T.TYPE_UINT32, label=T.LABEL_REPEATED)
    f.options.packed = True
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fd)
    Layer = message_factory.GetMessageClass(pool.FindMessageTypeByName("voxblox.LayerProto"))
    Block = message_factory.GetMessageClass(pool.FindMessageTypeByName("voxblox.BlockProto"))
    raw = open(path, "rb").read()

    def varint(pos):
        v = shift = 0
        while True:
            c = raw[pos]
            pos += 1
            v |= (c & 0x7F) << shift
            shift += 7
            if not c & 0x80:
                return v, pos
    n, pos = varint(0)
    size, pos = varint(pos)
    layer = Layer()
    layer.ParseFromString(raw[pos:pos + size])
    pos += size
    blocks = []
    for _ in range(n - 1):
        size, pos = varint(pos)
        b = Block()
        b.ParseFromString(raw[pos:pos + size])
        pos += size
        blocks.append(b)
    assert pos == len(raw)
    return layer, blocks


def esdf_words(b):
    """(distance [V] f32, observed, hallucinated, in_queue, fixed [V] bool) of an ESDF BlockProto"""
    w = np.array(b.voxel_data, np.uint64).astype(np.uint32).reshape(-1, 2)
    assert ((w[:, 1] & ~np.uint32(0x01010101)) == 0).all()
    return (w[:, 0].view(np.float32),) + tuple(((w[:, 1] >> s) & 1).astype(bool) for s in (0, 8, 16, 24))


def test_esdf_layer_file_parses_against_the_voxblox_schema(demo, tmp_path):  # noqa: F811
    path = tmp_path / "esdf.vxblx"
    r = subprocess.run([os.path.join(CPP, "esdf_io_test"), str(path)], capture_output=True, text=True)
    assert r.returncode == 0 and "esdf io ok" in r.stdout, r.stderr
    layer, blocks = parse_vxblx(path)
    assert layer.type == "esdf" and layer.voxels_per_side == 8 and abs(layer.voxel_size - 0.05) < 1e-7
    want = {(0, 0, 0): 0, (-1, 2, 3): 1, (5, -7, 1): 2}
    v = np.arange(8 ** 3)
    seen = []
    for b in blocks:
        assert b.voxels_per_side == 8 and abs(b.voxel_size - 0.05) < 1e-7
        assert len(b.voxel_data) == 2 * 8 ** 3                     # two words per voxel
        key = tuple(round(o / (8 * 0.05)) for o in (b.origin_x, b.origin_y, b.origin_z))
        k = want[key]
        seen.append(key)
        assert b.has_data == (k != 2)
        dist, obs, hal, inq, fixed = esdf_words(b)
        assert (dist == ((v.astype(np.float32) - np.float32(100)) * np.float32(0.01)) * np.float32(k + 1)).all()
        assert (obs == (v % 2 == 1)).all() and (hal == (v % 3 == 0)).all() and (inq == (v % 5 == 0)).all() and (fixed == (v % 7 == 0)).all()
    assert seen == sorted(want, key=lambda b: (b[2], b[1], b[0]))   # (z, y, x) order
