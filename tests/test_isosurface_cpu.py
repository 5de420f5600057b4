"""CPU: the marching-cubes mesh of next3d_b200.isosurface as tests/isosurface_oracle.py states it.  The table in csrc/isosurface.cu
is the one the face rule derives, every configuration's contour closes with at most five triangles, meshes of random and analytic
fields are closed, oriented outward and in the documented axis convention; the PLY writer, the MRC reader and the shape_utils
command's refusals."""
import os
import re
import struct

import numpy as np
import pytest

from tests import isosurface_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ the table
def cuda_table():
    src = open(os.path.join(ROOT, 'next3d_b200', 'csrc', 'isosurface.cu')).read()
    body = re.search(r'c_tri\[256\]\[16\] = \{(.*?)\n\};', src, re.S).group(1)
    rows = [[int(v) for v in r.split(',')] for r in re.findall(r'\{([-\d,\s]+)\}', body)]
    assert len(rows) == 256 and all(len(r) == 16 for r in rows)
    return rows


def test_cuda_table_equals_the_derivation():
    for config, row in enumerate(cuda_table()):
        tris = O.TABLE[config]
        assert row[15] == len(tris), config
        assert row[:3 * len(tris)] == [e for t in tris for e in t], config
        assert row[3 * len(tris):15] == [-1] * (15 - 3 * len(tris)), config


def _boundary(tris):
    """Directed edges of a cell's triangles whose reverse is not among them: the contour loops."""
    d = [(t[i], t[(i + 1) % 3]) for t in tris for i in range(3)]
    return {p for p in d if (p[1], p[0]) not in d}


@pytest.mark.parametrize('config', range(256))
def test_table_follows_the_face_rule(config):
    """Each face's contour segments join its two crossed edges, or on an ambiguous face cut off each inside corner; the segments
    close into loops; no fan diagonal joins two edges of one face; at most five triangles."""
    tris = O.TABLE[config]
    assert len(tris) <= 5
    inside = [(config >> k) & 1 for k in range(8)]
    bound = _boundary(tris)
    assert len(bound) == sum(len(O.face_segments(config, f)) for f in range(6))
    for corners, _ in O.FACES:
        edges = [e for e, (a, b) in enumerate(O.EDGES) if a in corners and b in corners]
        crossed = {e for e in edges if inside[O.EDGES[e][0]] != inside[O.EDGES[e][1]]}
        segs = {frozenset(p) for p in bound if set(p) <= set(edges)}
        if len(crossed) == 2:
            assert segs == {frozenset(crossed)}
        elif len(crossed) == 4:
            assert segs == {frozenset(e for e in crossed if k in O.EDGES[e]) for k in corners if inside[k]}
        else:
            assert not crossed and not segs
    heads = [a for a, _ in bound]
    tails = [b for _, b in bound]
    assert sorted(heads) == sorted(tails) and len(set(heads)) == len(heads)           # every crossed edge: one in, one out
    for t in tris:
        for i in range(3):
            a, b = t[i], t[(i + 1) % 3]
            if (a, b) not in bound:
                assert not any(a in f and b in f for f in O.FACE_EDGES), (config, t)


def test_single_corner_faces_outward():
    """Configuration 1 (corner 0 inside): the right-hand normal points away from corner 0."""
    (tri,) = O.TABLE[1]
    p = [O._mid(e) for e in tri]
    assert np.dot(np.cross(p[1] - p[0], p[2] - p[0]), np.ones(3)) > 0


# ------------------------------------------------------------------------------------------------ closed and oriented meshes
def random_grids():
    """Seeded random fields of 2-40 voxels per axis (cubic and not) with a -1000 border, level 10."""
    rng = np.random.default_rng(7)
    out = []
    for i in range(24):
        shape = (i % 3 + 2, 5, 3) if i < 3 else tuple(int(s) for s in rng.integers(2, 41, 3))
        g = (rng.standard_normal(shape) * 10 + 10).astype(np.float32)
        g[[0, -1]] = g[:, [0, -1]] = g[:, :, [0, -1]] = -1000
        out.append(g)
    return out


def configuration_grids():
    """All 256 configurations, each embedded in a 4x4x4 grid with a -1000 border, level 10."""
    rng = np.random.default_rng(8)
    out = []
    for config in range(256):
        g = np.full((4, 4, 4), -1000, np.float32)
        for k in range(8):
            dx, dy, dz = k & 1, (k >> 1) & 1, (k >> 2) & 1
            g[1 + dz, 1 + dy, 1 + dx] = 10 + (1 if (config >> k) & 1 else -1) * rng.uniform(0.5, 9)
        out.append(g)
    return out


def test_random_fields_are_closed_and_oriented():
    for g in random_grids():
        v, f = O.marching_cubes(g, 10.0)
        assert f.size == 0 or (f.min() >= 0 and f.max() < len(v))
        assert np.unique(f).size == len(v)                                            # every vertex is used
        assert O.directed_edges_closed(f), g.shape


def test_every_configuration_is_closed_and_oriented():
    for config, g in enumerate(configuration_grids()):
        v, f = O.marching_cubes(g, 10.0)
        assert O.directed_edges_closed(f), config
        if config not in (0, 255):
            assert O.area_volume(v, f)[1] > 0, config                                # encloses the inside corners


def _dist(shape, centre):
    z, y, x = np.meshgrid(*[np.arange(n, dtype=np.float64) for n in shape], indexing='ij')
    return np.sqrt((x - centre[0]) ** 2 + (y - centre[1]) ** 2 + (z - centre[2]) ** 2), (x, y, z)


def test_sphere():
    r = 20.0
    d, _ = _dist((64, 64, 64), (31.3, 32.1, 31.7))
    v, f = O.marching_cubes((r - d).astype(np.float32), 0.0)
    area, vol = O.area_volume(v, f)
    assert O.euler(v, f) == 2 and O.directed_edges_closed(f)
    assert abs(area / (4 * np.pi * r * r) - 1) < 0.01
    assert vol > 0 and abs(vol / (4 / 3 * np.pi * r ** 3) - 1) < 0.01


def test_torus():
    _, (x, y, z) = _dist((40, 64, 64), (0, 0, 0))
    rho = np.sqrt((x - 31.6) ** 2 + (y - 32.2) ** 2)
    g = (6.0 - np.sqrt((rho - 16.0) ** 2 + (z - 19.7) ** 2)).astype(np.float32)
    v, f = O.marching_cubes(g, 0.0)
    assert O.euler(v, f) == 0 and O.directed_edges_closed(f) and O.area_volume(v, f)[1] > 0


def test_two_spheres_one_voxel_apart():
    d1, _ = _dist((24, 24, 48), (12.0, 12.0, 12.0))
    d2, _ = _dist((24, 24, 48), (35.0, 12.0, 12.0))
    g = np.maximum(10.5 - d1, 10.5 - d2).astype(np.float32)                          # surfaces at x = 22.5 and 24.5
    v, f = O.marching_cubes(g, 0.0)
    assert O.components(len(v), f) == 2 and O.euler(v, f) == 4


def test_axis_convention():
    """A field of a2 alone is meshed as the plane x = const: y and z are the integer indices a1 and a0."""
    g = np.broadcast_to(np.arange(9, dtype=np.float32), (4, 6, 9)).copy()
    v, f = O.marching_cubes(g, 5.25)
    assert len(f) and np.all(v[:, 0] == np.float32(5.25))
    assert set(v[:, 1].tolist()) == set(range(6)) and set(v[:, 2].tolist()) == set(range(4))
    assert np.array_equal(v[:4], [[5.25, 0, 0], [5.25, 1, 0], [5.25, 2, 0], [5.25, 3, 0]])          # ascending (a0, a1, a2)


@pytest.mark.parametrize('row,xs', [([0, 10, 20], {1.0}), ([20, 10, 0], {1.0}), ([10, 20, 10], {0.0, 2.0})])
def test_voxels_at_the_level(row, xs):
    """A voxel equal to the level is outside (strict >): t = (level - s0) / (s1 - s0) is 0 on an edge that starts at it and 1 on
    an edge that ends at it, so the vertex lands on that voxel."""
    g = np.broadcast_to(np.array(row, np.float32), (2, 2, 3)).copy()
    v, f = O.marching_cubes(g, 10.0)
    assert len(f) and set(v[:, 0].tolist()) == xs


def test_grids_without_cells():
    for shape in ((1, 1, 1), (2, 1, 9), (1, 5, 5)):
        v, f = O.marching_cubes(np.full(shape, 20, np.float32) * (np.arange(shape[2]) % 2), 10.0)
        assert v.shape == (0, 3) and f.shape == (0, 3)


# ------------------------------------------------------------------------------------------------ PLY
HEADER = (b'ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n'
          b'element face %d\nproperty list uchar int vertex_indices\nend_header\n')


def parse_ply(data):
    """A strict reader of the two-element binary PLY files the reference writes: -> (verts [V, 3] float32, faces [F, 3] int32)."""
    end = data.index(b'end_header\n') + len(b'end_header\n')
    m = re.fullmatch(rb'ply\nformat binary_little_endian 1\.0\nelement vertex (\d+)\nproperty float x\nproperty float y\n'
                     rb'property float z\nelement face (\d+)\nproperty list uchar int vertex_indices\nend_header\n', data[:end])
    assert m, data[:end]
    nv, nf = int(m.group(1)), int(m.group(2))
    assert len(data) == end + 12 * nv + 13 * nf
    verts = np.frombuffer(data, '<f4', 3 * nv, end).reshape(nv, 3)
    rec = np.frombuffer(data, np.uint8, 13 * nf, end + 12 * nv).reshape(nf, 13)
    assert np.all(rec[:, 0] == 3)
    faces = np.ascontiguousarray(rec[:, 1:]).view('<i4').reshape(nf, 3)
    return verts, faces


def test_ply_header_and_round_trip(tmp_path):
    from next3d_b200.isosurface import ply_bytes, write_ply
    d, _ = _dist((16, 16, 16), (7.5, 7.2, 7.9))
    v, f = O.marching_cubes((5.5 - d).astype(np.float32), 0.0)
    data = ply_bytes(v, f)
    assert data.startswith(HEADER % (len(v), len(f)))
    gv, gf = parse_ply(data)
    assert np.array_equal(gv.view(np.int32), v.view(np.int32)) and np.array_equal(gf, f)
    write_ply(tmp_path / 'm.ply', v, f)
    assert (tmp_path / 'm.ply').read_bytes() == data


def test_ply_empty_mesh():
    from next3d_b200.isosurface import ply_bytes
    data = ply_bytes(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32))
    assert data == HEADER % (0, 0)
    assert [a.shape for a in parse_ply(data)] == [(0, 3), (0, 3)]


def test_ply_refuses_bad_arrays():
    from next3d_b200.isosurface import ply_bytes
    with pytest.raises(ValueError, match='verts'):
        ply_bytes(np.zeros((2, 3), np.float64), np.zeros((0, 3), np.int32))
    with pytest.raises(ValueError, match='faces'):
        ply_bytes(np.zeros((2, 3), np.float32), np.zeros((1, 4), np.int32))


# ------------------------------------------------------------------------------------------------ MRC
@pytest.mark.parametrize('shape', [(1, 1, 1), (3, 5, 7), (16, 9, 4), (32, 32, 32)])
def test_read_mrc_returns_what_write_mrc_wrote(tmp_path, shape):
    from next3d_b200.mrc import read_mrc, write_mrc
    x = np.random.default_rng(sum(shape)).standard_normal(shape).astype(np.float32)
    x.flat[0] = -1000
    write_mrc(tmp_path / 'a.mrc', x)
    y = read_mrc(tmp_path / 'a.mrc')
    assert y.shape == shape and y.dtype == np.float32 and np.array_equal(y.view(np.int32), x.view(np.int32))


def _mrc_file(path, x, nsymbt=0, mode=2, stamp=b'\x44\x44\x00\x00', order=(1, 2, 3), cut=0):
    from next3d_b200.mrc import write_mrc
    write_mrc(path, x)
    raw = bytearray(open(path, 'rb').read())
    struct.pack_into('<i', raw, 12, mode)
    struct.pack_into('<3i', raw, 64, *order)
    struct.pack_into('<i', raw, 92, nsymbt)
    raw[212:216] = stamp
    raw[1024:1024] = bytes(range(256)) * (nsymbt // 256) + bytes(nsymbt % 256)
    open(path, 'wb').write(bytes(raw[:len(raw) - cut]))


def test_read_mrc_skips_the_extended_header(tmp_path):
    from next3d_b200.mrc import read_mrc
    x = np.arange(60, dtype=np.float32).reshape(3, 4, 5)
    _mrc_file(tmp_path / 'e.mrc', x, nsymbt=1000)
    assert np.array_equal(read_mrc(tmp_path / 'e.mrc'), x)


@pytest.mark.parametrize('kw,field', [(dict(mode=0), 'mode'), (dict(stamp=b'\x11\x11\x00\x00'), 'machine stamp'),
                                      (dict(order=(3, 2, 1)), 'map order'), (dict(cut=4), 'truncated')])
def test_read_mrc_refuses(tmp_path, kw, field):
    from next3d_b200.mrc import read_mrc
    _mrc_file(tmp_path / 'b.mrc', np.zeros((3, 4, 5), np.float32), **kw)
    with pytest.raises(ValueError, match=field):
        read_mrc(tmp_path / 'b.mrc')


# ------------------------------------------------------------------------------------------------ shape_utils refusals
@pytest.fixture
def no_cuda(monkeypatch):
    """Any marching-cubes or CUDA work fails the test."""
    import torch
    from next3d_b200 import isosurface

    def fail(*a, **k):
        raise AssertionError('touched CUDA')
    monkeypatch.setattr(isosurface, 'marching_cubes', fail)
    monkeypatch.setattr(torch.cuda, 'set_device', fail)


def test_shape_utils_refusals(tmp_path, no_cuda):
    from next3d_b200.__main__ import main
    (tmp_path / 'a.ply').write_bytes(b'')
    write = tmp_path / 'g.mrc'
    write.write_bytes(b'')
    for argv, match in [([str(tmp_path / 'missing')], 'no such file'), ([str(tmp_path / 'a.ply')], r'\.mrc files'),
                        ([str(write), '--level', 'nan'], 'finite'), ([str(tmp_path), '--level', 'inf'], 'finite')]:
        with pytest.raises(SystemExit, match=match):
            main(['shape_utils', *argv])


def test_shape_utils_empty_directory(tmp_path, no_cuda, capsys):
    from next3d_b200.__main__ import main
    (tmp_path / 'x.ply').write_bytes(b'')
    main(['shape_utils', str(tmp_path)])
    assert 'nothing converted' in capsys.readouterr().out
    assert sorted(os.listdir(tmp_path)) == ['x.ply']
