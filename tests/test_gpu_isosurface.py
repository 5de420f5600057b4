"""GPU: the marching-cubes kernels of csrc/isosurface.cu write the counts, vertex bits and faces of tests/isosurface_oracle.py
exactly, on every CPU-suite grid and on shapes that stress the row decomposition, on two streams; non-finite grids are refused.
drivers.extract_mesh on generated heads is the oracle's mesh of extract_sigma_grid's grid, and `python -m next3d_b200 shape_utils`
on the .mrc files of `gen_samples --shapes True` writes the PLY files of the oracle's meshes, also as torchrun ranks."""
import os

import numpy as np
import pytest
import torch

from tests import isosurface_oracle as O
from tests.test_isosurface_cpu import _dist, configuration_grids, random_grids

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def kernel_mesh(g, level, stream=None):
    """The two passes through the C ABI on `stream` -> ([V, F, non-finite], verts, faces) on the host."""
    from next3d_b200 import _lib
    stream = stream or torch.cuda.current_stream()
    nz, ny, nx = g.shape
    nbytes = _lib.C.c_size_t()
    _lib.check(_lib.lib.n3d_isosurface_workspace_bytes(nz, ny, nx, _lib.C.byref(nbytes)))
    with torch.cuda.stream(stream):
        grid = torch.from_numpy(np.ascontiguousarray(g)).to(DEV)
        ws = torch.full((nbytes.value,), 0xA5, dtype=torch.uint8, device=DEV)           # stale workspace bytes must not matter
        counts = torch.empty(3, dtype=torch.int64, device=DEV)
        _lib.check(_lib.lib.n3d_isosurface_count(grid.data_ptr(), nz, ny, nx, level, ws.data_ptr(), counts.data_ptr(),
                                                 stream.cuda_stream))
        c = counts.tolist()
        verts = torch.full((max(c[0], 1), 3), float('nan'), device=DEV)
        faces = torch.full((max(c[1], 1), 3), -1, dtype=torch.int32, device=DEV)
        _lib.check(_lib.lib.n3d_isosurface_emit(grid.data_ptr(), nz, ny, nx, level, ws.data_ptr(), verts.data_ptr(), faces.data_ptr(),
                                                stream.cuda_stream))
        stream.synchronize()
    return c, verts[:c[0]].cpu().numpy(), faces[:c[1]].cpu().numpy()


def assert_equals_oracle(g, level):
    c, v, f = kernel_mesh(g, level)
    ov, of = O.marching_cubes(g, level)
    assert c == [len(ov), len(of), 0]
    assert np.array_equal(v.view(np.int32), ov.view(np.int32))
    assert np.array_equal(f, of)
    side = torch.cuda.Stream()
    c2, v2, f2 = kernel_mesh(g, level, side)
    assert c2 == c and v2.tobytes() == v.tobytes() and f2.tobytes() == f.tobytes()
    return ov, of


def smooth(shape, seed):
    """A seeded sum of random plane waves, in [-3, 3]."""
    rng = np.random.default_rng(seed)
    z, y, x = np.meshgrid(*[np.arange(n, dtype=np.float32) for n in shape], indexing='ij', sparse=True)
    g = np.zeros(shape, np.float32)
    for _ in range(3):
        k = rng.uniform(-0.2, 0.2, 3).astype(np.float32)
        g += np.sin(k[0] * x + k[1] * y + k[2] * z + np.float32(rng.uniform(0, 6)))
    return g


def analytic():
    d, (x, y, z) = _dist((64, 64, 64), (31.3, 32.1, 31.7))
    rho = np.sqrt((x - 31.6) ** 2 + (y - 32.2) ** 2)
    d1, _ = _dist((24, 24, 48), (12.0, 12.0, 12.0))
    d2, _ = _dist((24, 24, 48), (35.0, 12.0, 12.0))
    return {
        'sphere': ((20.0 - d).astype(np.float32), 0.0),
        'torus': ((6.0 - np.sqrt((rho - 16.0) ** 2 + (z - 19.7) ** 2)).astype(np.float32), 0.0),
        'two_spheres': (np.maximum(10.5 - d1, 10.5 - d2).astype(np.float32), 0.0),
        'axis': (np.broadcast_to(np.arange(9, dtype=np.float32), (4, 6, 9)).copy(), 5.25),
        'at_level_up': (np.broadcast_to(np.array([0, 10, 20], np.float32), (2, 2, 3)).copy(), 10.0),
        'at_level_peak': (np.broadcast_to(np.array([10, 20, 10], np.float32), (2, 2, 3)).copy(), 10.0),
    }


def shapes():
    rng = np.random.default_rng(11)
    return {
        '17x33x65': ((rng.standard_normal((17, 33, 65)) * 10 + 10).astype(np.float32), 10.0),
        '3x5x700': ((rng.standard_normal((3, 5, 700)) * 10 + 10).astype(np.float32), 10.0),
        '1x1x1': (np.full((1, 1, 1), 20, np.float32), 10.0),
        '2x1x9': ((np.arange(18, dtype=np.float32).reshape(2, 1, 9) % 3) * 10, 10.0),
        'all_inside': (np.full((9, 7, 40), 20, np.float32), 10.0),
        'all_outside': (np.full((9, 7, 40), -5, np.float32), 10.0),
        'smooth256': (smooth((256, 256, 256), 5), 0.5),
    }


def test_random_grids_equal_oracle():
    for g in random_grids():
        assert_equals_oracle(g, 10.0)


def test_configuration_grids_equal_oracle():
    for g in configuration_grids():
        assert_equals_oracle(g, 10.0)


@pytest.mark.parametrize('name', list(analytic()))
def test_analytic_fields_equal_oracle(name):
    g, level = analytic()[name]
    assert_equals_oracle(g, level)


@pytest.mark.parametrize('name', ['17x33x65', '3x5x700', '1x1x1', '2x1x9', 'all_inside', 'all_outside', 'smooth256'])
def test_shapes_equal_oracle(name):
    g, level = shapes()[name]
    v, f = assert_equals_oracle(g, level)
    if name in ('1x1x1', '2x1x9', 'all_inside', 'all_outside'):
        assert len(v) == 0 and len(f) == 0
    else:
        assert len(f) > 0


def test_marching_cubes_api():
    from next3d_b200.isosurface import marching_cubes
    g, level = analytic()['sphere']
    ov, of = O.marching_cubes(g, level)
    for src in (g, torch.from_numpy(g).to(DEV)):
        v, f = marching_cubes(src, level)
        assert v.is_cuda and f.is_cuda and v.dtype == torch.float32 and f.dtype == torch.int32
        assert np.array_equal(v.cpu().numpy().view(np.int32), ov.view(np.int32)) and np.array_equal(f.cpu().numpy(), of)
    v, f = marching_cubes(np.full((1, 4, 4), 20, np.float32))
    assert v.shape == (0, 3) and f.shape == (0, 3) and v.is_cuda


@pytest.mark.parametrize('bad', [float('nan'), float('inf')])
def test_non_finite_voxels_are_refused(bad):
    from next3d_b200.isosurface import marching_cubes
    g = np.zeros((6, 7, 8), np.float32)
    g[3, 2, 5] = bad
    with pytest.raises(ValueError, match='1 non-finite'):
        marching_cubes(torch.from_numpy(g).to(DEV))


def test_bad_arguments_are_refused():
    from next3d_b200.isosurface import marching_cubes
    for grid, level, match in [(np.zeros((4, 4), np.float32), 10, '3-D'), (np.zeros((4, 4, 4), np.float64), 10, 'float32'),
                               (torch.zeros(4, 4, 4, dtype=torch.float16, device=DEV), 10, 'float32'),
                               (np.zeros((4, 4, 4), np.float32), float('nan'), 'finite')]:
        with pytest.raises(ValueError, match=match):
            marching_cubes(grid, level)
    with pytest.raises(RuntimeError, match='CUDA tensor'):
        marching_cubes(torch.zeros(4, 4, 4))


# ------------------------------------------------------------------------------------------------ generated heads
@pytest.fixture(scope='module')
def tiny():
    from next3d_b200 import config, weights
    from tests.test_gpu_views import _generator
    cfg = config.tiny_config(512)
    _, G = _generator(cfg, 6)
    z, cc, _, v = weights.demo_inputs(cfg, 1, seed=3)
    ws = G.mapping(z.to(DEV), cc.to(DEV), truncation_psi=0.7, truncation_cutoff=14)
    return G, ws, v.to(DEV)


@pytest.mark.parametrize('res', [128, 256])
def test_extract_mesh_equals_oracle(tiny, res):
    from next3d_b200 import drivers
    G, ws, v = tiny
    grid = drivers.extract_sigma_grid(G, ws, v, shape_res=res)
    inner = grid[grid > -1000]
    level = float(np.quantile(inner, 0.7))             # the tiny generator's densities: a level that cuts the head
    verts, faces = drivers.extract_mesh(G, ws, v, shape_res=res, level=level)
    ov, of = O.marching_cubes(grid, level)
    assert len(of) > 1000
    assert np.array_equal(verts.cpu().numpy().view(np.int32), ov.view(np.int32)) and np.array_equal(faces.cpu().numpy(), of)
    assert O.directed_edges_closed(of)


# ------------------------------------------------------------------------------------------------ the shape_utils command
@pytest.fixture(scope='module')
def shapes_dir(tmp_path_factory):
    """The outdir of `gen_samples --shapes True` on the tiny generator: seedNNNN.png and seedNNNN.mrc for seeds 0-4."""
    from tests.test_gpu_sharded_cli import _cli
    from next3d_b200 import config, weights
    from tests.test_gpu_legacy import _mask
    from tests.test_legacy_cpu import _demo_args, generator_fields, persistence_pickle
    d = tmp_path_factory.mktemp('shapes')
    cfg = config.tiny_config(512)
    net = d / 'tiny.pkl'
    net.write_bytes(persistence_pickle(cfg, weights.make_state_dict(cfg, seed=9), generator_fields(cfg, _mask(10))))
    out = d / 'out'
    _cli(['gen_samples', '--network', str(net), '--seeds', '0-4', '--outdir', str(out), '--shapes', 'True', '--shape-res', '64',
          '--lms_cond', 'True', *_demo_args(d)], 1)
    return out


def _mrc_files(d):
    return sorted(n for n in os.listdir(d) if n.endswith('.mrc'))


def _copy_mrcs(src, dst):
    os.makedirs(dst, exist_ok=True)
    for n in _mrc_files(src):
        with open(os.path.join(src, n), 'rb') as f, open(os.path.join(dst, n), 'wb') as g:
            g.write(f.read())
    return str(dst)


def _cutting_level(d):
    """A level that cuts the tiny generator's heads: the 0.7 quantile of the first grid's densities inside the border."""
    from next3d_b200.mrc import read_mrc
    g = np.asarray(read_mrc(os.path.join(d, _mrc_files(d)[0])))
    return float(np.quantile(g[g > -1000], 0.7))


@pytest.mark.parametrize('level', ['default', '5', 'cutting'])
def test_shape_utils_writes_the_oracle_meshes(shapes_dir, tmp_path, level):
    from next3d_b200.isosurface import ply_bytes
    from next3d_b200.mrc import read_mrc
    from tests.test_gpu_sharded_cli import _cli
    d = _copy_mrcs(shapes_dir, tmp_path / 'd')
    cutting = level == 'cutting'
    level = {'default': None, '5': 5.0, 'cutting': _cutting_level(d)}[level]
    _cli(['shape_utils', d] + ([] if level is None else ['--level', repr(level)]), 1)
    names = _mrc_files(d)
    assert len(names) == 5
    assert sorted(os.listdir(d)) == sorted(names + [n[:-4] + '.ply' for n in names])
    faces = 0
    for n in names:
        ov, of = O.marching_cubes(np.asarray(read_mrc(os.path.join(d, n))), 10.0 if level is None else level)
        assert open(os.path.join(d, n[:-4] + '.ply'), 'rb').read() == ply_bytes(ov, of), n
        faces += len(of)
    assert faces > 0 or not cutting


def test_shape_utils_single_file(shapes_dir, tmp_path):
    from tests.test_gpu_sharded_cli import _cli
    d = _copy_mrcs(shapes_dir, tmp_path / 'all')
    _cli(['shape_utils', d], 1)
    one = _copy_mrcs(shapes_dir, tmp_path / 'one')
    name = _mrc_files(one)[2]
    _cli(['shape_utils', os.path.join(one, name)], 1)
    ply = name[:-4] + '.ply'
    assert sorted(n for n in os.listdir(one) if n.endswith('.ply')) == [ply]
    assert open(os.path.join(one, ply), 'rb').read() == open(os.path.join(d, ply), 'rb').read()


def test_shape_utils_at_world_2_and_3(shapes_dir, tmp_path):
    from tests.test_gpu_sharded_cli import _cli, _files
    want = None
    for w in (1, 2, 3):
        d = _copy_mrcs(shapes_dir, tmp_path / f'w{w}')
        _cli(['shape_utils', d, '--level', '8'], w)
        got = {n: b for n, b in _files(d).items() if n.endswith('.ply')}
        assert len(got) == 5, w
        if want is None:
            want = got
        assert got == want, w
