"""CPU: the vertex-colour bake of next3d_b200.bake as tests/bake_oracle.py states it.  The voxel -> world map reproduces
create_samples at integer voxels, before and after the grid's flip; the coloured PLY layout; the oracle on analytic scenes (a
sphere sees its front hemisphere with cos^2 weights, a vertex behind a nearer quad takes the fallback, constant images give their
colour exactly); the calls, head ids and rank split of drivers.coloured_meshes on the recording stub generator; and the gen_meshes
command's refusals, which come before the network is opened."""
import struct

import numpy as np
import pytest
import torch

from tests import bake_oracle as B
from tests import isosurface_oracle as O

F = np.float32


# ------------------------------------------------------------------------------------------------ the voxel -> world map
def _map_tolerance(R, cube):
    """create_samples rounds the flat index to float32 (a step of 2^(ceil(log2 R^3) - 24) above 2^24) and divides in float32:
    the reference's own rounding, in world units, plus a few ulps of the coordinates."""
    vs = cube / (R - 1)
    ulp_idx = 2.0 ** max(0, int(np.ceil(np.log2(R ** 3))) - 24)
    return vs * (ulp_idx / R + R * 2.0 ** -22) + 2.0 ** -21 * cube


@pytest.mark.parametrize('R', [2, 7, 64, 512])
def test_world_map_reproduces_create_samples(R):
    """Over the voxels the shape grid decodes (inside the border trim of int(30 R / 256)): at R = 512 the last indices round
    past R^3 - 1 in float32 and wrap around in the reference, but they all lie in the trimmed border."""
    from next3d_b200.drivers import create_samples
    cube = 1.0
    pad = int(30 * R / 256)
    rng = np.random.default_rng(R)
    heads = [0, R ** 3 - min(R ** 3, 4096)] + [int(h) for h in rng.integers(0, max(1, R ** 3 - 4096), 3)]
    if pad:
        heads.append((R - pad - 1) * R * R + (R - pad - 9) * R)            # the last decoded rows, where the index rounds most
    checked = 0
    for head in heads:
        count = min(R ** 3 - head, 4096)
        pts = create_samples(R, cube, head, count)[0].numpy()
        idx = np.arange(head, head + count)
        i, j, k = idx // (R * R), (idx // R) % R, idx % R
        # before the flip: grid index (i, j, k) of the reshaped samples; the mesh's vertex is (x, y, z) = (k, j, R - 1 - i)
        verts = np.stack([k, j, R - 1 - i], 1).astype(F)
        got = B.world_points(verts, R, cube)
        inner = ((np.stack([i, j, k], 1) >= pad) & (np.stack([i, j, k], 1) < R - pad)).all(1)
        assert np.abs(got.astype(np.float64) - pts)[inner].max(initial=0) <= _map_tolerance(R, cube), head
        checked += inner.sum()
    assert checked >= min(R ** 3, 4096)


@pytest.mark.parametrize('R', [2, 7, 64])
def test_world_map_after_the_flip(R):
    """The densities of a field sampled at create_samples points, flipped and trimmed as the shape grid is, sit at the world
    points the map gives their voxel (x, y, z) = (a2, a1, a0)."""
    from next3d_b200.drivers import create_samples, trim_sigma_grid
    cube = 0.9
    pts = create_samples(R, cube)[0]
    f = (pts[:, 0] * 3.0 - pts[:, 1] * 2.0 + pts[:, 2] * 5.0).reshape(R, R, R).double()
    grid = trim_sigma_grid(f.clone(), R, pad_value=float('nan'))
    a0, a1, a2 = np.meshgrid(np.arange(R), np.arange(R), np.arange(R), indexing='ij')
    verts = np.stack([a2, a1, a0], -1).reshape(-1, 3).astype(F)
    w = B.world_points(verts, R, cube).astype(np.float64)
    want = (w[:, 0] * 3.0 - w[:, 1] * 2.0 + w[:, 2] * 5.0).reshape(R, R, R)
    keep = ~torch.isnan(grid).numpy()
    assert keep.any()
    assert np.abs(grid.numpy()[keep] - want[keep]).max() <= 10 * _map_tolerance(R, cube)


def test_world_map_is_exact_at_the_corners():
    for R, cube in [(2, 1.0), (64, 1.0), (512, 1.0)]:
        w = B.world_points(np.array([[0, 0, R - 1], [R - 1, R - 1, 0]], F), R, cube)
        assert w[0].tolist() == [-0.5, -0.5, -0.5]
        assert np.allclose(w[1], [0.5 + (R - 1) / R * (1 / (R - 1)) + (R - 1) / R ** 2 * (1 / (R - 1)), 0.5 + (R - 1) / R / (R - 1), 0.5],
                           atol=1e-6)


# ------------------------------------------------------------------------------------------------ PLY with colours
def test_coloured_ply_layout():
    from next3d_b200.isosurface import ply_bytes
    rng = np.random.default_rng(0)
    v = rng.standard_normal((7, 3)).astype(F)
    f = rng.integers(0, 7, (5, 3)).astype(np.int32)
    c = rng.integers(0, 256, (7, 3)).astype(np.uint8)
    data = ply_bytes(v, f, c)
    head = (b'ply\nformat binary_little_endian 1.0\nelement vertex 7\nproperty float x\nproperty float y\nproperty float z\n'
            b'property uchar red\nproperty uchar green\nproperty uchar blue\nelement face 5\nproperty list uchar int vertex_indices\n'
            b'end_header\n')
    assert data.startswith(head)
    body = data[len(head):]
    assert len(body) == 7 * 15 + 5 * 13
    rec = np.frombuffer(body[:7 * 15], dtype=[('xyz', '<f4', 3), ('rgb', 'u1', 3)])
    assert np.array_equal(rec['xyz'], v) and np.array_equal(rec['rgb'], c)
    for t in range(5):
        n, *ids = struct.unpack_from('<B3i', body, 7 * 15 + 13 * t)
        assert n == 3 and ids == f[t].tolist()
    assert ply_bytes(v, f, None) == ply_bytes(v, f)
    assert ply_bytes(torch.from_numpy(v), torch.from_numpy(f), torch.from_numpy(c)) == data


def test_coloured_ply_refuses_bad_colours():
    from next3d_b200.isosurface import ply_bytes
    v, f = np.zeros((4, 3), F), np.zeros((1, 3), np.int32)
    for c in (np.zeros((4, 3), np.int32), np.zeros((3, 3), np.uint8), np.zeros((4, 4), np.uint8)):
        with pytest.raises(ValueError, match='colors'):
            ply_bytes(v, f, c)


# ------------------------------------------------------------------------------------------------ the oracle on analytic scenes
def sphere_scene(R=48, radius=15.0, centre=(23.3, 23.6, 23.1)):
    """A marching-cubes sphere (density radius - distance, level 0) of an R^3 grid, and its world centre and radius."""
    a0, a1, a2 = np.meshgrid(*[np.arange(R, dtype=np.float64)] * 3, indexing='ij')
    d = np.sqrt((a2 - centre[0]) ** 2 + (a1 - centre[1]) ** 2 + (a0 - centre[2]) ** 2)
    grid = (radius - d).astype(F)
    verts, faces = O.marching_cubes(grid, 0.0)
    c = B.world_points(np.array([centre], F), R, 1.0)[0].astype(np.float64)
    return grid, verts, faces, c, radius / (R - 1)


def test_sphere_sees_its_front_hemisphere():
    grid, verts, faces, c, r = sphere_scene(radius=12.0)
    R = grid.shape[0]
    cam = B.camera(np.pi / 2 + 0.3, np.pi / 2 - 0.2)
    H = W = 96
    world = B.world_points(verts, R, 1.0)
    zb = B.zbuffer(world, faces, [cam], H, W)
    assert (zb != B.EMPTY).mean() > 0.1
    images = np.zeros((1, 3, H, W), F)
    colors, vis, w = B.bake(verts, world, grid, [cam], images, zb, np.zeros((len(verts), 3), F))
    origin = cam[:16].reshape(4, 4)[:3, 3].astype(np.float64)
    p = world.astype(np.float64)
    n = (p - c) / np.linalg.norm(p - c, axis=1, keepdims=True)
    to_cam = (origin - p) / np.linalg.norm(origin - p, axis=1, keepdims=True)
    cos = (n * to_cam).sum(1)
    # every front-facing vertex is seen; behind the silhouette the depth tolerance of two voxels lets a thin band through
    u, v, _ = B.project(cam, world, H, W)
    assert u.min() > 0 and u.max() < W - 1 and v.min() > 0 and v.max() < H - 1             # the whole sphere is in the image
    assert vis[0][cos > 0.02].all()
    assert not vis[0][cos < -0.25].any()
    front = vis[0] & (cos > 0)
    assert np.abs(w[0][front] - cos[front] ** 2).max() < 0.025
    assert (w[0][~vis[0]] == 0).all()


def quad_scene(R=16):
    """A quad (two triangles) at voxel x = 12 over y, z in [5, 10] in front of a small triangle at x = 4, seen by the frontal
    camera (world +z, which is voxel +x); the grid falls along x, so every normal faces that camera."""
    verts = np.array([[12, 5, 5], [12, 10, 5], [12, 10, 10], [12, 5, 10], [4, 7, 7], [4, 8, 7], [4, 7, 8]], F)
    faces = np.array([[0, 1, 2], [0, 2, 3], [4, 5, 6]], np.int32)
    grid = np.broadcast_to(-np.arange(R, dtype=F), (R, R, R)).copy()
    return grid, verts, faces


def test_hidden_vertex_takes_the_fallback():
    grid, verts, faces = quad_scene()
    R = grid.shape[0]
    cam = B.camera(np.pi / 2, np.pi / 2)
    H = W = 64
    world = B.world_points(verts, R, 1.0)
    zb = B.zbuffer(world, faces, [cam], H, W)
    ids = zb[zb != B.EMPTY] & np.uint64(0xFFFFFFFF)
    assert set(ids.tolist()) == {0, 1}                                 # the quad hides the far triangle entirely
    images = np.full((1, 3, H, W), 0.5, F)
    fallback = np.full((len(verts), 3), 0.375, F)                    # the decoder's 0.375 shows as 2 * 0.375 - 1 = -0.25
    colors, vis, w = B.bake(verts, world, grid, [cam], images, zb, fallback)
    assert vis[0].tolist() == [True] * 4 + [False] * 3
    assert (w[0][:4] > 0.9).all()
    assert (colors[:4] == 191).all()                                   # 0.5 * 127.5 + 128 = 191.75
    assert (colors[4:] == 96).all()                                    # -0.25 * 127.5 + 128 = 96.125


def test_constant_images_give_their_colour_exactly():
    """Dyadic colours: w * c and its sums scale exactly, so the weighted mean of several views is c itself."""
    grid, verts, faces, _, _ = sphere_scene(R=32, radius=10.0, centre=(15.4, 15.7, 15.2))
    R = grid.shape[0]
    cams = [B.camera(np.pi / 2 + yaw, np.pi / 2 + pitch) for yaw, pitch in [(-0.4, -0.2), (0.0, -0.2), (0.4, 0.2)]]
    H = W = 64
    world = B.world_points(verts, R, 1.0)
    zb = B.zbuffer(world, faces, cams, H, W)
    rgb = np.array([0.25, -0.5, 0.75], F)
    images = np.broadcast_to(rgb[None, :, None, None], (3, 3, H, W)).copy()
    colors, vis, w = B.bake(verts, world, grid, cams, images, zb, np.zeros((len(verts), 3), F))
    seen = w.sum(0) > 0
    assert seen.mean() > 0.4 and (~seen).any()
    assert (colors[seen] == [159, 64, 223]).all()
    assert (colors[~seen] == 0).all()                                  # decoder 0 -> -1 -> -1 * 127.5 + 128 = 0.5


def test_zbuffer_skips_near_and_degenerate_triangles():
    cam = B.camera(np.pi / 2, np.pi / 2, radius=1.0)
    origin = cam[:16].reshape(4, 4)[:3, 3]
    verts = np.array([[0, 0, 0], [0.1, 0, 0], [0, 0.1, 0],              # a visible triangle
                      [0, 0, 0.995], [0.1, 0, 0.995], [0, 0.1, 0.995],   # within the near plane (camera at z = 1)
                      [0, 0, 0.2], [0.1, 0.1, 0.2], [0.2, 0.2, 0.2]], F)   # zero area
    faces = np.array([[0, 1, 2], [3, 4, 5], [6, 7, 8], [0, 1, 9]], np.int32)
    assert np.allclose(origin, [0, 0, 1], atol=1e-6)
    zb = B.zbuffer(verts, faces, [cam], 32, 32)
    ids = set((zb[zb != B.EMPTY] & np.uint64(0xFFFFFFFF)).tolist())
    assert ids == {0}


# ------------------------------------------------------------------------------------------------ the coloured-mesh driver
def _run_coloured_meshes(monkeypatch, ws, v, seed, plan=None, batch=3):
    """(calls, [(head, what reached the bake)]) of drivers.coloured_meshes on the recording stub generator, with host stand-ins
    for marching cubes, the world map, the decoder at the vertices, the z-buffer and the bake (the last returns its inputs)."""
    from next3d_b200 import bake, drivers, isosurface
    from tests.test_driver_calls_cpu import _StubG
    G = _StubG()
    G.rendering_kwargs['box_warp'] = 0.5
    monkeypatch.setattr(isosurface, 'marching_cubes', lambda grid, level: (grid.reshape(-1, 1)[:4] * torch.tensor([1., 2., 3.]) + level,
                                                                           torch.tensor([[0, 1, 2], [1, 2, 3]], dtype=torch.int32)))
    monkeypatch.setattr(bake, 'world_points', lambda verts, R, cube: verts * cube + R)
    G.cached_sample_points = lambda b, world: (None, G.cached[0][b].mean() + world)
    monkeypatch.setattr(bake, 'mesh_zbuffer', lambda world, faces, cams, H, W: (world.sum() + faces.sum() + cams.sum()).expand(len(cams), H, W))
    monkeypatch.setattr(bake, 'bake_vertex_colors', lambda verts, world, grid, cams, images, zbuf, feat, cube:
                        dict(verts=verts, world=world, grid=grid.clone(), cams=cams, images=images.clone(), zbuf=zbuf, feat=feat, cube=cube))
    out = [(i, colors) for i, _, _, colors in drivers.coloured_meshes(G, ws, v, plan, batch=batch, shape_res=2, level=0.25, seed=seed)]
    return G.calls, out


@pytest.mark.parametrize('S,batch', [(5, 2), (7, 3), (1, 3)])
def test_coloured_meshes_calls_and_heads(monkeypatch, S, batch):
    """Per call of `batch` heads (the last repeats its last head): one caching synthesis of view 0 (seed + 2 c), one render_views
    of the other seven views of each head (seed + 2 c + 1), then one grid per head the call owns; every head is baked from its own
    views, grid and decoder features.  At world sizes 1-3 the ranks' whole-call plans make exactly the single-process calls."""
    from next3d_b200 import drivers
    from tests.test_driver_calls_cpu import RES, _StubG, _image, _sigmas
    g = torch.Generator().manual_seed(S * 10 + batch)
    ws, v = torch.randn(S, drivers.NUM_WS, 512, generator=g), torch.randn(1, 7, 3, generator=g)
    calls, out = _run_coloured_meshes(monkeypatch, ws, v, 3, batch=batch)
    n = len(drivers.BAKE_VIEWS)
    want = []
    for c in range(-(-S // batch)):
        want += [('synthesis', batch, True, False, 3 + 2 * c, None), ('render_views', batch * (n - 1), False, False, 4 + 2 * c, None)]
        want += [('grid', b) for b in range(min(batch, S - c * batch))]
    assert calls == want
    assert [i for i, _ in out] == list(range(S))
    cams = drivers.bake_cameras(_StubG())
    for i, got in out:
        assert torch.equal(got['images'], _image(ws[i:i + 1].expand(n, -1, -1), cams, v.expand(n, -1, -1), None, RES)), i
        assert torch.equal(got['cams'], cams) and got['zbuf'].shape == (n, RES, RES)
        assert torch.equal(got['grid'], _sigmas(ws[i], 2)), i
        assert torch.equal(got['verts'][:, 0], _sigmas(ws[i], 2).reshape(-1)[:4] + 0.25) and got['cube'] == 0.5
        assert torch.equal(got['feat'], ws[i].mean() + got['world']), i
    for world in (1, 2, 3):
        rank_calls, rank_out = [], []
        for r in range(world):
            c, o = _run_coloured_meshes(monkeypatch, ws, v, 3, plan=drivers.head_plan(S, batch, r, world), batch=batch)
            rank_calls += c
            rank_out += o
        assert rank_calls == calls, world                                 # whole calls: none repeated, none missing
        assert [i for i, _ in rank_out] == list(range(S))
        assert all(torch.equal(a['images'], b['images']) and torch.equal(a['grid'], b['grid']) for (_, a), (_, b) in zip(rank_out, out))


# ------------------------------------------------------------------------------------------------ the gen_meshes refusals
@pytest.mark.parametrize('extra,match', [
    (['--level', 'nan'], '--level'),
    (['--level', 'inf'], '--level'),
    (['--shape-res', '1'], '--shape-res'),
    (['--no-obj'], '--obj_path'),
    (['--no-lms'], '--lms_path'),
    (['--missing-obj'], '--obj_path'),
    (['--lms_cond', 'False'], 'lms_cond'),
])
def test_gen_meshes_refuses_before_loading(tmp_path, extra, match):
    from next3d_b200.__main__ import main
    from tests.test_legacy_cpu import _demo_args
    mesh = _demo_args(tmp_path)
    if extra == ['--no-obj']:
        mesh, extra = mesh[2:], []
    elif extra == ['--no-lms']:
        mesh, extra = mesh[:2], []
    elif extra == ['--missing-obj']:
        mesh, extra = ['--obj_path', str(tmp_path / 'none.obj')] + mesh[2:], []
    argv = ['gen_meshes', '--network', str(tmp_path / 'missing.pkl'), '--seeds', '0', '--outdir', str(tmp_path / 'o')] + mesh
    argv += extra if '--lms_cond' in extra else ['--lms_cond', 'True'] + extra
    with pytest.raises(SystemExit, match=match):
        main(argv)
    assert not (tmp_path / 'o').exists()
