"""GPU: the bake kernels of csrc/bake.cu write the world points, z-buffers, visibility, weights and colours of
tests/bake_oracle.py exactly: random triangle soups, triangles across the image border and the near plane, degenerate triangles
and marching-cubes spheres.  drivers.extract_coloured_mesh on generated heads has extract_mesh's geometry (and that of shape_utils
on gen_samples' .mrc grid), colours that repeat run to run, and vertices the frontal view sees at the depth it renders; the
gen_meshes command writes the same files at world sizes 1 to 3."""
import os

import numpy as np
import pytest
import torch

from tests import bake_oracle as B
from tests import isosurface_oracle as O
from tests.test_bake_cpu import quad_scene, sphere_scene

pytestmark = pytest.mark.gpu
DEV = 'cuda'
F = np.float32


def _t(a, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dtype)


def kernel_zbuffer(verts, faces, cams, H, W):
    from next3d_b200.bake import mesh_zbuffer
    zb = mesh_zbuffer(_t(verts, torch.float32), _t(faces, torch.int32), torch.from_numpy(np.stack(cams)), H, W)
    return zb.cpu().numpy().view(np.uint64)


def assert_zbuffer_equals_oracle(verts, faces, cams, H, W):
    got = kernel_zbuffer(verts, faces, cams, H, W)
    want = B.zbuffer(verts, faces, cams, H, W)
    assert np.array_equal(got, want), f'{(got != want).sum()} pixels differ'
    return got


def cameras(radius=2.7):
    return [B.camera(np.pi / 2 + yaw, np.pi / 2 + pitch, radius) for yaw, pitch in [(0.0, 0.0), (-0.5, -0.2), (0.7, 0.3)]]


# ------------------------------------------------------------------------------------------------ world points and z-buffers
@pytest.mark.parametrize('R', [2, 7, 64, 512])
def test_world_points_equal_oracle(R):
    from next3d_b200.bake import world_points
    v = (np.random.default_rng(R).random((5000, 3)) * (R - 1)).astype(F)
    v[:8] = np.array([[x, y, z] for x in (0, R - 1) for y in (0, R - 1) for z in (0, R - 1)], F)
    got = world_points(_t(v), R, 1.0).cpu().numpy()
    assert np.array_equal(got.view(np.int32), B.world_points(v, R, 1.0).view(np.int32))


@pytest.mark.parametrize('seed', range(4))
def test_zbuffer_random_soups_equal_oracle(seed):
    """Small and large triangles (the large ones take the warp-wide path), indices outside the vertices skipped."""
    rng = np.random.default_rng(seed)
    verts = (rng.random((300, 3)) - 0.5).astype(F) * F(0.8)
    faces = rng.integers(0, 300, (400, 3)).astype(np.int32)
    near = rng.integers(0, 300, (200, 1))
    faces[200:] = (near + rng.integers(-3, 4, (200, 3))).clip(0, 299)            # small triangles of nearby vertices
    faces[5] = [0, 1, 300]
    faces[6] = [-1, 2, 3]
    zb = assert_zbuffer_equals_oracle(verts, faces, cameras(), 96, 80)
    assert (zb != B.EMPTY).mean() > 0.05


def test_zbuffer_across_border_and_near_plane_equals_oracle():
    """Cameras 0.6 from the pivot: triangles straddle the image border, reach out of the image and cross the near plane."""
    rng = np.random.default_rng(7)
    verts = (rng.random((400, 3)) - 0.5).astype(F) * F(1.4)
    faces = rng.integers(0, 400, (300, 3)).astype(np.int32)
    cams = cameras(radius=0.6)
    zb = assert_zbuffer_equals_oracle(verts, faces, cams, 64, 64)
    assert (zb != B.EMPTY).any()
    for cam in cams:
        _, _, z = B.project(cam, verts, 64, 64)
        assert (z <= 0.01).any() and (z > 0.01).any()


def test_zbuffer_degenerate_triangles_equal_oracle():
    rng = np.random.default_rng(3)
    verts = (rng.random((50, 3)) - 0.5).astype(F) * F(0.5)
    verts[40:] = verts[30:40]                                            # duplicated points
    faces = np.concatenate([rng.integers(0, 50, (60, 3)), [[1, 1, 2], [3, 3, 3], [30, 40, 5], [31, 41, 31]]]).astype(np.int32)
    line = np.array([[0, 0, 0], [0.1, 0.1, 0.1], [0.2, 0.2, 0.2]], F)                  # collinear
    verts = np.concatenate([verts, line])
    faces = np.concatenate([faces, [[50, 51, 52]]]).astype(np.int32)
    assert_zbuffer_equals_oracle(verts, faces, cameras(), 64, 64)


def test_zbuffer_marching_cubes_sphere_equals_oracle():
    grid, verts, faces, _, _ = sphere_scene(R=40, radius=14.0, centre=(19.3, 19.6, 19.1))
    world = B.world_points(verts, grid.shape[0], 1.0)
    zb = assert_zbuffer_equals_oracle(world, faces, cameras(), 128, 128)
    assert (zb != B.EMPTY).mean() > 0.1


def test_zbuffer_empty_mesh():
    zb = kernel_zbuffer(np.zeros((0, 3), F), np.zeros((0, 3), np.int32), cameras()[:1], 8, 8)
    assert (zb == B.EMPTY).all()


# ------------------------------------------------------------------------------------------------ the bake
def kernel_bake(verts, faces, grid, cams, images, fallback, cube=1.0):
    """world points, then (colors, visible, weights) of the kernels, on the z-buffer the kernel draws."""
    from next3d_b200.bake import bake_vertex_colors, mesh_zbuffer, world_points
    v = _t(verts)
    world = world_points(v, grid.shape[0], cube)
    cams_t = torch.from_numpy(np.stack(cams))
    zb = mesh_zbuffer(world, _t(faces), cams_t, images.shape[2], images.shape[3])
    return world, bake_vertex_colors(v, world, _t(grid), cams_t, _t(images), zb, _t(fallback), cube, per_view=True)


def assert_bake_equals_oracle(grid, verts, faces, cams, images, fallback, cube=1.0):
    world, (colors, vis, w) = kernel_bake(verts, faces, grid, cams, images, fallback, cube)
    world = world.cpu().numpy()
    assert np.array_equal(world.view(np.int32), B.world_points(verts, grid.shape[0], cube).view(np.int32))
    zb = B.zbuffer(world, faces, cams, images.shape[2], images.shape[3])
    oc, ovis, ow = B.bake(verts, world, grid, cams, images, zb, fallback, cube=cube)
    vis = vis.cpu().numpy().astype(bool)
    # visibility may only differ where the depth test is within 1e-6 of its threshold (it does not: every operation rounds alike)
    R = grid.shape[0]
    eps = F(2 * cube / (R - 1))
    depth = B.zbuffer_depth(zb)
    for v, cam in enumerate(cams):
        u, wv, z = B.project(cam, world, images.shape[2], images.shape[3])
        r = np.clip(np.floor(wv + F(0.5)), 0, images.shape[2] - 1).astype(np.int64)
        c = np.clip(np.floor(u + F(0.5)), 0, images.shape[3] - 1).astype(np.int64)
        margin = np.abs(z.astype(np.float64) - (depth[v, r, c].astype(np.float64) + eps))
        assert not (vis[v] != ovis[v])[~(margin < 1e-6)].any()
    assert np.array_equal(vis, ovis)
    assert np.array_equal(w.cpu().numpy().view(np.int32), ow.view(np.int32))
    assert np.array_equal(colors.cpu().numpy(), oc)
    return oc, ovis, ow


def test_bake_sphere_equals_oracle():
    grid, verts, faces, _, _ = sphere_scene(R=40, radius=12.0, centre=(19.3, 19.6, 19.1))
    cams = cameras()
    rng = np.random.default_rng(0)
    images = (rng.random((3, 3, 96, 96)) * 2 - 1).astype(F)
    fallback = (rng.random((len(verts), 5)) * 1.002 - 0.001).astype(F)              # the decoder's range
    oc, ovis, ow = assert_bake_equals_oracle(grid, verts, faces, cams, images, fallback)
    seen = ow.sum(0) > 0
    assert 0.3 < seen.mean() < 1


def test_bake_hidden_vertex_equals_oracle():
    grid, verts, faces = quad_scene()
    cams = [B.camera(np.pi / 2, np.pi / 2)]
    images = np.full((1, 3, 64, 64), 0.5, F)
    oc, ovis, _ = assert_bake_equals_oracle(grid, verts, faces, cams, images, np.full((len(verts), 3), 0.375, F))
    assert ovis[0].tolist() == [True] * 4 + [False] * 3


def test_bake_refuses_bad_arguments():
    from next3d_b200.bake import bake_vertex_colors, mesh_zbuffer
    v, f = torch.zeros(4, 3, device=DEV), torch.zeros(2, 3, dtype=torch.int32, device=DEV)
    cams = torch.from_numpy(np.stack(cameras()[:1]))
    with pytest.raises(ValueError, match='int32'):
        mesh_zbuffer(v, f.long(), cams, 8, 8)
    with pytest.raises(ValueError, match='shape'):
        mesh_zbuffer(v[:, :2], f, cams, 8, 8)
    with pytest.raises(RuntimeError, match='CUDA tensor'):
        mesh_zbuffer(v.cpu(), f, cams, 8, 8)
    with pytest.raises(ValueError, match='cams'):
        mesh_zbuffer(v, f, cams[:, :16], 8, 8)
    zb = mesh_zbuffer(v, f, cams, 8, 8)
    grid = torch.zeros(4, 4, 4, device=DEV)
    images = torch.zeros(1, 3, 8, 8, device=DEV)
    fb = torch.zeros(4, 3, device=DEV)
    bake_vertex_colors(v, v, grid, cams, images, zb, fb, 1.0)
    for args, match in [((v, v, grid[:, :, :3], cams, images, zb, fb), 'cube'), ((v, v, grid, cams, images[:, :2], zb, fb), 'images'),
                        ((v, v, grid, cams, images, zb[:, :4], fb), 'zbuf'), ((v, v, grid, cams, images, zb, fb[:, :2]), '3 channels'),
                        ((v, v[:3], grid, cams, images, zb, fb), 'world')]:
        with pytest.raises(ValueError, match=match):
            bake_vertex_colors(*args, 1.0)


# ------------------------------------------------------------------------------------------------ generated heads
@pytest.fixture(scope='module')
def tiny():
    from next3d_b200 import config, drivers
    from tests.test_gpu_views import _generator
    cfg = config.tiny_config(512)
    _, G = _generator(cfg, 6)
    from next3d_b200 import weights
    _, _, _, v = weights.demo_inputs(cfg, 1, seed=3)
    ws = drivers.sample_sheet_ws(G, [0, 1], 0.7)
    return G, ws, v.to(DEV)


def _cutting_level(G, ws, v, res):
    from next3d_b200 import drivers
    grid = drivers.extract_sigma_grid(G, ws, v, shape_res=res)
    return float(np.quantile(grid[grid > -1000], 0.7))


def test_extract_coloured_mesh_has_extract_mesh_geometry(tiny):
    from next3d_b200 import drivers
    G, ws, v = tiny
    level = _cutting_level(G, ws[:1], v, 96)
    verts, faces, colors = drivers.extract_coloured_mesh(G, ws[:1], v, shape_res=96, level=level)
    ev, ef = drivers.extract_mesh(G, ws[:1], v, shape_res=96, level=level)
    assert len(faces) > 1000
    assert torch.equal(verts.view(torch.int32), ev.view(torch.int32)) and torch.equal(faces, ef)
    assert colors.dtype == torch.uint8 and colors.shape == verts.shape
    v2, f2, c2 = drivers.extract_coloured_mesh(G, ws[:1], v, shape_res=96, level=level)
    assert torch.equal(c2, colors) and torch.equal(f2, faces)
    assert len(torch.unique(colors, dim=0)) > 50
    # a batch of two heads gives the first head's mesh of its own call
    out = list(drivers.coloured_meshes(G, ws, v, shape_res=96, level=level, batch=2))
    assert [i for i, *_ in out] == [0, 1]
    assert torch.equal(out[0][1].view(torch.int32), verts.view(torch.int32)) and torch.equal(out[0][2], faces)


def test_unseen_vertices_take_the_decoders_colour(tiny):
    """A vertex no bake view sees has the decoder's colour at its world point as image_raw shows it: G.sample_mixed's first three
    channels f, rescaled 2 f - 1 and converted to uint8 as the images are.  The views and weights are recomputed with the calls
    and sampler seeds of extract_coloured_mesh, which must give its colours."""
    from next3d_b200 import bake, drivers
    G, ws, v = tiny
    res = 96
    level = _cutting_level(G, ws[:1], v, res)
    verts, faces, colors = drivers.extract_coloured_mesh(G, ws[:1], v, shape_res=res, level=level)
    eng = G._get_engine()
    cams = drivers.bake_cameras(G).to(DEV)
    front = G.synthesis(ws[:1], cams[:1], v, noise_mode='const', cache_backbone=True, seed=0)['image']
    images = torch.cat([front, G.render_views(cams[1:], seed=1)['image']])
    grid = torch.empty(res, res, res, device=DEV)
    eng.cached_sigma_grid(0, res, grid)
    box = G.rendering_kwargs['box_warp']
    world = bake.world_points(verts, res, box)
    _, feat = eng.cached_sample_points(0, world)
    zb = bake.mesh_zbuffer(world, faces, cams, images.shape[2], images.shape[3])
    again, _, w = bake.bake_vertex_colors(verts, world, grid, cams, images, zb, feat, box, per_view=True)
    assert torch.equal(again, colors)
    unseen = w.sum(0) == 0
    assert 0 < int(unseen.sum()) < len(verts)
    rgb = G.sample_mixed(world[None], None, ws[:1], v, noise_mode='const')['rgb'][0, :, :3]
    want = ((rgb * 2 - 1) * 127.5 + 128).clamp(0, 255).to(torch.uint8)
    assert torch.equal(colors[unseen], want[unseen])
    # the decoder's range is about 0..1: as it was written before the rescale, the unseen colours would all be >= 127
    assert int((want[unseen] < 120).sum()) > 0


@pytest.mark.parametrize('yaw,pitch,quantile', [(0.0, -0.2, 0.99), (0.0, 0.2, 0.97)], ids=['frontal', 'below'])
def test_views_see_vertices_at_their_rendered_depth(yaw, pitch, quantile):
    """A full-config random-weight head: the distances to the camera of the vertices the bake marks visible in a bake view follow
    that view's rendered depth at their pixels, and three wrong conventions each break that: the mesh's x and z axes exchanged,
    the image rows flipped (w -> H - 1 - w), and the grid's a0 flip undone (z -> R - 1 - z).  The random weights give a density
    without a sharp surface (rendered depth is an expectation through a fog), so the mesh is taken at the dense core and the check
    is the correlation, with a median offset of under 20 voxels of the 128^3 grid, not agreement to a few voxels.  The head is
    nearly mirror-symmetric left to right, which hides the undone a0 flip (a left-right mirror of the mesh) from the frontal
    view at the sheets' pitch; the frontal view from below (pitch +0.2) shows it."""
    from next3d_b200 import bake, config, drivers, weights
    from next3d_b200.isosurface import marching_cubes
    from tests.test_gpu_views import _generator
    cfg = config.full_config(512)
    _, G = _generator(cfg, 1)
    _, _, _, v = weights.demo_inputs(cfg, 1, seed=1)
    v = v.to(DEV)
    ws = drivers.sample_sheet_ws(G, [4], 0.7)
    res = 128
    eng = G._get_engine()
    cams = drivers.bake_cameras(G).to(DEV)
    view = drivers.BAKE_VIEWS.index((yaw, pitch))
    cam_t = cams[view:view + 1]
    out = G.synthesis(ws, cam_t, v, noise_mode='const', cache_backbone=True, seed=0, depth_range='image')
    grid = torch.empty(res, res, res, device=DEV)
    eng.cached_sigma_grid(0, res, grid)
    inner = grid[grid > -1000]
    level = float(torch.quantile(inner[::max(1, inner.numel() // 1000000)], quantile))
    verts, faces = marching_cubes(grid, level)
    box = G.rendering_kwargs['box_warp']
    H = W = out['image'].shape[-1]
    vs = box / (res - 1)
    cam = cams[view].cpu().numpy()
    depth = out['image_depth'][0, 0].cpu().numpy()

    def compare(verts, flip_rows=False):
        """(correlation, median |distance - rendered depth| in voxels) over the visible vertices."""
        verts = verts.contiguous()
        world = bake.world_points(verts, res, box)
        _, feat = eng.cached_sample_points(0, world)
        zb = bake.mesh_zbuffer(world, faces, cam_t, H, W)
        _, vis, _ = bake.bake_vertex_colors(verts, world, grid, cam_t, out['image'], zb, feat, box, per_view=True)
        w = world.cpu().numpy()[vis[0].cpu().numpy().astype(bool)]
        assert len(w) > 1000
        Rn = depth.shape[0]
        u, wv, _ = B.project(cam, w, Rn, Rn)
        r, c = np.clip(np.rint(wv), 0, Rn - 1).astype(int), np.clip(np.rint(u), 0, Rn - 1).astype(int)
        d = depth[Rn - 1 - r if flip_rows else r, c]
        dist = np.linalg.norm(w - cam[:16].reshape(4, 4)[:3, 3], axis=1)
        return np.corrcoef(dist, d)[0, 1], np.median(np.abs(dist - d)) / vs

    corr, med = compare(verts)
    swapped, _ = compare(verts[:, [2, 1, 0]])
    rows, _ = compare(verts, flip_rows=True)
    unflipped, _ = compare(torch.stack([verts[:, 0], verts[:, 1], res - 1 - verts[:, 2]], 1))
    print(f'view ({yaw}, {pitch}): correlation {corr:.3f}, median offset {med:.1f} voxels; axes exchanged {swapped:.3f}, '
          f'rows flipped {rows:.3f}, a0 flip undone {unflipped:.3f}')
    assert corr > 0.85 and med < 20
    assert swapped < 0.6 and rows < 0.6
    if view != drivers.BAKE_VIEWS.index((0.0, drivers.SHEET_PITCH)):
        assert unflipped < 0.6


# ------------------------------------------------------------------------------------------------ the gen_meshes command
def read_ply(data):
    head, body = data.split(b'end_header\n', 1)
    lines = head.decode().split('\n')
    nv = int(next(l for l in lines if l.startswith('element vertex')).split()[-1])
    nf = int(next(l for l in lines if l.startswith('element face')).split()[-1])
    coloured = 'property uchar red' in lines
    vt = np.dtype([('xyz', '<f4', 3)] + ([('rgb', 'u1', 3)] if coloured else []))
    rec = np.frombuffer(body[:nv * vt.itemsize], vt)
    ft = np.dtype([('n', 'u1'), ('ids', '<i4', 3)])
    faces = np.frombuffer(body[nv * vt.itemsize:], ft)
    assert len(faces) == nf and (faces['n'] == 3).all()
    return rec['xyz'], faces['ids'], rec['rgb'] if coloured else None


@pytest.fixture(scope='module')
def net(tmp_path_factory):
    from next3d_b200 import config, weights
    from tests.test_gpu_legacy import _mask
    from tests.test_legacy_cpu import _demo_args, generator_fields, persistence_pickle
    d = tmp_path_factory.mktemp('meshes')
    cfg = config.tiny_config(512)
    path = d / 'tiny.pkl'
    path.write_bytes(persistence_pickle(cfg, weights.make_state_dict(cfg, seed=9), generator_fields(cfg, _mask(10))))
    return str(path), _demo_args(d), d


@pytest.fixture(scope='module')
def shapes(net):
    """gen_samples --shapes True of seeds 3 and 5 at --shape-res 48, and a level that cuts the tiny generator's heads (the 0.7
    quantile of seed 3's densities inside the border)."""
    from next3d_b200.mrc import read_mrc
    from tests.test_gpu_sharded_cli import _cli
    path, demo, d = net
    out = d / 'shapes'
    _cli(['gen_samples', '--network', path, '--seeds', '3,5', '--outdir', str(out), '--shapes', 'True', '--shape-res', '48',
          '--lms_cond', 'True', *demo], 1)
    g = np.asarray(read_mrc(str(out / 'seed0003.mrc')))
    return out, float(np.quantile(g[g > -1000], 0.7))


def test_gen_meshes_matches_shape_utils_on_gen_samples(net, shapes, tmp_path):
    from tests.test_gpu_sharded_cli import _cli
    path, demo, _ = net
    shapes, level = shapes
    _cli(['shape_utils', str(shapes), '--level', repr(level)], 1)
    meshes = tmp_path / 'meshes'
    _cli(['gen_meshes', '--network', path, '--seeds', '3,5', '--outdir', str(meshes), '--shape-res', '48', '--level', repr(level),
          '--lms_cond', 'True', *demo], 1)
    assert sorted(os.listdir(meshes)) == ['seed0003.ply', 'seed0005.ply']
    for name in ('seed0003', 'seed0005'):
        sv, sf, sc = read_ply((shapes / f'{name}.ply').read_bytes())
        mv, mf, mc = read_ply((meshes / f'{name}.ply').read_bytes())
        assert sc is None and mc is not None and len(mf) > 0
        assert np.array_equal(sv.view(np.int32), mv.view(np.int32)) and np.array_equal(sf, mf), name
        assert O.directed_edges_closed(mf)


def test_gen_meshes_at_world_2_and_3(net, shapes, tmp_path):
    from tests.test_gpu_sharded_cli import _same_files_at
    path, demo, _ = net
    level = shapes[1]
    files = _same_files_at((2, 3), lambda out: ['gen_meshes', '--network', path, '--seeds', '0-4', '--outdir', out, '--shape-res', '48',
                                                '--level', repr(level), '--lms_cond', 'True', *demo], tmp_path)
    assert sorted(files) == [f'seed{s:04d}.ply' for s in range(5)]
    assert sum(read_ply(b)[1].size > 0 for b in files.values()) >= 3
