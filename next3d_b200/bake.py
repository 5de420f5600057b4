"""Vertex colours of shape meshes on the device (csrc/bake.cu; DESIGN.md section 3.8): `world_points` maps marching-cubes
vertices of the flipped shape grid to the world points the densities were sampled at, `mesh_zbuffer` rasterises a mesh into the
renderer's camera views, and `bake_vertex_colors` blends those views onto the vertices.  The colours are a function of the mesh,
the grid, the images, the cameras and the fallback colours alone; tests/bake_oracle.py restates them in numpy."""
import math

import torch

from . import _lib

INDEX_LIMIT = 1 << 31           # vertex and triangle counts must fit int32 indices and the z-buffer's 32-bit triangle ids
NEAR = 0.01                     # near plane (world units) of the z-buffer and the bake; the heads sit ~2.7 from the cameras
EMPTY = -1                      # a z-buffer pixel no triangle covers (~0 as int64)


def _check(t, name, dtype, shape):
    """Refuse t unless it is a CUDA tensor of `dtype` whose shape matches `shape` (None = any size there)."""
    _lib.require_cuda(t, name)
    if t.dtype != dtype:
        raise ValueError(f'{name} must be {dtype}, got {t.dtype}')
    if t.dim() != len(shape) or any(s is not None and s != n for s, n in zip(shape, t.shape)):
        want = ', '.join('*' if s is None else str(s) for s in shape)
        raise ValueError(f'{name} must have shape [{want}], got {list(t.shape)}')
    return t.contiguous()


def _cameras(cams, device):
    """cams [views, 25] (cam2world 16 + intrinsics 9, the generator's camera_params) -> (cam2world, intrinsics) on `device`."""
    cams = torch.as_tensor(cams)
    if cams.dim() != 2 or cams.shape[1] != 25 or cams.shape[0] < 1:
        raise ValueError(f'cams must be [views >= 1, 25] camera_params, got {list(cams.shape)}')
    cams = cams.to(device, torch.float32)
    return cams[:, :16].contiguous(), cams[:, 16:].contiguous()


def voxel_size(grid_n, cube):
    return cube / (grid_n - 1)


def world_points(verts, grid_n, cube):
    """World points float32 [V, 3] of verts float32 [V, 3] (CUDA; voxel units (x, y, z) = (a2, a1, a0) of the flipped grid of
    drivers.create_samples(grid_n, cube)).  The sheared map of create_samples' float division, exact at integer voxels."""
    verts = _check(verts, 'verts', torch.float32, (None, 3))
    if grid_n < 2 or not (math.isfinite(cube) and cube > 0):
        raise ValueError(f'need grid_n >= 2 and a finite positive cube, got {grid_n}, {cube}')
    world = torch.empty_like(verts)
    with torch.cuda.device(verts.device):
        _lib.check(_lib.lib.n3d_bake_world_points(verts.data_ptr(), verts.shape[0], int(grid_n), float(cube), world.data_ptr(),
                                                  _lib.stream_ptr(verts.device)), 'n3d_bake_world_points')
    return world


def mesh_zbuffer(verts, faces, cams, height, width, near=NEAR):
    """Z-buffer int64 [views, height, width] of the mesh (verts float32 [V, 3] world points, faces int32 [F, 3]; CUDA) in the
    views cams [views, 25]: pixel = (camera depth bits << 32) | triangle id of the nearest triangle covering its centre, EMPTY
    where none does (the uint64 keys of n3d_mesh_zbuffer, viewed as int64)."""
    verts = _check(verts, 'verts', torch.float32, (None, 3))
    faces = _check(faces, 'faces', torch.int32, (None, 3))
    if faces.device != verts.device:
        raise ValueError(f'verts are on {verts.device}, faces on {faces.device}')
    if verts.shape[0] >= INDEX_LIMIT or faces.shape[0] >= INDEX_LIMIT:
        raise ValueError(f'{verts.shape[0]} vertices and {faces.shape[0]} triangles: int32 indices stop at 2^31 - 1')
    if height < 1 or width < 1:
        raise ValueError(f'the image must be at least 1x1, got {height}x{width}')
    c2w, intr = _cameras(cams, verts.device)
    zbuf = torch.empty(c2w.shape[0], height, width, dtype=torch.int64, device=verts.device)
    with torch.cuda.device(verts.device):
        _lib.check(_lib.lib.n3d_mesh_zbuffer(verts.data_ptr(), verts.shape[0], faces.data_ptr(), faces.shape[0], c2w.data_ptr(),
                                             intr.data_ptr(), c2w.shape[0], height, width, float(near), zbuf.data_ptr(),
                                             _lib.stream_ptr(verts.device)), 'n3d_mesh_zbuffer')
    return zbuf


def zbuffer_depth(zbuf):
    """Camera depth float32 of every z-buffer pixel (inf where empty) and its triangle id int64 (-1 where empty)."""
    empty = zbuf == EMPTY
    depth = (zbuf >> 32).to(torch.int32).view(torch.float32).masked_fill(empty, float('inf'))
    return depth, (zbuf & 0xffffffff).masked_fill(empty, -1)


def bake_vertex_colors(verts, world, grid, cams, images, zbuf, fallback, cube, near=NEAR, eps=None, per_view=False):
    """uint8 colours [V, 3] of the vertices verts float32 [V, 3] (voxel units of `grid`) at world points `world`
    (world_points(verts, R, cube)), from images float32 [views, 3, H, W] (-1..1) rendered with cams [views, 25], their z-buffer
    zbuf (mesh_zbuffer) and the density grid float32 [R, R, R] the mesh came from.  A vertex with no visible, front-facing view
    takes the decoder's colour: fallback float32 [V, >= 3] holds the decoder's output at the vertices as n3d_sample_points writes
    it (Engine.cached_sample_points; its first three channels, sigmoid(x) * 1.002 - 0.001), and the kernel rescales it by
    2 f - 1 to the images' range, as the ray marcher rescales its composite for image_raw.  eps: the visibility tolerance in
    camera depth, by default two voxels (2 cube / (R - 1)).  per_view: also return visible uint8 [views, V] and weights float32
    [views, V]."""
    verts = _check(verts, 'verts', torch.float32, (None, 3))
    dev, V = verts.device, verts.shape[0]
    world = _check(world, 'world', torch.float32, (V, 3))
    grid = _check(grid, 'grid', torch.float32, (None, None, None))
    R = grid.shape[0]
    if tuple(grid.shape) != (R, R, R) or R < 2:
        raise ValueError(f'grid must be a cube [R, R, R] with R >= 2, got {list(grid.shape)}')
    c2w, intr = _cameras(cams, dev)
    n = c2w.shape[0]
    images = _check(images, 'images', torch.float32, (n, 3, None, None))
    H, W = images.shape[2:]
    zbuf = _check(zbuf, 'zbuf', torch.int64, (n, H, W))
    fallback = _check(fallback, 'fallback', torch.float32, (V, None))
    if fallback.shape[1] < 3:
        raise ValueError(f'fallback needs at least 3 channels, got {fallback.shape[1]}')
    if V >= INDEX_LIMIT:
        raise ValueError(f'{V} vertices: int32 indices stop at 2^31 - 1')
    for t, name in ((world, 'world'), (grid, 'grid'), (images, 'images'), (zbuf, 'zbuf'), (fallback, 'fallback')):
        if t.device != dev:
            raise ValueError(f'verts are on {dev}, {name} on {t.device}')
    eps = 2 * voxel_size(R, cube) if eps is None else eps
    colors = torch.empty(V, 3, dtype=torch.uint8, device=dev)
    visible = torch.empty(n, V, dtype=torch.uint8, device=dev) if per_view else None
    weights = torch.empty(n, V, dtype=torch.float32, device=dev) if per_view else None
    with torch.cuda.device(dev):
        _lib.check(_lib.lib.n3d_bake_vertex_colors(verts.data_ptr(), world.data_ptr(), V, grid.data_ptr(), R, c2w.data_ptr(),
                                                   intr.data_ptr(), n, images.data_ptr(), H, W, zbuf.data_ptr(), float(near), float(eps),
                                                   fallback.data_ptr(), fallback.shape[1], colors.data_ptr(), _lib.ptr(visible),
                                                   _lib.ptr(weights), _lib.stream_ptr(dev)), 'n3d_bake_vertex_colors')
    return (colors, visible, weights) if per_view else colors
