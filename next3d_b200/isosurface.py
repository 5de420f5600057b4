"""Meshes of density grids on the device: `marching_cubes` runs the sm_90a marching cubes of csrc/isosurface.cu on a float32 grid
[nz, ny, nx], and `ply_bytes` / `write_ply` write the mesh as the binary PLY file the reference's shape_utils.py writes with
plyfile.  The mesh is a function of the grid and the level alone (DESIGN.md section 3.7; tests/isosurface_oracle.py restates
it in numpy)."""
import math

import numpy as np
import torch

from . import _lib

INDEX_LIMIT = 1 << 31           # vertex and triangle counts must fit the int32 indices of the faces


def marching_cubes(grid, level=10.0):
    """Mesh of the level set of `grid` (float32 [nz, ny, nx]; a CUDA tensor, or a numpy array copied to the current device) ->
    (verts float32 [V, 3], faces int32 [F, 3]) CUDA tensors.  Vertex (x, y, z) = (a2, a1, a0) in voxel units, as the reference
    meshes np.transpose(grid, (2, 1, 0)); a voxel is inside when grid > level, and triangles wind with their right-hand normal
    pointing outward (down the density).  One host read of the counts between the two passes."""
    if isinstance(grid, np.ndarray):
        if grid.dtype != np.float32:
            raise ValueError(f'marching_cubes needs a float32 grid, got {grid.dtype}')
        grid = torch.from_numpy(np.ascontiguousarray(grid)).to(torch.device('cuda', torch.cuda.current_device()))
    _lib.require_cuda(grid, 'grid')
    if grid.dim() != 3:
        raise ValueError(f'marching_cubes needs a 3-D grid [nz, ny, nx], got shape {list(grid.shape)}')
    if grid.dtype != torch.float32:
        raise ValueError(f'marching_cubes needs a float32 grid, got {grid.dtype}')
    level = float(level)
    if not math.isfinite(level):
        raise ValueError(f'the level must be finite, got {level}')
    dev = grid.device
    empty = (torch.zeros(0, 3, dtype=torch.float32, device=dev), torch.zeros(0, 3, dtype=torch.int32, device=dev))
    if grid.numel() == 0:
        return empty
    grid = grid.contiguous()
    nz, ny, nx = grid.shape
    nbytes = _lib.C.c_size_t()
    _lib.check(_lib.lib.n3d_isosurface_workspace_bytes(nz, ny, nx, _lib.C.byref(nbytes)), 'n3d_isosurface_workspace_bytes')
    with torch.cuda.device(dev):
        stream = _lib.stream_ptr(dev)
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        counts = torch.empty(3, dtype=torch.int64, device=dev)
        _lib.check(_lib.lib.n3d_isosurface_count(grid.data_ptr(), nz, ny, nx, level, ws.data_ptr(), counts.data_ptr(), stream),
                   'n3d_isosurface_count')
        V, F, nonfinite = counts.tolist()
        if nonfinite:
            raise ValueError(f'the grid has {nonfinite} non-finite voxels')
        if V >= INDEX_LIMIT or F >= INDEX_LIMIT:
            raise ValueError(f'the mesh has {V} vertices and {F} triangles: int32 indices stop at 2^31 - 1')
        if V == 0:
            return empty
        verts = torch.empty(V, 3, dtype=torch.float32, device=dev)
        faces = torch.empty(F, 3, dtype=torch.int32, device=dev)
        _lib.check(_lib.lib.n3d_isosurface_emit(grid.data_ptr(), nz, ny, nx, level, ws.data_ptr(), verts.data_ptr(),
                                                faces.data_ptr(), stream), 'n3d_isosurface_emit')
    return verts, faces


def ply_header(nverts, nfaces, colors=False):
    """The header plyfile writes for the reference's two elements (shape_utils.py:89-96); with `colors`, the vertex element also
    has uchar red, green and blue after z."""
    rgb = 'property uchar red\nproperty uchar green\nproperty uchar blue\n' if colors else ''
    return (f'ply\nformat binary_little_endian 1.0\nelement vertex {nverts}\nproperty float x\nproperty float y\nproperty float z\n'
            f'{rgb}element face {nfaces}\nproperty list uchar int vertex_indices\nend_header\n').encode('ascii')


def ply_bytes(verts, faces, colors=None):
    """Binary little-endian PLY file of verts float32 [V, 3] and faces int32 [F, 3] (tensors on any device, or numpy arrays):
    the header, V x 12 bytes of vertices, then F x 13 bytes of faces (the count byte 3 and three int32 indices).  The face
    records are packed where the faces are, and each array is read back once.  colors: uint8 [V, 3] vertex colours, written as
    uchar red, green, blue after each vertex's z (15-byte vertex records); None writes the plain file."""
    verts, faces = torch.as_tensor(verts), torch.as_tensor(faces)
    if verts.dtype != torch.float32 or verts.dim() != 2 or verts.shape[1] != 3:
        raise ValueError(f'verts must be float32 [V, 3], got {verts.dtype} {list(verts.shape)}')
    if faces.dtype != torch.int32 or faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError(f'faces must be int32 [F, 3], got {faces.dtype} {list(faces.shape)}')
    if faces.device != verts.device:
        raise ValueError(f'verts are on {verts.device}, faces on {faces.device}')
    count = torch.full((faces.shape[0], 1), 3, dtype=torch.uint8, device=faces.device)
    records = torch.cat([count, faces.reshape(-1).view(torch.uint8).reshape(-1, 12)], 1)          # [F, 13]
    if colors is None:
        vbytes = verts.contiguous().cpu().numpy().astype('<f4').tobytes()
    else:
        colors = torch.as_tensor(colors)
        if colors.dtype != torch.uint8 or tuple(colors.shape) != (verts.shape[0], 3):
            raise ValueError(f'colors must be uint8 [{verts.shape[0]}, 3], got {colors.dtype} {list(colors.shape)}')
        if colors.device != verts.device:
            raise ValueError(f'verts are on {verts.device}, colors on {colors.device}')
        vrec = torch.cat([verts.contiguous().reshape(-1).view(torch.uint8).reshape(-1, 12), colors], 1)   # [V, 15]
        vbytes = vrec.cpu().numpy().tobytes()
    return ply_header(verts.shape[0], faces.shape[0], colors is not None) + vbytes + records.cpu().numpy().tobytes()


def write_ply(path, verts, faces, colors=None):
    data = ply_bytes(verts, faces, colors)
    with open(path, 'wb') as f:
        f.write(data)
