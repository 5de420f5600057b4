"""numpy restatement of the vertex-colour bake of next3d_b200.bake (DESIGN.md section 3.8): the voxel -> world map of the shape
grid, the renderer's projection, the mesh z-buffer, the outward normal and the per-vertex blend, in float32 operations that round
as the kernels' (each product, sum and quotient rounded on its own, no fused multiply-add), so that the kernels match bit for bit.

Cameras are camera_params rows [views, 25] (cam2world 16, intrinsics 9).  Vertices are (x, y, z) = (a2, a1, a0) in voxel units of
the flipped grid g[a0, a1, a2]."""
import numpy as np

F = np.float32
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


def world_points(verts, R, cube):
    """s2 = x, s1 = y + x / R, s0 = (R - 1 - z) + s1 / R; p = s * cube / (R - 1) - cube / 2 (create_samples' float division)."""
    v = np.asarray(verts, F)
    inv, vs, h = F(1) / F(R), F(cube) / F(R - 1), F(cube) * F(0.5)
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    s1 = y + x * inv
    s0 = (F(R - 1) - z) + s1 * inv
    return np.stack([s0 * vs - h, s1 * vs - h, x * vs - h], 1).astype(F)


def project(cam, p, H, W):
    """(u, w, z) of world points p [P, 3] in the view cam [25]: camera depth z and pixel coordinates with centres at integers."""
    C = np.asarray(cam[:16], F).reshape(4, 4)
    I = np.asarray(cam[16:], F)
    d = [p[:, a] - C[a, 3] for a in range(3)]
    q = [(C[0, j] * d[0] + C[1, j] * d[1]) + C[2, j] * d[2] for j in range(3)]
    with np.errstate(divide='ignore', invalid='ignore'):
        xl, yl = q[0] / q[2], q[1] / q[2]
    xc = (I[0] * xl + I[1] * yl) + I[2]
    yc = I[4] * yl + I[5]
    return xc * F(W) - F(0.5), yc * F(H) - F(0.5), q[2]


def _edge(ua, wa, ub, wb, px, py):
    return (ub - ua) * (py - wa) - (wb - wa) * (px - ua)


def zbuffer(verts, faces, cams, H, W, near=0.01):
    """uint64 [views, H, W]: per pixel the least (depth bits << 32) | triangle id over the triangles covering its centre (edges
    included), EMPTY where none does; triangles with a vertex at z <= near, an index outside the vertices, zero area or non-finite
    corners are skipped."""
    verts = np.asarray(verts, F)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    out = np.full((len(cams), H, W), EMPTY, np.uint64)
    near = F(near)
    for v, cam in enumerate(cams):
        u, w, z = project(cam, verts, H, W)
        with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
            iz = F(1) / z
            zb = out[v]
            for f, tri in enumerate(faces):
                if (tri < 0).any() or (tri >= len(verts)).any():
                    continue
                tu, tw, tz = u[tri], w[tri], z[tri]
                if not (tz > near).all() or not np.isfinite(tu).all() or not np.isfinite(tw).all():
                    continue
                area = (tu[1] - tu[0]) * (tw[2] - tw[0]) - (tw[1] - tw[0]) * (tu[2] - tu[0])
                if not (area != 0) or not np.isfinite(area):
                    continue
                c0 = int(min(max(np.ceil(tu.min()), F(0)), F(W)))
                c1 = int(min(max(np.floor(tu.max()), F(-1)), F(W - 1)))
                r0 = int(min(max(np.ceil(tw.min()), F(0)), F(H)))
                r1 = int(min(max(np.floor(tw.max()), F(-1)), F(H - 1)))
                if c0 > c1 or r0 > r1:
                    continue
                py, px = np.meshgrid(np.arange(r0, r1 + 1, dtype=F), np.arange(c0, c1 + 1, dtype=F), indexing='ij')
                e = [_edge(tu[1], tw[1], tu[2], tw[2], px, py), _edge(tu[2], tw[2], tu[0], tw[0], px, py),
                     _edge(tu[0], tw[0], tu[1], tw[1], px, py)]
                a = area
                if a < 0:
                    e, a = [-x for x in e], -a
                inside = (e[0] >= 0) & (e[1] >= 0) & (e[2] >= 0)
                if not inside.any():
                    continue
                izp = ((e[0] / a) * iz[tri[0]] + (e[1] / a) * iz[tri[1]]) + (e[2] / a) * iz[tri[2]]
                depth = (F(1) / izp).astype(F)
                key = (depth.view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.uint64(f)
                rr, cc = py[inside].astype(np.int64), px[inside].astype(np.int64)
                zb[rr, cc] = np.minimum(zb[rr, cc], key[inside])
    return out


def zbuffer_depth(zb):
    """Camera depth float32 of every pixel of a z-buffer, inf where empty."""
    d = (zb >> np.uint64(32)).astype(np.uint32).view(F)
    return np.where(zb == EMPTY, F(np.inf), d).astype(F)


def _lerp(a, b, t):
    return a + (b - a) * t


def normals(verts, grid):
    """Unit outward normals [V, 3] in world space: the trilinear interpolation (along x, then y, then z) of the grid's central
    differences at the nodes (neighbours clamped), taken through the inverse transpose of the voxel -> world map; 0 where the
    gradient vanishes."""
    g = np.asarray(grid, F)
    R = g.shape[0]
    v = np.asarray(verts, F)

    def cell(c):
        i = np.clip(np.floor(c), 0, R - 2).astype(np.int64)
        return i, c - i.astype(F)

    i2, fx = cell(v[:, 0])
    i1, fy = cell(v[:, 1])
    i0, fz = cell(v[:, 2])

    def node(a0, a1, a2):
        h = F(0.5)
        return [(g[a0, a1, np.minimum(a2 + 1, R - 1)] - g[a0, a1, np.maximum(a2 - 1, 0)]) * h,
                (g[a0, np.minimum(a1 + 1, R - 1), a2] - g[a0, np.maximum(a1 - 1, 0), a2]) * h,
                (g[np.minimum(a0 + 1, R - 1), a1, a2] - g[np.maximum(a0 - 1, 0), a1, a2]) * h]

    gz = []
    for dz in (0, 1):
        gy = []
        for dy in (0, 1):
            g0, g1 = node(i0 + dz, i1 + dy, i2), node(i0 + dz, i1 + dy, i2 + 1)
            gy.append([_lerp(g0[k], g1[k], fx) for k in range(3)])
        gz.append([_lerp(gy[0][k], gy[1][k], fy) for k in range(3)])
    gv = [_lerp(gz[0][k], gz[1][k], fz) for k in range(3)]
    inv = F(1) / F(R)
    n = [gv[2], -(gv[1] + gv[2] * inv), gv[1] * inv - gv[0]]
    ln = np.sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2]).astype(F)
    with np.errstate(divide='ignore', invalid='ignore'):
        out = np.stack([np.where(ln > 0, x / ln, F(0)) for x in n], 1)
    return out.astype(F)


def bake(verts, world, grid, cams, images, zb, fallback, near=0.01, eps=None, cube=1.0):
    """(colors uint8 [V, 3], visible bool [views, V], weights float32 [views, V]) of n3d_bake_vertex_colors.  images float32
    [views, 3, H, W]; zb the z-buffer; fallback [V, >= 3] the decoder's colour (sigmoid range), used as 2 f - 1 where no view
    sees a vertex; eps defaults to two voxels of the grid."""
    verts, world, images = np.asarray(verts, F), np.asarray(world, F), np.asarray(images, F)
    V = len(verts)
    R = np.asarray(grid).shape[0]
    H, W = images.shape[2:]
    eps = F(2 * cube / (R - 1)) if eps is None else F(eps)
    n = normals(verts, grid)
    depth = zbuffer_depth(zb)
    sw = np.zeros(V, F)
    sc = np.zeros((V, 3), F)
    vis_all = np.zeros((len(cams), V), bool)
    w_all = np.zeros((len(cams), V), F)
    for v, cam in enumerate(cams):
        C = np.asarray(cam[:16], F).reshape(4, 4)
        u, w, z = project(cam, world, H, W)
        with np.errstate(invalid='ignore'):
            cr, cc = np.floor(w + F(0.5)), np.floor(u + F(0.5))
            ok = (z > F(near)) & (cr >= 0) & (cr < H) & (cc >= 0) & (cc < W)
        ri, ci = np.where(ok, cr, 0).astype(np.int64), np.where(ok, cc, 0).astype(np.int64)
        vis = ok & (z <= depth[v, ri, ci] + eps)
        e = [C[a, 3] - world[:, a] for a in range(3)]
        dl = np.sqrt((e[0] * e[0] + e[1] * e[1]) + e[2] * e[2]).astype(F)
        cos = np.maximum(((n[:, 0] * e[0] + n[:, 1] * e[1]) + n[:, 2] * e[2]) / dl, F(0))
        wt = np.where(vis, cos * cos, F(0)).astype(F)
        vis_all[v], w_all[v] = vis, wt
        use = wt > 0
        u0, w0 = np.floor(u), np.floor(w)
        tu, tw = u - u0, w - w0
        u0i, w0i = np.where(use, u0, 0).astype(np.int64), np.where(use, w0, 0).astype(np.int64)
        ca, cb = np.clip(u0i, 0, W - 1), np.clip(u0i + 1, 0, W - 1)
        ra, rb = np.clip(w0i, 0, H - 1), np.clip(w0i + 1, 0, H - 1)
        sw = np.where(use, sw + wt, sw)
        for k in range(3):
            im = images[v, k]
            top = _lerp(im[ra, ca], im[ra, cb], tu)
            bot = _lerp(im[rb, ca], im[rb, cb], tu)
            sc[:, k] = np.where(use, sc[:, k] + wt * _lerp(top, bot, tw), sc[:, k])
    fb = np.asarray(fallback, F)[:, :3] * F(2) - F(1)                   # the decoder's colour, rescaled as image_raw is
    with np.errstate(divide='ignore', invalid='ignore'):
        c = np.where((sw > 0)[:, None], sc / sw[:, None], fb).astype(F)
    colors = np.clip(c * F(127.5) + F(128), 0, 255).astype(np.uint8)
    return colors, vis_all, w_all


def camera(horizontal, vertical, radius=2.7, fov_deg=18.837, lookat=(0.0, 0.0, 0.0)):
    """camera_params [25] float32 of next3d_b200.camera.look_at_pose and fov_to_intrinsics (the renderer's convention)."""
    import torch
    from next3d_b200 import camera as cam
    pose = cam.look_at_pose(horizontal, vertical, torch.tensor(lookat, dtype=torch.float32), radius).reshape(16)
    return torch.cat([pose, cam.fov_to_intrinsics(fov_deg).reshape(9)]).numpy().astype(F)
