"""numpy restatement of the marching-cubes mesh of next3d_b200.isosurface (DESIGN.md section 3.7): the triangle table derived
from the face rule, the classification, the vertex and triangle orders and the fp32 vertex positions.

Grid g[a0, a1, a2] of shape [nz, ny, nx]; output (x, y, z) = (a2, a1, a0) in voxel units.  A voxel is inside when g > level.
Cell corner k = dx + 2 dy + 4 dz (dx along a2, dy along a1, dz along a0).  Edges 0-3 run along x at (dy, dz) = (0,0), (1,0),
(0,1), (1,1); edges 4-7 along y at (dx, dz) in that order; edges 8-11 along z at (dx, dy) in that order."""
import numpy as np

# (corner a, corner b) of every cell edge, a the lower endpoint
EDGES = ([(2 * dy + 4 * dz, 2 * dy + 4 * dz + 1) for dz in (0, 1) for dy in (0, 1)]
         + [(dx + 4 * dz, dx + 4 * dz + 2) for dz in (0, 1) for dx in (0, 1)]
         + [(dx + 2 * dy, dx + 2 * dy + 4) for dy in (0, 1) for dx in (0, 1)])
AXIS = [0] * 4 + [1] * 4 + [2] * 4                       # 0 = x, 1 = y, 2 = z
MAX_TRIANGLES = 5


def corner_xyz(k):
    return np.array([k & 1, (k >> 1) & 1, (k >> 2) & 1], np.float64)


def _faces():
    """The six cube faces: (corners, outward normal)."""
    out = []
    for axis in range(3):
        for side in (0, 1):
            corners = [k for k in range(8) if (k >> axis) & 1 == side]
            n = np.zeros(3)
            n[axis] = 1.0 if side else -1.0
            out.append((corners, n))
    return out


FACES = _faces()


def _mid(e):
    a, b = EDGES[e]
    return (corner_xyz(a) + corner_xyz(b)) / 2


def face_segments(config, face):
    """Directed contour segments (edge, edge) of one face under the face rule: two crossed edges are joined; on a face with four
    (two inside corners on a diagonal) each inside corner is cut off on its own.  Each segment runs so that the inside corner of
    its first edge lies to its left seen from outside the cube: the right-hand normal of a loop then points from the inside
    corners to the outside ones."""
    corners, n = FACES[face]
    inside = [(config >> k) & 1 for k in range(8)]
    edges = [e for e, (a, b) in enumerate(EDGES) if a in corners and b in corners]
    crossed = [e for e in edges if inside[EDGES[e][0]] != inside[EDGES[e][1]]]
    if len(crossed) == 2:
        pairs = [tuple(crossed)]
    elif len(crossed) == 4:
        pairs = [tuple(e for e in crossed if k in EDGES[e]) for k in corners if inside[k]]
    else:
        assert not crossed
        pairs = []
    out = []
    for ea, eb in pairs:
        q = next(k for k in EDGES[ea] if inside[k])
        pa, d = _mid(ea), _mid(eb) - _mid(ea)
        side = np.dot(np.cross(corner_xyz(q) - pa, d), n)
        assert side != 0
        out.append((ea, eb) if side > 0 else (eb, ea))
    return out


def cell_loops(config):
    """Closed contour loops of a configuration, each starting at its smallest edge, in order of that edge."""
    nxt = {}
    for f in range(6):
        for a, b in face_segments(config, f):
            assert a not in nxt, (config, a)
            nxt[a] = b
    assert sorted(nxt) == sorted(nxt.values())
    loops, seen = [], set()
    for e in sorted(nxt):
        if e in seen:
            continue
        loop = [e]
        while nxt[loop[-1]] != e:
            loop.append(nxt[loop[-1]])
        seen.update(loop)
        loops.append(loop)
    return loops


FACE_EDGES = [{e for e, (a, b) in enumerate(EDGES) if a in c and b in c} for c, _ in FACES]


def fan_start(loop):
    """Index in `loop` of the vertex its fan starts from: the first (from the smallest edge, in loop order) whose diagonals join
    no two edges of one cube face.  Such a diagonal lies on an ambiguous face that the loop crosses twice, and the cell across
    that face may fan the same diagonal: the edge would then belong to four triangles."""
    n = len(loop)
    for r in range(n):
        v0 = loop[r]
        if not any(v0 in f and loop[(r + i) % n] in f for f in FACE_EDGES for i in range(2, n - 1)):
            return r
    raise AssertionError(loop)


def derive_table():
    """[256] lists of triangles (edge, edge, edge): each loop, rotated to start at fan_start, fanned as (v0, vi, vi+1)."""
    table = []
    for config in range(256):
        tris = []
        for lp in cell_loops(config):
            r = fan_start(lp)
            lp = lp[r:] + lp[:r]
            tris += [(lp[0], lp[i], lp[i + 1]) for i in range(1, len(lp) - 1)]
        table.append(tris)
    assert max(len(t) for t in table) == MAX_TRIANGLES
    return table


TABLE = derive_table()
NTRI = np.array([len(t) for t in TABLE], np.int64)
TRI = np.full((256, MAX_TRIANGLES, 3), -1, np.int64)
for _c, _t in enumerate(TABLE):
    if _t:
        TRI[_c, :len(_t)] = _t


def _edge_flags(inside):
    """[nz, ny, nx, 3] bool: the voxel's x-, y- and z-edge (toward +a2, +a1, +a0) crosses the surface."""
    f = np.zeros(inside.shape + (3,), bool)
    f[:, :, :-1, 0] = inside[:, :, :-1] != inside[:, :, 1:]
    f[:, :-1, :, 1] = inside[:, :-1, :] != inside[:, 1:, :]
    f[:-1, :, :, 2] = inside[:-1] != inside[1:]
    return f


def counts(g, level=10.0):
    """(vertices, triangles, non-finite voxels) of the mesh of g."""
    v, f = marching_cubes(g, level)
    return len(v), len(f), int((~np.isfinite(g)).sum())


def marching_cubes(g, level=10.0):
    """g float32 [nz, ny, nx] -> (verts float32 [V, 3], faces int32 [F, 3]) in the orders of DESIGN.md section 3.7."""
    g = np.ascontiguousarray(g, np.float32)
    assert g.ndim == 3
    lv = np.float32(level)
    nz, ny, nx = g.shape
    if min(g.shape) < 2:
        return np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32)
    inside = g > lv
    flags = _edge_flags(inside)
    ids = np.cumsum(flags.reshape(-1)).reshape(flags.shape) - 1            # vertex id of every crossed (voxel, axis)
    a0, a1, a2, ax = np.nonzero(flags)                                     # ascending (a0, a1, a2), then x, y, z
    s0 = g[a0, a1, a2]
    s1 = g[a0 + (ax == 2), a1 + (ax == 1), a2 + (ax == 0)]
    with np.errstate(divide='ignore', invalid='ignore'):
        t = (lv - s0) / (s1 - s0)
    verts = np.stack([a2, a1, a0], 1).astype(np.float32)
    rows = np.arange(len(ax))
    verts[rows, ax] = verts[rows, ax] + t.astype(np.float32)

    ins = inside.astype(np.int64)
    config = np.zeros((nz - 1, ny - 1, nx - 1), np.int64)
    for k in range(8):
        dx, dy, dz = k & 1, (k >> 1) & 1, (k >> 2) & 1
        config |= ins[dz:nz - 1 + dz, dy:ny - 1 + dy, dx:nx - 1 + dx] << k
    c0, c1, c2 = np.nonzero(NTRI[config] > 0)
    cfg = config[c0, c1, c2]
    # vertex id of each of the 12 edges of the active cells: the edge's lower endpoint and axis
    eid = np.empty((len(cfg), 12), np.int64)
    for e, (a, _) in enumerate(EDGES):
        dx, dy, dz = a & 1, (a >> 1) & 1, (a >> 2) & 1
        eid[:, e] = ids[c0 + dz, c1 + dy, c2 + dx, AXIS[e]]
    tri = TRI[cfg]                                                         # [C, 5, 3] edge numbers
    vid = np.take_along_axis(eid[:, None, :].repeat(MAX_TRIANGLES, 1), np.maximum(tri, 0), 2)
    faces = vid[np.arange(MAX_TRIANGLES)[None, :] < NTRI[cfg][:, None]]
    return verts, faces.astype(np.int32)


# ------------------------------------------------------------------------------------------------ mesh properties for the tests
def euler(verts, faces):
    e = {tuple(sorted(p)) for f in faces.tolist() for p in ((f[0], f[1]), (f[1], f[2]), (f[2], f[0]))}
    return len(verts) - len(e) + len(faces)


def directed_edges_closed(faces):
    """True when every undirected edge is in exactly two triangles, once in each direction."""
    f = faces.astype(np.int64)
    d = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    key = d[:, 0] * (1 << 32) + d[:, 1]
    if len(np.unique(key)) != len(key):
        return False
    rev = d[:, 1] * (1 << 32) + d[:, 0]
    return bool(np.isin(rev, key).all())


def components(nverts, faces):
    parent = np.arange(nverts)

    def find(i):
        while parent[i] != i:
            parent[i] = parent[parent[i]]
            i = parent[i]
        return i
    for a, b, c in faces.tolist():
        for u, w in ((a, b), (b, c)):
            ru, rw = find(u), find(w)
            if ru != rw:
                parent[ru] = rw
    return len({find(i) for i in np.unique(faces)})


def area_volume(verts, faces):
    p = verts.astype(np.float64)[faces]
    cr = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    return 0.5 * np.linalg.norm(cr, axis=1).sum(), np.einsum('ij,ij->i', p[:, 0], np.cross(p[:, 1], p[:, 2])).sum() / 6
