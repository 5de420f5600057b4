"""Per-head time of a coloured mesh (drivers.coloured_meshes) at shape_res 512 on a seeded full-width generator, split into its
steps: the caching synthesis and render_views of the bake views, the density grid from the cached planes, marching cubes, the
world points and decoder colours, the z-buffer, the bake and the PLY write (device events around each step, after a warm-up
head).  Also the triangle count and the z-buffer fill rate (covered pixels over all views).  The level is the 0.7 quantile of the
densities inside the border, which cuts the random-weight head.  Prints the card name and power limit of the run, then one JSON
line.

    python tools/bench_bake.py [--res 512] [--iters 3]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--res', type=int, default=512)
    ap.add_argument('--iters', type=int, default=3)
    args = ap.parse_args()
    from next3d_b200 import bake, config, drivers, isosurface, weights
    from next3d_b200.triplane_next3d import TriPlaneGenerator
    print(card())
    cfg = config.full_config(512)
    G = TriPlaneGenerator.from_config(cfg, weights.make_state_dict(cfg, seed=0), device='cuda')
    _, _, _, v = weights.demo_inputs(cfg, 1, seed=0)
    v = v.cuda()
    ws = drivers.sample_sheet_ws(G, [0], 0.7)
    eng = G._get_engine()
    cams = drivers.bake_cameras(G).cuda()
    n = cams.shape[0]
    res = args.res
    grid = torch.empty(res, res, res, device='cuda')
    box = G.rendering_kwargs['box_warp']
    G.synthesis(ws, cams[:1], v, noise_mode='const', cache_backbone=True, seed=0)
    eng.cached_sigma_grid(0, res, grid)
    inner = grid[grid > -1000]
    level = float(torch.quantile(inner[::max(1, inner.numel() // 4000000)], 0.7))
    times = {}
    out_dir = tempfile.mkdtemp()
    for it in range(args.iters + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(9)]
        ev[0].record()
        front = G.synthesis(ws, cams[:1], v, noise_mode='const', cache_backbone=True, seed=0)['image']
        more = G.render_views(cams[1:], seed=1)['image']
        images = torch.cat([front, more])
        ev[1].record()
        eng.cached_sigma_grid(0, res, grid)
        ev[2].record()
        verts, faces = isosurface.marching_cubes(grid, level)
        ev[3].record()
        world = bake.world_points(verts, res, box)
        _, feat = eng.cached_sample_points(0, world)
        ev[4].record()
        zb = bake.mesh_zbuffer(world, faces, cams, images.shape[2], images.shape[3])
        ev[5].record()
        colors = bake.bake_vertex_colors(verts, world, grid, cams, images, zb, feat, box)
        ev[6].record()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        isosurface.write_ply(os.path.join(out_dir, 'head.ply'), verts, faces, colors)
        t_ply = (time.perf_counter() - t0) * 1e3
        if it == 0:
            continue                                                                   # warm-up head
        for k, name in enumerate(['views', 'grid', 'mesh', 'world_and_fallback', 'zbuffer', 'bake']):
            times.setdefault(name, []).append(ev[k].elapsed_time(ev[k + 1]))
        times.setdefault('ply_write', []).append(t_ply)
    fill = float((zb != bake.EMPTY).float().mean())
    result = {'bench': 'bake', 'card': card(), 'shape_res': res, 'views': n, 'image': list(images.shape[2:]), 'level': level,
              'vertices': int(verts.shape[0]), 'triangles': int(faces.shape[0]), 'zbuffer_fill': round(fill, 4),
              'ms': {k: round(float(np.median(t)), 3) for k, t in times.items()}}
    result['ms']['total'] = round(sum(result['ms'].values()), 3)
    print(json.dumps(result))


if __name__ == '__main__':
    main()
