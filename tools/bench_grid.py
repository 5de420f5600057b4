"""Frames/s of the grid video drivers against separate single-identity passes, on the C4 shapes (full FFHQ-512 widths, random weights
from weights.make_state_dict, 64^2 neural render, 96 + 96 samples per ray, 512^2 output, CUDA-graph replay).
python tools/bench_grid.py [--tiny]

  reenact   drivers.reenact_grid_frames: S = 3 identities + the driving photo in a 2x2 grid, 3 heads x 8 frames per call, heads
            cached once -- against three drivers.reenact_frames passes (batch 8), one per identity, over the same driving directory
            (a synthetic one written to a temporary directory: the demo mesh with jitter, 512^2 PNG photos, dataset.json).
  interp    drivers.render_grid_frames: a 2x2 interpolation grid (8 seeds, 2 keyframes per cell), batch 8 -- against four
            drivers.render_frames passes (batch 8), one per cell, with the same latents, cameras and mesh.
A rate is grid frames per second of host wall time around the whole clip (every frame read back to the host); for the separate
passes, the grid's frame count over the summed time of the passes.  Each variant has its own generator (same weights): the backbone
cache of a generator holds one batch size, and a caching call with another one drops the graphs that use the cache, so variants
sharing a generator would re-capture inside their timed rounds.  Each variant runs once untimed (graph capture), then the variants
alternate for three rounds and the best round counts; a timed round that captures a graph aborts the run."""
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from next3d_b200 import config, drivers, weights
from next3d_b200.triplane_next3d import TriPlaneGenerator


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader', '-i',
                        str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    print(f'card {torch.cuda.get_device_name()}  (name, power limit, SM clock, max SM clock): {q or "unknown"}', flush=True)


def drive_root(path, v, c, n):
    from PIL import Image
    rng = np.random.RandomState(0)
    labels = []
    for k in range(n):
        name = f'{k:04d}'
        Image.fromarray(rng.randint(0, 256, (512, 512, 3), dtype=np.uint8)).save(os.path.join(path, f'{name}.png'))
        vk = v + rng.randn(*v.shape).astype(np.float32) * 1e-4
        with open(os.path.join(path, f'{name}.obj'), 'w') as f:
            f.write(''.join(f'v {a!r} {b!r} {c_!r}\n' for a, b, c_ in vk[:5023].tolist()))
        with open(os.path.join(path, f'{name}_kpt2d.txt'), 'w') as f:
            f.write('\n'.join(f'{a!r} {b!r} {c_!r}' for a, b, c_ in vk[5023:].tolist()) + '\n')
        cam = c.astype(np.float64)
        cam[3] += 0.002 * k
        labels.append([f'{name}.png', cam.tolist()])
    with open(os.path.join(path, 'dataset.json'), 'w') as f:
        json.dump({'labels': labels}, f)


def clock(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = fn()
    torch.cuda.synchronize()
    return n, time.perf_counter() - t0


def graphs(G):
    """The captured graphs of G's engine by key (a snapshot: holding it keeps the entries alive, so identity comparisons hold)."""
    return dict(G._get_engine()._graphs)


def same_graphs(a, b):
    return a.keys() == b.keys() and all(a[k] is b[k] for k in a)


def compare(title, variants):
    """variants: {name: (generator, fn() -> grid frames produced)}; returns {name: best frames/s}."""
    for _, fn in variants.values():
        fn()
    best = {k: 0.0 for k in variants}
    for _ in range(3):
        for name, (G, fn) in variants.items():
            before = graphs(G)
            n, t = clock(fn)
            if not same_graphs(before, graphs(G)):
                raise RuntimeError(f'{title} {name}: a CUDA graph was captured inside a timed round')
            best[name] = max(best[name], n / t)
    base = list(variants)[1]
    for name in variants:
        print(f'{title} {name:18s}: {best[name]:8.2f} frames/s ({best[name] / best[base]:.2f}x of {base})', flush=True)
    return best


def main():
    tiny = '--tiny' in sys.argv
    import dataclasses
    base = config.tiny_config(512) if tiny else config.full_config(512)
    rk = dict(base.rendering_kwargs, depth_resolution=96, depth_resolution_importance=96)
    cfg = dataclasses.replace(base, neural_rendering_resolution=64, rendering_kwargs=rk)
    card()
    print(f'config {"tiny" if tiny else "full"}: {cfg.neural_rendering_resolution}^2 neural render, 96 + 96 samples, '
          f'{cfg.img_resolution}^2 output, CUDA graphs', flush=True)
    sd = weights.make_state_dict(cfg, seed=0)
    G, Gs = (TriPlaneGenerator.from_config(cfg, sd, device='cuda') for _ in range(2))         # grid drivers / separate passes
    G.use_cuda_graph = Gs.use_cuda_graph = True
    z, c_cond, c, v = weights.demo_inputs(cfg, 3, seed=0)
    ws = G.mapping(z.cuda(), c_cond.cuda(), truncation_psi=0.7, truncation_cutoff=14)

    with tempfile.TemporaryDirectory() as tmp:
        drive_root(tmp, v[0].numpy(), c[0].numpy(), 50)                    # 48 frames (the schedule drops the first and last)

        def grid():
            return sum(1 for _ in drivers.reenact_grid_frames(G, ws, tmp, 1000, (2, 2), batch=24, seed=1))

        def separate():
            n = [sum(1 for _ in drivers.reenact_frames(Gs, ws[s:s + 1], tmp, 1000, batch=8, seed=1)) for s in range(3)]
            return n[0]
        compare('reenact S=3 2x2', {'reenact_grid': (G, grid), '3x reenact_frames': (Gs, separate)})

    ws_grid = drivers.grid_keyframes(G, list(range(8)), (2, 2), truncation_psi=0.7)
    w_frames = 24
    vs = v[:1]
    rk_ = G.rendering_kwargs
    F = ws_grid.shape[2] * w_frames
    cams = drivers.orbit_camera_params(F, torch.tensor(rk_['avg_camera_pivot']), rk_['avg_camera_radius'])
    cell_ws = [drivers.interpolate_ws_device(ws_grid[yi, xi], w_frames) for yi in range(2) for xi in range(2)]

    def igrid():
        return sum(1 for _ in drivers.render_grid_frames(G, ws_grid, vs, w_frames, batch=8, seed=1))

    def iseparate():
        n = [sum(1 for _ in drivers.render_frames(Gs, w, cams, vs, batch=8, seed=1)) for w in cell_ws]
        return n[0]
    compare('interp 2x2', {'render_grid_frames': (G, igrid), '4x render_frames': (Gs, iseparate)})


if __name__ == '__main__':
    main()
