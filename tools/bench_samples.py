"""Seeds/s of the sample-sheet drivers against the script's own loop, on the full FFHQ-512 widths (random weights from
weights.make_state_dict, the default 64^2 neural render and 48 + 48 samples per ray, 512^2 output, CUDA-graph replay), S = 16 seeds,
one mesh, three yaws per sheet and a density grid per seed at shape_res 256 and 512.
python tools/bench_samples.py [--tiny] [--seeds S]

  script    gen_samples_next3d.py:182-238 restated: per seed, three synthesis calls (one per yaw, the sheet read back with .cpu())
            and drivers.extract_sigma_grid (the planes computed again, one grid launch, read back).
  driver    drivers.render_sample_sheets, batch 9 (3 heads per call): one caching synthesis call and one render_views call per 3
            heads, each grid decoded from the cached planes, read-back overlapped with the next call.
  sharded   drivers.render_sample_sheets_sharded at world size 1 (sheets gathered into one pinned host tensor).
A rate is seeds per second of host wall time around the whole run, every sheet and grid on the host at the end.  Each variant has its
own generator (same weights), so that no variant evicts another's cached graphs; each runs once untimed (graph capture), then the
variants alternate for three rounds and the best round counts; a timed round that captures a graph aborts the run."""
import dataclasses
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch

from bench_grid import card, clock, graphs, same_graphs
from next3d_b200 import config, drivers, weights
from next3d_b200.triplane_next3d import TriPlaneGenerator


def script_loop(G, ws, v, shape_res):
    """One seed at a time, as the script: three full synthesis calls, then the shape from freshly computed planes."""
    cams = drivers.sample_sheet_cameras(G)[0].cuda()
    for i in range(ws.shape[0]):
        imgs = [(G.synthesis(ws[i:i + 1], cams[j:j + 1], v, noise_mode='const', seed=1)['image'].permute(0, 2, 3, 1) * 127.5 + 128)
                .clamp(0, 255).to(torch.uint8) for j in range(3)]
        torch.cat(imgs, dim=2)[0].cpu().numpy()
        drivers.extract_sigma_grid(G, ws[i:i + 1], v, shape_res)
    return ws.shape[0]


def driver(G, ws, v, shape_res):
    return sum(1 for _ in drivers.render_sample_sheets(G, ws, v, batch=9, shapes=True, shape_res=shape_res, seed=1))


def sharded(G, ws, v, shape_res):
    sheets, grids = drivers.render_sample_sheets_sharded(G, ws, v, batch=9, shapes=True, shape_res=shape_res, seed=1)
    torch.cuda.current_stream().synchronize()
    return len(grids)


def main():
    tiny = '--tiny' in sys.argv
    S = int(sys.argv[sys.argv.index('--seeds') + 1]) if '--seeds' in sys.argv else 16
    cfg = config.tiny_config(512) if tiny else config.full_config(512)
    card()
    print(f'config {"tiny" if tiny else "full"}: {cfg.neural_rendering_resolution}^2 neural render, '
          f'{cfg.rendering_kwargs["depth_resolution"]} + {cfg.rendering_kwargs["depth_resolution_importance"]} samples, '
          f'{cfg.img_resolution}^2 output, CUDA graphs, S = {S} seeds', flush=True)
    sd = weights.make_state_dict(cfg, seed=0)
    variants = {'script': script_loop, 'driver': driver, 'sharded': sharded}
    gens = {name: TriPlaneGenerator.from_config(cfg, sd, device='cuda') for name in variants}
    for G in gens.values():
        G.use_cuda_graph = True
    v = weights.demo_inputs(cfg, 1, seed=0)[3].cuda()
    ws = drivers.sample_sheet_ws(gens['driver'], list(range(S)), truncation_psi=0.7)
    for shape_res in (256, 512):
        for name, fn in variants.items():
            fn(gens[name], ws, v, shape_res)
        best = {k: 0.0 for k in variants}
        for _ in range(3):
            for name, fn in variants.items():
                before = graphs(gens[name])
                n, t = clock(lambda: fn(gens[name], ws, v, shape_res))
                if not same_graphs(before, graphs(gens[name])):
                    raise RuntimeError(f'{name}: a CUDA graph was captured inside a timed round')
                assert n == S, (name, n)
                best[name] = max(best[name], n / t)
        for name in variants:
            print(f'shape_res {shape_res} {name:8s}: {best[name]:7.2f} seeds/s ({best[name] / best["script"]:.2f}x of script)', flush=True)
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
