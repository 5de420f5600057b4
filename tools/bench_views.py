"""Time new camera views of a cached head against full synthesis on the C2 shapes (batch 8, 64^2 neural render, 48 + 48 samples,
512^2 output; random weights from weights.make_state_dict).  python tools/bench_views.py [--tiny]

Per frame, CUDA-graph replay, alternated in rounds:
  synthesis          G.synthesis on 8 heads
  use_cached         G.synthesis(use_cached_backbone=True) on the same 8 heads (cache of batch 8): everything but the two ws-only backbones
  render_views       G.render_views of 8 cameras of one cached head (B = 1, V = 8): volume rendering + super-resolution only
and n3d_render_rays with views = 8 on one plane set against views = 1 on eight copies of it.  Then one eager call of synthesis and of
render_views with the engine's per-launch profile, which says where the time of each goes (conv = every convolution, i.e. the
backbones, StyleUNets and super-resolution; render = the fused renderer)."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from next3d_b200 import config, kernels as K, weights
from next3d_b200.triplane_next3d import TriPlaneGenerator


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader', '-i',
                        str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    print(f'card {torch.cuda.get_device_name()}  (name, power limit, SM clock, max SM clock): {q or "unknown"}', flush=True)


def timed(fn, reps):
    """Median and minimum ms of `reps` calls, each between CUDA events and followed by a synchronise."""
    ts = []
    for i in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn(i)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def main():
    tiny = '--tiny' in sys.argv
    base = config.tiny_config(512) if tiny else config.full_config(512)
    rk = dict(base.rendering_kwargs, depth_resolution=48, depth_resolution_importance=48)
    import dataclasses
    cfg = dataclasses.replace(base, neural_rendering_resolution=64, rendering_kwargs=rk)
    card()
    print(f'config {"tiny" if tiny else "full"}: batch 8, {cfg.neural_rendering_resolution}^2 neural render, 48 + 48 samples, '
          f'{cfg.img_resolution}^2 output', flush=True)
    G = TriPlaneGenerator.from_config(cfg, weights.make_state_dict(cfg, seed=0), device='cuda')
    G.use_cuda_graph = True
    B = 8
    z, c_cond, c, v = weights.demo_inputs(cfg, B, seed=0)
    ws = G.mapping(z.cuda(), c_cond.cuda(), truncation_psi=0.7, truncation_cutoff=14)
    c, v = c.cuda(), v.cuda()

    # each variant: (set-up run before its block, untimed: fills the cache it reads), timed call
    variants = {
        'synthesis': (None, lambda i: G.synthesis(ws, c, v, noise_mode='const', seed=i)),
        'use_cached': (lambda: G.synthesis(ws, c, v, noise_mode='const', seed=0, cache_backbone=True),
                       lambda i: G.synthesis(ws, c, v, noise_mode='const', seed=i, use_cached_backbone=True)),
        'render_views': (lambda: G.synthesis(ws[:1], c[:1], v[:1], noise_mode='const', seed=0, cache_backbone=True),
                         lambda i: G.render_views(c, seed=i)),
    }
    med = {k: [] for k in variants}
    for rnd in range(3):
        for name, (setup, fn) in variants.items():
            if setup is not None:
                setup()
            fn(0); fn(1)                                    # capture (the cache's batch size changed) + warm replay
            torch.cuda.synchronize()
            med[name].append(timed(fn, 20)[0])
    full = min(med['synthesis']) / B
    for name in variants:
        per = min(med[name]) / B
        print(f'{name:13s} per frame: {per:.3f} ms (block medians {" / ".join(f"{m / B:.3f}" for m in med[name])}), '
              f'{per / full * 100:.1f} % of synthesis', flush=True)

    # the renderer alone: one plane set seen from 8 cameras, against 8 copies of it
    eng = G._get_engine()
    R = cfg.neural_rendering_resolution
    g = torch.Generator().manual_seed(0)
    one = torch.randn(1, 3, 256, 256, cfg.plane_ch, generator=g).cuda() * 0.5
    eight = one.repeat(B, 1, 1, 1, 1)
    cam, intr = c[:, :16].contiguous(), c[:, 16:25].contiguous()
    rgb = torch.empty(B, R * R, 32, device='cuda'); depth = torch.empty(B, R * R, device='cuda'); wsum = torch.empty_like(depth)
    mm = torch.tensor([float('inf'), 0.0], device='cuda')
    rays = {'views=8, 1 set': lambda i: K.render_rays(one, cam, intr, R, rk, eng.dec, rgb, depth, wsum, mm, seed=i, views=B),
            'views=1, 8 sets': lambda i: K.render_rays(eight, cam, intr, R, rk, eng.dec, rgb, depth, wsum, mm, seed=i)}
    rmed = {k: [] for k in rays}
    for f in rays.values():
        f(0); f(1)
    for rnd in range(3):
        for name, f in rays.items():
            rmed[name].append(timed(f, 30)[0])
    for name in rays:
        print(f'n3d_render_rays {name:16s}: {min(rmed[name]):.3f} ms per 8 images (block medians '
              f'{" / ".join(f"{m:.3f}" for m in rmed[name])})', flush=True)

    # where the time goes: one eager call each with the per-launch profile
    G.use_cuda_graph = False
    for name, fn in (('synthesis', lambda: G.synthesis(ws, c, v, noise_mode='const', seed=1)),
                     ('render_views', lambda: G.render_views(c, seed=1))):
        fn()
        eng.prof = []
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        summary = eng.profile_summary()
        eng.prof = None
        parts = ', '.join(f'{kind} {n} launches {ms:.2f} ms' for kind, (n, ms, _) in sorted(summary.items()))
        print(f'eager {name}: {e0.elapsed_time(e1):.2f} ms for 8 images, {eng.launches} launches; {parts}', flush=True)


if __name__ == '__main__':
    main()
