"""Time the sharded video drivers and the renderer's per-image depth range.  python tools/bench_sharded.py [--tiny] [--frames F]

C4 shapes (full FFHQ-512 widths, random weights from weights.make_state_dict, 64^2 neural render, 96 + 96 samples, 512^2 output,
batch 8), CUDA-graph replay, one head driven by F synthetic frames read from a memory-mapped .n3dpack in a temporary directory:
  reenact_frames           the single-GPU driver (backbones cached on the first batch)
  reenact_frames_sharded   the sharded driver at world size 1 (same work + the staging / gather loop)
  render_orbit_sharded     F orbit cameras of the head through render_views
each as frames/s of whole-clip runs (host clock around a run that ends in a device synchronise; the best of 3 after a warm-up run),
then the same at world size N = every visible GPU (one spawned process per GPU, NCCL) when more than one is visible.  Finally
n3d_render_rays alone at the C2 (batch 8, 64^2, 48 + 48) and C3 (batch 16, 128^2, 96 + 96) shapes with depth_range_per_image 0 and
1, alternated in rounds (CUDA events, median of 30 launches per block).  Anything that did not run is reported as not measured.

python tools/bench_sharded.py --cli [--frames F] instead times whole `python -m next3d_b200 gen_videos --encoder n3d` runs (a 4x2
grid of one keyframe per cell, F frames, default 120, `--gop 30`; loading, graph capture and the MP4 included) of a tiny and of
a full-width random-weight pickle, at a constant QP and with `--bitrate script`, as frames/s at world 1 and at world N = every
visible GPU (torchrun-style ranks, one per GPU), with the card's name and power limit from the same run."""
import dataclasses
import os
import socket
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from next3d_b200 import config, drivers, inputs, kernels as K, weights
from next3d_b200.triplane_next3d import TriPlaneGenerator


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader', '-i',
                        str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    print(f'card {torch.cuda.get_device_name()}  (name, power limit, SM clock, max SM clock): {q or "unknown"}', flush=True)


def make_config(tiny, res=64, depth=96):
    base = config.tiny_config(512) if tiny else config.full_config(512)
    rk = dict(base.rendering_kwargs, depth_resolution=depth, depth_resolution_importance=depth)
    return dataclasses.replace(base, neural_rendering_resolution=res, rendering_kwargs=rk)


def setup(tiny, frames, tmp, device='cuda'):
    """Generator (graphed), one head (ws [1, L, D], mesh [1, V, 3]), orbit cameras and the clip's pack of `frames` meshes."""
    cfg = make_config(tiny)
    G = TriPlaneGenerator.from_config(cfg, weights.make_state_dict(cfg, seed=0), device=device)
    G.use_cuda_graph = True
    z, c_cond, c, v = weights.demo_inputs(cfg, 1, seed=0)
    ws = G.mapping(z.to(device), c_cond.to(device), truncation_psi=0.7, truncation_cutoff=14)
    cams = drivers.orbit_camera_params(frames, torch.tensor([0, 0, 0.2]), 2.7)
    pack = os.path.join(tmp, 'clip.n3dpack')
    if not os.path.exists(pack):
        rng = np.random.RandomState(0)
        verts = v[0].numpy()[None] + rng.randn(frames, *v.shape[1:]).astype(np.float32) * 1e-4
        inputs.write_frame_pack(pack, verts, cams.numpy())
    return cfg, G, ws, v, cams, pack


def fps(run, frames, barrier=lambda: None):
    """Frames/s of the best of 3 timed runs after one warm-up run (graph capture, allocator)."""
    run()
    best = float('inf')
    for _ in range(3):
        barrier()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run()
        torch.cuda.synchronize()
        barrier()
        best = min(best, time.perf_counter() - t0)
    return frames / best


def drivers_fps(G, ws, v, cams, pack, frames, batch, barrier=lambda: None):
    out = torch.empty(frames, G.img_resolution, G.img_resolution, 3, dtype=torch.uint8).pin_memory()
    return {
        'reenact_frames_sharded': fps(lambda: drivers.reenact_frames_sharded(G, ws, pack, frames, batch=batch, seed=1, out=out), frames, barrier),
        'render_orbit_sharded': fps(lambda: drivers.render_orbit_sharded(G, ws, cams, v, batch=batch, seed=1, out=out), frames, barrier),
    }


def _rank(rank, world, port, tiny, frames, batch, tmp, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    from next3d_b200 import distributed as D
    D.init_from_env('nccl')
    try:
        _, G, ws, v, cams, pack = setup(tiny, frames, tmp, f'cuda:{rank}')
        res = drivers_fps(G, ws, v, cams, pack, frames, batch, torch.distributed.barrier)
        if rank == 0:
            q.put(res)
    finally:
        torch.distributed.destroy_process_group()


def render_rays_flag(tiny):
    """n3d_render_rays at C2 and C3 with depth_range_per_image 0 / 1, alternated -> {(name, flag): ms per launch}."""
    out = {}
    for name, batch, res, depth in (('C2', 8, 64, 48), ('C3', 16, 128, 96)):
        cfg = make_config(tiny, res, depth)
        rk = cfg.rendering_kwargs
        g = torch.Generator().manual_seed(0)
        dec = tuple((torch.randn(*shape, generator=g) * scale).cuda().contiguous()
                    for shape, scale in (((64, 32), 32 ** -0.5), ((64,), 0.1), ((33, 64), 64 ** -0.5), ((33,), 0.1)))
        _, _, c, _ = weights.demo_inputs(cfg, batch, seed=0)
        planes = torch.randn(batch, 3, 256, 256, cfg.plane_ch, generator=g).cuda() * 0.5
        cam, intr = c[:, :16].contiguous().cuda(), c[:, 16:25].contiguous().cuda()
        M = res * res
        rgb = torch.empty(batch, M, 32, device='cuda')
        depth_t, wsum = torch.empty(batch, M, device='cuda'), torch.empty(batch, M, device='cuda')
        mm = {0: torch.tensor([float('inf'), 0.0], device='cuda'),
              1: torch.tensor([float('inf'), float('-inf')], device='cuda').repeat(batch, 1)}
        run = {f: (lambda i, f=f: K.render_rays(planes, cam, intr, res, rk, dec, rgb, depth_t, wsum, mm[f], seed=i, depth_range_per_image=f))
               for f in (0, 1)}
        for f in (0, 1):
            run[f](0)
        med = {0: [], 1: []}
        for _ in range(3):
            for f in (0, 1):
                ts = []
                for i in range(30):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    run[f](i)
                    e1.record()
                    torch.cuda.synchronize()
                    ts.append(e0.elapsed_time(e1))
                med[f].append(sorted(ts)[len(ts) // 2])
        for f in (0, 1):
            out[(name, f)] = med[f]
    return out


def _cli_run(argv, world):
    """Seconds of one `python -m next3d_b200 argv` run as `world` ranks, one per GPU."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    t0 = time.perf_counter()
    procs = [subprocess.Popen([sys.executable, '-m', 'next3d_b200', *argv], cwd=root, stdout=subprocess.DEVNULL,
                              env=dict(os.environ, PYTHONPATH=root, **({} if world == 1 else dict(
                                  RANK=str(r), WORLD_SIZE=str(world), LOCAL_RANK=str(r), MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port)))))
             for r in range(world)]
    codes = [p.wait() for p in procs]
    if any(codes):
        raise SystemExit(f'gen_videos exited with {codes}')
    return time.perf_counter() - t0


def cli_main(frames):
    """Frames/s of whole gen_videos --encoder n3d runs at world 1 and N."""
    from tests.test_legacy_cpu import _demo_args, generator_fields, persistence_pickle
    import pathlib
    card()
    world = torch.cuda.device_count()
    with tempfile.TemporaryDirectory() as tmp:
        demo = _demo_args(pathlib.Path(tmp))
        for tiny in (True, False):
            cfg = config.tiny_config(512) if tiny else config.full_config(512)
            net = os.path.join(tmp, 'net.pkl')
            with open(net, 'wb') as f:
                f.write(persistence_pickle(cfg, weights.make_state_dict(cfg, seed=0), generator_fields(cfg, torch.ones(1, 1, 256, 256))))
            for name, stream in (('QP 18', ['--qp', '18']), ('bitrate script', ['--bitrate', 'script'])):
                argv = ['gen_videos', '--network', net, '--seeds', '0-7', '--grid', '4x2', '--w-frames', str(frames), '--gop', '30',
                        '--outdir', os.path.join(tmp, 'out'), '--lms_cond', 'True', '--encoder', 'n3d', *stream, *demo]
                fps1 = frames / _cli_run(argv, 1)
                line = f'gen_videos {"tiny" if tiny else "full"} 4x2 grid, {frames} frames, {name}: world 1 {fps1:.2f} frames/s'
                if world > 1:
                    fpsN = frames / _cli_run(argv, world)
                    line += f', world {world} {fpsN:.2f} frames/s ({fpsN / fps1:.2f}x)'
                else:
                    line += ', world N not measured (one GPU visible)'
                print(line, flush=True)


def main():
    if '--cli' in sys.argv:
        return cli_main(int(sys.argv[sys.argv.index('--frames') + 1]) if '--frames' in sys.argv else 120)
    tiny = '--tiny' in sys.argv
    frames = int(sys.argv[sys.argv.index('--frames') + 1]) if '--frames' in sys.argv else 96
    batch = 8
    if not torch.cuda.is_available():
        raise SystemExit('bench_sharded.py needs a CUDA device')
    card()
    print(f'config {"tiny" if tiny else "full"}: {frames}-frame clip, one head, 64^2 neural render, 96 + 96 samples, 512^2 output, '
          f'batch {batch}', flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        cfg, G, ws, v, cams, pack = setup(tiny, frames, tmp)
        single = fps(lambda: [f for f in drivers.reenact_frames(G, ws, pack, frames, batch=batch, seed=1)], frames)
        print(f'world 1  reenact_frames           {single:8.1f} frames/s', flush=True)
        res = drivers_fps(G, ws, v, cams, pack, frames, batch)
        for name, r in res.items():
            print(f'world 1  {name:24s} {r:8.1f} frames/s', flush=True)
        del G
        torch.cuda.empty_cache()
        world = torch.cuda.device_count()
        if world > 1:
            s = socket.socket()
            s.bind(('127.0.0.1', 0))
            port = s.getsockname()[1]
            s.close()
            ctx = torch.multiprocessing.get_context('spawn')
            q = ctx.Queue()
            procs = [ctx.Process(target=_rank, args=(r, world, port, tiny, frames, batch, tmp, q)) for r in range(world)]
            for p in procs:
                p.start()
            resN = q.get(timeout=1800)
            for p in procs:
                p.join()
            for name, r in resN.items():
                print(f'world {world}  {name:24s} {r:8.1f} frames/s ({r / res[name]:.2f}x world 1)', flush=True)
        else:
            print('world N  multi-GPU scaling: not measured (one GPU visible)', flush=True)
    for (name, f), med in render_rays_flag(tiny).items():
        print(f'n3d_render_rays {name} depth_range_per_image={f}: {min(med):.3f} ms per launch (block medians '
              f'{" / ".join(f"{m:.3f}" for m in med)})', flush=True)


if __name__ == '__main__':
    main()
