"""The fp16 super-resolution head (TriPlaneGenerator.sr_precision = 'fp16') against the default fp32 head, in one session with the
two modes alternated: images/s of bench.py's configurations (graphed synthesis), render_views ms per frame (graphed, --views
cameras of one cached head), and the per-launch times of the four SR convolutions (eager, CUDA events around every
launch, as tools/profile_convs.py times them).  The header names the GPU and its power limit.

--parent DIR (a checkout of the parent commit with its library built) first runs bench.py's C2 in the default mode there and here,
alternated --rounds times, and reports both img/s and whether the outputs of the two builds are bit-identical (bench.py
--dump-outputs, into a temporary directory).

Usage (GPU box): python tools/bench_sr_fp16.py [--configs c2,c3] [--steps 30] [--rounds 3] [--views 8] [--parent DIR] [--json PATH]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MODES = ('fp32', 'fp16')


def _gpu_header(torch):
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                      # the numbers still need the device name beside them
        q = f'{torch.cuda.get_device_name(0)} (nvidia-smi unavailable: {e})'
    return q


def _timed(torch, fn, steps):
    """Seconds per call of fn over `steps` calls, host clock around work that ends in a device synchronise."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps


def _bench_py(tree, steps, warmup, dump):
    """bench.py C2 (default mode, graphed) of the tree at `tree`, outputs dumped to `dump` -> its img/s."""
    out = subprocess.run([sys.executable, os.path.join(tree, 'bench.py'), '--gpus', '1', '--steps', str(steps), '--warmup', str(warmup),
                          '--no-other-configs', '--no-cpu-baseline', '--dump-outputs', dump], cwd=tree, capture_output=True, text=True,
                         check=True).stdout
    return json.loads([ln for ln in out.splitlines() if ln.startswith('{')][-1])['value']


def compare_with_parent(parent, steps, warmup, rounds):
    """bench.py C2 of the parent tree and of this one, alternated: img/s of each run and the bit-identity of their outputs."""
    import numpy as np
    res = {'parent_img_s': [], 'this_img_s': [], 'bit_identical': {}}
    with tempfile.TemporaryDirectory() as tmp:
        dumps = {k: os.path.join(tmp, k) for k in ('parent', 'this')}
        for _ in range(rounds):
            res['parent_img_s'].append(_bench_py(os.path.abspath(parent), steps, warmup, dumps['parent']))
            res['this_img_s'].append(_bench_py(ROOT, steps, warmup, dumps['this']))
        for f in sorted(os.listdir(dumps['parent'])):
            a, b = np.load(os.path.join(dumps['parent'], f)), np.load(os.path.join(dumps['this'], f))
            res['bit_identical'][f] = a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--configs', default='c2,c3')
    ap.add_argument('--steps', type=int, default=30, help='graphed steps per timed window (about 1 s at C2)')
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rounds', type=int, default=3, help='alternations of the two modes per measurement (median reported)')
    ap.add_argument('--views', type=int, default=8, help='render_views cameras per cached head')
    ap.add_argument('--parent', metavar='DIR', default=None, help='parent checkout to compare bench.py C2 (default mode) with')
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    result = {}
    if args.parent:                                         # before this process takes GPU memory
        result['bench_py_c2_vs_parent'] = p = compare_with_parent(args.parent, args.steps, args.warmup, args.rounds)
        print(f'# bench.py C2, default mode: parent {", ".join(f"{v:.1f}" for v in p["parent_img_s"])} img/s, this build '
              f'{", ".join(f"{v:.1f}" for v in p["this_img_s"])} img/s; outputs bit-identical: {p["bit_identical"]}')

    import torch
    import bench
    from next3d_b200 import drivers, weights
    from next3d_b200.triplane_next3d import TriPlaneGenerator

    assert torch.cuda.is_available(), 'bench_sr_fp16.py needs a CUDA device'
    dev = torch.device('cuda', 0)
    result.update(gpu=_gpu_header(torch), configs={})
    print(f'# {result["gpu"]}')
    for name in args.configs.split(','):
        cfg = bench.config_for(name)
        B = bench.CONFIGS[name]['batch']
        G = TriPlaneGenerator.from_config(cfg, weights.make_state_dict(cfg, seed=0), device=dev)
        G.use_cuda_graph = True
        z, c_cond, c_cam, v = weights.demo_inputs(cfg, B, seed=0)
        with torch.no_grad():
            ws = G.mapping(z.to(dev), c_cond.to(dev), truncation_psi=0.7, truncation_cutoff=14)
        c_d, v_d = c_cam.to(dev), v.to(dev)
        R = cfg.neural_rendering_resolution
        cams = drivers.orbit_camera_params(args.views, torch.tensor([0, 0, 0.2]), 2.7).to(dev)
        row = {'batch': B, 'views_per_head': args.views}

        def synth():
            return G.synthesis(ws, c_d, v_d, noise_mode='const', seed=5)

        def views():
            return G.render_views(cams, seed=5)

        with torch.no_grad():
            for mode in MODES:                                  # warm-up: captures, module loads, the backbone cache
                G.sr_precision = mode
                G.synthesis(ws[:1], c_d[:1], v_d[:1], noise_mode='const', seed=0, cache_backbone=True)
                for _ in range(args.warmup):
                    synth()
                    views()
            ts = {m: [] for m in MODES}
            tv = {m: [] for m in MODES}
            for _ in range(args.rounds):
                for mode in MODES:
                    G.sr_precision = mode
                    ts[mode].append(_timed(torch, synth, args.steps))
                    tv[mode].append(_timed(torch, views, args.steps))
            # per-launch SR times, eager on one stream
            G.use_cuda_graph = False
            eng = G._get_engine()
            eng.concurrent = False
            launches = {}
            for mode in MODES:
                G.sr_precision = mode
                synth()
                per = {}
                for _ in range(args.rounds):
                    eng.prof = []
                    synth()
                    torch.cuda.synchronize()
                    for kind, e0, e1, fl, info in eng.prof:
                        if kind == 'conv_gemm' and info and str(info[0]).startswith('superresolution'):
                            per.setdefault(info[0], []).append(e0.elapsed_time(e1))
                eng.prof = None
                launches[mode] = {k: statistics.median(v) for k, v in per.items()}
            eng.concurrent = True
            G.use_cuda_graph = True
        for mode in MODES:
            s, sv = statistics.median(ts[mode]), statistics.median(tv[mode])
            row[mode] = {'images_per_s': B / s, 'synthesis_ms': s * 1e3, 'render_views_ms_per_frame': sv * 1e3 / cams.shape[0],
                         'sr_launch_ms': launches[mode], 'spread_synthesis_ms': [t * 1e3 for t in ts[mode]]}
        result['configs'][name] = row
        print(f'## {name}: batch {B}, {R}^2 render')
        for mode in MODES:
            r = row[mode]
            print(f'  {mode}: {r["images_per_s"]:8.2f} img/s  synthesis {r["synthesis_ms"]:8.2f} ms  render_views '
                  f'{r["render_views_ms_per_frame"]:7.3f} ms/frame  (synthesis runs: {", ".join(f"{t:.2f}" for t in r["spread_synthesis_ms"])})')
        for layer in sorted(row['fp32']['sr_launch_ms']):
            a, b = row['fp32']['sr_launch_ms'][layer], row['fp16']['sr_launch_ms'].get(layer, float('nan'))
            print(f'    {layer:40s} fp32 {a:7.3f} ms  fp16 {b:7.3f} ms  ratio {b / a:5.2f}')
        del G
        torch.cuda.empty_cache()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
