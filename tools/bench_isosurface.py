"""Time of the sm_90a marching cubes (next3d_b200.isosurface.marching_cubes: count pass, one host read of the counts, emit pass)
on the density grids of seeded tiny- and full-width generators at shape_res 256 and 512, from grids already on the device:
ms per grid (device events, after warm-up), vertices, triangles and the grid-read rate (two passes x 4 B x R^3 over the time),
at the scripts' level 10 and at a level that cuts the head (the 0.7 quantile of the densities inside the border).  With --cli,
also `python -m next3d_b200 shape_utils` end to end on a directory of 512^3 .mrc files, split into MRC read, mesh and PLY write.
Prints the card name and power limit of the run, then one JSON line.

    python tools/bench_isosurface.py [--iters 20] [--cli]
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
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def grid(width, res, seed=0):
    """float32 numpy [res]^3: drivers.extract_sigma_grid of a seeded generator."""
    from next3d_b200 import config, drivers, weights
    from next3d_b200.triplane_next3d import TriPlaneGenerator
    cfg = config.tiny_config(512) if width == 'tiny' else config.full_config(512)
    G = TriPlaneGenerator.from_config(cfg, weights.make_state_dict(cfg, seed=0), device='cuda')
    z, cc, _, v = weights.demo_inputs(cfg, 1, seed=seed, device='cuda')
    ws = G.mapping(z, cc, truncation_psi=0.7, truncation_cutoff=14)
    return drivers.extract_sigma_grid(G, ws, v, shape_res=res)


def time_mesh(g, level, iters):
    from next3d_b200.isosurface import marching_cubes
    for _ in range(3):
        verts, faces = marching_cubes(g, level)
    torch.cuda.synchronize()
    ms = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        marching_cubes(g, level)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    t = float(np.median(ms))
    return {'ms': round(t, 3), 'ms_min': round(min(ms), 3), 'vertices': verts.shape[0], 'triangles': faces.shape[0],
            'grid_read_GB_per_s': round(2 * 4 * g.numel() / (t * 1e-3) / 1e9, 1)}


def cli(grids, tmp):
    """shape_utils on a directory of the .mrc files of `grids`: whole-process time, and the in-process split per file."""
    from next3d_b200 import isosurface, mrc
    for i, g in enumerate(grids):
        mrc.write_mrc(os.path.join(tmp, f'seed{i:04d}.mrc'), g)
    t = time.perf_counter()
    subprocess.run([sys.executable, '-m', 'next3d_b200', 'shape_utils', tmp], cwd=ROOT, check=True, stdout=subprocess.DEVNULL)
    whole = time.perf_counter() - t
    split = {'read_s': 0.0, 'mesh_s': 0.0, 'write_s': 0.0}
    for i in range(len(grids)):
        path = os.path.join(tmp, f'seed{i:04d}.mrc')
        t0 = time.perf_counter()
        data = np.array(mrc.read_mrc(path))
        t1 = time.perf_counter()
        verts, faces = isosurface.marching_cubes(data, 10.0)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        isosurface.write_ply(path[:-4] + '.ply', verts, faces)
        t3 = time.perf_counter()
        split['read_s'] += t1 - t0
        split['mesh_s'] += t2 - t1
        split['write_s'] += t3 - t2
    return {'files': len(grids), 'process_s': round(whole, 2), 'per_file_in_process': {k: round(v / len(grids), 3) for k, v in split.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--cli', action='store_true')
    a = ap.parse_args()
    print('card:', card(), flush=True)
    out = {'card': card()}
    big = []
    for width in ('tiny', 'full'):
        for res in (256, 512):
            host = grid(width, res)
            if res == 512:
                big.append(host)
            g = torch.from_numpy(host).cuda()
            inner = host[host > -1000]
            for name, level in (('level10', 10.0), ('cutting', float(np.quantile(inner, 0.7)))):
                row = time_mesh(g, level, a.iters)
                row['level'] = level
                out[f'{width}_{res}_{name}'] = row
                print(f'{width} {res}^3 level {level:.4g}: {row["ms"]:.3f} ms (min {row["ms_min"]:.3f}), {row["vertices"]} vertices, '
                      f'{row["triangles"]} triangles, grid read {row["grid_read_GB_per_s"]} GB/s', flush=True)
            del g
    if a.cli:
        with tempfile.TemporaryDirectory() as tmp:
            out['cli'] = cli(big, tmp)
        print('shape_utils:', out['cli'], flush=True)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
