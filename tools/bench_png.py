"""Throughput of the sm_90a PNG encoder (next3d_b200.png.PngEncoder) against PIL on the same frames: images/s and bytes/image
for frames rendered by the tiny- and full-width generators at 512x512 and at sample-sheet size (three 512x512 views side by
side, 1536x512), from frames already on the device; PIL at compress_level 1 and 6 on the host copies of the same frames.
Prints the card name and power limit of the run, then one JSON line.

    python tools/bench_png.py [--images 64] [--batch 16]
"""
import argparse
import io
import json
import os
import subprocess
import sys
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


def rendered(width, n):
    """n distinct 512x512 uint8 frames [n, 512, 512, 3] on the device: an orbit of one head of a seeded generator."""
    from next3d_b200 import config, drivers, weights
    from next3d_b200.triplane_next3d import TriPlaneGenerator
    cfg = config.tiny_config(512) if width == 'tiny' else config.full_config(512)
    G = TriPlaneGenerator.from_config(cfg, weights.make_state_dict(cfg, seed=0), device='cuda')
    *_, v = weights.demo_inputs(cfg, 1, seed=0, device='cuda')
    rk = G.rendering_kwargs
    ws = drivers.grid_keyframes(G, [3], (1, 1), truncation_psi=0.7)[0, 0]
    cams = drivers.orbit_camera_params(n, torch.tensor(rk['avg_camera_pivot']), rk['avg_camera_radius'])
    return torch.stack([torch.as_tensor(f) for f in drivers.render_orbit(G, ws[:1], cams, v, seed=0)]).cuda()


def encoder_rate(frames, batch):
    from next3d_b200.png import PngEncoder
    H, W = frames.shape[1:3]
    enc = PngEncoder(W, H, batch=batch)
    enc.write(frames[:batch])                                   # warm-up: module load, first launches
    enc.flush()
    torch.cuda.synchronize()
    t = time.perf_counter()
    files = enc.write(frames) + enc.flush()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t
    return {'images_per_s': len(files) / dt, 'bytes_per_image': sum(map(len, files)) / len(files)}


def pil_rate(frames, level, n=8):
    from PIL import Image
    host = frames[:n].cpu().numpy()
    sizes, t = [], time.perf_counter()
    for f in host:
        buf = io.BytesIO()
        Image.fromarray(f).save(buf, format='png', compress_level=level)
        sizes.append(len(buf.getvalue()))
    dt = time.perf_counter() - t
    return {'images_per_s': len(host) / dt, 'bytes_per_image': sum(sizes) / len(sizes)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=64)
    ap.add_argument('--batch', type=int, default=16)
    a = ap.parse_args()
    print('card:', card(), flush=True)
    out = {'card': card()}
    for width in ('tiny', 'full'):
        views = rendered(width, a.images + 2)
        sheets = torch.cat([views[:-2], views[1:-1], views[2:]], dim=2).contiguous()         # [n, 512, 1536, 3]
        for name, frames in (('512x512', views[:a.images]), ('sheet1536x512', sheets)):
            row = {'encoder': encoder_rate(frames, a.batch), 'pil_level1': pil_rate(frames, 1), 'pil_level6': pil_rate(frames, 6)}
            out[f'{width}_{name}'] = row
            print(f'{width} {name}: ' + ', '.join(f'{k} {v["images_per_s"]:.1f} images/s, {v["bytes_per_image"]:.0f} B'
                                                  for k, v in row.items()), flush=True)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
