"""Throughput of the sm_90a H.264 encoder (next3d_b200.video.H264Writer): encode frames/s and bits/frame at 512x512 and
2048x1024 (the frame of a --grid 4x2 interpolation video) from frames already on the device, for the constant-QP stream and the
rate-controlled one (achieved against target bitrate, luma PSNR against the input), and render + encode of a --grid 4x2
interpolation run of the tiny generator at both.  Prints the card name and power limit of the run, then one JSON line.

    python tools/bench_video.py [--frames 120] [--qp 18] [--bitrate 12M]
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


def frames_on_device(W, H, n):
    """A moving, textured RGB sequence [n, H, W, 3] uint8 (a pattern panned 3 px right and 1 px up per frame)."""
    y, x = torch.meshgrid(torch.arange(H + n, device='cuda'), torch.arange(W + 3 * n, device='cuda'), indexing='ij')
    img = torch.stack([torch.sin(x * 0.05 + y * 0.02) * 60 + torch.sin(x * 0.21) * 20, torch.cos(y * 0.07 - x * 0.03) * 70,
                       torch.sin((x + y) * 0.11) * 50], -1) + 128
    img = img.clamp(0, 255).to(torch.uint8)
    return torch.stack([img[n - t:n - t + H, 3 * t:3 * t + W] for t in range(n)])


def luma(frames):
    f = frames.double()
    return ((66 * f[..., 0] + 129 * f[..., 1] + 25 * f[..., 2] + 128) / 256).floor() + 16


def encode_rate(W, H, n, qp, out, bitrate=None):
    from next3d_b200.video import H264Writer
    frames = frames_on_device(W, H, n)
    kw = dict(qp=qp) if bitrate is None else dict(bitrate=bitrate)
    with H264Writer(os.path.join(out, 'warm.mp4'), W, H, 60, **kw) as w:       # warm-up: module load, first launches
        w.write(frames[:8])
    path = os.path.join(out, f'{W}x{H}.mp4')
    torch.cuda.synchronize()
    t = time.perf_counter()
    with H264Writer(path, W, H, 60, **kw) as w:
        w.write(frames)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t
    bits = 8 * (os.path.getsize(path) - 1000) / n
    res = {'fps': n / dt, 'bits_per_frame': bits}
    mse = 0.0                                                                 # luma PSNR against the input, frame by frame
    with H264Writer(os.path.join(out, 'psnr.mp4'), W, H, 60, **kw) as w:
        for i in range(n):
            w.write(frames[i])
            mse += ((w.recon[0][:H, :W].double() - luma(frames[i])) ** 2).mean().item() / n
    res['luma_psnr_db'] = 10 * np.log10(255 ** 2 / max(mse, 1e-12))
    if bitrate is not None:
        res['target_bits_per_s'] = bitrate
        res['achieved_bits_per_s'] = bits * 60
    return res


def render_encode_grid(n_frames, qp, out, bitrate=None):
    from next3d_b200 import config, drivers, weights
    from next3d_b200.triplane_next3d import TriPlaneGenerator
    from next3d_b200.video import H264Writer
    cfg = config.tiny_config(256)
    G = TriPlaneGenerator.from_config(cfg, weights.make_state_dict(cfg, seed=0), device='cuda')
    _, _, _, v = weights.demo_inputs(cfg, 1, seed=0, device='cuda')
    ws = drivers.grid_keyframes(G, list(range(16)), (4, 2), truncation_psi=0.7)
    w_frames = max(1, n_frames // 2)
    list(drivers.render_grid_frames(G, ws, v, 1, seed=0))                         # warm-up
    torch.cuda.synchronize()
    t = time.perf_counter()
    frames = list(drivers.render_grid_frames(G, ws, v, w_frames, seed=0))
    render = time.perf_counter() - t
    H, W, _ = frames[0].shape
    t = time.perf_counter()
    with H264Writer(os.path.join(out, 'grid.mp4'), W, H, 60, **(dict(qp=qp) if bitrate is None else dict(bitrate=bitrate))) as w:
        for f in drivers.render_grid_frames(G, ws, v, w_frames, seed=0):
            w.write(f)
    both = time.perf_counter() - t
    return {'frame': f'{W}x{H}', 'frames': len(frames), 'render_fps': len(frames) / render, 'render_encode_fps': len(frames) / both}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=120)
    ap.add_argument('--qp', type=int, default=18)
    ap.add_argument('--bitrate', default='12M', help="the rate-controlled arm's rate (the grid run uses the scripts' 10M)")
    args = ap.parse_args()
    from next3d_b200.video import parse_bitrate
    rate = parse_bitrate(args.bitrate)
    print('card, power limit:', card())
    with tempfile.TemporaryDirectory() as out:
        res = {'qp': args.qp, 'bitrate': rate, 'card': card()}
        for W, H in [(512, 512), (2048, 1024)]:
            res[f'encode_{W}x{H}'] = encode_rate(W, H, args.frames, args.qp, out)
            res[f'encode_{W}x{H}_bitrate'] = encode_rate(W, H, args.frames, args.qp, out, rate)
        res['grid4x2_tiny'] = render_encode_grid(16, args.qp, out)
        res['grid4x2_tiny_bitrate_script'] = render_encode_grid(16, args.qp, out, 10 * 10 ** 6)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
