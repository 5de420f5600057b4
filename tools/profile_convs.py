"""Per-launch table of the convolution GEMMs of one synthesis of a bench.py configuration: --config c2 (the default: FFHQ-512
widths, 64^2 neural render, batch 8) or c3 (128^2 render, batch 16); --batch overrides the configuration's batch size.  One row
per conv_gemm launch (layer, Cin -> Cout, M-space, taps, ms, algorithmic TFLOP/s), sorted by time, and the total; the header
names the GPU, configuration and batch.  The synthesis runs eagerly on one stream with CUDA events around every launch, the way
bench.py measures `roofline.achieved` of conv_gemm_kernel.
Usage (GPU box): python tools/profile_convs.py [--config c2|c3] [--batch B] [--top K]"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', default='c2', choices=['c2', 'c3'])
    ap.add_argument('--batch', type=int, default=None)
    ap.add_argument('--top', type=int, default=0, help='print only the K slowest launches (0 = all)')
    args = ap.parse_args()

    import torch
    import bench
    from next3d_b200 import weights
    from next3d_b200.triplane_next3d import TriPlaneGenerator

    assert torch.cuda.is_available(), 'profile_convs.py needs a CUDA device'
    dev = torch.device('cuda', 0)
    cfg = bench.config_for(args.config)
    B = args.batch or bench.CONFIGS[args.config]['batch']
    G = TriPlaneGenerator.from_config(cfg, weights.make_state_dict(cfg, seed=0), device=dev)
    G.use_cuda_graph = False
    z, c_cond, c_cam, v = weights.demo_inputs(cfg, B, seed=0)
    with torch.no_grad():
        ws = G.mapping(z.to(dev), c_cond.to(dev), truncation_psi=0.7, truncation_cutoff=14)
        c_d, v_d = c_cam.to(dev), v.to(dev)
        eng = G._get_engine()
        eng.concurrent = False
        for _ in range(2):                                   # warm-up: module load, allocator, every launch shape once
            G.synthesis(ws, c_d, v_d, noise_mode='const', seed=5)
        eng.prof = []
        G.synthesis(ws, c_d, v_d, noise_mode='const', seed=5)
        torch.cuda.synchronize(dev)
        rows = [(e0.elapsed_time(e1), fl, info) for kind, e0, e1, fl, info in eng.prof if kind == 'conv_gemm']
        eng.prof = None

    print(f'# {torch.cuda.get_device_name(dev)}  config {args.config}  batch {B}  conv_gemm launches {len(rows)}')
    print(f'{"layer":40s} {"Cin":>5s} {"Cout":>5s} {"MH":>4s} {"MW":>4s} {"taps":>4s} {"ms":>8s} {"TFLOP/s":>8s}')
    tot_ms = sum(r[0] for r in rows)
    tot_fl = sum(r[1] for r in rows)
    shown = sorted(rows, key=lambda r: -r[0])
    if args.top:
        shown = shown[:args.top]
    for ms, fl, (layer, cin, cout, mh, mw, taps) in shown:
        tf = fl / (ms * 1e-3) / 1e12 if fl else 0.0
        print(f'{str(layer):40s} {cin:5d} {cout:5d} {mh:4d} {mw:4d} {taps:4d} {ms:8.3f} {tf:8.1f}')
    print(f'{"total":40s} {"":5s} {"":5s} {"":4s} {"":4s} {"":4s} {tot_ms:8.3f} {tot_fl / (tot_ms * 1e-3) / 1e12:8.1f}')


if __name__ == '__main__':
    main()
