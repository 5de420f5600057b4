"""Per-launch table of the convolution GEMMs of one synthesis of a bench.py configuration: --config c2 (the default: FFHQ-512
widths, 64^2 neural render, batch 8) or c3 (128^2 render, batch 16); --batch overrides the configuration's batch size.  One row
per conv_gemm launch (layer, Cin -> Cout, M-space, taps, ms, algorithmic TFLOP/s), sorted by time, and the total; the header
names the GPU, configuration and batch.  The synthesis runs eagerly on one stream with CUDA events around every launch, the way
bench.py measures `roofline.achieved` of conv_gemm_kernel.

--classes adds, for every distinct stride-2 transposed (up-sampling conv0) shape of the synthesis, the one-launch
n3d_conv_transposed_gemm against its four output-parity classes (a, b) run as separate n3d_conv_gemm launches, on random operands
of the same shape: median ms over --reps launches each, and TFLOP/s of the useful work (taps x output positions of the class).

--nprod 1 runs every launch with one MMA product (hi x hi) instead of three: the same stage ring, half the bytes loaded and a
third of the MMAs.  A layer's time ratio t(nprod 1) / t(nprod 3) near 1/2 says that feeding the operands bounds it, near 1/3
that the tensor pipe does.  (The TFLOP/s column stays algorithmic, i.e. it counts the 3-product work.)
Usage (GPU box): python tools/profile_convs.py [--config c2|c3] [--batch B] [--top K] [--classes] [--reps R] [--nprod 1|3]"""
import argparse
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _time_ms(torch, fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts)


def parity_classes(torch, K, dev, N, Cin, Cout, H, reps):
    """Rows (label, ms, useful FLOPs) for one transposed layer: the one-launch form, then each parity class alone."""
    g = torch.Generator(device=dev).manual_seed(Cin * 7 + Cout + H)
    a_hi, a_lo = K.split_bf16(torch.randn(N, H, H, Cin, device=dev, generator=g))
    w_hi, w_lo = K.split_bf16(torch.randn(9, Cout, Cin, device=dev, generator=g) / (3 * Cin ** 0.5))
    raw = torch.empty(N, 2 * H + 1, 2 * H + 1, Cout, device=dev)
    total = 2.0 * Cin * Cout * N * (3 * H + 2) ** 2
    rows = [('one launch', _time_ms(torch, lambda: K.conv_transposed_gemm(a_hi, a_lo, w_hi, w_lo, N, H, H, raw), reps), total)]
    for a in (0, 1):
        for b in (0, 1):
            taps = K.taps_transposed(a, b)
            mh, mw = H + 1 - a, H + 1 - b

            def run():
                K.conv_gemm(a_hi, a_lo, w_hi, w_lo, taps, N, mh, mw, mode=1, out_f32=raw, f32_cstride=Cout, oy_mul=2, oy_off=a,
                            ox_mul=2, ox_off=b, OH=2 * H + 1, OW=2 * H + 1)
            rows.append((f'class ({a},{b}) {len(taps)} taps', _time_ms(torch, run, reps), 2.0 * Cin * Cout * N * len(taps) * mh * mw))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', default='c2', choices=['c2', 'c3'])
    ap.add_argument('--batch', type=int, default=None)
    ap.add_argument('--top', type=int, default=0, help='print only the K slowest launches (0 = all)')
    ap.add_argument('--classes', action='store_true', help='also time the four parity classes of every transposed layer shape')
    ap.add_argument('--reps', type=int, default=20, help='launches per timing of --classes (median)')
    ap.add_argument('--nprod', type=int, default=3, choices=[1, 3],
                    help='MMA products per k-step of the synthesis launches: 3 = bf16x3 (what the engine runs), 1 = hi*hi only '
                         '(the same stage ring with half the bytes loaded and a third of the MMAs)')
    args = ap.parse_args()

    import torch
    import bench
    from next3d_b200 import kernels as K
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
        eng.nprod = args.nprod
        for _ in range(2):                                   # warm-up: module load, allocator, every launch shape once
            G.synthesis(ws, c_d, v_d, noise_mode='const', seed=5)
        eng.prof = []
        G.synthesis(ws, c_d, v_d, noise_mode='const', seed=5)
        torch.cuda.synchronize(dev)
        rows = [(e0.elapsed_time(e1), fl, info) for kind, e0, e1, fl, info in eng.prof if kind == 'conv_gemm']
        eng.prof = None

    def transposed(info):
        L = eng.mod.get(info[0])
        return L is not None and L.up == 2

    print(f'# {torch.cuda.get_device_name(dev)}  config {args.config}  batch {B}  nprod {args.nprod}  conv_gemm launches {len(rows)}')
    print(f'{"layer":40s} {"Cin":>5s} {"Cout":>5s} {"MH":>4s} {"MW":>4s} {"taps":>4s} {"ms":>8s} {"TFLOP/s":>8s}')
    tot_ms = sum(r[0] for r in rows)
    tot_fl = sum(r[1] for r in rows)
    shown = sorted(rows, key=lambda r: -r[0])
    if args.top:
        shown = shown[:args.top]
    for ms, fl, (layer, cin, cout, mh, mw, taps) in shown:
        tf = fl / (ms * 1e-3) / 1e12 if fl else 0.0
        print(f'{str(layer):40s} {cin:5d} {cout:5d} {mh:4d} {mw:4d} {taps:4d} {ms:8.3f} {tf:8.1f}')
    up = [r for r in rows if transposed(r[2])]
    up_ms, up_fl = sum(r[0] for r in up), sum(r[1] for r in up)
    print(f'{f"transposed ({len(up)} launches)":40s} {"":5s} {"":5s} {"":4s} {"":4s} {"":4s} {up_ms:8.3f} {up_fl / (up_ms * 1e-3) / 1e12:8.1f}')
    print(f'{"total":40s} {"":5s} {"":5s} {"":4s} {"":4s} {"":4s} {tot_ms:8.3f} {tot_fl / (tot_ms * 1e-3) / 1e12:8.1f}')

    if args.classes:
        shapes = sorted({(info[1], info[2], info[3] - 1) for _, _, info in up}, key=lambda s: -s[0] * s[1] * s[2] ** 2)
        print(f'\n# parity classes, batch {B}, median of {args.reps} launches')
        print(f'{"Cin":>5s} {"Cout":>5s} {"H":>4s}  {"launch":24s} {"ms":>8s} {"TFLOP/s":>8s}')
        with torch.no_grad():
            for cin, cout, h in shapes:
                cls = parity_classes(torch, K, dev, B, cin, cout, h, args.reps)
                for label, ms, fl in cls:
                    print(f'{cin:5d} {cout:5d} {h:4d}  {label:24s} {ms:8.3f} {fl / (ms * 1e-3) / 1e12:8.1f}')
                print(f'{cin:5d} {cout:5d} {h:4d}  {"sum of the classes":24s} {sum(r[1] for r in cls[1:]):8.3f}')
                torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
