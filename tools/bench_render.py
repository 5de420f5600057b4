"""Time the fused renderer alone on a benchmark workload (random planes).  python tools/bench_render.py [c2|c3]"""
import sys, os, math
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from next3d_b200 import config, weights, kernels as K
cfg = config.full_config(512)
which = sys.argv[1] if len(sys.argv) > 1 else 'c2'
N, R, D = (8, 64, 48) if which == 'c2' else (16, 128, 96)
opts = dict(cfg.rendering_kwargs, depth_resolution=D, depth_resolution_importance=D)
g = torch.Generator().manual_seed(0)
planes = torch.randn(N, 3, 256, 256, 32, generator=g).cuda()
dec = (torch.randn(64, 32, generator=g).cuda() / math.sqrt(32), torch.randn(64, generator=g).cuda() * 0.1,
       torch.randn(33, 64, generator=g).cuda() / math.sqrt(64), torch.randn(33, generator=g).cuda() * 0.1)
_, _, c, _ = weights.demo_inputs(cfg, N)
cam, intr = c[:, :16].contiguous().cuda(), c[:, 16:25].contiguous().cuda()
rgb = torch.zeros(N, R * R, 32, device='cuda'); depth = torch.zeros(N, R * R, device='cuda'); wsum = torch.zeros_like(depth)
mm = torch.tensor([float('inf'), 0.0], device='cuda')
flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
for _ in range(3):
    K.render_rays(planes, cam, intr, R, opts, dec, rgb, depth, wsum, mm, seed=1)
ts = []
for i in range(10):
    flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    K.render_rays(planes, cam, intr, R, opts, dec, rgb, depth, wsum, mm, seed=i)
    e1.record(); torch.cuda.synchronize()
    ts.append(e0.elapsed_time(e1))
ts.sort()
print(which, 'render_fused_kernel median', ts[len(ts) // 2], 'ms  min', ts[0], 'ms', flush=True)
if which == 'c2' and os.environ.get('N3D_BENCH_GRID', '1') == '1':
    Rg = 256
    out = torch.empty(Rg, Rg, Rg, device='cuda')
    for pad in (0, int(30 * Rg / 256)):
        for _ in range(2):
            K.sample_grid(planes[0], Rg, 1.0, 1.0, dec, out, pad=pad)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            K.sample_grid(planes[0], Rg, 1.0, 1.0, dec, out, pad=pad)
        e1.record(); torch.cuda.synchronize()
        print(f'c5 grid {Rg}^3 pad {pad}: {e0.elapsed_time(e1) / 5:.3f} ms per grid', flush=True)
