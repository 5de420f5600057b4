"""Time the fused renderer alone on a benchmark workload (random planes).  python tools/bench_render.py [c2|c3] [--normals | --long]
--normals: n3d_render_rays_normals (renderer + normal pass) against n3d_render_rays on both the C2 and the C3 workload, and the
normal pass alone (n3d_render_normals_pass) and the gather-only floor.
--long: both entry points at 96 + 96, 144 + 144 and 192 + 192 samples per ray on the C2 and the C3 workload, alternated, in ms
and ms per million decoded samples."""
import sys, os, math, subprocess
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from next3d_b200 import config, weights, kernels as K
cfg = config.full_config(512)
args = [a for a in sys.argv[1:] if not a.startswith('--')]
which = args[0] if args else 'c2'


def _events(fn, reps, flush):
    ts = []
    for i in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn(i)
        e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def _card():
    power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                           capture_output=True, text=True).stdout.strip()
    print(f'card {torch.cuda.get_device_name()}  power limit {power or "unknown"}', flush=True)


if '--long' in sys.argv:
    # long rays (gen_videos_next3d.py --sample_mult 2 / 3 / 4): 96 + 96 runs the 32-lane layout, 144 + 144 and 192 + 192 the
    # 64-lane one.  Per workload the three counts are timed in alternated blocks (two rounds), for n3d_render_rays and
    # n3d_render_rays_normals; cost per million decoded samples = ms / (N * r^2 * (Dc + Df) / 1e6).
    _card()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
    for name, (N, R) in (('c2', (8, 64)), ('c3', (16, 128))):
        g = torch.Generator().manual_seed(0)
        planes = torch.randn(N, 3, 256, 256, 32, generator=g).cuda()
        dec = (torch.randn(64, 32, generator=g).cuda() / math.sqrt(32), torch.randn(64, generator=g).cuda() * 0.1,
               torch.randn(33, 64, generator=g).cuda() / math.sqrt(64), torch.randn(33, generator=g).cuda() * 0.1)
        _, _, c, _ = weights.demo_inputs(cfg, N)
        cam, intr = c[:, :16].contiguous().cuda(), c[:, 16:25].contiguous().cuda()
        rgb = torch.zeros(N, R * R, 32, device='cuda'); depth = torch.zeros(N, R * R, device='cuda'); wsum = torch.zeros_like(depth)
        mm = torch.tensor([float('inf'), 0.0], device='cuda')
        normal = torch.zeros(N, R * R, 3, device='cuda')
        counts = (96, 144, 192)
        opts = {D: dict(cfg.rendering_kwargs, depth_resolution=D, depth_resolution_importance=D) for D in counts}
        work = torch.empty(K.normals_workspace_floats(N, R, opts[counts[-1]]), device='cuda')
        fns = {}
        for D in counts:
            fns[D, 'rays'] = lambda i, o=opts[D]: K.render_rays(planes, cam, intr, R, o, dec, rgb, depth, wsum, mm, seed=i)
            fns[D, 'normals'] = lambda i, o=opts[D]: K.render_rays_normals(planes, cam, intr, R, o, dec, rgb, depth, wsum, mm, normal, work,
                                                                         seed=i)
        for f in fns.values():
            f(0); f(1)
        med = {key: [] for key in fns}
        for _ in range(2):                                  # alternated blocks: every (count, entry) once per round
            for key, f in fns.items():
                med[key].append(_events(f, 15, flush)[0])
        for entry in ('rays', 'normals'):
            base = None
            for D in counts:
                m = min(med[D, entry])
                per = m / (N * R * R * 2 * D / 1e6)
                base = per if base is None else base
                print(f'{name} N={N} r={R} {D}+{D} n3d_render_{entry if entry == "rays" else "rays_normals"}: median '
                      f'{" / ".join(f"{x:.3f}" for x in med[D, entry])} ms, {per:.4f} ms per 1e6 samples ({per / base:.2f}x the 96+96 cost)',
                      flush=True)
    sys.exit(0)

if '--normals' in sys.argv:
    _card()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
    for name, (N, R, D) in (('c2', (8, 64, 48)), ('c3', (16, 128, 96))):
        opts = dict(cfg.rendering_kwargs, depth_resolution=D, depth_resolution_importance=D)
        g = torch.Generator().manual_seed(0)
        planes = torch.randn(N, 3, 256, 256, 32, generator=g).cuda()
        dec = (torch.randn(64, 32, generator=g).cuda() / math.sqrt(32), torch.randn(64, generator=g).cuda() * 0.1,
               torch.randn(33, 64, generator=g).cuda() / math.sqrt(64), torch.randn(33, generator=g).cuda() * 0.1)
        _, _, c, _ = weights.demo_inputs(cfg, N)
        cam, intr = c[:, :16].contiguous().cuda(), c[:, 16:25].contiguous().cuda()
        rgb = torch.zeros(N, R * R, 32, device='cuda'); depth = torch.zeros(N, R * R, device='cuda'); wsum = torch.zeros_like(depth)
        mm = torch.tensor([float('inf'), 0.0], device='cuda')
        normal = torch.zeros(N, R * R, 3, device='cuda')
        work = torch.empty(K.normals_workspace_floats(N, R, opts), device='cuda')
        plain = lambda i: K.render_rays(planes, cam, intr, R, opts, dec, rgb, depth, wsum, mm, seed=i)
        normals = lambda i: K.render_rays_normals(planes, cam, intr, R, opts, dec, rgb, depth, wsum, mm, normal, work, seed=i)
        for i in range(3):
            plain(i); normals(i)
        tp = _events(plain, 15, flush)          # alternated blocks: plain, normals, plain, normals
        tn = _events(normals, 15, flush)
        tp2 = _events(plain, 15, flush)
        tn2 = _events(normals, 15, flush)
        p_med, n_med = min(tp[0], tp2[0]), min(tn[0], tn2[0])
        print(f'{name} N={N} r={R} D={D}+{D}: n3d_render_rays median {tp[0]:.3f} / {tp2[0]:.3f} ms, n3d_render_rays_normals median '
              f'{tn[0]:.3f} / {tn2[0]:.3f} ms, normal pass ~{n_med - p_med:.3f} ms ({n_med / p_med:.2f}x)', flush=True)
        # the normal pass alone on the samples the last call exported
        normals(0)
        alone = lambda i: K.render_normals_pass(planes, cam, intr, R, opts, dec, normal, work)
        alone(0)
        tr, tr2 = _events(alone, 15, flush), _events(alone, 15, flush)
        print(f'{name} normal pass alone: median {tr[0]:.3f} / {tr2[0]:.3f} ms; gather-only floor (n3d_render_floor kind 0, both passes) '
              f'{_events(lambda i: K.render_floor(planes, cam, intr, R, opts, 0, seed=i), 15, flush)[0]:.3f} ms', flush=True)
    sys.exit(0)
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
