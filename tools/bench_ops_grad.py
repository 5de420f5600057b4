"""Forward + backward of torch_utils.ops.conv2d_resample (+ bias_act) on generator-shaped layers, against the reference route on
the same GPU: torch.nn.functional conv / conv_transpose autograd (cuDNN, fp32, TF32 off) with the impl='ref' ops.  Reports the wall
time of one forward + backward, and the n3d_conv_wgrad kernel's time (CUDA events around the launch) and achieved rate counting
3 bf16 products per multiply-add.  Prints the card name and power limit first.
Usage (GPU box): python tools/bench_ops_grad.py [--reps R]"""
import argparse
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import next3d_b200.torch_utils.ops as ops                       # noqa: E402
from next3d_b200 import kernels as K                            # noqa: E402
from next3d_b200.torch_utils.ops import conv2d_resample as cr   # noqa: E402

DEV = 'cuda'

# name, N, groups, Cin per group, Cout per group, resolution (input), k, up, down
LAYERS = [
    ('backbone 3x3 128->128 @256', 1, 1, 128, 128, 256, 3, 1, 1),
    ('SR 3x3 128->128 @512 N=1', 1, 1, 128, 128, 512, 3, 1, 1),
    ('modconv 3x3 256->256 @64 groups=N=8', 1, 8, 256, 256, 64, 3, 1, 1),
    ('up-conv 3x3 256->128 @128->256', 1, 1, 256, 128, 128, 3, 2, 1),
    ('down-conv 3x3 128->256 @256->128', 1, 1, 128, 256, 256, 3, 1, 2),
    ('ToRGB 1x1 128->3 @256 groups=N=8', 1, 8, 128, 3, 256, 1, 1, 1),
]


def ref_conv(x, w, f, up, down, groups, k):
    """The reference route: conv2d_resample.py through torch autograd, the FIR steps as impl='ref' upfirdn2d."""
    p = k // 2
    if up == 2:
        cout_g, cin_g = w.shape[0] // groups, w.shape[1]
        wt = w.reshape(groups, cout_g, cin_g, k, k).transpose(1, 2).reshape(groups * cin_g, cout_g, k, k).flip([2, 3])
        y = F.conv_transpose2d(x, wt, stride=2, groups=groups)
        return ops.upfirdn2d.upfirdn2d(y, f, padding=[1, 1, 1, 1], gain=4, impl='ref')
    if down == 2:
        x = ops.upfirdn2d.upfirdn2d(x, f, padding=[2, 2, 2, 2], impl='ref')
        return F.conv2d(x, w, stride=2, groups=groups)
    return F.conv2d(x, w, padding=p, groups=groups)


def wall(fn, reps):
    fn(); torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def wgrad_kernel_ms(x, dy, f, kind, k, groups, reps):
    """Median time of the n3d_conv_wgrad launch(es) alone on the operands the backward builds."""
    calls = []
    orig = K.conv_wgrad

    def capture(*a, **kw):
        calls.append((a, kw))
        return orig(*a, **kw)

    K.conv_wgrad = capture
    try:
        with torch.no_grad():
            cr._weight_grad(x, dy, f, kind, k, groups)
    finally:
        K.conv_wgrad = orig
    a, kw = calls[0]
    ts = []
    for _ in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); orig(*a, **kw); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts = sorted(ts[1:])
    G, M, Nn, Kp, a_off = a[4], a[5], a[6], a[7], a[8]
    macs = G * len(a_off) * M * Nn * Kp
    return ts[len(ts) // 2], 3 * 2 * macs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    args = ap.parse_args()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    print(f'# card: {q.stdout.strip() or torch.cuda.get_device_name()}')
    f = ops.upfirdn2d.setup_filter([1, 3, 3, 1], device=DEV)
    g = torch.Generator(device=DEV).manual_seed(0)
    print(f'{"layer":40s} {"ours fwd+bwd ms":>16s} {"ref fwd+bwd ms":>15s} {"wgrad ms":>9s} {"wgrad TFLOP/s":>14s}')
    for name, N, groups, cin, cout, res, k, up, down in LAYERS:
        x = torch.randn(N, cin * groups, res, res, device=DEV, generator=g)
        w = torch.randn(cout * groups, cin, k, k, device=DEV, generator=g) / (cin * k * k) ** 0.5
        b = torch.randn(cout * groups, device=DEV, generator=g)
        res_out = res * up // down
        dy = torch.randn(N, cout * groups, res_out, res_out, device=DEV, generator=g)
        xg, wg, bg = x.clone().requires_grad_(), w.clone().requires_grad_(), b.clone().requires_grad_()

        def ours():
            y = ops.conv2d_resample.conv2d_resample(xg, wg, f=f, up=up, down=down, padding=k // 2, groups=groups, flip_weight=(up == 1))
            y = ops.bias_act.bias_act(y, bg, act='lrelu')
            torch.autograd.grad(y, [xg, wg, bg], dy)

        def ref():
            y = ref_conv(xg, wg, f, up, down, groups, k)
            y = ops.bias_act.bias_act(y, bg, act='lrelu', impl='ref')
            torch.autograd.grad(y, [xg, wg, bg], dy)

        t_ours, t_ref = wall(ours, args.reps), wall(ref, args.reps)
        kind = 'up' if up == 2 else 'down' if down == 2 else 'same'
        with torch.no_grad():
            d = torch.nn.functional.leaky_relu(dy, 0.2)          # a stand-in output gradient of the conv (same shape)
        t_w, flops = wgrad_kernel_ms(x, d, f, kind, k, groups, args.reps)
        print(f'{name:40s} {t_ours:16.3f} {t_ref:15.3f} {t_w:9.3f} {flops / t_w / 1e9:14.1f}')


if __name__ == '__main__':
    main()
