"""A/B of the small-layer convolution launches (batch 8): one conv_gemm launch with the fused epilogue vs split-K (S K-slices writing raw
partial sums + n3d_splitk_epilogue).  CUDA-event timing, L2 flushed before every timed launch.  Usage (GPU box): python tools/bench_splitk.py"""
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from next3d_b200 import kernels as K

DEV = 'cuda'
flush = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)


def timeit(fn, reps=7):
    fn(); torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        flush.fill_(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def main():
    g = torch.Generator(device=DEV).manual_seed(1)
    N = int(os.environ.get('BATCH', '8'))
    for cin, cout, res in [(512, 512, 4), (512, 512, 8), (1024, 512, 8), (512, 512, 16), (1024, 512, 16), (512, 512, 32), (1024, 512, 32)]:
        x = torch.randn(N, res, res, cin, device=DEV, generator=g)
        hi, lo = K.split_bf16(x)
        w = torch.randn(cout, cin, 3, 3, device=DEV, generator=g) / (cin * 9) ** 0.5
        w_hi, w_lo = K.pack_conv_weight(w)
        o_hi = torch.empty(N, res, res, cout, device=DEV, dtype=torch.bfloat16)
        o_lo = torch.empty_like(o_hi)
        d = torch.rand(N, cout, device=DEV) + 0.5
        b = torch.randn(cout, device=DEV)
        st = torch.randn(N, cout, device=DEV)
        outs = [K.make_split_out(o_hi, o_lo, st, cout, 0)]
        base = timeit(lambda: K.conv_gemm(hi, lo, w_hi, w_lo, K.taps_conv3x3(), N, res, res, dcoef=d, bias=b, gain=math.sqrt(2), slope=0.2, clamp=256.0, outs=outs))
        ref_hi = o_hi.clone()
        line = f'{cin:4d}->{cout:3d} @{res:2d}^2 N={N}: fused {base:6.1f} us |'
        for S in (3, 9):
            part = torch.empty(S, N, res, res, cout, device=DEV)

            def run():
                K.conv_gemm(hi, lo, w_hi, w_lo, K.taps_conv3x3(), N, res, res, mode=1, out_f32=part, f32_cstride=cout, splits=S, split_stride=N * res * res * cout)
                K.splitk_epilogue(part, d, b, None, math.sqrt(2), 0.2, 256.0, outs=outs)
            t = timeit(run)
            diff = (o_hi.float() - ref_hi.float()).abs().max().item() / ref_hi.float().abs().max().item()
            line += f' S{S} {t:6.1f} ({diff:.0e})'
        print(line, flush=True)


if __name__ == '__main__':
    main()
