"""CPU: the fp16 super-resolution statement (oracle/sr_fp16.py) against the reference's own SR blocks run in fp16.

The reference runs an SR block in fp16 only on a CUDA device (networks_stylegan2.py:547-548: `if ws.device.type != 'cuda':
force_fp32 = True`).  Here its blocks run on CPU with that one check answered 'cuda' (a ws whose `device` says so and that is a
plain tensor to every op), which is otherwise the reference's fp16 forward: fp16 activations, pre-normalised fp16 modulated weights,
fp16 convolutions, the clamp at 256.  On CPU its ops take their reference fallbacks, which round at the points
`sr_fp16.superresolution(..., plugins=False)` follows (the module docstring names the one difference from the CUDA plugins:
_bias_act_ref rounds after each op).  What the reference computed is stored in tests/golden/reference_sr_fp16.npz (every 4th pixel
of `image`, tests.helpers.ReferenceVectors; N3D_RECORD_REFERENCE=1 recomputes it where the reference can be imported).

Two fp16 computations of the same head that round at slightly different points differ by whole fp16 ulps at a few pixels, so the
max error cannot pin one to the other; the mean error does.  Measured on the stored pixels (4X / 8XDC): statement mean 4.0e-5 /
5.1e-5 of the range (max 5.2e-4 / 8.2e-4), the fp32 oracle 2.3e-4 / 2.7e-4; on the full image, the statement with the CUDA plugins'
rounding is 1.8e-4 / 2.6e-4."""
import pytest
import torch

from next3d_b200 import config, weights
from oracle import generator as og
from oracle import ref_shim, sr_fp16
from tests.helpers import ReferenceVectors

REF = ReferenceVectors('reference_sr_fp16')
MEAN_BOUND = 1e-4           # mean |statement - reference| / max|reference|
MAX_BOUND = 2e-3            # max, the same normalisation: a few fp16 ulps of the ToRGB output


class _ReportsCuda(torch.Tensor):
    """A tensor whose `device` reads as CUDA and that is a plain CPU tensor to every op (results are plain tensors)."""

    @property
    def device(self):
        return torch.device('cuda')

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        plain = lambda a: a.as_subclass(torch.Tensor) if isinstance(a, cls) else a   # noqa: E731
        with torch._C.DisableTorchFunctionSubclass():
            return func(*(plain(a) for a in args), **{k: plain(v) for k, v in (kwargs or {}).items()})


def _case(res):
    cfg = config.tiny_config(res)
    sd = weights.make_state_dict(cfg, seed=2)
    g = torch.Generator().manual_seed(5)
    feat = torch.rand(1, 32, 64, 64, generator=g)
    ws = torch.randn(1, 14, 512, generator=g)
    return cfg, sd, feat, ws


def _reference(res):
    """SuperresolutionHybrid8XDC / 4X.forward (superresolution.py:279-290, :77-88) with the blocks called directly, so that they
    receive the ws whose device reads as CUDA (the forward's own slicing of ws would drop it)."""
    cfg, sd, feat, ws = _case(res)
    G = ref_shim.build_reference_generator(cfg)
    G.load_state_dict(sd)
    sr = G.superresolution
    w3 = ws[:, -1:, :].repeat(1, 3, 1).as_subclass(_ReportsCuda)
    x, rgb = feat, feat[:, :3]
    if (x.shape[-1] != 128) if res == 512 else (x.shape[-1] < 128):
        x = torch.nn.functional.interpolate(x, size=(128, 128), mode='bilinear', align_corners=False, antialias=True)
        rgb = torch.nn.functional.interpolate(rgb, size=(128, 128), mode='bilinear', align_corners=False, antialias=True)
    with torch.no_grad():
        x, rgb = sr.block0(x, rgb, w3, noise_mode='none')
        assert x.dtype == torch.float16                  # the block did run in fp16
        _, img = sr.block1(x, rgb, w3, noise_mode='none')
    return img


def _errs(a, ref):
    d = (a.double() - ref.double()).abs() / ref.double().abs().max()
    return d.mean().item(), d.max().item()


@pytest.mark.parametrize('res', [256, 512])
def test_fp16_statement_matches_reference_fp16_forward(res):
    ref = REF.get(f'image_s4_{res}', lambda: _reference(res)[..., ::4, ::4])
    cfg, sd, feat, ws = _case(res)
    with torch.no_grad():
        st = sr_fp16.superresolution(sd, cfg, feat[:, :3], feat, ws, plugins=False)[..., ::4, ::4]
        f32 = og.superresolution(sd, cfg, feat[:, :3], feat, ws)[..., ::4, ::4]
    mean, mx = _errs(st, ref)
    mean32, _ = _errs(f32, ref)
    print(f'{res}: statement vs reference fp16: mean {mean:.2e} max {mx:.2e}; fp32 oracle mean {mean32:.2e}')
    assert mean < MEAN_BOUND and mx < MAX_BOUND, (mean, mx)
    assert mean < mean32 / 3, (mean, mean32)                 # the pin tells the fp16 forward from the fp32 one
