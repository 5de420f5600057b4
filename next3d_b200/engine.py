"""Generator engine: packs a reference state dict once and runs `TriPlaneGenerator.synthesis` as a fixed sequence of
libnext3d_b200 kernel launches (no ATen compute on the hot path; torch only owns the device buffers and the stream).

Execution model (see DESIGN.md):
  * all style vectors and demodulation coefficients of the ~70 modulated layers: 2 launches (n3d_styles, n3d_demod);
  * every convolution: n3d_conv_gemm (wgmma implicit GEMM, shared weights for the whole batch -- the algebraically
    equivalent non-fused form of networks_stylegan2.py:70-79: activations are pre-multiplied by the consumer's style,
    demodulation is applied in the epilogue), with noise / bias / lrelu / clamp / next-layer modulation / bf16 split fused;
  * up-convs: 4 parity-class GEMMs (stride-2 transposed conv, conv2d_resample.py:114-127) + one FIR-epilogue kernel;
  * down-convs: FIR + parity split kernel, then one GEMM over 9 unit-stride taps;
  * mesh path, volume renderer, resizes, blending: one kernel each (raster.cu, render_fused.cu);
  * super-resolution in fp16 (Engine.sr_precision = 'fp16', opt-in): the same launches on fp16 single activations and weights, one
    product per k-step: the reference's SR precision on CUDA with sr_num_fp16_res > 0, rounded at the engine's own points
    (INTEGRATION.md section 1).
Reference call order: triplane_next3d.py:117-188.
"""
import contextlib
import dataclasses
import math

import numpy as np
import torch

from . import config as _config
from . import kernels as K

SQRT2 = math.sqrt(2.0)
VIEWS = ((0, 0, 0), (0, 90, 0), (0, -90, 0), (90, 0, 0))      # triplane_next3d.py:140-145


def _angle2matrix(angles_deg):
    """fp32 sin/cos of angle*pi/180, rows [cz*cy, ...] (volumetric_rendering/renderer.py:518-547)."""
    a = torch.tensor(angles_deg, dtype=torch.float32).reshape(1, 3) * np.pi / 180.
    s, c = torch.sin(a), torch.cos(a)
    cx, cy, cz = c[0, 0], c[0, 1], c[0, 2]
    sx, sy, sz = s[0, 0], s[0, 1], s[0, 2]
    return torch.stack([cz * cy, cz * sy * sx - sz * cx, cz * sy * cx + sz * sx,
                        sz * cy, sz * sy * sx + cz * cx, sz * sy * cx - cz * sx,
                        -sy, cy * sx, cy * cx]).reshape(3, 3)


class Split:
    """bf16 (hi, lo) NHWC activation pair."""
    __slots__ = ('hi', 'lo')

    def __init__(self, shape, device):
        self.hi = torch.empty(shape, dtype=torch.bfloat16, device=device)
        self.lo = torch.empty(shape, dtype=torch.bfloat16, device=device)

    @property
    def C(self):
        return self.hi.shape[-1]


class Half:
    """fp16 single NHWC activation of the fp16 super-resolution head (lo is None: no second tensor)."""
    __slots__ = ('hi', 'lo')

    def __init__(self, shape, device):
        self.hi = torch.empty(shape, dtype=torch.float16, device=device)
        self.lo = None

    @property
    def C(self):
        return self.hi.shape[-1]


@dataclasses.dataclass(eq=False)
class _Layer:
    """A packed convolution layer, with the part of its epilogue that its place in the network fixes.  Engine.mod holds the
    modulated ones: SynthesisLayer (networks_stylegan2.py:311-330) and ToRGBLayer (:353-357, a 1x1 modulated conv without
    demodulation, linear bias + clamp).  Engine.plain holds the StyleUNet Conv2dLayers (networks_stylegan2_styleunet.py:198-207),
    their weight_gain folded into the packed weights."""
    name: str
    cin: int
    cout: int
    k: int
    w_hi: torch.Tensor                      # split bf16 [k*k, Cout, Cin]
    w_lo: torch.Tensor
    bias: torch.Tensor = None
    w_f32: torch.Tensor = None              # fp32 [Cout, Cin] of a ToRGB layer of <= 4 channels: the fused-ToRGB epilogue operand
    w16: torch.Tensor = None                # fp16 [k*k, Cout, Cin] of an SR conv, pre-normalised as for fp16 (Engine._pack)
    noise: torch.Tensor = None              # noise_const * noise_strength
    noise_strength: torch.Tensor = None
    clamp: float = -1.0                     # -1: no conv_clamp
    gain: float = 1.0                       # activation: lrelu (sqrt 2, 0.2) or linear (1, 1)
    slope: float = 1.0
    up: int = 1                             # 2: stride-2 transposed conv (SynthesisBlock conv0)
    down: int = 1                           # 2: stride-2 conv over the parity-split input (EncoderResBlock conv2)
    widx: int = -1                          # ws index of a modulated layer's style
    is_rgb: bool = False
    sbase: int = -1                         # element offsets (per N=1) of a modulated layer's style / dcoef blocks
    dbase: int = -1


class _BackboneCache(dict):
    """What synthesis(cache_backbone=True) keeps for a batch of B heads: (a) the two ws-only backbone outputs 'textures' and
    'static', (b) the blended 'planes' and (c) the call's 'ws' and 'noise_mode', in engine-owned buffers at fixed addresses, so that
    captured graphs can read and write them and no graph replay overwrites them.  use_cached_backbone=True re-runs everything but
    (a) (triplane.py:120-128 of EG3D); render_views renders new cameras from (b).  The cache lives until the next cache_backbone
    call with another batch size or the engine is rebuilt."""

    def __init__(self, B=0, textures=None, static=None, planes=None, ws=None):
        # noise_mode: the caching call's; None while nothing is cached
        super().__init__(B=B, textures=textures, static=static, planes=planes, ws=ws, noise_mode=None)

    @property
    def filled(self):
        return self['noise_mode'] is not None

    def fill(self, noise_mode):
        """Record that a caching call with `noise_mode` has written the buffers (run eagerly or replayed from a graph)."""
        self['noise_mode'] = noise_mode

    def views(self, N, views, mismatch):
        """Images per cached head for a call with N images, None while nothing is cached.  N must equal B or, where `views` are
        allowed, be a multiple B * V of it (image n reads head n // V); any other N raises RuntimeError(mismatch % (N, B))."""
        if not self.filled:
            return None
        B = self['B']
        if N % B if views else N != B:
            raise RuntimeError(mismatch % (N, B))
        return N // B


class Engine:
    # Split-K for the 3x3 layers up to 16^2: a batch of 8 gives 1-4 tiles of 128 pixels and a 72-step serial K loop (9 taps x 512
    # channels): the nine taps become nine concurrent work items per tile writing raw partial sums, summed in fixed order by
    # n3d_splitk_epilogue (deterministic; an atomics-based variant was rejected for run-to-run differences).  Chosen by resolution
    # only: the summation order of a sample must not depend on the batch size.
    splitk_maxres = 16

    def __init__(self, cfg, state_dict, device='cuda', nprod=3, uv_face_mask=None):
        if not torch.cuda.is_available():
            raise RuntimeError('next3d_b200.Engine needs a CUDA device (sm_90a); there is no CPU path')
        self.cfg, self.device, self.nprod = cfg, torch.device(device), nprod
        self.rk = cfg.rendering_kwargs
        self.mod, self.plain, self.consts = {}, {}, {}
        self.launches = 0                       # kernels launched by the last synthesis() / compute_planes() call (counted in kernels.py)
        self.conv_flops = 0.0
        self.prof = None
        self._cur_layer = ''                    # the layer whose launch is being set up (hooks on _noise read it)
        sd = {k: v.to(self.device, non_blocking=True) if isinstance(v, torch.Tensor) else v for k, v in state_dict.items()}
        self._pack(sd)
        self._tables = {}
        mask = torch.ones(1, 1, 256, 256) if uv_face_mask is None else uv_face_mask
        self.eye_mask = mask.reshape(mask.shape[-2], mask.shape[-1]).to(self.device, torch.float32).contiguous()
        self._mm_init = torch.tensor([float('inf'), 0.0], device=self.device)
        self._mm_init_image = torch.tensor([[float('inf'), float('-inf')]], device=self.device)     # one pair per image: repeat(N, 1)
        self._graphs = {}                       # key[0]: the graph reads or writes the backbone cache
        self._cache = _BackboneCache()          # allocated by the first cache_backbone call, see _cache_buffers
        self._side = None                      # side streams of the concurrent branches (compute_planes)
        self.concurrent = True                  # False: the three branches of compute_planes run on one stream (per-kernel timing)
        self.splitk = True                      # False: every conv runs as one conv_gemm pass (the reference of the split-K test)
        self.sr_precision = 'fp32'              # 'fp16': the super-resolution head on fp16 operands (TriPlaneGenerator.sr_precision)

    # ------------------------------------------------------------------------------------------ packing (one-time)
    def _add_mod(self, sd, name, cin, cout, k, up, widx, is_rgb=False, clamp=None, noise=True):
        w = sd[f'{name}.weight'].float()
        noise = noise and not is_rgb
        strength = sd[f'{name}.noise_strength'].float() if noise else None
        self.mod[name] = _Layer(
            name, cin, cout, k, *K.pack_conv_weight(w),
            bias=sd[f'{name}.bias'].float().contiguous(),
            w_f32=w.reshape(cout, cin).contiguous() if is_rgb and cout <= 4 else None,
            noise=(sd[f'{name}.noise_const'].float() * strength).contiguous() if noise else None,
            noise_strength=strength,
            clamp=-1.0 if clamp is None else clamp,
            gain=1.0 if is_rgb else SQRT2, slope=1.0 if is_rgb else 0.2,          # ToRGBLayer: linear, SynthesisLayer: lrelu
            up=up, widx=widx, is_rgb=is_rgb)

    def _add_plain(self, sd, name, k, lrelu=False, down=1):
        w = sd[f'{name}.weight'].float()
        cout, cin = w.shape[:2]
        b = sd.get(f'{name}.bias')
        self.plain[name] = _Layer(
            name, cin, cout, k, *K.pack_conv_weight(w, gain=1.0 / math.sqrt(cin * k * k)),      # Conv2dLayer.weight_gain
            bias=b.float().contiguous() if b is not None else None,
            gain=SQRT2 if lrelu else 1.0, slope=0.2 if lrelu else 1.0,
            down=down)

    def _pack_synthesis(self, sd, prefix, cimg, ws_off, first_res=4):
        cfg = self.cfg
        for res in _config.block_resolutions(cfg.plane_res):
            k = int(math.log2(res)) - 2
            start = 0 if res == 4 else 1 + 2 * (k - 1)
            cin = cfg.channels(res // 2) if res > 4 else 0
            cout = cfg.channels(res)
            p = f'{prefix}.b{res}'
            if res < first_res:
                continue                                   # e.g. mouth_backbone.b4 / neural_blending.b4..b32: never executed
            if res > 4:
                self._add_mod(sd, f'{p}.conv0', cin, cout, 3, 2, ws_off + start)
                self._add_mod(sd, f'{p}.conv1', cout, cout, 3, 1, ws_off + start + 1)
                self._add_mod(sd, f'{p}.torgb', cout, cimg, 1, 1, ws_off + start + 2, is_rgb=True)
            else:
                self._add_mod(sd, f'{p}.conv1', cout, cout, 3, 1, ws_off + 0)
                self._add_mod(sd, f'{p}.torgb', cout, cimg, 1, 1, ws_off + 1, is_rgb=True)
                self.consts[prefix] = sd[f'{p}.const'].float().permute(1, 2, 0).contiguous()      # [4,4,C] NHWC

    def _pack_unet(self, sd, prefix, in_size, final_size):
        enc = _config.encoder_resolutions(in_size, final_size)
        for i, _ in enumerate(enc[:-1]):
            self._add_plain(sd, f'{prefix}.encoder.{i}.fromrgb', 1)
            self._add_plain(sd, f'{prefix}.encoder.{i}.conv1', 3, lrelu=True)
            self._add_plain(sd, f'{prefix}.encoder.{i}.conv2', 3, lrelu=True, down=2)
        n_fusion = len(enc) - 1                            # the last fusion module (highest res) is never executed
        for i in range(n_fusion):
            self._add_plain(sd, f'{prefix}.fusion.{i}', 3)
        self._pack_synthesis(sd, prefix, self.cfg.plane_ch, 0, first_res=final_size * 2)

    def _pack(self, sd):
        cfg = self.cfg
        self._pack_synthesis(sd, 'texture_backbone.synthesis', cfg.plane_ch, 14)
        self._pack_synthesis(sd, 'backbone.synthesis', cfg.plane_ch * 3, 0)
        self._pack_unet(sd, 'mouth_backbone.synthesis', 64, 4)
        self._pack_unet(sd, 'neural_blending.synthesis', 256, 32)
        c0, c1 = _config.sr_channels(cfg)
        sr_up0 = 2 if cfg.sr_module == '8XDC' else 1
        for blk, (cin, cout, up) in enumerate([(cfg.plane_ch, c0, sr_up0), (c0, c1, 2)]):
            p = f'superresolution.block{blk}'
            noise = self.rk['superresolution_noise_mode'] != 'none'
            # ws = eg3d_ws[:, -1:].repeat(1, 3, 1) (superresolution.py:280): every SR layer reads ws index 13
            self._add_mod(sd, f'{p}.conv0', cin, cout, 3, up, 13, clamp=cfg.sr_clamp, noise=noise)
            self._add_mod(sd, f'{p}.conv1', cout, cout, 3, 1, 13, clamp=cfg.sr_clamp, noise=noise)
            self._add_mod(sd, f'{p}.torgb', cout, 3, 1, 1, 13, is_rgb=True, clamp=cfg.sr_clamp)
        # decoder (OSGDecoder, triplane_next3d.py:348-357): FullyConnectedLayer gains folded like its forward does
        self.dec = ((sd['decoder.net.0.weight'].float() * (1.0 / math.sqrt(32))).contiguous(), sd['decoder.net.0.bias'].float().contiguous(),
                    (sd['decoder.net.2.weight'].float() * (1.0 / math.sqrt(64))).contiguous(), sd['decoder.net.2.bias'].float().contiguous())
        # topology
        self.faces = sd['faces'][0][:, [0, 2, 1]].to(torch.int32).contiguous()                       # :207
        self.face_uv = sd['face_uvcoords'][0][:, [0, 2, 1], :2].float().contiguous()                # :208 (u, v)
        self.rot = torch.stack([_angle2matrix(a) for a in VIEWS]).to(self.device).contiguous()
        # concatenated affine tables (layer order fixed here)
        order = list(self.mod.values())
        sb = db = 0
        for L in order:
            L.sbase = sb
            sb += L.cin
            if not L.is_rgb:
                L.dbase = db
                db += L.cout
        self.style_elems, self.dcoef_elems = sb, db
        self.aff_w = torch.cat([sd[f'{L.name}.affine.weight'].float() for L in order], 0).contiguous()
        self.aff_b = torch.cat([sd[f'{L.name}.affine.bias'].float() for L in order], 0).contiguous()
        self.row_widx = torch.cat([torch.full((L.cin,), L.widx, dtype=torch.int32) for L in order]).to(self.device)
        self.row_scale = torch.cat([torch.full((L.cin,), (1.0 / math.sqrt(L.cin * L.k * L.k)) if L.is_rgb else 1.0) for L in order]).to(self.device)
        self.row_cin = torch.cat([torch.full((L.cin,), L.cin, dtype=torch.int32) for L in order]).to(self.device)
        dl = [L for L in order if not L.is_rgb]
        self.wsq = torch.cat([sd[f'{L.name}.weight'].float().square().sum(dim=[2, 3]).reshape(-1) for L in dl]).contiguous()   # [Cout, Cin] each
        woff, acc = [], 0
        for L in dl:
            woff.append(torch.arange(L.cout, dtype=torch.int64) * L.cin + acc)
            acc += L.cout * L.cin
        self.d_woff = torch.cat(woff).to(self.device)
        # fp16 SR: the reference pre-normalises each SR conv's weights for fp16, W * (1 / sqrt(Cin k^2) / max|W[o]|)
        # (networks_stylegan2.py:54-56).  The gain is folded into the fp16 weights and into their demodulation table wsq16;
        # demodulation cancels it, so only the fp16 rounding sees it.
        wsq16 = []
        for L in dl:
            w = sd[f'{L.name}.weight'].float()
            if L.name.startswith('superresolution.'):
                g = 1.0 / math.sqrt(L.cin * L.k * L.k) / w.abs().amax(dim=[1, 2, 3])
                L.w16 = K.pack_conv_weight_f16(w, g)
                w = w * g.reshape(-1, 1, 1, 1)
            wsq16.append(w.square().sum(dim=[2, 3]).reshape(-1))
        self.wsq16 = torch.cat(wsq16).contiguous()
        self.d_cin = torch.cat([torch.full((L.cout,), L.cin, dtype=torch.int32) for L in dl]).to(self.device)
        self.d_cout = torch.cat([torch.full((L.cout,), L.cout, dtype=torch.int32) for L in dl]).to(self.device)

    def _batch_tables(self, N):
        """Per-batch-size offset tables: every layer's style / dcoef block is dense [N, C] at base*N."""
        t = self._tables.get(N)
        if t is None:
            order = list(self.mod.values())
            s_ooff = torch.cat([torch.arange(L.cin, dtype=torch.int64) + L.sbase * N for L in order]).to(self.device)
            dl = [L for L in order if not L.is_rgb]
            d_soff = torch.cat([torch.full((L.cout,), L.sbase * N, dtype=torch.int64) for L in dl]).to(self.device)
            d_ooff = torch.cat([torch.arange(L.cout, dtype=torch.int64) + L.dbase * N for L in dl]).to(self.device)
            t = self._tables[N] = (s_ooff, d_soff, d_ooff)
        return t

    # ------------------------------------------------------------------------------------------ instrumentation
    def _prof_begin(self):
        if self.prof is None:
            return None
        e0 = torch.cuda.Event(enable_timing=True)
        e0.record()
        return e0

    def _prof_end(self, e0, kind, flops=0, info=None):
        if e0 is None:
            return
        e1 = torch.cuda.Event(enable_timing=True)
        e1.record()
        self.prof.append((kind, e0, e1, flops, info))

    def _timed(self, L, flops, M, ntaps, launch, *args, **kw):
        """launch(*args, **kw), one pass of layer L over an M x M space: adds its FLOPs to conv_flops and records it as a conv_gemm
        profiler entry with info (layer, Cin, Cout, MH, MW, taps), the row tools/profile_convs.py prints."""
        self.conv_flops += flops
        ev = self._prof_begin()
        launch(*args, **kw)
        self._prof_end(ev, 'conv_gemm', flops, (L.name, L.cin, L.cout, M, M, ntaps))

    def profile_summary(self):
        """After a synthesis() with self.prof = []: {kind: (launches, total_ms, total_flops)} (synchronises)."""
        torch.cuda.synchronize(self.device)
        out = {}
        for kind, e0, e1, fl, _ in self.prof or []:
            n, ms, f = out.get(kind, (0, 0.0, 0.0))
            out[kind] = (n + 1, ms + e0.elapsed_time(e1), f + fl)
        return out

    # ------------------------------------------------------------------------------------------ small helpers
    def _style(self, L):
        return self._styles[L.sbase * self._N: (L.sbase + L.cin) * self._N]

    def _dcoef(self, L):
        return self._dcoefs[L.dbase * self._N: (L.dbase + L.cout) * self._N]

    def _f32(self, *shape):
        return torch.empty(shape, dtype=torch.float32, device=self.device)

    def _noise(self, L, noise_mode):
        if L.noise is None or noise_mode == 'none':
            return None, 0
        if noise_mode == 'const':
            return L.noise, 0
        res = L.noise.shape[0]                               # 'random': per-sample noise (networks_stylegan2.py:318-319)
        return (torch.randn(self._N, res, res, device=self.device) * L.noise_strength).contiguous(), res * res

    def _out(self, buf, consumer=None, coff=0):
        """SplitOut descriptor writing into `buf` (Split, or Half: fp16 single) pre-multiplied by `consumer`'s style (None = unmodulated)."""
        style = self._style(self.mod[consumer]) if consumer else None
        return K.make_split_out(buf.hi, buf.lo, style, buf.C, coff, f16=buf.lo is None)

    # ------------------------------------------------------------------------------------------ layers
    def _epilogue(self, L, noise_mode='none', outs=(), f32=None, accumulate=False):
        """Layer L's epilogue under the keyword names conv_gemm, splitk_epilogue and fir_up_epilogue share: demodulation (SynthesisLayer),
        bias, noise, activation and clamp, then the split bf16 outputs `outs` and the fp32 NHWC output `f32`, which conv_gemm adds
        to with `accumulate`."""
        self._cur_layer = L.name
        noise, nstride = self._noise(L, noise_mode)
        return dict(dcoef=self._dcoef(L) if L.dbase >= 0 else None, bias=L.bias, noise=noise, noise_nstride=nstride, gain=L.gain,
                    slope=L.slope, clamp=L.clamp, outs=outs, out_f32=f32, f32_cstride=L.cout if f32 is not None else 0,
                    f32_accumulate=accumulate)

    def _fused_rgb(self, L, img, nchw=False):
        """Descriptor that folds ToRGBLayer L (<= 4 image channels) into the epilogue of the conv producing its input: img += torgb."""
        return dict(out=img, weight=L.w_f32, style=self._style(L), bias=L.bias, clamp=L.clamp, nchw=nchw, accumulate=True)

    def _conv(self, L, a, res, epi, rgb=None):
        """Layer L on the activation `a` (Split, or Half with L's fp16 weights; modulated layers: already pre-multiplied by L's style) at input resolution `res`, with
        the epilogue `epi` of _epilogue and the fused ToRGB `rgb` of _fused_rgb: a stride-2 transposed conv (4 parity classes into a
        raw sum, then the FIR-up epilogue), a stride-2 conv over the parity-split input, split-K (splitk_maxres), or one pass.
        Algorithmic FLOPs = 2 * Cin * Cout * taps * M-space positions (one product)."""
        N = self._N
        accumulate = epi.pop('f32_accumulate')                 # conv_gemm's alone: the split-K and FIR-up epilogues overwrite
        w_hi, w_lo, nprod = (L.w16, None, 1) if a.lo is None else (L.w_hi, L.w_lo, self.nprod)
        if L.up == 2:
            assert rgb is None and not accumulate
            raw = self._f32(N, 2 * res + 1, 2 * res + 1, L.cout)
            self._timed(L, 2.0 * L.cin * L.cout * N * (3 * res + 2) ** 2, res + 1, 9,       # taps x positions over the 4 parity classes
                        K.conv_transposed_gemm, a.hi, a.lo, w_hi, w_lo, N, res, res, raw, nprod=nprod)
            K.fir_up_epilogue(raw, L.cout, **epi)
            return
        M = res // L.down
        taps = K.taps_stride2() if L.down == 2 else K.taps_conv3x3() if L.k == 3 else K.taps_conv1x1()
        flops = 2.0 * L.cin * L.cout * len(taps) * N * M * M
        if L.k == 3 and L.down == 1 and self.splitk and res <= self.splitk_maxres and rgb is None and not accumulate:
            S = 9
            part = self._f32(S, N, res, res, L.cout)
            self._timed(L, flops, M, len(taps), K.conv_gemm, a.hi, a.lo, w_hi, w_lo, taps, N, M, M, nprod=nprod, mode=1,
                        out_f32=part, f32_cstride=L.cout, splits=S, split_stride=N * res * res * L.cout)
            self._timed(L, 0.0, M, 0, K.splitk_epilogue, part, **epi)         # the reduction is conv time (0 extra FLOPs)
            return
        self._timed(L, flops, M, len(taps), K.conv_gemm, a.hi, a.lo, w_hi, w_lo, taps, N, M, M, a_img_mul=N if L.down == 2 else 0,
                    nprod=nprod, rgb=rgb, f32_accumulate=accumulate, **epi)

    # ------------------------------------------------------------------------------------------ networks
    def _synthesis_blocks(self, prefix, x, res_list, cimg, noise_mode, concat_next=None, img=None):
        """Run SynthesisBlocks `res_list` (all with conv0 up) starting from split activation `x` (modulated for the first
        conv0) at resolution res_list[0]//2.  concat_next: {res: (concat Split buffer, fusion runner)} -- when the output of
        block `res` feeds a fusion conv (StyleUNet) instead of the next conv0 directly."""
        N, dev = self._N, self.device
        for i, res in enumerate(res_list):
            p = f'{prefix}.b{res}'
            conv0, conv1, torgb = self.mod[f'{p}.conv0'], self.mod[f'{p}.conv1'], self.mod[f'{p}.torgb']
            c = conv1.cout
            x1 = Split((N, res, res, c), dev)
            self._conv(conv0, x, res // 2, self._epilogue(conv0, noise_mode, [self._out(x1, f'{p}.conv1')]))
            nxt = res_list[i + 1] if i + 1 < len(res_list) else None
            rgb_in = Split((N, res, res, c), dev)
            outs = [self._out(rgb_in, f'{p}.torgb')]
            x = None
            if concat_next and res in concat_next:
                cat_buf, _ = concat_next[res]
                outs.append(K.make_split_out(cat_buf.hi, cat_buf.lo, None, cat_buf.C, 0))
            elif nxt is not None:
                x = Split((N, res, res, c), dev)
                outs.append(self._out(x, f'{prefix}.b{nxt}.conv0'))
            self._conv(conv1, x1, res, self._epilogue(conv1, noise_mode, outs))
            if img is None:
                img = self._f32(N, res, res, cimg)
                self._conv(torgb, rgb_in, res, self._epilogue(torgb, f32=img))
            else:
                up = self._f32(N, res, res, cimg)
                K.upsample2d_nhwc(img, up)
                self._conv(torgb, rgb_in, res, self._epilogue(torgb, f32=up, accumulate=True))
                img = up
            if concat_next and res in concat_next:
                x = concat_next[res][1]()                      # run the fusion conv, returns the next conv0's input
        return img

    def _backbone(self, prefix, cimg, noise_mode):
        """StyleGAN2 SynthesisNetwork (networks_stylegan2.py:630-645), 4 -> 256."""
        N, dev, cfg = self._N, self.device, self.cfg
        c4 = cfg.channels(4)
        const = self.consts[prefix][None].expand(N, -1, -1, -1).contiguous()
        conv1, torgb = self.mod[f'{prefix}.b4.conv1'], self.mod[f'{prefix}.b4.torgb']
        x0 = Split((N, 4, 4, c4), dev)
        K.modulate_split(const, self._style(conv1), x0.hi, x0.lo)
        rgb_in = Split((N, 4, 4, c4), dev)
        x = Split((N, 4, 4, c4), dev)
        self._conv(conv1, x0, 4, self._epilogue(conv1, noise_mode, [self._out(rgb_in, f'{prefix}.b4.torgb'), self._out(x, f'{prefix}.b8.conv0')]))
        img = self._f32(N, 4, 4, cimg)
        self._conv(torgb, rgb_in, 4, self._epilogue(torgb, f32=img))
        return self._synthesis_blocks(prefix, x, _config.block_resolutions(cfg.plane_res)[1:], cimg, noise_mode, img=img)

    def _styleunet(self, prefix, x_in, in_size, final_size, num_cond_res, noise_mode):
        """StyleUNet SynthesisNetwork.forward (networks_stylegan2_styleunet.py:554-588).  x_in: fp32 NHWC [N,in,in,32]."""
        N, dev, cfg = self._N, self.device, self.cfg
        enc_res = _config.encoder_resolutions(in_size, final_size)
        res_list = _config.block_resolutions(cfg.plane_res)
        start = int(math.log2(final_size)) - 1
        dec_res = res_list[start:]
        # which decoder levels get a condition: index j (block dec_res[j]) iff 2**(j + log2(final)) < num_cond_res
        n_cond = sum(1 for j in range(len(dec_res)) if 2 ** (j + int(math.log2(final_size))) < num_cond_res)
        # fusion j consumes cond_list[j] at resolution final_size * 2**j; for j >= 1 it is concatenated after the decoder's x
        cat = {}
        for j in range(1, n_cond):
            r = final_size * 2 ** j
            cat[j] = Split((N, r, r, 2 * cfg.channels(r)), dev)
        cond0 = Split((N, final_size, final_size, cfg.channels(final_size)), dev)
        # ---- encoder (EncoderResBlock.forward :107-115)
        skip = None
        x = x_in
        n_enc = len(enc_res) - 1
        for i, r in enumerate(enc_res[:-1]):
            p = f'{prefix}.encoder.{i}'
            fromrgb, conv1, conv2 = self.plain[f'{p}.fromrgb'], self.plain[f'{p}.conv1'], self.plain[f'{p}.conv2']
            cin = cfg.channels(r)
            if i > 0:
                xd = self._f32(N, r, r, cfg.plane_ch)
                K.downsample2d_nhwc(x, xd)
                x = xd
            xs = Split((N, r, r, cfg.plane_ch), dev)
            K.modulate_split(x, None, xs.hi, xs.lo)
            h = Split((N, r, r, cin), dev)
            if skip is None:
                self._conv(fromrgb, xs, r, self._epilogue(fromrgb, outs=[K.make_split_out(h.hi, h.lo, None, cin, 0)]))
            else:
                self._conv(fromrgb, xs, r, self._epilogue(fromrgb, f32=skip, accumulate=True))       # out = fromrgb(x) + skip
                K.modulate_split(skip, None, h.hi, h.lo)
            c1 = self._f32(N, r, r, cin)
            self._conv(conv1, h, r, self._epilogue(conv1, f32=c1))
            sh = (r + 2) // 2
            par = Split((4 * N, sh, sh, cin), dev)
            K.fir_down_split(c1, par.hi, par.lo)
            # cond of this block lives at resolution r/2; cond_list (reversed) index:
            j = n_enc - 1 - i
            cout = cfg.channels(r // 2)
            outs = []
            if j == 0:
                outs.append(K.make_split_out(cond0.hi, cond0.lo, None, cond0.C, 0))
            elif j < n_cond:
                outs.append(K.make_split_out(cat[j].hi, cat[j].lo, None, cat[j].C, cat[j].C - cout))
            skip = self._f32(N, r // 2, r // 2, cout) if i + 1 < n_enc else None
            self._conv(conv2, par, r, self._epilogue(conv2, outs=outs, f32=skip))
        # ---- decoder with fusion
        first = dec_res[0]
        x = Split((N, final_size, final_size, cfg.channels(final_size)), dev)
        fusion = self.plain[f'{prefix}.fusion.0']
        self._conv(fusion, cond0, final_size, self._epilogue(fusion, outs=[self._out(x, f'{prefix}.b{first}.conv0')]))
        concat_next = {}
        for j in range(1, n_cond):
            r = final_size * 2 ** j

            def run_fusion(j=j, r=r):
                y = Split((N, r, r, cfg.channels(r)), dev)
                fusion = self.plain[f'{prefix}.fusion.{j}']
                self._conv(fusion, cat[j], r, self._epilogue(fusion, outs=[self._out(y, f'{prefix}.b{2 * r}.conv0')]))
                return y
            concat_next[r] = (cat[j], run_fusion)
        return self._synthesis_blocks(prefix, x, dec_res, cfg.plane_ch, noise_mode, concat_next=concat_next)

    def _superresolution(self, feat, noise_mode_sr, image_out):
        """SuperresolutionHybrid8XDC / 4X (superresolution.py:77-88, 279-290).  feat: fp32 NHWC [N,R,R,32].  With sr_precision 'fp16'
        the activations between the SR convolutions are fp16 single tensors (x.to(float16) at each block's entry, networks_stylegan2.py:557)
        and the convolutions take the fp16 weights; the ToRGB sums, the skip image and `image_out` stay fp32."""
        N, dev, cfg = self._N, self.device, self.cfg
        f16 = self.sr_precision == 'fp16'
        Act = Half if f16 else Split
        R = feat.shape[1]
        p0, p1 = 'superresolution.block0', 'superresolution.block1'
        c0, c1 = _config.sr_channels(cfg)
        need = (R != 128) if cfg.sr_module == '8XDC' else (R < 128)
        r0 = 128 if need else R
        if need and R > 128 and not self.rk.get('sr_antialias', True):
            raise RuntimeError('next3d_b200: sr_antialias=False with a neural rendering resolution above 128 (a plain bilinear minification) is not '
                               'implemented')
        (b0_conv0, b0_conv1, b0_torgb), (b1_conv0, b1_conv1, b1_torgb) = [[self.mod[f'{p}.{n}'] for n in ('conv0', 'conv1', 'torgb')] for p in (p0, p1)]
        x = Act((N, r0, r0, cfg.plane_ch), dev)
        rgb_lo = feat[..., :3].contiguous()                                    # image_raw channels (tiny copy)
        if need:
            if f16:
                K.resize_aa_f16(feat, x.hi, style=self._style(b0_conv0))
            else:
                K.resize_aa(feat, None, r0, r0, style=self._style(b0_conv0), hi=x.hi, lo=x.lo)
            rgb = self._f32(N, r0, r0, 3)
            K.resize_aa(rgb_lo, rgb)
        else:
            if f16:
                K.modulate_f16(feat, self._style(b0_conv0), x.hi)
            else:
                K.modulate_split(feat, self._style(b0_conv0), x.hi, x.lo)
            rgb = rgb_lo
        # block0
        res0 = r0 * (2 if cfg.sr_module == '8XDC' else 1)
        x1 = Act((N, res0, res0, c0), dev)
        self._conv(b0_conv0, x, r0, self._epilogue(b0_conv0, noise_mode_sr, [self._out(x1, f'{p0}.conv1')]))
        x2 = Act((N, res0, res0, c0), dev)
        if cfg.sr_module == '8XDC':
            img = self._f32(N, res0, res0, 3)
            K.upsample2d_nhwc(rgb, img)
        else:
            img = rgb.clone()                                                   # SynthesisBlockNoUp: no image upsample
        # the two ToRGB layers (3 channels) run inside the conv1 epilogues: img += torgb(conv1 output)
        self._conv(b0_conv1, x1, res0, self._epilogue(b0_conv1, noise_mode_sr, [self._out(x2, f'{p1}.conv0')]), rgb=self._fused_rgb(b0_torgb, img))
        # block1
        res1 = res0 * 2
        x3 = Act((N, res1, res1, c1), dev)
        self._conv(b1_conv0, x2, res0, self._epilogue(b1_conv0, noise_mode_sr, [self._out(x3, f'{p1}.conv1')]))
        K.upsample2d_nhwc(img, image_out, y_nchw=True)
        self._conv(b1_conv1, x3, res1, self._epilogue(b1_conv1, noise_mode_sr, []), rgb=self._fused_rgb(b1_torgb, image_out, nchw=True))

    # ------------------------------------------------------------------------------------------ planes + synthesis
    def _on_device(self, **tensors):
        """Inputs must live on the engine's device: raw device pointers are handed to the C ABI, so a CPU or other-GPU tensor
        would become an illegal address instead of a clean error."""
        for name, t in tensors.items():
            if t is not None and t.device != self.device:
                raise RuntimeError(f'next3d_b200: `{name}` is on {t.device} but the generator runs on {self.device}; move it there '
                                   f'(there is no CPU path)')

    @contextlib.contextmanager
    def _entry(self, **inputs):
        """The bracket of an eager entry point: its tensor inputs must be on the engine's device, which is made current, and
        `launches` / `conv_flops` count what the call issues."""
        self._on_device(**inputs)
        with torch.cuda.device(self.device):
            n0, self.conv_flops = K.launches, 0.0
            yield
            self.launches = K.launches - n0

    def compute_planes(self, ws, v, noise_mode='const', return_intermediates=False):
        """Everything up to the blended tri-planes (triplane_next3d.py:137-174) -> [N,3,256,256,32] channels-last fp32."""
        with self._entry(ws=ws, v=v):
            return self._compute_planes(ws, v, noise_mode, return_intermediates)

    # ------------------------------------------------------------------------------------------ backbone cache (_BackboneCache)
    def _cache_buffers(self, B, ws_shape):
        """The cache buffers for batch B; a new B (or ws shape) reallocates them, which empties the cache and drops every graph that
        reads or writes them."""
        c = self._cache
        if c['ws'] is None or c['B'] != B or tuple(c['ws'].shape[1:]) != tuple(ws_shape[1:]):
            P, C = self.cfg.plane_res, self.cfg.plane_ch
            self._graphs = {k: g for k, g in self._graphs.items() if not k[0]}
            c = self._cache = _BackboneCache(B, textures=self._f32(B, P, P, C), static=self._f32(B, P, P, 3 * C),
                                             planes=self._f32(B, 3, P, P, C), ws=self._f32(B, *ws_shape[1:]))
        return c

    def _reused_views(self, N, use_cached_backbone, cache_backbone):
        """Images per cached head when a call of N images takes its backbones from the cache, None when it computes them.  A call
        that also refills the cache keeps N = B (the cache holds one set of planes per head)."""
        if not use_cached_backbone:
            return None
        return self._cache.views(N, not cache_backbone, 'next3d_b200: use_cached_backbone with batch %d, but the cached backbone holds batch %d')

    def _render_views_per_head(self, N):
        """Views per cached head for render_views of N cameras."""
        if not self._cache.filled:
            raise RuntimeError('next3d_b200: render_views needs cached planes: run synthesis(..., cache_backbone=True) first')
        return self._cache.views(N, True, 'next3d_b200: render_views got %d cameras, not a multiple of the cached batch %d')

    def _set_styles(self, ws):
        """Style vectors and demodulation coefficients of every modulated layer for the batch ws [N, L, D]."""
        N = ws.shape[0]
        self._N = N
        ws = ws.to(torch.float32).contiguous()
        s_ooff, d_soff, d_ooff = self._batch_tables(N)
        self._styles = self._f32(self.style_elems * N)
        self._dcoefs = self._f32(self.dcoef_elems * N)
        K.styles(ws, self.aff_w, self.aff_b, self.row_widx, self.row_scale, s_ooff, self.row_cin, self._styles)
        K.demod(self._styles, self.wsq16 if self.sr_precision == 'fp16' else self.wsq, self.d_woff, self.d_cin, d_soff, d_ooff, self.d_cout, self._dcoefs, N)

    def _compute_planes(self, ws, v, noise_mode='const', return_intermediates=False, cache_backbone=False, use_cached_backbone=False):
        cfg, dev = self.cfg, self.device
        N = ws.shape[0]
        P = cfg.plane_res
        # N = B * V images on a cache of B heads: image n takes its texture and static planes from head n // V
        reuse = self._reused_views(N, use_cached_backbone, cache_backbone)
        V = reuse or 1
        v = v.to(torch.float32)
        verts, lms = v[:, :5023].contiguous(), v[:, 5023:].contiguous()
        self._set_styles(ws)
        # Three independent branches (triplane_next3d.py:137-170): (1) neural texture -> UV lookup -> mouth / blending UNets,
        # (2) mesh rasterization + mouth box (needs only the vertices), (3) the static tri-plane backbone (needed only by the final
        # blend).  (2) and (3) run on side streams: their latency-bound kernels (4^2..32^2 layers on a few dozen SMs, the flood
        # fill, the rasterizer) fill SMs the main branch leaves idle and vice versa.  Captured as parallel graph branches.
        main = torch.cuda.current_stream(dev)
        if self.concurrent:
            if self._side is None:
                self._side = (torch.cuda.Stream(dev), torch.cuda.Stream(dev))
            s_rast, s_static = self._side
            s_rast.wait_stream(main)
            s_static.wait_stream(main)
        else:
            s_rast = s_static = main
        with torch.cuda.stream(s_rast):
            tv = self._f32(N, 4, verts.shape[1], 3)
            K.transform_points(verts, self.rot, 10.0, True, tv)
            tl = self._f32(N, 4, lms.shape[1], 3)
            K.transform_points(lms, self.rot, 0.0, False, tl)
            p2f = torch.empty(N * 4, P, P, dtype=torch.int32, device=dev)
            bary = self._f32(N * 4, P, P, 3)
            K.rasterize(tv.view(N * 4, -1, 3), self.faces, P, P, p2f, bary)
            boxes = torch.empty(N, 4, dtype=torch.int32, device=dev)
            lm2d = tl[:, 0, :, :2].contiguous()
            K.mouth_box(lm2d, boxes)
        if reuse is None:
            with torch.cuda.stream(s_static):
                static = self._backbone('backbone.synthesis', cfg.plane_ch * 3, noise_mode)         # [N,256,256,96]
            textures = self._backbone('texture_backbone.synthesis', cfg.plane_ch, noise_mode)      # [N,256,256,32]
        else:
            static, textures = self._cache['static'], self._cache['textures']
        if self.concurrent:
            main.wait_stream(s_rast)
            for t in (p2f, bary, boxes, lm2d):
                t.record_stream(main)
        # look up texture + eye mask at the rasterized UVs, fill the mouth hole; the side plane's alpha (images N .. 2N - 1 of
        # alpha) ends binary, as the reference's (alpha.bool() | alpha.bool()).float() leaves it (triplane_next3d.py:226)
        tex_planes = self._f32(3, N, P, P, cfg.plane_ch)
        alpha = self._f32(3, N, P, P)
        K.uv_sample(p2f, bary, self.face_uv, textures, self.eye_mask, tex_planes, alpha, views=V)
        K.fill_mouth(alpha, binarize=(N, 2 * N))
        # mouth crop -> StyleUNet -> paste back -> neural blending
        front = tex_planes[0]
        crop = self._f32(N, 64, 64, cfg.plane_ch)
        K.resize_aa(front, crop, src_box=boxes)
        mouth = self._styleunet('mouth_backbone.synthesis', crop, 64, 4, 64, noise_mode)
        stitched = front.clone()
        K.resize_aa(mouth, stitched, dst_box=boxes)
        blended = self._styleunet('neural_blending.synthesis', stitched, 256, 32, 256, noise_mode)
        if self.concurrent and reuse is None:
            main.wait_stream(s_static)
            static.record_stream(main)
        planes = self._f32(N, 3, P, P, cfg.plane_ch)
        K.blend_planes(blended, tex_planes, alpha, static, planes, views=V)
        if cache_backbone:
            c = self._cache_buffers(N, ws.shape)
            if reuse is None:
                c['textures'].copy_(textures)
                c['static'].copy_(static)
                c.fill(noise_mode)
            c['planes'].copy_(planes)
            c['ws'].copy_(ws)
        if return_intermediates:
            return planes, dict(textures=textures, pix_to_face=p2f.view(N, 4, P, P), tex_planes=tex_planes, alpha=alpha, boxes=boxes,
                                mouth_crop=crop, mouth_plane=mouth, stitched=stitched, blended_front=blended, static=static, lm2d=lm2d)
        return planes

    def synthesis(self, ws, c, v, noise_mode='const', neural_rendering_resolution=None, sampler_noise=None, seed=0,
                  return_intermediates=False, seed_ptr=None, cache_backbone=False, use_cached_backbone=False, depth_range='batch'):
        """cache_backbone: also keep the backbone outputs, planes and ws (see _cache_buffers); use_cached_backbone: take the two
        ws-only backbones from that cache (no cache = computed as usual): N = B * V images on a cache of batch B, image n reading
        head n // V (N = B when cache_backbone is also set; any other batch raises).  depth_range: 'batch'
        clamps every image's depth to the range of the whole call (ray_marcher.py:54 on a batch), 'image' to the image's own range
        (what a call per image gives)."""
        with self._entry(ws=ws, c=c, v=v):
            depth_range = _depth_range(depth_range)
            R = neural_rendering_resolution or self.cfg.neural_rendering_resolution
            out = self._compute_planes(ws, v, noise_mode, return_intermediates, cache_backbone, use_cached_backbone)
            planes, inter = out if return_intermediates else (out, None)
            result, feat, wsum, ws_normals = self._render(planes, c, R, sampler_noise, seed, seed_ptr, depth_range=depth_range)
        if return_intermediates:
            inter.update(planes=planes, feature_image=feat, weights_sum=wsum)
            if ws_normals is not None:                                      # per ray: D sorted sample depths, then D - 1 final weights
                inter['normal_samples'] = ws_normals.view(feat.shape[0], R * R, -1)
            result['intermediates'] = inter
        return result

    def _render(self, planes, c, R, sampler_noise, seed, seed_ptr, views=1, depth_range='batch'):
        """Volume rendering, depth clamp and super-resolution of N = planes.shape[0] * views images (image n reads plane set
        n // views) with the current batch's styles -> (synthesis output dict, feature image, weight sums, normal workspace).
        depth_range 'image': one (min, max) pair per image, each image clamped to its own."""
        cfg, dev = self.cfg, self.device
        N = planes.shape[0] * views
        c = c.to(torch.float32)
        cam = c[:, :16].contiguous()
        intr = c[:, 16:25].contiguous()
        M = R * R
        feat = self._f32(N, R, R, cfg.plane_ch)                                 # [N, M, 32] == NHWC feature image
        depth = self._f32(N, 1, R, R)
        wsum = self._f32(N, M)
        per_image = int(depth_range == 'image')
        if per_image:                                                       # running (min, max) of each image's sample depths
            mm = self._mm_init_image.repeat(N, 1)
        else:
            mm = self._mm_init.clone()                                      # running (min, max) of all sample depths
        u_c, u_f = sampler_noise if sampler_noise is not None else (None, None)
        if u_c is not None:
            u_c, u_f = u_c.to(dev, torch.float32).contiguous(), u_f.to(dev, torch.float32).contiguous()
        normal = self._f32(N, M, 3) if self.rk.get('return_normal', False) else None
        ws_normals = None
        ev = self._prof_begin()
        if normal is None:
            K.render_rays(planes, cam, intr, R, self.rk, self.dec, feat, depth, wsum, mm, u_coarse=u_c, u_fine=u_f, seed=seed, seed_ptr=seed_ptr,
                          views=views, depth_range_per_image=per_image)
        else:                                                               # return_normal (renderer.py:271-355, ray_marcher.py:61-64)
            ws_normals = self._f32(K.normals_workspace_floats(N, R, self.rk))
            K.render_rays_normals(planes, cam, intr, R, self.rk, self.dec, feat, depth, wsum, mm, normal, ws_normals, u_coarse=u_c, u_fine=u_f,
                                  seed=seed, seed_ptr=seed_ptr, views=views, depth_range_per_image=per_image)
        self._prof_end(ev, 'render_rays')
        if per_image:
            K.depth_clamp_images(depth, mm)
        else:
            K.depth_clamp(depth, mm)
        image = self._f32(N, 3, cfg.img_resolution, cfg.img_resolution)
        self._superresolution(feat, self.rk['superresolution_noise_mode'], image)
        result = {'image': image, 'image_raw': feat.permute(0, 3, 1, 2)[:, :3], 'image_depth': depth}
        if normal is not None:
            result['image_normal'] = normal.view(N, R, R, 3).permute(0, 3, 1, 2)          # ray m = i * R + j -> pixel (i, j)
        return result, feat, wsum, ws_normals

    def render_views(self, c, neural_rendering_resolution=None, sampler_noise=None, seed=0, seed_ptr=None, depth_range='batch'):
        """New camera views of the cached heads: c [N, 25] with N = B * V for a cache of batch B; view n belongs to head n // V.
        Renders from the cached planes and runs super-resolution with the cached ws; returns what synthesis returns (depth_range as
        there: 'image' gives every view its own depth range)."""
        with self._entry(c=c):
            depth_range = _depth_range(depth_range)
            V = self._render_views_per_head(c.shape[0])
            R = neural_rendering_resolution or self.cfg.neural_rendering_resolution
            ws = self._cache['ws']
            self._set_styles(ws[:, None].expand(ws.shape[0], V, *ws.shape[1:]).reshape(-1, *ws.shape[1:]))     # ws of head n // V
            return self._render(self._cache['planes'], c, R, sampler_noise, seed, seed_ptr, views=V, depth_range=depth_range)[0]

    def cached_sigma_grid(self, b, shape_res, sigma):
        """The shape-extraction density grid of cached head b (gen_samples_next3d.py:208-238: create_samples at box_warp, sigma
        flipped along axis 0 and trimmed) written into sigma, float32 [shape_res]^3 on the engine's device, from the planes the
        caching call kept: one n3d_sample_grid launch, no backbone.  Raises RuntimeError when nothing is cached or b is not a cached head."""
        c = self._cache
        if not c.filled:
            raise RuntimeError('next3d_b200: cached_sigma_grid needs cached planes: run synthesis(..., cache_backbone=True) first')
        if not 0 <= b < c['B']:
            raise RuntimeError(f'next3d_b200: cached_sigma_grid of head {b}, but the cache holds {c["B"]} head(s)')
        self._on_device(sigma=sigma)
        if sigma.dtype != torch.float32 or tuple(sigma.shape) != (shape_res,) * 3 or not sigma.is_contiguous():
            raise RuntimeError(f'next3d_b200: cached_sigma_grid needs a contiguous float32 [{shape_res}]^3 output, got {sigma.dtype} '
                               f'{tuple(sigma.shape)}')
        box = self.rk['box_warp']
        with torch.cuda.device(self.device):
            K.sample_grid(c['planes'][b], shape_res, box * 1, box, self.dec, sigma, pad=int(30 * shape_res / 256))

    def cached_sample_points(self, b, coords):
        """The decoder at world points coords float32 [P, 3] of cached head b (G.sample's run_model on the planes the caching call
        kept) -> (sigma [P], features [P, K.POINT_FEATURES], the width n3d_sample_points writes whatever the plane channels).  The
        first three features are the decoder's colour, sigmoid(x) * 1.002 - 0.001; image_raw shows them as 2 f - 1 (the ray
        marcher's rescaling of its composite).  One n3d_sample_points launch."""
        c = self._cache
        if not c.filled:
            raise RuntimeError('next3d_b200: cached_sample_points needs cached planes: run synthesis(..., cache_backbone=True) first')
        if not 0 <= b < c['B']:
            raise RuntimeError(f'next3d_b200: cached_sample_points of head {b}, but the cache holds {c["B"]} head(s)')
        self._on_device(coords=coords)
        coords = coords.to(torch.float32).contiguous()
        P = coords.shape[0]
        sigma, feat = self._f32(1, P), self._f32(1, P, K.POINT_FEATURES)
        if P:
            with torch.cuda.device(self.device):
                K.sample_points(c['planes'][b:b + 1], coords.view(1, P, 3), self.rk['box_warp'], self.dec, sigma, feat)
        return sigma[0], feat[0]

    # ------------------------------------------------------------------------------------------ CUDA graph replay
    def _render_key(self, R):
        """The part of a graph key every graphed call shares: the rendering options a captured graph bakes in and the SR precision.
        It first refuses the options the renderer lacks, which the eager call would refuse."""
        rk = self.rk
        K.check_render_options(rk)
        return (R, rk['depth_resolution'], rk['depth_resolution_importance'], float(rk['ray_start']), float(rk['ray_end']), float(rk['box_warp']),
                bool(rk.get('white_back', False)), rk['superresolution_noise_mode'], bool(rk.get('sr_antialias', True)),
                bool(rk.get('return_normal', False)), self.sr_precision)

    def _settings_key(self):
        """The convolution settings a captured graph bakes in (each changes the result).  `concurrent` is not part of any key: the
        branches' stream layout does not change the result."""
        return (bool(self.splitk), self.splitk_maxres, self.nprod)

    def _replay(self, key, inputs, run, seed):
        """Capture run(static inputs) once per key into a CUDA graph and replay it: inputs are copied into static buffers (plus a
        device seed counter for the in-kernel sampler RNG); the returned tensors are the graph's static outputs and are overwritten
        by the next call with the same key."""
        g = self._graphs.get(key)
        if g is None:
            st = {k: torch.empty(t.shape, dtype=torch.float32, device=self.device) for k, t in inputs.items()}
            st['seed'] = torch.zeros(1, dtype=torch.int64, device=self.device)
            for k, t in inputs.items():
                st[k].copy_(t)
            side = torch.cuda.Stream(self.device)
            side.wait_stream(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(side):                                   # warm-up outside capture (lazy attribute setup, allocator)
                run(st)
            torch.cuda.current_stream(self.device).wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                out = run(st)
            g = self._graphs[key] = (graph, st, out, self.launches, self.conv_flops)
        graph, st, out, launches, flops = g
        for k, t in inputs.items():
            st[k].copy_(t, non_blocking=True)
        bits = K.seed_bits(seed)                                            # the int64 counter holds the seed's 64-bit pattern
        st['seed'].fill_(bits - (1 << 64) if bits >> 63 else bits)
        graph.replay()
        self.launches, self.conv_flops = launches, flops
        return out

    # The graphed entry points capture the eager one (its Python does not run on a replay, so what it records on the engine --
    # launches, conv_flops, a filled cache -- is restored or re-recorded after each replay).
    def synthesis_graphed(self, ws, c, v, noise_mode='const', neural_rendering_resolution=None, seed=0, cache_backbone=False,
                          use_cached_backbone=False, depth_range='batch'):
        """Same as synthesis() (in-kernel sampler RNG) but the ~200 launches of one forward are captured once per
        (batch, cached batch, resolution, noise_mode, cache use) into a CUDA graph and replayed: removes the host-side launch latency that otherwise
        leaves the GPU idle between kernels.  The cache-using graphs read and write the engine's cache buffers in place."""
        depth_range = _depth_range(depth_range)
        self._on_device(ws=ws, c=c, v=v)
        with torch.cuda.device(self.device):
            N = ws.shape[0]
            R = neural_rendering_resolution or self.cfg.neural_rendering_resolution
            render_key = self._render_key(R) + self._settings_key()      # refuses unsupported options before the cache is touched
            reuse = self._reused_views(N, use_cached_backbone, cache_backbone) is not None
            if cache_backbone:
                self._cache_buffers(N, ws.shape)          # allocated before capture: the graph writes the cache at fixed addresses
            B = self._cache['B'] if reuse else N             # (N, B): the images per cached head of a reusing graph
            key = (cache_backbone or reuse, cache_backbone, reuse, N, B, noise_mode, tuple(v.shape), depth_range) + render_key

            def run(st):
                return self.synthesis(st['ws'], st['c'], st['v'], noise_mode, R, seed=0, seed_ptr=st['seed'], cache_backbone=cache_backbone,
                                      use_cached_backbone=reuse, depth_range=depth_range)
            out = self._replay(key, dict(ws=ws, c=c, v=v), run, seed)
            if cache_backbone and not reuse:
                self._cache.fill(noise_mode)
            return out

    def render_views_graphed(self, c, neural_rendering_resolution=None, seed=0, depth_range='batch'):
        """render_views() replayed from a CUDA graph per (N, V, resolution, depth range, rendering options); in-kernel sampler RNG."""
        self._on_device(c=c)
        depth_range = _depth_range(depth_range)
        with torch.cuda.device(self.device):
            V = self._render_views_per_head(c.shape[0])
            R = neural_rendering_resolution or self.cfg.neural_rendering_resolution
            key = (True, 'views', c.shape[0], V, depth_range) + self._render_key(R) + self._settings_key()
            return self._replay(key, dict(c=c), lambda st: self.render_views(st['c'], R, seed=0, seed_ptr=st['seed'], depth_range=depth_range),
                                seed)


def _depth_range(depth_range):
    """The `depth_range` keyword: 'batch' (one depth range per call) or 'image' (one per image)."""
    if depth_range not in ('batch', 'image'):
        raise ValueError(f"depth_range must be 'batch' or 'image', got {depth_range!r}")
    return depth_range
