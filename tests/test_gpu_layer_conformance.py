"""Every layer the engine runs, checked as it runs against an fp64 statement of the reference's layer on the inputs the engine gave it.

`TriPlaneGenerator.synthesis` runs eagerly on one stream (Engine.concurrent = False) with hooks on Engine._conv, kernels.make_split_out
and the glue entry points the engine calls between its convolutions (modulate_split, modulate_f16, fir_down_split, upsample2d_nhwc,
downsample2d_nhwc, resize_aa, resize_aa_f16).  Each step clones what it reads, runs, and is compared at once with fp64 statements of

    SynthesisLayer   y = bias_act(conv2d_resample(a, W, up) * d + noise, b, lrelu, sqrt 2, clamp),  a = x * s,
                     d = rsqrt(sum (W * s)^2 + 1e-8)                                  (networks_stylegan2.py:311-330)
    ToRGBLayer       bias_act(conv1x1(a, W), b, linear, clamp), s with the 1 / sqrt(Cin) gain     (:353-357)
    Conv2dLayer      bias_act(conv2d_resample(x, W / sqrt(Cin k^2), down), b, linear | lrelu)   (networks_stylegan2_styleunet.py:198-207)

and of the glue (oracle.ops upsample2d / downsample2d / upfirdn2d, fp64 antialiased F.interpolate).  The styles are fp64 affine
outputs of the ws row the oracle feeds each layer (tests.helpers.oracle_widx), never the engine's.  Each step starts from the engine's
own input, so errors do not compound and the bounds sit near the kernels' own.

What the engine decides, and how it is checked:
  * which buffer a step reads: every traced write labels its buffer with the step's name (a glue write with kind(label of its input));
    a step's input must carry the label producer_table names, built from the reference's data flow.  Buffers no traced step wrote (the
    const input, the mouth crop, the rendered feature image, ...) read as INPUT.  The trace holds every buffer it labels, so no address
    is reused while it runs;
  * which style a split output is pre-multiplied by: a split output must equal the reference times the fp64 style of the layer that
    reads it, and the layer that reads it must be one the reference feeds from that producer (a plain or concat consumer: no style);
  * concat halves: a concat buffer's label is the tuple of its writers in channel order, which must be (decoder x, encoder cond);
  * each epilogue's demodulation, bias, noise, gain, slope and clamp: part of the statement the output is compared with;
  * accumulation: an accumulating fp32 output equals its previous contents (cloned before the step) plus the reference, and those
    contents must carry the label the reference adds onto; the fused ToRGB image equals the previous image plus clamp(torgb(y));
  * each traced synthesis runs every executed convolutional layer exactly once, and every split output is read exactly once.

CPU tests pin the statements to oracle.generator in fp64, check that producer_table names every convolution of config.param_spec, and that
the hot super-resolution biases make the clamp fire on both sides in every SR layer.
"""
import copy
import dataclasses
import math

import pytest
import torch
import torch.nn.functional as F

from next3d_b200 import config, weights
from oracle import ops as oo
from tests.helpers import HOT_CONV_BIAS, HOT_RGB_BIAS, RangeErr, hot_sr_state_dict, oracle_widx, record_errors

DEV = 'cuda'
INPUT = '<input>'               # the label of a buffer no traced step wrote

# Error bounds, range-relative (max |got - ref| / max |ref|) per output of a step, each at most 4x the worst case measured over the
# workloads below on an H100 80GB HBM3 (700 W power limit), which is given beside it.  N3D_LAYER_ERRORS=<file> appends every measured
# worst case to that file as JSON lines.
BOUNDS = {
    'split': 8e-5,          # bf16 (hi, lo) outputs times the consumer's style.  Worst: 3.9e-5 (full512, fusion.3 -> b64.conv0 of the mouth)
    'f32': 5e-5,            # fp32 outputs, accumulated ones included.  Worst: 2.2e-5 (full512, mouth encoder.0.conv2: from the fp32
                            # input of its FIR-down, through the bf16 split of the parity images)
    'rgb': 3e-5,            # the fused-ToRGB skip image.  Worst: 1.2e-5 (full512, superresolution.block0.torgb)
    'glue': 2e-5,           # modulate, FIR-down split, up/downsample, resize.  Worst: 7.4e-6 (tiny512_random, the mouth's encoder.0
                            # FIR-down split)
    # The fp16 super-resolution head against the same fp64 statement: the bounds follow from fp16 rounding (unit roundoff u = 2^-11 =
    # 4.9e-4), not from the split.  A glue output is rounded once (<= u).  A convolution's output is rounded once, and its weights are
    # rounded to fp16 (each <= u, through the sum); its input is the engine's own, so its rounding does not count.
    'split16': 3 * 2 ** -11,    # 3u = 1.5e-3.  Worst: 6.7e-4 (hot_fp16, superresolution.block1.conv0 -> block1.conv1)
    'rgb16': 2 * 2 ** -11,      # 2u: the fp32 ToRGB of an fp16 convolution's fp32 output (weights rounded, output not).  Worst: 2.6e-4
                                # (hot_fp16, superresolution.block0.torgb)
    'glue16': 6e-4,             # u, plus the fp32 resize / modulation before the rounding.  Worst: 3.8e-4 (tiny512_fp16, resize_aa_f16)
}


# ------------------------------------------------------------------------------------------------ fp64 layer statements
def synthesis_layer(a, weight, s, bias, f, up=1, noise=None, clamp=None):
    """SynthesisLayer on the pre-modulated input a = x * s (NCHW): conv2d_resample(a, W, up) * d + noise, then lrelu * sqrt 2 and the
    clamp, with d = rsqrt(sum (W * s)^2 + 1e-8).  up = 2 is the transposed conv + FIR of conv2d_resample with flip_weight False, as
    modulated_conv2d calls it."""
    d = ((weight[None] * s[:, None, :, None, None]).square().sum(dim=[2, 3, 4]) + 1e-8).rsqrt()
    y = oo.conv2d_resample(a, weight, f=f, up=up, padding=weight.shape[-1] // 2, flip_weight=(up == 1)) * d[:, :, None, None]
    if noise is not None:
        y = y + noise
    return oo.bias_act(y, bias, act='lrelu', clamp=clamp)


def torgb_layer(a, weight, bias, clamp=None):
    """ToRGBLayer on a = x * s, s including the 1 / sqrt(Cin) style gain: a 1x1 conv without demodulation, bias, the clamp."""
    return oo.bias_act(F.conv2d(a, weight), bias, clamp=clamp)


def conv2d_layer(x, weight, bias, f, down=1, lrelu=False):
    """StyleUNet Conv2dLayer: weight gain 1 / sqrt(Cin k^2), FIR then stride 2 for down = 2, linear or lrelu * sqrt 2."""
    k = weight.shape[-1]
    w = weight * (1.0 / math.sqrt(weight.shape[1] * k * k))
    y = oo.conv2d_resample(x, w, f=f, down=down, padding=k // 2, flip_weight=True)
    return oo.bias_act(y, bias, act='lrelu' if lrelu else 'linear')


def fir_down_split_reference(x, f):
    """n3d_fir_down_split of x (NCHW): FIR pad 2 -> (H+1) x (W+1), a zero row and column appended, split by pixel parity ->
    [4, N, C, SH, SW] (parity (y & 1) * 2 + (x & 1))."""
    fo = F.pad(oo.upfirdn2d(x, f, padding=2), (0, 1, 0, 1))
    return torch.stack([fo[:, :, a::2, b::2] for a in (0, 1) for b in (0, 1)])


def resize_reference(x, size):
    """The SR head's antialiased bilinear resize in fp64 (on the CPU, where F.interpolate's antialias path takes fp64)."""
    return F.interpolate(x.cpu(), size=size, mode='bilinear', align_corners=False, antialias=True).to(x.device)


# ------------------------------------------------------------------------------------------------ the reference's data flow
def conv_layers(cfg):
    """Every convolution weight of config.param_spec, by layer name."""
    return [name[:-len('.weight')] for name, shape, kind, _ in config.param_spec(cfg) if kind == 'weight' and len(shape) == 4]


def producer_table(cfg, R=None, sr_fp16=False):
    """{convolutional layer of config.param_spec: None when the reference never runs it, else dict(inp=what it reads, onto=the fp32
    buffer it adds into, or None)}.  What a layer reads is named as the trace labels it: the name of the layer that wrote it, kind(x)
    for a glue launch on x, INPUT for a buffer no layer wrote, and a tuple (first half, second half) for a torch.cat.  Follows
    oracle.generator: backbone / synthesis_block, styleunet and superresolution.  R: the neural rendering resolution."""
    R = R or cfg.neural_rendering_resolution
    res_list = config.block_resolutions(cfg.plane_res)
    table = dict.fromkeys(conv_layers(cfg))

    def block(p, res, x, img):
        """synthesis_block: conv0 (up) on x, conv1, torgb onto the upsampled image.  -> (x, img) labels after the block."""
        table[f'{p}.b{res}.conv0'] = dict(inp=x, onto=None)
        table[f'{p}.b{res}.conv1'] = dict(inp=f'{p}.b{res}.conv0', onto=None)
        table[f'{p}.b{res}.torgb'] = dict(inp=f'{p}.b{res}.conv1', onto=f'upsample2d({img})' if img else None)
        return f'{p}.b{res}.conv1', f'{p}.b{res}.torgb'

    def backbone(p):
        table[f'{p}.b4.conv1'] = dict(inp=f'modulate_split({INPUT})', onto=None)          # the const, modulated
        table[f'{p}.b4.torgb'] = dict(inp=f'{p}.b4.conv1', onto=None)
        x, img = f'{p}.b4.conv1', f'{p}.b4.torgb'
        for res in res_list[1:]:
            x, img = block(p, res, x, img)

    def styleunet(p, in_size, final_size, num_cond_res):
        enc = config.encoder_resolutions(in_size, final_size)
        x, cond, cond_list = INPUT, None, []
        for i, res in enumerate(enc[:-1]):
            e = f'{p}.encoder.{i}'
            if res < in_size:
                x = f'downsample2d({x})'
            table[f'{e}.fromrgb'] = dict(inp=f'modulate_split({x})', onto=cond)           # out = fromrgb(x) + cond
            table[f'{e}.conv1'] = dict(inp=f'{e}.fromrgb' if cond is None else f'modulate_split({e}.fromrgb)', onto=None)
            table[f'{e}.conv2'] = dict(inp=f'fir_down_split({e}.conv1)', onto=None)
            cond = f'{e}.conv2'
            cond_list.append(cond)
        cond_list = cond_list[::-1]
        start = int(math.log2(final_size)) - 1
        x = img = None
        for index, res in enumerate(res_list[start:]):
            if 2 ** (index + int(math.log2(final_size))) < num_cond_res:
                table[f'{p}.fusion.{index}'] = dict(inp=cond_list[0] if index == 0 else (x, cond_list[index]), onto=None)
                x = f'{p}.fusion.{index}'
            x, img = block(p, res, x, img)

    def superresolution():
        need = R != 128 if cfg.sr_module == '8XDC' else R < 128
        if sr_fp16:
            x = f'resize_aa_f16({INPUT})' if need else f'modulate_f16({INPUT})'
        else:
            x = f'resize_aa({INPUT})' if need else f'modulate_split({INPUT})'
        rgb = f'resize_aa({INPUT})' if need else INPUT
        # 8XDC: the image is upsampled into block0; 4X: block0 (SynthesisBlockNoUp) adds onto a copy of the resized image
        img = f'upsample2d({rgb})' if cfg.sr_module == '8XDC' else INPUT
        p = 'superresolution'
        table[f'{p}.block0.conv0'] = dict(inp=x, onto=None)
        table[f'{p}.block0.conv1'] = dict(inp=f'{p}.block0.conv0', onto=None)
        table[f'{p}.block0.torgb'] = dict(inp=f'{p}.block0.conv1', onto=img)
        table[f'{p}.block1.conv0'] = dict(inp=f'{p}.block0.conv1', onto=None)
        table[f'{p}.block1.conv1'] = dict(inp=f'{p}.block1.conv0', onto=None)
        table[f'{p}.block1.torgb'] = dict(inp=f'{p}.block1.conv1', onto=f'upsample2d({p}.block0.torgb)')

    backbone('texture_backbone.synthesis')
    styleunet('mouth_backbone.synthesis', 64, 4, 64)
    styleunet('neural_blending.synthesis', 256, 32, 256)
    backbone('backbone.synthesis')
    superresolution()
    return table


def consumers(table, label):
    """The layers that read the buffer labelled `label` in the reference."""
    return [c for c, e in table.items() if e and (e['inp'] == label or isinstance(e['inp'], tuple) and label in e['inp'])]


# ------------------------------------------------------------------------------------------------ the trace
class Trace:
    """Hooks that check each step of one synthesis call as it runs (see the module docstring).  kinds: {kind: [worst error, step]};
    problems: what disagreed with the reference's data flow; ran: {layer: times run}; clamped: {SR layer: (fraction >= 256, fraction
    <= -256)} of the reference's outputs."""

    def __init__(self, cfg, sd, ws, noise_mode, R, sr_fp16):
        self.cfg, self.noise_mode, self.sr_fp16 = cfg, noise_mode, sr_fp16
        self.table = producer_table(cfg, R, sr_fp16)
        self.sd = sd
        self.ws = ws.double()
        self.widx = oracle_widx(cfg)
        self.f = oo.setup_filter([1, 3, 3, 1]).double().to(DEV)
        self.labels = {}                    # data_ptr -> [record]; a record: dict(label, coff, width, kind, errs, reads, src)
        self.keep = []                      # every labelled buffer: no address is reused while the trace runs
        self.descs = {}                     # id(SplitOut) -> (hi, lo, coff, f16)
        self.kinds, self.problems, self.ran, self.clamped = {}, [], {}, {}
        self.net = None                     # the network being run (Engine._backbone, _styleunet, _superresolution)
        self._p64 = {}

    # ---- reference inputs
    def p64(self, key):
        t = self._p64.get(key)
        if t is None:
            t = self._p64[key] = self.sd[key].to(DEV, torch.float64)
        return t

    def style(self, name):
        """fp64 style of modulated layer `name` from the ws row the oracle feeds it (ToRGB: times 1 / sqrt(Cin)); None for a plain layer."""
        if name not in self.widx:
            return None
        s = oo.fully_connected(self.ws[:, self.widx[name]], self.p64(f'{name}.affine.weight'), self.p64(f'{name}.affine.bias'))
        if name.endswith('.torgb'):
            s = s / math.sqrt(self.sd[f'{name}.weight'].shape[1])
        return s

    def clamp(self, name):
        return self.cfg.sr_clamp if name.startswith('superresolution.') else None

    def sr16(self, name):
        return self.sr_fp16 and name.startswith('superresolution.')

    # ---- bookkeeping
    def problem(self, msg):
        self.problems.append(msg)

    @staticmethod
    def err(got, ref):
        e = RangeErr()
        e.add(got, ref)
        return e.value()

    def count(self, kind, step, e):
        worst = self.kinds.setdefault(kind, [0.0, None])
        if not e <= worst[0]:
            worst[:] = [e, step]

    def label(self, t):
        recs = self.labels.get(t.data_ptr())
        if not recs:
            return INPUT
        recs = sorted(recs, key=lambda r: r['coff'])
        return recs[0]['label'] if len(recs) == 1 else tuple(r['label'] for r in recs)

    def put(self, t, label, kind, coff=0, width=None, errs=None, src=None, holders=()):
        width = t.shape[-1] if width is None else width
        old = [r for r in self.labels.get(t.data_ptr(), []) if r['coff'] + r['width'] <= coff or r['coff'] >= coff + width]
        self.labels[t.data_ptr()] = old + [dict(label=label, kind=kind, coff=coff, width=width, errs=errs, reads=0, src=src)]
        self.keep += [t, *holders]

    def forget(self, t):
        self.labels.pop(t.data_ptr(), None)

    def read(self, t, reader, expected):
        """A step `reader` reads split buffer t: its label must be `expected`, its channels must be tiled by its writes, and each write's
        error against `reader`'s style counts."""
        got = self.label(t)
        if got != expected:
            self.problem(f'{reader} reads {got!r}; the reference feeds it {expected!r}')
            return []
        recs = sorted(self.labels[t.data_ptr()], key=lambda r: r['coff'])
        edges = [0] + [r['coff'] + r['width'] for r in recs]
        if [r['coff'] for r in recs] != edges[:-1] or edges[-1] != t.shape[-1]:
            self.problem(f'{reader} reads a buffer of {t.shape[-1]} channels written at {[(r["coff"], r["width"]) for r in recs]}')
        for r in recs:
            r['reads'] += 1
            if r['errs'] is not None:
                e = r['errs'].get(reader)
                if e is None:
                    self.problem(f'{reader} reads the output of {r["label"]}, which the reference feeds to {list(r["errs"])}')
                else:
                    self.count(r['kind'], f'{r["label"]} -> {reader}', e)
        return recs

    # ---- split outputs
    def split_value(self, hi, lo, coff, width, f16):
        v = hi[..., coff:coff + width].double()
        return v if f16 else v + lo[..., coff:coff + width].double()

    def write_split(self, writer, label, kind, hi, lo, coff, f16, ref_nhwc, src=None):
        """A split output of `writer` holding ref_nhwc (fp64 NHWC, before any style): its error against every layer the reference feeds
        from `label`, each times that layer's style."""
        width = ref_nhwc.shape[-1]
        if tuple(hi.shape[:-1]) != tuple(ref_nhwc.shape[:-1]):
            self.problem(f'{writer} writes a {tuple(hi.shape)} buffer; the reference output is {tuple(ref_nhwc.shape)}')
            return
        got = self.split_value(hi, lo, coff, width, f16)
        errs = {}
        for c in consumers(self.table, label):
            s = self.style(c)
            if s is not None and s.shape[-1] != width:
                continue                    # another network's layer with the same kind of input: it cannot read this one
            errs[c] = self.err(got, ref_nhwc * s[:, None, None, :] if s is not None else ref_nhwc)
        if not errs:
            self.problem(f'{writer} writes a split output, but the reference reads {label} nowhere')
        self.put(hi, label, kind, coff, width, errs, src, holders=(lo,) if lo is not None else ())

    # ---- hooks
    def conv(self, orig, E, L, a, res, epi, rgb=None):
        name = L.name
        self.ran[name] = self.ran.get(name, 0) + 1
        entry = self.table.get(name)
        if entry is None:
            self.problem(f'{name} runs, but the reference never runs it')
            return orig(E, L, a, res, epi, rgb)
        accumulate = epi['f32_accumulate']
        recs = self.read(a.hi, name, entry['inp'])
        out32 = epi['out_f32']
        prev32 = out32.double() if accumulate else None
        if accumulate != (entry['onto'] is not None):
            self.problem(f'{name}: accumulate={accumulate}; the reference adds onto {entry["onto"]}')
        if accumulate and self.label(out32) != entry['onto']:
            self.problem(f'{name} adds onto {self.label(out32)!r}; the reference adds onto {entry["onto"]!r}')
        if L.down == 2:
            src = recs[0]['src'] if recs else None          # the fp32 input of the fir_down_split that made the parity images
            a64 = None
        else:
            a64 = (a.hi.double() if a.lo is None else a.hi.double() + a.lo.double()).permute(0, 3, 1, 2)
        noise = epi['noise'].double() if epi['noise'] is not None and epi['noise_nstride'] else None
        rgb_prev = rgb['out'].double() if rgb is not None else None
        rgb_label = self.label(rgb['out']) if rgb is not None else None
        outs = [self.descs[id(o)] for o in epi['outs']]
        orig(E, L, a, res, epi, rgb)

        # the reference output of the layer, fp64 NCHW
        W = self.p64(f'{name}.weight')
        bias = self.p64(f'{name}.bias') if f'{name}.bias' in self.sd else None
        if name in self.widx and not name.endswith('.torgb'):
            mode = self.cfg.rendering_kwargs['superresolution_noise_mode'] if name.startswith('superresolution.') else self.noise_mode
            if mode == 'const':
                ref_noise = (self.p64(f'{name}.noise_const') * self.p64(f'{name}.noise_strength'))[None, None]
            elif mode == 'random':
                if noise is None:
                    self.problem(f'{name} draws no per-sample noise in noise_mode random')
                ref_noise = noise[:, None] if noise is not None else None
            else:
                ref_noise = None
            y = synthesis_layer(a64, W, self.style(name), bias, self.f, up=L.up, noise=ref_noise, clamp=self.clamp(name))
        elif name.endswith('.torgb'):
            y = torgb_layer(a64, W, bias, clamp=self.clamp(name))
        else:
            leaf = name.rsplit('.', 1)[1]
            lrelu = leaf in ('conv1', 'conv2')
            if L.down == 2:
                if src is None:
                    self.problem(f'{name} reads parity images no fir_down_split made')
                    return
                y = conv2d_layer(src, W, bias, self.f, down=2, lrelu=True)
            else:
                y = conv2d_layer(a64, W, bias, self.f, lrelu=lrelu)
        y_nhwc = y.permute(0, 2, 3, 1)
        if name.startswith('superresolution.'):
            self.clamped[name] = ((y >= 256).double().mean().item(), (y <= -256).double().mean().item())
        sr16 = self.sr16(name)

        for hi, lo, coff, f16 in outs:
            self.write_split(name, name, 'split16' if sr16 else 'split', hi, lo, coff, f16, y_nhwc)
        if out32 is not None:
            ref = y_nhwc + prev32 if accumulate else y_nhwc
            if out32.shape != ref.shape:
                self.problem(f'{name} writes fp32 {tuple(out32.shape)}; the reference output is {tuple(ref.shape)}')
            else:
                self.count('f32', name, self.err(out32, ref))
            self.put(out32, name, 'f32')
        if rgb is not None:
            t = name.rsplit('.', 1)[0] + '.torgb'
            self.ran[t] = self.ran.get(t, 0) + 1
            te = self.table.get(t)
            if te is None or te['inp'] != name:
                self.problem(f'the ToRGB fused into {name} is {t}, which the reference does not feed from {name}')
                return
            if rgb_label != te['onto']:
                self.problem(f'{t} adds onto {rgb_label!r}; the reference adds onto {te["onto"]!r}')
            tr = torgb_layer(y * self.style(t)[:, :, None, None], self.p64(f'{t}.weight'), self.p64(f'{t}.bias'), clamp=self.clamp(t))
            self.clamped[t] = ((tr >= 256).double().mean().item(), (tr <= -256).double().mean().item())
            img = rgb_prev.permute(0, 2, 3, 1) + tr.permute(0, 2, 3, 1) if rgb['nchw'] else rgb_prev + tr.permute(0, 2, 3, 1)
            got = rgb['out'].permute(0, 2, 3, 1) if rgb['nchw'] else rgb['out']
            self.count('rgb16' if sr16 else 'rgb', t, self.err(got, img))
            self.put(rgb['out'], t, 'rgb')

    def glue_split(self, kind, x, ref_nhwc, hi, lo, coff, f16, src=None):
        label = f'{kind}({self.label(x)})'
        self.write_split(kind, label, 'glue16' if f16 else 'glue', hi, lo, coff, f16, ref_nhwc, src)

    def glue_f32(self, kind, x, y, ref):
        label = f'{kind}({self.label(x)})'
        self.count('glue', label, self.err(y, ref))
        self.put(y, label, 'f32')


def _nchw(x):
    return x.double().permute(0, 3, 1, 2)


def install(monkeypatch, tr):
    """Hook the engine and the glue entry points it calls into trace `tr`."""
    from next3d_b200 import engine as eng_mod, kernels as K
    Engine = eng_mod.Engine

    orig_conv = Engine._conv
    monkeypatch.setattr(Engine, '_conv', lambda self, L, a, res, epi, rgb=None: tr.conv(orig_conv, self, L, a, res, epi, rgb))

    def network(fn_name):
        orig = getattr(Engine, fn_name)

        def run(self, *args, **kw):
            tr.net = fn_name
            try:
                return orig(self, *args, **kw)
            finally:
                tr.net = None
        monkeypatch.setattr(Engine, fn_name, run)
    for fn_name in ('_backbone', '_styleunet', '_superresolution'):
        network(fn_name)

    make = K.make_split_out

    def make_split_out(hi=None, lo=None, style=None, cstride=0, coff=0, f16=False):
        d = make(hi, lo, style, cstride, coff, f16)
        tr.descs[id(d)] = (hi, lo, coff, bool(f16))
        tr.keep.append(d)                   # keeps id(d) unique while the trace runs
        return d
    monkeypatch.setattr(K, 'make_split_out', make_split_out)

    def hook(fn_name, traced):
        orig = getattr(K, fn_name)

        def run(*args, **kw):
            if tr.net is None:              # the mouth crop and paste-back resizes: not part of the convolutional networks
                out = orig(*args, **kw)
                for t in list(args) + list(kw.values()):
                    if isinstance(t, torch.Tensor):
                        tr.forget(t)
                return out
            return traced(orig, *args, **kw)
        monkeypatch.setattr(K, fn_name, run)

    def modulate_split(orig, x, style, hi, lo, cstride=None, coff=0):
        x64 = x.double()
        orig(x, style, hi, lo, cstride, coff)
        tr.glue_split('modulate_split', x, x64, hi, lo, coff, False)

    def modulate_f16(orig, x, style, out, cstride=None, coff=0):
        x64 = x.double()
        orig(x, style, out, cstride, coff)
        tr.glue_split('modulate_f16', x, x64, out, None, coff, True)

    def fir_down_split(orig, x, hi, lo):
        x64 = _nchw(x)
        orig(x, hi, lo)
        N = x.shape[0]
        ref = fir_down_split_reference(x64, tr.f)                           # [4, N, C, SH, SW]
        ref = ref.permute(0, 1, 3, 4, 2).reshape(4 * N, *ref.shape[3:], ref.shape[2])
        tr.glue_split('fir_down_split', x, ref, hi, lo, 0, False, src=x64)

    def upsample2d_nhwc(orig, x, y, y_nchw=False):
        x64 = _nchw(x)
        orig(x, y, y_nchw)
        ref = oo.upsample2d(x64, tr.f).permute(0, 2, 3, 1)
        tr.glue_f32('upsample2d', x, y.permute(0, 2, 3, 1) if y_nchw else y, ref)

    def downsample2d_nhwc(orig, x, y):
        x64 = _nchw(x)
        orig(x, y)
        tr.glue_f32('downsample2d', x, y, oo.downsample2d(x64, tr.f).permute(0, 2, 3, 1))

    def resize_aa(orig, src, dst=None, DH=None, DW=None, src_box=None, dst_box=None, style=None, hi=None, lo=None):
        assert src_box is None and dst_box is None
        x64 = _nchw(src)
        orig(src, dst, DH, DW, src_box, dst_box, style, hi, lo)
        size = tuple(dst.shape[1:3]) if dst is not None else (DH, DW)
        ref = resize_reference(x64, size).permute(0, 2, 3, 1)
        if hi is not None:
            tr.glue_split('resize_aa', src, ref, hi, lo, 0, False)
        if dst is not None:
            tr.glue_f32('resize_aa', src, dst, ref)

    def resize_aa_f16(orig, src, out, src_box=None, dst_box=None, style=None):
        assert src_box is None and dst_box is None
        x64 = _nchw(src)
        orig(src, out, src_box, dst_box, style)
        tr.glue_split('resize_aa_f16', src, resize_reference(x64, tuple(out.shape[1:3])).permute(0, 2, 3, 1), out, None, 0, True)

    for fn_name, traced in (('modulate_split', modulate_split), ('modulate_f16', modulate_f16), ('fir_down_split', fir_down_split),
                            ('upsample2d_nhwc', upsample2d_nhwc), ('downsample2d_nhwc', downsample2d_nhwc), ('resize_aa', resize_aa),
                            ('resize_aa_f16', resize_aa_f16)):
        hook(fn_name, traced)


# ------------------------------------------------------------------------------------------------ workloads
def _cfg(factory, res, R=None, sr_noise=None, sr_num_fp16_res=4):
    cfg = factory(res)
    rk = copy.deepcopy(cfg.rendering_kwargs)
    if sr_noise:
        rk['superresolution_noise_mode'] = sr_noise
    return dataclasses.replace(cfg, neural_rendering_resolution=R or cfg.neural_rendering_resolution, rendering_kwargs=rk,
                               sr_num_fp16_res=sr_num_fp16_res)


# name: (config, noise_mode, sr_precision, hot SR weights).  The noise cases run the SR head with the same noise mode.
WORKLOADS = {
    'tiny512_const': (lambda: _cfg(config.tiny_config, 512, sr_noise='const'), 'const', 'fp32', False),
    'tiny512_random': (lambda: _cfg(config.tiny_config, 512, sr_noise='random'), 'random', 'fp32', False),
    'tiny512_none': (lambda: _cfg(config.tiny_config, 512), 'none', 'fp32', False),
    'tiny512_fp16': (lambda: _cfg(config.tiny_config, 512, sr_noise='const'), 'const', 'fp16', False),
    'tiny256': (lambda: _cfg(config.tiny_config, 256, sr_noise='const'), 'const', 'fp32', False),
    'tiny512_r128': (lambda: _cfg(config.tiny_config, 512, R=128), 'const', 'fp32', False),
    'tiny512_r128_fp16': (lambda: _cfg(config.tiny_config, 512, R=128), 'const', 'fp16', False),
    'full512': (lambda: _cfg(config.full_config, 512), 'const', 'fp32', False),
    'hot_fp32': (lambda: _cfg(config.tiny_config, 512), 'const', 'fp32', True),
    'hot_fp16': (lambda: _cfg(config.tiny_config, 512), 'const', 'fp16', True),
    'hot_noclamp': (lambda: _cfg(config.tiny_config, 512, sr_num_fp16_res=0), 'const', 'fp32', True),
}
BATCH = 2
# Fraction of each SR layer's reference outputs at or beyond +256 and at or beyond -256 with the hot weights: 1/8 of the conv channels
# carry each hot bias, but the convolution sums move some of their pixels back inside (fewest on the CPU oracle: 0.079 of the outputs at
# -256, without the clamp at 256^2); 1/3 of the ToRGB channels carry each hot bias.
HOT_CONV_FRACTION = 0.07
HOT_RGB_FRACTION = 0.3


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(WORKLOADS))
def test_every_layer_matches_fp64(name, monkeypatch):
    from next3d_b200.triplane_next3d import TriPlaneGenerator
    make_cfg, noise_mode, precision, hot = WORKLOADS[name]
    cfg = make_cfg()
    sd = hot_sr_state_dict(cfg, seed=3) if hot else weights.make_state_dict(cfg, seed=3)
    G = TriPlaneGenerator.from_config(cfg, sd, device=DEV)
    G.sr_precision = precision
    E = G._get_engine()
    E.concurrent = False
    _, _, c_cam, v = weights.demo_inputs(cfg, BATCH, seed=3)
    ws = torch.randn(BATCH, 28, 512, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))   # 28 distinct rows
    tr = Trace(cfg, sd, ws, noise_mode, cfg.neural_rendering_resolution, precision == 'fp16')
    install(monkeypatch, tr)
    with torch.no_grad():
        out = G.synthesis(ws, c_cam.to(DEV), v.to(DEV), noise_mode=noise_mode, seed=1)
    torch.cuda.synchronize()
    assert torch.isfinite(out['image']).all()

    assert not tr.problems, tr.problems
    executed = {k for k, e in tr.table.items() if e is not None}
    assert tr.ran == dict.fromkeys(executed, 1), {k: tr.ran.get(k, 0) for k in executed | set(tr.ran) if tr.ran.get(k, 0) != 1}
    unread = [(r['label'], r['reads']) for recs in tr.labels.values() for r in recs if r['errs'] is not None and r['reads'] != 1]
    assert not unread, unread
    if hot:
        for layer, (pos, neg) in tr.clamped.items():
            want = HOT_RGB_FRACTION if layer.endswith('.torgb') else HOT_CONV_FRACTION
            assert pos >= want and neg >= want, (layer, pos, neg)
    rows = [{'case': name, 'kind': k, 'err': e, 'step': step, 'bound': BOUNDS[k]} for k, (e, step) in sorted(tr.kinds.items())]
    record_errors('N3D_LAYER_ERRORS', rows)
    expect = {'split', 'f32', 'rgb' if precision == 'fp32' else 'rgb16', 'glue'} | ({'split16', 'glue16'} if precision == 'fp16' else set())
    assert expect <= set(tr.kinds), sorted(tr.kinds)
    bad = [r for r in rows if not r['err'] < r['bound']]
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ CPU: the statements, pinned
def _layer_sd(cin, cout, k, res, wdim, g, bias=None):
    p = {'weight': torch.randn(cout, cin, k, k, generator=g), 'bias': torch.randn(cout, generator=g) if bias is None else bias,
         'affine.weight': torch.randn(cin, wdim, generator=g), 'affine.bias': 1 + 0.1 * torch.randn(cin, generator=g),
         'noise_const': torch.randn(res, res, generator=g), 'noise_strength': torch.tensor(0.3, dtype=torch.float64),
         'resample_filter': oo.setup_filter([1, 3, 3, 1])}
    return {f'L.{n}': t.double() for n, t in p.items()}


def _hot_bias(cout, g, big):
    b = torch.randn(cout, generator=g)
    b[0::4], b[1::4] = big, -big
    return b


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max()).item()


@pytest.mark.parametrize('up', [1, 2])
@pytest.mark.parametrize('noise', ['const', 'none', 'per_sample'])
@pytest.mark.parametrize('clamp', [None, 2.0])
def test_synthesis_layer_statement_matches_oracle(up, noise, clamp):
    from oracle import generator as og
    g = torch.Generator().manual_seed(up * 10 + len(noise))
    N, cin, cout, H, wdim = 2, 6, 8, 5, 16
    sd = _layer_sd(cin, cout, 3, H * up, wdim, g, bias=_hot_bias(cout, g, 20.0) if clamp else None)
    x = torch.randn(N, cin, H, H, generator=g).double()
    w = torch.randn(N, wdim, generator=g).double()
    mode = {'L': torch.randn(N, 1, H * up, H * up, generator=g).double()} if noise == 'per_sample' else noise
    ref = og.synthesis_layer(sd, 'L', x, w, up=up, noise_mode=mode, clamp=clamp)
    s = oo.fully_connected(w, sd['L.affine.weight'], sd['L.affine.bias'])
    nz = mode['L'] if noise == 'per_sample' else sd['L.noise_const'] * sd['L.noise_strength'] if noise == 'const' else None
    got = synthesis_layer(x * s[:, :, None, None], sd['L.weight'], s, sd['L.bias'], sd['L.resample_filter'], up=up, noise=nz, clamp=clamp)
    assert got.shape == (N, cout, H * up, H * up)
    assert _rel(got, ref) < 1e-12
    if clamp:
        assert (ref == clamp).any() and (ref == -clamp).any()


@pytest.mark.parametrize('clamp', [None, 2.0])
def test_torgb_statement_matches_oracle(clamp):
    from oracle import generator as og
    g = torch.Generator().manual_seed(7)
    N, cin, wdim = 2, 12, 16
    sd = _layer_sd(cin, 3, 1, 6, wdim, g, bias=torch.tensor([20.0, -20.0, 0.1]))
    x = torch.randn(N, cin, 6, 6, generator=g).double()
    w = torch.randn(N, wdim, generator=g).double()
    ref = og.torgb(sd, 'L', x, w, clamp=clamp)
    s = oo.fully_connected(w, sd['L.affine.weight'], sd['L.affine.bias']) / math.sqrt(cin)
    got = torgb_layer(x * s[:, :, None, None], sd['L.weight'], sd['L.bias'], clamp=clamp)
    assert _rel(got, ref) < 1e-12
    if clamp:
        assert (ref == clamp).any() and (ref == -clamp).any()


@pytest.mark.parametrize('k, down, act', [(1, 1, 'linear'), (3, 1, 'linear'), (3, 1, 'lrelu'), (3, 2, 'lrelu')])
def test_conv2d_layer_statement_matches_oracle(k, down, act):
    from oracle import generator as og
    g = torch.Generator().manual_seed(k * 10 + down)
    sd = {'L.weight': torch.randn(8, 6, k, k, generator=g).double(), 'L.bias': torch.randn(8, generator=g).double(),
          'L.resample_filter': oo.setup_filter([1, 3, 3, 1]).double()}
    x = torch.randn(2, 6, 8, 8, generator=g).double()
    ref = og.conv2d_layer(sd, 'L', x, k, activation=act, down=down)
    got = conv2d_layer(x, sd['L.weight'], sd['L.bias'], sd['L.resample_filter'], down=down, lrelu=act == 'lrelu')
    assert got.shape == (2, 8, 8 // down, 8 // down)
    assert _rel(got, ref) < 1e-12


def test_fir_down_split_reference_is_conv2d_resample():
    """The parity images, convolved at unit stride over the nine taps of a stride-2 conv, give conv2d_resample(down=2): the statement
    of the engine's FIR-down launch is the first half of the reference's down-conv."""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 4, 8, 8, generator=g).double()
    w = torch.randn(5, 4, 3, 3, generator=g).double()
    f = oo.setup_filter([1, 3, 3, 1]).double()
    par = fir_down_split_reference(x, f)                               # [4, N, C, SH, SW]
    out = sum(F.conv2d(par[(ky & 1) * 2 + (kx & 1)][:, :, (ky >> 1):(ky >> 1) + 4, (kx >> 1):(kx >> 1) + 4], w[:, :, ky:ky + 1, kx:kx + 1])
              for ky in range(3) for kx in range(3))
    assert _rel(out, oo.conv2d_resample(x, w, f=f, down=2, padding=1)) < 1e-12


# ------------------------------------------------------------------------------------------------ CPU: the producer table
@pytest.mark.parametrize('factory, res', [(config.tiny_config, 512), (config.full_config, 512), (config.tiny_config, 256),
                                          (config.full_config, 256)])
@pytest.mark.parametrize('R', [64, 128])
def test_producer_table_names_every_conv_layer_once(factory, res, R):
    cfg = factory(res)
    layers = conv_layers(cfg)
    assert len(layers) == len(set(layers))
    table = producer_table(cfg, R)
    assert list(table) == layers                          # no layer the state dict lacks, none added twice
    executed = {k for k, e in table.items() if e is not None}
    # the layers the reference never runs: mouth b4, blending b4..b32, and the last fusion module of each StyleUNet
    never = {k for k in layers if k.startswith('mouth_backbone.synthesis.b4.') or
             any(k.startswith(f'neural_blending.synthesis.b{r}.') for r in (4, 8, 16, 32))} | \
        {'mouth_backbone.synthesis.fusion.4', 'neural_blending.synthesis.fusion.3'}
    assert set(layers) - executed == never
    assert executed >= set(oracle_widx(cfg))              # every modulated layer the oracle feeds a ws row
    # every input and accumulation target is made by an executed layer (through glue launches) or is INPUT
    for k in executed:
        for src in (table[k]['inp'] if isinstance(table[k]['inp'], tuple) else (table[k]['inp'],)) + (table[k]['onto'] or INPUT,):
            inner = src
            while inner.endswith(')'):
                inner = inner[inner.index('(') + 1:-1]
            assert inner == INPUT or inner in executed, (k, src)
    # the concat of fusion j: the decoder's x first, the encoder's cond second (torch.cat([x, cond_list[j]], 1))
    assert table['neural_blending.synthesis.fusion.1']['inp'] == ('neural_blending.synthesis.b64.conv1',
                                                                   'neural_blending.synthesis.encoder.1.conv2')
    assert table['mouth_backbone.synthesis.fusion.0']['inp'] == 'mouth_backbone.synthesis.encoder.3.conv2'


# ------------------------------------------------------------------------------------------------ CPU: the hot SR weights
@pytest.mark.parametrize('res', [512, 256])
def test_hot_sr_weights_clamp_every_sr_layer_at_both_signs(res, monkeypatch):
    """On the CPU oracle at tiny widths (a 64^2 random feature image, seeded weights with the hot biases): every SR conv and ToRGB
    puts at least the stated fraction of its bias_act outputs on each side of +-256."""
    from oracle import generator as og
    cfg = config.tiny_config(res)
    sd = hot_sr_state_dict(cfg, seed=3)
    for b in (0, 1):
        for n in ('conv0', 'conv1'):
            bias = sd[f'superresolution.block{b}.{n}.bias']
            assert (bias[0::8] == HOT_CONV_BIAS[0]).all() and (bias[4::8] == HOT_CONV_BIAS[1]).all()
        assert sd[f'superresolution.block{b}.torgb.bias'][:2].tolist() == list(HOT_RGB_BIAS)
    seen = []
    bias_act = oo.bias_act

    def record(x, b=None, dim=1, act='linear', alpha=None, gain=None, clamp=None):
        y = bias_act(x, b, dim, act, alpha, gain)
        seen.append((act, clamp, (y >= 256).double().mean().item(), (y <= -256).double().mean().item()))
        return bias_act(x, b, dim, act, alpha, gain, clamp)
    monkeypatch.setattr(oo, 'bias_act', record)
    g = torch.Generator().manual_seed(3)
    feat = torch.randn(1, cfg.plane_ch, 64, 64, generator=g)
    ws = torch.randn(1, 14, 512, generator=g)
    with torch.no_grad():
        og.superresolution(sd, cfg, feat[:, :3], feat, ws)
    assert len(seen) == 6                                  # conv0, conv1, torgb of the two blocks, in order
    for i, (act, clamp, pos, neg) in enumerate(seen):
        want = HOT_RGB_FRACTION if act == 'linear' else HOT_CONV_FRACTION
        assert clamp == 256.0 and pos >= want and neg >= want, (i, act, pos, neg)
