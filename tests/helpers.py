"""Shared helpers for the parity tests and the kernel conformance suites."""
import json
import math
import os
import re

import numpy as np
import pytest
import torch

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def load_golden(name):
    with np.load(os.path.join(GOLDEN_DIR, f'{name}.npz')) as z:
        return {k: z[k] for k in z.files}


class ReferenceVectors:
    """What a test compares against in the original project, computed by the original project's own code on the test's seeded
    inputs and stored as tests/golden/<name>.npz, so that the comparison runs wherever the repository does.  get(key, compute)
    returns the stored array; with N3D_RECORD_REFERENCE=1 it calls compute() (which imports the original project through
    oracle.ref_shim), stores the result under key and rewrites the file."""

    def __init__(self, name):
        self.path = os.path.join(GOLDEN_DIR, f'{name}.npz')
        self.record = os.environ.get('N3D_RECORD_REFERENCE') == '1'
        self.data = load_golden(name) if os.path.exists(self.path) or not self.record else {}

    def get(self, key, compute):
        if self.record:
            v = compute()
            self.data[key] = v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
            np.savez_compressed(self.path, **self.data)
        a = self.data[key]
        return torch.from_numpy(a.copy()) if a.dtype.kind in 'biuf' else a


def golden_planes(g):
    """(stride, texels) of the stored tri-plane sample of a golden fixture: every 8th texel, or every 16th in batch fixtures."""
    return (8, g['planes_s8']) if 'planes_s8' in g else (16, g['planes_s16'])


def range_rel_err(a, ref):
    """max|a - ref| / max|ref| -- the parity metric used everywhere in this repo (SURVEY.md section 7: per-pixel
    relative error is ill-conditioned at zero crossings, so errors are normalised by the reference's range)."""
    a = torch.as_tensor(a, dtype=torch.float64)
    ref = torch.as_tensor(ref, dtype=torch.float64)
    return ((a - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def pixel_rel_err(a, ref, floor=1e-3):
    """north_star's literal metric: max over elements of |a - ref| / max(|ref|, floor * max|ref|) -- per-pixel relative error with an
    absolute floor so that zero crossings do not divide by ~0.  Returned together with the fraction of elements above 1e-3."""
    a = torch.as_tensor(a, dtype=torch.float64)
    ref = torch.as_tensor(ref, dtype=torch.float64)
    den = ref.abs().clamp_min(floor * ref.abs().max().clamp_min(1e-30))
    e = (a - ref).abs() / den
    return e.max().item(), (e > 1e-3).double().mean().item()


def report_parity(name, a, ref):
    """Both parity metrics of one output; appended to gpurun_out/parity_report.jsonl when that directory exists (so a GPU run
    leaves the numbers behind for the design notes).  -> (range_rel, pixel_rel_max, pixel_rel_frac_above_1e-3)."""
    r = range_rel_err(a, ref)
    pmax, pfrac = pixel_rel_err(a, ref)
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'gpurun_out')
    if os.path.isdir(out):
        with open(os.path.join(out, 'parity_report.jsonl'), 'a') as f:
            f.write(json.dumps({'case': name, 'range_rel_err': r, 'pixel_rel_err_max_floor1e-3': pmax, 'pixel_frac_above_1e-3': pfrac}) + '\n')
    return r, pmax, pfrac


# ------------------------------------------------------------------------------------------------ kernel conformance suites
GUARD = 64                  # sentinel elements on each side of an output view: keeps the view's base alignment that of a fresh allocation
SENTINEL = {torch.float32: (torch.int32, 0x7FC01234), torch.int32: (torch.int32, 0x7FC01234),      # NaN bit patterns no store produces
            torch.bfloat16: (torch.int16, 0x7FC1), torch.float16: (torch.int16, 0x7E01)}


class Guarded:
    """An output tensor as a view into a larger allocation filled with a sentinel.  The launch owns the elements `own` selects: all of
    the view (None), a slice of the last dimension, or a bool tensor broadcastable to the view; `own` may be assigned after
    construction.  `init`: initial content of the view, in place of the sentinel."""

    def __init__(self, shape, dtype=torch.float32, own=None, init=None):
        n = math.prod(shape)
        self.int_dtype, self.sentinel = SENTINEL[dtype]
        self.buf = torch.empty(GUARD + n + GUARD, dtype=dtype, device='cuda')
        self.view = self.buf[GUARD:GUARD + n].view(shape)
        self.own = own
        self.reset()
        if init is not None:
            self.view.copy_(init)

    def reset(self):
        self.buf.view(self.int_dtype).fill_(self.sentinel)

    def bits(self):
        return self.view.view(self.int_dtype)

    def _own_mask(self):
        if isinstance(self.own, slice):
            m = torch.zeros(self.view.shape[-1], dtype=torch.bool, device=self.view.device)
            m[self.own] = True
            return m
        return self.own

    def untouched_ok(self):
        """The guard bands and every element outside `own` still hold the sentinel's bits."""
        b, own = self.buf.view(self.int_dtype), self._own_mask()
        ok = bool((b[:GUARD] == self.sentinel).all()) and bool((b[-GUARD:] == self.sentinel).all())
        return ok and (own is None or bool(((self.bits() == self.sentinel) | own).all()))

    def written(self):
        """No element of `own` holds the sentinel's bits."""
        kept, own = self.bits() == self.sentinel, self._own_mask()
        return not bool((kept if own is None else kept & own).any())

    def snapshot(self):
        """The bits of the whole allocation, guards included, on the host."""
        return self.buf.view(self.int_dtype).cpu()


class RangeErr:
    """max |got - ref| / max |ref| accumulated over reference chunks; a NaN difference counts as infinite."""

    def __init__(self):
        self.diff = self.range = 0.0

    def add(self, got, ref):
        d = (got.double() - ref).abs().max().item()
        self.diff = max(self.diff, d if d == d else math.inf)
        self.range = max(self.range, ref.abs().max().item())

    def value(self):
        return self.diff / max(self.range, 1e-30)


def record_errors(env_var, rows):
    """Append each row (a dict) as a JSON line to the file named by the environment variable `env_var`, when it is set: scripts that
    re-measure the worst cases beside a suite's bounds read these files."""
    path = os.environ.get(env_var)
    if path:
        with open(path, 'a') as f:
            for r in rows:
                f.write(json.dumps(r) + '\n')


def rerun_identical(outputs, launch):
    """Reset the guarded outputs to the sentinel, call launch() and synchronise -> whether every output holds the same bits as
    before the call."""
    before = [t.snapshot() for t in outputs]
    for t in outputs:
        t.reset()
    launch()
    torch.cuda.synchronize()
    return all(torch.equal(a, t.snapshot()) for a, t in zip(before, outputs))


def launched_kernels(run, pattern, tmp_path):
    """Call run() twice under torch.profiler; run() launches kernels and returns a list with one entry per launch whose kernel name
    `pattern` matches.  -> (what the second call returned, the chrome-trace events of its matching launches in launch order, each
    with the launch's 'grid' and 'cluster' in its 'args' where the trace records them).  A profiler session that follows another
    one in the same process can drop its first kernel records, so only the second call is compared; skips the test when CUDA
    activity tracing is unavailable."""
    from torch.profiler import ProfilerActivity, profile
    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run()
            expected = run()
            torch.cuda.synchronize()
    except RuntimeError as e:              # CUPTI missing or busy
        pytest.skip(f'CUDA activity tracing unavailable: {e}')
    trace = tmp_path / 'trace.json'
    prof.export_chrome_trace(str(trace))
    events = [e for e in json.loads(trace.read_text()).get('traceEvents', []) if e.get('cat') == 'kernel' and re.search(pattern, e.get('name', ''))]
    if not events:
        pytest.skip('the trace recorded no kernel activity (CUPTI unavailable)')
    events.sort(key=lambda e: e['ts'])
    n = len(expected)
    assert n <= len(events) <= 2 * n, [e['name'] for e in events]
    return expected, events[-n:]


def cdiv(a, b):
    return -(-a // b)


def grid_stride(work, sms, per_sm, threads=256):
    """n3d_grid (common.cuh): one block per `threads` work items, at least 1 and at most `per_sm` blocks per SM."""
    return max(1, min(cdiv(work, threads), sms * per_sm))


def lib():
    from next3d_b200 import _lib as L
    return L


def refused(rc, what):
    """The entry point returned -1 and its last error contains `what`."""
    msg = lib().lib.n3d_last_error().decode()
    assert rc == -1 and what in msg, (rc, msg)


def offset_view(t, nbytes):
    """A view of `t` (a fresh, 64-byte aligned allocation) that starts `nbytes` later."""
    assert t.data_ptr() % 64 == 0
    return t.view(-1)[nbytes // t.element_size():]


# ------------------------------------------------------------------------------------------------ generator-level helpers
def oracle_widx(cfg):
    """{modulated layer: the ws index oracle.generator.synthesis feeds it}, read off the oracle's own slicing of a ws whose entries
    are their index: the texture backbone takes ws[:, 14:], the other backbones ws[:, :14] (the StyleUNets from their first executed
    block on), the super-resolution blocks ws[:, 13]."""
    from next3d_b200 import config
    from oracle import generator as og
    idx = torch.arange(28)[None, :, None]
    eg3d, tex = idx[:, :14], idx[:, 14:]
    res_list = config.block_resolutions(cfg.plane_res)
    out = {}

    def blocks(prefix, ws, start):
        for res, cur in list(zip(res_list, og._split_ws(ws, res_list)))[start:]:
            names = ('conv1', 'torgb') if res == 4 else ('conv0', 'conv1', 'torgb')
            for name, w in zip(names, cur.unbind(1)):
                out[f'{prefix}.b{res}.{name}'] = int(w)

    blocks('texture_backbone.synthesis', tex, 0)
    blocks('backbone.synthesis', eg3d, 0)
    blocks('mouth_backbone.synthesis', eg3d, int(math.log2(4)) - 1)            # styleunet(..., 64, 4, 64)
    blocks('neural_blending.synthesis', eg3d, int(math.log2(32)) - 1)          # styleunet(..., 256, 32, 256)
    sr = eg3d[:, -1:].repeat(1, 3, 1)
    for b in (0, 1):
        for name, w in zip(('conv0', 'conv1', 'torgb'), sr.unbind(1)):
            out[f'superresolution.block{b}.{name}'] = int(w)
    return out


# "Hot" super-resolution biases that push outputs past the +-256 conv_clamp of the SR layers.  Every 8th output channel of each SR
# convolution gets +400, every 8th (offset 4) -1200: lrelu(400) * sqrt 2 = 566 and lrelu(-1200) * sqrt 2 = -339.  ToRGB channel 0 gets
# +2000 and channel 1 -2000: the ToRGB sums of the hot activations alone reach +-1000 at the seeded weights, which +-300 would not
# outweigh.  So about 1/8 of every SR conv's outputs and 1/3 of every SR ToRGB's outputs reach each side of the clamp.
HOT_CONV_BIAS = (400.0, -1200.0)
HOT_RGB_BIAS = (2000.0, -2000.0)


def hot_sr_state_dict(cfg, seed=0):
    """weights.make_state_dict(cfg, seed) with the hot super-resolution biases above."""
    from next3d_b200 import weights
    sd = weights.make_state_dict(cfg, seed=seed)
    for b in (0, 1):
        for name in ('conv0', 'conv1'):
            bias = sd[f'superresolution.block{b}.{name}.bias'].clone()
            bias[0::8], bias[4::8] = HOT_CONV_BIAS
            sd[f'superresolution.block{b}.{name}.bias'] = bias
        bias = sd[f'superresolution.block{b}.torgb.bias'].clone()
        bias[0], bias[1] = HOT_RGB_BIAS
        sd[f'superresolution.block{b}.torgb.bias'] = bias
    return sd


# ------------------------------------------------------------------------------------------------ the renderer's in-kernel sampler RNG
HASH_GAMMA = 0x9E3779B97F4A7C15         # hash_uniform (render_common.cuh): splitmix64 of seed + idx * gamma
HASH_MIX = (0xBF58476D1CE4E5B9, 0x94D049BB133111EB)
FINE_SEED_XOR = 0xA5A5A5A5DEADBEEF      # the fine (importance) stream's seed: seed ^ this (render_fused.cu)


def hash_uniform(seed, idx):
    """The renderer's counter RNG in numpy uint64 arithmetic: uniform float32 number `idx` (an integer array) of stream `seed` (any
    integer, taken modulo 2^64).  The top 24 bits of the mixed word over 2^24: the 2^-24 grid in [0, 1 - 2^-24], torch.rand's range."""
    u64 = np.uint64
    with np.errstate(over='ignore'):
        z = u64(int(seed) & ((1 << 64) - 1)) + np.asarray(idx, dtype=u64) * u64(HASH_GAMMA)
        z = (z ^ (z >> u64(30))) * u64(HASH_MIX[0])
        z = (z ^ (z >> u64(27))) * u64(HASH_MIX[1])
        z ^= z >> u64(31)
    return (z >> u64(40)).astype(np.float32) * np.float32(2.0 ** -24)


def sampler_uniforms(seed, N, M, Dc, Df):
    """The uniforms a render launch of N images of M rays draws in the kernel with `seed` (the descriptor's seed plus *seed_ptr), in
    the layouts of injected ones: u_coarse [N, M, Dc, 1] with number gr * Dc + k of stream seed for sample k of global ray
    gr = n * M + m, and u_fine [N * M, max(Df, 1)] with number gr * Df + j of stream seed ^ FINE_SEED_XOR (zeros when Df is 0)."""
    rays = np.arange(N * M, dtype=np.uint64)[:, None]
    u_c = hash_uniform(seed, rays * np.uint64(Dc) + np.arange(Dc, dtype=np.uint64))
    if Df:
        u_f = hash_uniform((int(seed) & ((1 << 64) - 1)) ^ FINE_SEED_XOR, rays * np.uint64(Df) + np.arange(Df, dtype=np.uint64))
    else:
        u_f = np.zeros((N * M, 1), np.float32)
    return torch.from_numpy(u_c).reshape(N, M, Dc, 1), torch.from_numpy(u_f)
