"""The mode bench.py times against the mode the layer suite holds to fp64: `synthesis` with concurrent branches (Engine.concurrent,
two side streams) and replayed from CUDA graphs with the in-kernel sampler RNG, against the eager single-stream forward.

Per workload row and call: (a) eager with concurrent = False, (b) eager with concurrent = True, (c) the first graphed call (it
captures) and (d) a replay with other ws, c, v and seed against (a) on those inputs, every output bit for bit: the kernels use no
order-dependent atomics (the depth range is a min / max), so equality is the contract, not a tolerance.

Stream order without luck: (b) and (c) run once more under StreamDelay, which fills every new CUDA tensor with a sentinel on the
stream current at its allocation and then delays that stream (torch.cuda._sleep), either the main stream or the side streams.  The
producers on the delayed streams start late, so a consumer on another stream that is not ordered after its producer reads the sentinel
or stale memory in one run, and the outputs differ from (a).  These runs take inputs no earlier run used, so stale memory does not
hold the right answer either.

Then graph families (interleaved keys, a refilled cache), the seed range, and key completeness: every rendering option and engine
setting a forward reads is part of a graph key, of the engine rebuild key, refused on every call, or shown not to change the outputs,
and flipping it after a capture gives what the eager call gives.  The in-kernel RNG is pinned by tests.helpers.hash_uniform, a host
statement checked here on the CPU (uniformity, grid, independence of the streams) and on the GPU against synthesis, render_views and
drivers.render_frames.
"""
import copy
import dataclasses
import math
import time

import numpy as np
import pytest
import torch
from torch.overrides import TorchFunctionMode
from torch.utils._pytree import tree_leaves

from tests.helpers import FINE_SEED_XOR, hash_uniform, sampler_uniforms

DEV = 'cuda'
OUTPUTS = ('image', 'image_raw', 'image_depth', 'image_normal')


# ------------------------------------------------------------------------------------------------ the workload table
def _row(name, cfg='tiny512', N=2, res=64, depth=48, noise_mode='const', sr='fp32', rk=None, depth_range='batch', calls=None):
    """A generator setup and its calls: ('synthesis', N, flags) or ('views', N, {}); by default one plain synthesis of N images."""
    return dict(name=name, cfg=cfg, N=N, res=res, depth=depth, noise_mode=noise_mode, sr=sr, rk=rk or {}, depth_range=depth_range,
                calls=calls or [('synthesis', N, {})])


ROWS = [
    _row('tiny512_n2'),
    _row('tiny512_n3', N=3),
    _row('tiny256_n2', cfg='tiny256'),
    _row('tiny512_r128', res=128),
    _row('c2_full_n8', cfg='full512', N=8),                                     # bench.py c2
    _row('c3_full_n16', cfg='full512', N=16, res=128, depth=96),                # bench.py c3, its batch
    _row('c2_full_n8_sr_fp16', cfg='full512', N=8, sr='fp16'),
    _row('tiny512_normal_white_image', rk=dict(return_normal=True, white_back=True), depth_range='image'),
    _row('tiny512_sample_mult4', depth=192),                                    # --sample_mult 4
    _row('tiny512_noise_none', noise_mode='none'),
    _row('tiny512_cache_views', calls=[('synthesis', 2, dict(cache_backbone=True)), ('synthesis', 6, dict(use_cached_backbone=True)),
                                       ('views', 4, {})]),
]
ROW_IDS = [r['name'] for r in ROWS]


def _calls(rows):
    return [(r, kind, N, flags) for r in rows for kind, N, flags in r['calls']]


COVERAGE = {
    'tiny512 at N 2 and 3': lambda rs: {2, 3} <= {r['N'] for r in rs if r['cfg'] == 'tiny512'},
    'tiny256 (4X super-resolution)': lambda rs: any(r['cfg'] == 'tiny256' for r in rs),
    'tiny512 at a 128^2 render': lambda rs: any(r['cfg'] == 'tiny512' and r['res'] == 128 for r in rs),
    'full width C2: 64^2, 48 + 48, N 8': lambda rs: any((r['cfg'], r['res'], r['depth'], r['N'], r['sr']) == ('full512', 64, 48, 8, 'fp32') for r in rs),
    'full width C3: 128^2, 96 + 96, N 16': lambda rs: any((r['cfg'], r['res'], r['depth'], r['N']) == ('full512', 128, 96, 16) for r in rs),
    "sr_precision 'fp16' at C2": lambda rs: any((r['cfg'], r['res'], r['depth'], r['sr']) == ('full512', 64, 48, 'fp16') for r in rs),
    'return_normal': lambda rs: any(r['rk'].get('return_normal') for r in rs),
    'white_back': lambda rs: any(r['rk'].get('white_back') for r in rs),
    "depth_range 'image'": lambda rs: any(r['depth_range'] == 'image' for r in rs),
    '192 + 192 samples (--sample_mult 4)': lambda rs: any(r['depth'] == 192 for r in rs),
    "noise_mode 'const' and 'none'": lambda rs: {'const', 'none'} <= {r['noise_mode'] for r in rs},
    'cache_backbone, then use_cached_backbone at V 3, then render_views at V 2':
        lambda rs: any([(k, N // r['N'], tuple(f)) for k, N, f in r['calls']] == [('synthesis', 1, ('cache_backbone',)),
                                                                                   ('synthesis', 3, ('use_cached_backbone',)), ('views', 2, ())]
                       for r in rs),
    # the fields of the synthesis key (engine.py, synthesis_graphed) that the table varies; the others are varied by the key test
    'cache flags, N, B, noise_mode, v shape and depth_range of the synthesis key take two values or more':
        lambda rs: all(len({f(r, N, fl) for r, k, N, fl in _calls(rs) if k == 'synthesis'}) >= 2
                       for f in (lambda r, N, fl: fl.get('cache_backbone', False), lambda r, N, fl: fl.get('use_cached_backbone', False),
                                 lambda r, N, fl: N, lambda r, N, fl: r['noise_mode'], lambda r, N, fl: r['depth_range'])),
    'R, sample counts, white_back, return_normal and sr_precision of the render key take two values or more':
        lambda rs: all(len({f(r) for r in rs}) >= 2 for f in (lambda r: r['res'], lambda r: r['depth'], lambda r: r['rk'].get('white_back', False),
                                                                lambda r: r['rk'].get('return_normal', False), lambda r: r['sr'])),
}


def test_workload_table_covers_every_configuration():
    """CPU: the rows reach everything listed in COVERAGE."""
    missing = [k for k, ok in COVERAGE.items() if not ok(ROWS)]
    assert not missing, missing
    assert len(set(ROW_IDS)) == len(ROW_IDS)
    for r in ROWS:
        for kind, N, _ in r['calls']:
            assert N % r['N'] == 0


# ------------------------------------------------------------------------------------------------ the host statement of the RNG (CPU)
DRAWS = 1 << 20


def test_hash_uniform_is_uniform_on_torch_rand_grid():
    """10^6 draws of one stream: a KS test against U[0, 1), and every value on the 2^-24 grid in [0, 1 - 2^-24]."""
    from scipy import stats
    u = hash_uniform(0x5EED, np.arange(DRAWS, dtype=np.uint64)).astype(np.float64)
    assert stats.kstest(u, 'uniform').pvalue > 1e-3
    k = u * 2.0 ** 24
    assert (k == np.floor(k)).all() and u.min() >= 0.0 and u.max() <= 1.0 - 2.0 ** -24
    assert abs(u.mean() - 0.5) < 5 / math.sqrt(12 * DRAWS)


@pytest.mark.parametrize('seed', [0, 7, 2 ** 63 + 11])
def test_hash_uniform_streams_are_uncorrelated(seed):
    """No measurable correlation (|r| < 5 / sqrt(n)) between the coarse and fine streams of one call, between seeds s and s + 1 (the
    drivers' consecutive batches), or between neighbouring numbers of one stream (neighbouring samples of a ray)."""
    idx = np.arange(DRAWS, dtype=np.uint64)
    coarse = hash_uniform(seed, idx).astype(np.float64)
    pairs = {'coarse / fine': hash_uniform((seed & (2 ** 64 - 1)) ^ FINE_SEED_XOR, idx),
             'seed / seed + 1': hash_uniform(seed + 1, idx),
             'number / number + 1': hash_uniform(seed, idx + np.uint64(1))}
    for name, other in pairs.items():
        r = np.corrcoef(coarse, other.astype(np.float64))[0, 1]
        assert abs(r) < 5 / math.sqrt(DRAWS), (name, r)


def test_sampler_uniforms_layout():
    """u_coarse [N, M, Dc, 1] holds number (n M + m) Dc + k of the seed's stream; u_fine [N M, Df] number (n M + m) Df + j of the fine
    stream; seeds are taken modulo 2^64."""
    N, M, Dc, Df = 2, 5, 3, 4
    u_c, u_f = sampler_uniforms(-1, N, M, Dc, Df)
    assert u_c.shape == (N, M, Dc, 1) and u_f.shape == (N * M, Df)
    assert u_c[1, 2, 1, 0].item() == hash_uniform(2 ** 64 - 1, [(1 * M + 2) * Dc + 1])[0]
    assert u_f[7, 3].item() == hash_uniform((2 ** 64 - 1) ^ FINE_SEED_XOR, [7 * Df + 3])[0]
    a, b = sampler_uniforms(2 ** 64 + 5, N, M, Dc, Df), sampler_uniforms(5, N, M, Dc, Df)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


# ------------------------------------------------------------------------------------------------ generators and inputs
_GENERATORS = {}


def _config(row):
    from next3d_b200 import config
    base = {'tiny512': lambda: config.tiny_config(512), 'tiny256': lambda: config.tiny_config(256),
            'full512': lambda: config.full_config(512)}[row['cfg']]()
    rk = copy.deepcopy(base.rendering_kwargs)
    rk.update(depth_resolution=row['depth'], depth_resolution_importance=row['depth'], **row['rk'])
    return dataclasses.replace(base, neural_rendering_resolution=row['res'], rendering_kwargs=rk)


def _generator(row):
    """The row's generator in its default state (one per configuration, reused: weights packed once), no graphs captured."""
    from next3d_b200 import weights
    from next3d_b200.triplane_next3d import TriPlaneGenerator
    cfg = _config(row)
    G = _GENERATORS.get(row['cfg'])
    if G is None:
        if row['cfg'] == 'full512':                 # at most one full-width generator alive
            _GENERATORS.clear()
            torch.cuda.empty_cache()
        G = _GENERATORS[row['cfg']] = TriPlaneGenerator.from_config(cfg, weights.make_state_dict(cfg, seed=31), device=DEV)
    G.rendering_kwargs = cfg.rendering_kwargs
    G.neural_rendering_resolution = cfg.neural_rendering_resolution
    G.sr_precision = row['sr']
    G.use_cuda_graph = False
    eng = G._get_engine()
    eng.concurrent, eng.splitk, eng.nprod = True, True, 3
    eng._graphs = {}
    return G


def _inputs(G, N, seed):
    """ws, c, v of N images, all depending on `seed`: latents, a jittered camera and a jittered mesh."""
    from next3d_b200 import weights
    z, c_cond, c_cam, v = weights.demo_inputs(G.cfg, N, seed=seed, jitter=1e-3)
    g = torch.Generator().manual_seed(seed)
    c_cam = c_cam.clone()
    c_cam[:, :16] += 1e-3 * torch.randn(N, 16, generator=g)
    ws = G.mapping(z.to(DEV), c_cond.to(DEV), truncation_psi=0.7, truncation_cutoff=14)
    return ws, c_cam.to(DEV), v.to(DEV)


def _snap(out):
    return {k: out[k].clone() for k in OUTPUTS if k in out}


def _call(G, row, kind, N, flags, inp, seed, concurrent=True, graph=False):
    """One call -> a copy of its outputs."""
    G._get_engine().concurrent = concurrent
    G.use_cuda_graph = graph
    try:
        if kind == 'views':
            out = G.render_views(inp[1], seed=seed, depth_range=row['depth_range'])
        else:
            out = G.synthesis(*inp, noise_mode=row['noise_mode'], seed=seed, depth_range=row['depth_range'], **flags)
        return _snap(out)
    finally:
        G.use_cuda_graph = False
        G._get_engine().concurrent = True


def _assert_same(a, b, what):
    assert a.keys() == b.keys(), what
    for k in a:
        assert torch.isfinite(b[k]).all(), (what, k)
        assert torch.equal(a[k], b[k]), (what, k, (a[k] - b[k]).abs().max().item())


# ------------------------------------------------------------------------------------------------ deterministic stream-order check
SENTINEL_FILL = {torch.float32: float('nan'), torch.bfloat16: float('nan'), torch.float16: float('nan'), torch.int32: -2 ** 31,
                 torch.int64: -2 ** 63}
_EMPTY = {torch.empty, torch.empty_like, torch.Tensor.new_empty}
CYCLES_PER_MS = 2_000_000               # torch.cuda._sleep counts SM clock cycles: <= 2 GHz on the H100


class StreamDelay(TorchFunctionMode):
    """Every new CUDA tensor of the calls under this mode is filled with a sentinel on the stream current at its allocation, and
    then, when that stream is a delayed one, the stream sleeps `ms`.  `delay` 'side': the engine's side streams are delayed after
    each of their new tensors, so whatever the main stream reads from the branches is produced late.  'main': the main stream is
    delayed after each new tensor it makes before the branches' first one in each forward (Engine._compute_planes), which is where
    everything the branches read from it is produced: the vertices, the landmarks and the styles.  A fresh tensor computed by a
    torch op (.contiguous(), .clone(), ...) is returned as a copy made the same way (sentinel, sleep, copy), so its producer also
    starts late.  Views and in-place results are passed through."""

    def __init__(self, eng, delay, ms):
        super().__init__()
        self.eng, self.delay, self.cycles = eng, delay, int(ms * CYCLES_PER_MS)
        self.sleeps = 0
        self.before_branches = False
        compute_planes = eng._compute_planes

        def forward(*args, **kwargs):               # the start of a forward: the branches have not allocated yet
            self.before_branches = True
            return compute_planes(*args, **kwargs)
        self.forward = forward

    def __enter__(self):
        self.eng._compute_planes = self.forward
        return super().__enter__()

    def __exit__(self, *exc):
        del self.eng._compute_planes
        return super().__exit__(*exc)

    def _poison(self, t):
        fill = SENTINEL_FILL.get(t.dtype)
        if fill is not None:
            t.fill_(fill)
        side = self.eng._side
        on_side = side is not None and torch.cuda.current_stream() in side
        if on_side:
            self.before_branches = False
        if (on_side if self.delay == 'side' else self.before_branches):
            torch.cuda._sleep(self.cycles)
            self.sleeps += 1

    def __torch_function__(self, func, types, args=(), kwargs=None):
        out = func(*args, **(kwargs or {}))
        if not isinstance(out, torch.Tensor) or not out.is_cuda or out.numel() == 0:
            return out
        if func in _EMPTY:
            self._poison(out)
            return out
        inputs = {t.untyped_storage().data_ptr() for t in tree_leaves((args, kwargs)) if isinstance(t, torch.Tensor)}
        if out.untyped_storage().data_ptr() in inputs:
            return out
        fresh = torch.empty_like(out)
        self._poison(fresh)
        fresh.copy_(out)
        return fresh


MAIN_DELAY_MS = 25.0        # far longer than the host takes from the fork's producers to the branches' first launch


def _timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, time.perf_counter() - t0


def _instrumented(G, row, kind, N, flags, inp, seed, delay, ms, graph):
    """(b) or (c) under StreamDelay, the graphed one captured afresh (and dropped afterwards) -> (outputs, sleeps, seconds)."""
    eng = G._get_engine()
    saved = eng._graphs
    if graph:
        eng._graphs = {}
    mode = StreamDelay(eng, delay, ms)
    try:
        with mode:
            out, sec = _timed(lambda: _call(G, row, kind, N, flags, inp, seed, graph=graph))
    finally:
        eng._graphs = saved
    return out, mode.sleeps, sec


# ------------------------------------------------------------------------------------------------ per row: (a) == (b) == (c), (d)
TIMES = {}


@pytest.mark.gpu
@pytest.mark.parametrize('row', ROWS, ids=ROW_IDS)
def test_concurrent_and_graphed_forward_equal_the_serial_one(row):
    G = _generator(row)
    base = 1000 * (ROW_IDS.index(row['name']) + 1)
    for i, (kind, N, flags) in enumerate(row['calls']):
        s = base + 100 * i
        x, y = _inputs(G, N, s + 1), _inputs(G, N, s + 2)
        seed_x, seed_y = s + 3, 2 ** 40 + s
        a, t_serial = _timed(lambda: _call(G, row, kind, N, flags, x, seed_x, concurrent=False))
        # instrumented (b) and (c) first, on inputs no earlier run used; each against the serial call on its inputs
        # render_views runs on one stream: nothing to order
        delays = [('main', MAIN_DELAY_MS), ('side', max(2.0, 1000 * t_serial / 5))] if kind == 'synthesis' else []
        for graph in (False, True):
            for j, (delay, ms) in enumerate(delays):
                if not graph:       # warm the allocator: a cudaMalloc in the checked run would synchronise the device and hide a race
                    _instrumented(G, row, kind, N, flags, _inputs(G, N, s + 50 + j), seed_x + j, delay, ms, graph)
                xi = _inputs(G, N, s + 10 + 2 * j + graph)
                got, sleeps, sec = _instrumented(G, row, kind, N, flags, xi, seed_x + j, delay, ms, graph)
                assert sleeps > 0
                TIMES[(row['name'], i, delay, graph)] = sec
                _assert_same(_call(G, row, kind, N, flags, xi, seed_x + j, concurrent=False), got,
                             f'{kind} {N}: {"graphed" if graph else "concurrent"} with the {delay} stream delayed')
        _assert_same(a, _call(G, row, kind, N, flags, x, seed_x), f'{kind} {N}: concurrent')
        _assert_same(a, _call(G, row, kind, N, flags, x, seed_x, graph=True), f'{kind} {N}: graph capture')
        d = _call(G, row, kind, N, flags, y, seed_y, graph=True)
        _assert_same(_call(G, row, kind, N, flags, y, seed_y, concurrent=False), d, f'{kind} {N}: graph replay on new inputs')
        assert not torch.equal(d['image'], a['image'])
    print(row['name'], {k[1:]: round(v, 3) for k, v in TIMES.items() if k[0] == row['name']})


@pytest.mark.gpu
def test_random_noise_replays_are_finite_and_differ():
    """noise_mode 'random' draws new torch RNG noise per call: two replays differ and are finite (no bit-identity to check)."""
    row = _row('tiny512_noise_random', noise_mode='random')
    G = _generator(row)
    x = _inputs(G, 2, 77)
    r1 = _call(G, row, 'synthesis', 2, {}, x, 5, graph=True)
    r2 = _call(G, row, 'synthesis', 2, {}, x, 5, graph=True)
    for k in r1:
        assert torch.isfinite(r1[k]).all() and torch.isfinite(r2[k]).all(), k
    assert not torch.equal(r1['image'], r2['image'])


# ------------------------------------------------------------------------------------------------ graph families and state
@pytest.mark.gpu
def test_interleaved_keys_replay_their_own_graphs():
    """N 2 (caching), N 3, N 2 (caching, new inputs), views, N 3 again: each graphed call equals eager on its own inputs, and
    replaying one key leaves the outputs of the other keys' graphs as they were."""
    row = _row('interleave')
    G = _generator(row)
    seq = [('synthesis', 2, dict(cache_backbone=True)), ('synthesis', 3, {}), ('synthesis', 2, dict(cache_backbone=True)),
           ('views', 4, {}), ('synthesis', 3, {})]
    held = {}                                        # key -> (the graph's own output tensors, a copy of them)
    for i, (kind, N, flags) in enumerate(seq):
        inp = _inputs(G, N, 500 + i)
        G.use_cuda_graph = True
        out = G.render_views(inp[1], seed=40 + i) if kind == 'views' else G.synthesis(*inp, noise_mode='const', seed=40 + i, **flags)
        G.use_cuda_graph = False
        key = (kind, N, tuple(flags))
        held[key] = (out, _snap(out))
        _assert_same(_call(G, row, kind, N, flags, inp, 40 + i), held[key][1], f'step {i}: {kind} {N}')
        for k, (live, copy_) in held.items():
            if k != key:
                _assert_same(copy_, _snap(live), f'step {i}: outputs of {k}')


@pytest.mark.gpu
def test_refilling_the_cache_at_another_batch_drops_the_cache_graphs():
    """cache_backbone at B 2, use_cached_backbone and render_views at V 2, then cache_backbone at B 3 (new buffers: the graphs that
    read the old ones are dropped) and the same calls at V 2: every graphed call equals eager on its inputs."""
    row = _row('refill')
    G = _generator(row)
    for B in (2, 3, 2):
        seq = [('synthesis', B, dict(cache_backbone=True)), ('synthesis', 2 * B, dict(use_cached_backbone=True)), ('views', 2 * B, {})]
        for i, (kind, N, flags) in enumerate(seq):
            inp = _inputs(G, N, 600 + 10 * B + i)
            g = _call(G, row, kind, N, flags, inp, 9 + i, graph=True)
            _assert_same(_call(G, row, kind, N, flags, inp, 9 + i), g, f'B {B}: {kind} {N}')
        eng = G._get_engine()
        cache_graphs = [k for k in eng._graphs if k[0]]                 # views keys: (True, 'views', N, V, ...); synthesis: B at 4
        assert eng._cache['B'] == B and all((k[2] // k[3] if k[1] == 'views' else k[4]) == B for k in cache_graphs), cache_graphs


SEEDS = [0, 2 ** 31 - 2, 2 ** 32 + 7, 2 ** 63 - 1, -1, 2 ** 63, 2 ** 64 - 1, 2 ** 64 + 5]


@pytest.mark.gpu
def test_seed_range_is_the_same_on_both_paths():
    """Graphed == eager for every seed; seeds are taken modulo 2^64 on both paths (-1 and 2^64 - 1 draw the same, 2^64 + 5 as 5)."""
    row = _row('seeds')
    G = _generator(row)
    x = _inputs(G, 2, 700)
    got = {}
    for s in SEEDS:
        e = _call(G, row, 'synthesis', 2, {}, x, s)
        _assert_same(e, _call(G, row, 'synthesis', 2, {}, x, s, graph=True), f'seed {s}')
        got[s] = e
    _assert_same(got[-1], got[2 ** 64 - 1], 'seed -1 against 2^64 - 1')
    _assert_same(_call(G, row, 'synthesis', 2, {}, x, 5), got[2 ** 64 + 5], 'seed 5 against 2^64 + 5')
    assert not torch.equal(got[0]['image'], got[2 ** 63]['image'])


# ------------------------------------------------------------------------------------------------ key completeness
class _Reads(dict):
    """rendering_kwargs that records every key read."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.read = set()

    def __getitem__(self, k):
        self.read.add(k)
        return super().__getitem__(k)

    def get(self, k, default=None):
        self.read.add(k)
        return super().get(k, default)

    def __contains__(self, k):
        self.read.add(k)
        return super().__contains__(k)


SETTINGS = ('splitk', 'splitk_maxres', 'nprod', 'concurrent', 'sr_precision')       # the Engine attributes a forward reads
# each name a forward reads: how a captured graph stays right when it changes, and the value the test flips it to
GROUPS = {
    'graph key': dict(depth_resolution=24, depth_resolution_importance=40, ray_start=2.2, ray_end=3.4, box_warp=0.9, white_back=True,
                      sr_antialias=False, return_normal=True, sr_precision='fp16', splitk=False, splitk_maxres=8, nprod=1),
    'engine rebuild key': dict(superresolution_noise_mode='const'),
    'refused on every call': dict(disparity_space_sampling=True, density_noise=1.0, clamp_mode='relu'),
    'does not change the outputs': dict(concurrent=False),
}
FLIPS = {k: v for g in GROUPS.values() for k, v in g.items()}


def _run_or_raise(fn):
    try:
        return fn(), None
    except RuntimeError as e:
        return None, str(e)


@pytest.mark.gpu
def test_every_option_a_forward_reads_is_keyed_refused_or_inert():
    from next3d_b200.engine import Engine
    row = _row('keys')
    G = _generator(row)
    x = _inputs(G, 2, 800)
    # what an eager and a graphed forward read
    rk = _Reads(G.rendering_kwargs)
    G.rendering_kwargs = rk
    eng = G._get_engine()
    read = set()

    class Recording(Engine):
        def __getattribute__(self, name):
            if name in SETTINGS:
                read.add(name)
            return object.__getattribute__(self, name)

    eng.__class__ = Recording
    try:
        _call(G, row, 'synthesis', 2, {}, x, 1)
        _call(G, row, 'synthesis', 2, {}, x, 1, graph=True)
    finally:
        eng.__class__ = Engine
    read |= rk.read
    assert set(SETTINGS) <= read
    assert sum(len(g) for g in GROUPS.values()) == len(FLIPS)             # every name in exactly one group
    assert read <= set(FLIPS), sorted(read - set(FLIPS))

    # flip each after a capture: the graphed call must give what the eager call gives, or raise what it raises
    wrong = []
    for name in sorted(read):
        G = _generator(row)
        eng = G._get_engine()
        _call(G, row, 'synthesis', 2, {}, x, 3, graph=True)
        before = {n: getattr(eng, n) for n in SETTINGS}
        if name == 'sr_precision':
            G.sr_precision = FLIPS[name]
        elif name in SETTINGS:
            setattr(eng, name, FLIPS[name])
        else:
            G.rendering_kwargs[name] = FLIPS[name]
        try:
            # _call sets `concurrent` itself: flip it through the graphed call's own argument
            conc = FLIPS[name] if name == 'concurrent' else True
            g, g_err = _run_or_raise(lambda: _call(G, row, 'synthesis', 2, {}, x, 3, concurrent=conc, graph=True))
            e, e_err = _run_or_raise(lambda: _call(G, row, 'synthesis', 2, {}, x, 3, concurrent=conc))
        finally:
            eng = G._get_engine()
            for n, v in before.items():
                setattr(eng, n, v)
            G.sr_precision = row['sr']
            G.rendering_kwargs = _config(row).rendering_kwargs
        if (g_err is None) != (e_err is None) or (g_err is not None and g_err != e_err):
            wrong.append((name, g_err, e_err))
        elif g is not None and (g.keys() != e.keys() or not all(torch.equal(g[k], e[k]) for k in g)):
            wrong.append((name, 'graphed output differs from eager'))
    assert not wrong, ('names: ' + ', '.join(w[0] for w in wrong), wrong)


# ------------------------------------------------------------------------------------------------ the in-kernel RNG at generator level
def _host_noise(G, N, seed):
    rk, R = G.rendering_kwargs, G.neural_rendering_resolution
    u_c, u_f = sampler_uniforms(seed, N, R * R, rk['depth_resolution'], rk['depth_resolution_importance'])
    return u_c.to(DEV), u_f.to(DEV)


@pytest.mark.gpu
def test_in_kernel_rng_equals_the_host_statement_in_synthesis_and_render_views():
    """synthesis(seed=s) eager and graphed, and render_views(seed=s) eager and graphed, equal the calls fed
    sampler_noise=host statement(s), bit for bit."""
    row = _row('rng')
    G = _generator(row)
    ws, c, v = _inputs(G, 2, 900)
    for s in (0, 12345, 2 ** 63 + 3):
        ref = _snap(G.synthesis(ws, c, v, noise_mode='const', sampler_noise=_host_noise(G, 2, s), cache_backbone=True))
        _assert_same(ref, _call(G, row, 'synthesis', 2, dict(cache_backbone=True), (ws, c, v), s), f'synthesis seed {s}')
        _assert_same(ref, _call(G, row, 'synthesis', 2, dict(cache_backbone=True), (ws, c, v), s, graph=True), f'graphed synthesis seed {s}')
        cams = _inputs(G, 4, 901)[1]
        ref = _snap(G.render_views(cams, sampler_noise=_host_noise(G, 4, s + 1)))
        _assert_same(ref, _call(G, row, 'views', 4, {}, (None, cams, None), s + 1), f'render_views seed {s + 1}')
        _assert_same(ref, _call(G, row, 'views', 4, {}, (None, cams, None), s + 1, graph=True), f'graphed render_views seed {s + 1}')


@pytest.mark.gpu
@pytest.mark.parametrize('graph', [False, True], ids=['eager', 'graphed'])
def test_render_frames_batch_k_draws_seed_plus_k(graph):
    """drivers.render_frames(seed=s): batch k draws seed s + k, so its frames equal those rendered from the host statement's
    uniforms of s + k, image by image."""
    from next3d_b200 import drivers
    row = _row('frames')
    G = _generator(row)
    F, batch, s = 6, 2, 2 ** 33 + 1
    ws, c, v = _inputs(G, F, 950)
    M = G.neural_rendering_resolution ** 2
    parts = [_host_noise(G, batch, s + k) for k in range(F // batch)]
    u_c = torch.cat([p[0] for p in parts])
    u_f = torch.cat([p[1].reshape(batch, M, -1) for p in parts])
    G.use_cuda_graph = graph
    try:
        got = list(drivers.render_frames(G, ws, c, v[:1], batch=batch, seed=s))
        ref = list(drivers.render_frames(G, ws, c, v[:1], batch=batch, sampler_noise=(u_c, u_f)))
    finally:
        G.use_cuda_graph = False
    assert len(got) == len(ref) == F
    for f, (a, b) in enumerate(zip(got, ref)):
        assert np.array_equal(a, b), f
