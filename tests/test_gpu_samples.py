"""GPU: sample sheets and shapes for many seeds (drivers.render_sample_sheets and its sharded twin) against the script's own loop,
gen_samples_next3d.py:182-238 restated: per seed, G.mapping and one synthesis call per yaw, the uint8 images concatenated along the
width, and the density grid of extract_sigma_grid.  Also sample_sheet_ws against per-seed mapping, graph replay against eager
launches, and a profiler count of the backbone passes."""
import numpy as np
import pytest
import torch

from tests.test_gpu_views import _generator, _inputs

pytestmark = pytest.mark.gpu
DEV = 'cuda'
OWN = r'_kernel'                     # the library's kernels are all named *_kernel; PyTorch's own are excluded by namespace below


@pytest.fixture(scope='module')
def tiny():
    from next3d_b200 import config
    cfg = config.tiny_config(512)
    _, G = _generator(cfg, 8)
    _, _, v, _ = _inputs(cfg, G, 1, 50)
    return cfg, G, v


def _noise(G, S, seed):
    """Per-image sampler uniforms of the 3 S sheet images, rows 3 i + yaw."""
    R = G.neural_rendering_resolution
    rk = G.rendering_kwargs
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(3 * S, R * R, rk['depth_resolution'], 1, generator=g).to(DEV),
            torch.rand(3 * S, R * R, rk['depth_resolution_importance'], generator=g).to(DEV))


def _script_sheets(G, seeds, v, noise, truncation_psi=0.7, truncation_cutoff=14, fov_deg=18.837):
    """gen_samples_next3d.py:182-206 with the sampler's uniforms injected: per seed, per yaw, mapping and a full synthesis call."""
    from next3d_b200 import drivers
    cams, cond = drivers.sample_sheet_cameras(G, fov_deg)                    # the script's camera_params / conditioning_params
    sheets = []
    for seed_idx, seed in enumerate(seeds):
        z = torch.from_numpy(np.random.RandomState(seed).randn(1, G.z_dim)).to(DEV)
        imgs = []
        for yaw in range(3):
            camera_params, conditioning_params = cams[yaw:yaw + 1].to(DEV), cond.to(DEV)
            ws = G.mapping(z, conditioning_params, truncation_psi=truncation_psi, truncation_cutoff=truncation_cutoff)
            r = 3 * seed_idx + yaw
            img = G.synthesis(ws, camera_params, v, noise_mode='const', sampler_noise=(noise[0][r:r + 1], noise[1][r]))['image']
            img = (img.permute(0, 2, 3, 1) * 127.5 + 128).clamp(0, 255).to(torch.uint8)
            imgs.append(img)
        img = torch.cat(imgs, dim=2)
        sheets.append(img[0].cpu().numpy())
    return sheets


def _assert_sheets(got, ref):
    assert len(got) == len(ref)
    for i, ((j, a, _), b) in enumerate(zip(got, ref)):
        assert j == i and a.shape == b.shape and a.dtype == np.uint8, (j, a.shape, b.shape)
        assert np.array_equal(a, b), f'seed {i}: {(a != b).sum()} bytes differ, max |diff| {np.abs(a.astype(int) - b.astype(int)).max()}'


def test_sample_sheet_ws_equals_per_seed_mapping(tiny):
    from next3d_b200 import drivers
    _, G, _ = tiny
    seeds = [0, 3, 17, 10720, 99]
    _, cond = drivers.sample_sheet_cameras(G)
    for psi, cutoff in ((1, 14), (0.7, 14), (0.5, None)):
        ws = drivers.sample_sheet_ws(G, seeds, truncation_psi=psi, truncation_cutoff=cutoff)
        assert ws.shape == (len(seeds), 28, 512) and ws.dtype == torch.float32
        for s, seed in enumerate(seeds):
            z = torch.from_numpy(np.random.RandomState(seed).randn(1, G.z_dim)).to(DEV)
            assert torch.equal(ws[s:s + 1], G.mapping(z, cond.to(DEV), truncation_psi=psi, truncation_cutoff=cutoff)), (psi, seed)


@pytest.mark.parametrize('S,batch', [(1, 3), (4, 6), (7, 9), (4, 9)])
def test_sheets_equal_the_script_loop(tiny, S, batch):
    """Heads per call B = batch // 3: (1, 3) one head per call; (4, 6) two full calls; (7, 9) and (4, 9) a padded last call."""
    from next3d_b200 import drivers
    _, G, v = tiny
    seeds = list(range(200, 200 + S))
    noise = _noise(G, S, S * 10 + batch)
    ws = drivers.sample_sheet_ws(G, seeds, truncation_psi=0.7)
    got = list(drivers.render_sample_sheets(G, ws, v, batch=batch, sampler_noise=noise))
    assert all(sig is None for _, _, sig in got)
    _assert_sheets(got, _script_sheets(G, seeds, v, noise))


def test_graph_replay_equals_eager(tiny):
    """G.use_cuda_graph: the caching call and the views replay graphs; the sheets and grids equal the eager driver's with the same
    sampler seeds, bit for bit, and a second graphed run (no capture) gives them again."""
    from next3d_b200 import drivers
    _, G, v = tiny
    ws = drivers.sample_sheet_ws(G, [5, 6, 7, 8, 9], truncation_psi=0.7)
    eager = list(drivers.render_sample_sheets(G, ws, v, batch=6, shapes=True, shape_res=64, seed=21))
    G.use_cuda_graph = True
    try:
        graphed = [list(drivers.render_sample_sheets(G, ws, v, batch=6, shapes=True, shape_res=64, seed=21)) for _ in range(2)]
    finally:
        G.use_cuda_graph = False
    for run in graphed:
        assert len(run) == len(eager) == 5
        for (i, a, sa), (j, b, sb) in zip(run, eager):
            assert i == j and np.array_equal(a, b) and np.array_equal(sa, sb), i
    assert np.abs(eager[0][1].astype(int) - eager[1][1].astype(int)).max() > 0


@pytest.mark.parametrize('shape_res', [64, 128])
def test_shapes_equal_extract_sigma_grid(tiny, shape_res):
    """3 seeds, 2 heads per call (a padded last call): every grid equals extract_sigma_grid of its seed alone, bit for bit."""
    from next3d_b200 import drivers
    _, G, v = tiny
    seeds = [31, 32, 33]
    noise = _noise(G, 3, shape_res)
    ws = drivers.sample_sheet_ws(G, seeds, truncation_psi=0.7)
    got = list(drivers.render_sample_sheets(G, ws, v, batch=6, shapes=True, shape_res=shape_res, sampler_noise=noise))
    _assert_sheets(got, _script_sheets(G, seeds, v, noise))
    for i, _, sig in got:
        ref = drivers.extract_sigma_grid(G, ws[i:i + 1], v, shape_res)
        assert sig.shape == (shape_res,) * 3 and sig.dtype == np.float32
        assert np.array_equal(sig, ref), f'seed {i}: {(sig != ref).sum()} voxels differ'
    pad = int(30 * shape_res / 256)
    assert (got[0][2][:pad] == -1000).all() and got[0][2][pad:-pad, pad:-pad, pad:-pad].std() > 0


def test_sharded_twin_at_world_size_one_equals_the_driver(tiny):
    from next3d_b200 import drivers
    _, G, v = tiny
    S = 5
    noise = _noise(G, S, 77)
    ws = drivers.sample_sheet_ws(G, list(range(40, 40 + S)), truncation_psi=0.7)
    got = list(drivers.render_sample_sheets(G, ws, v, batch=9, shapes=True, shape_res=64, sampler_noise=noise))
    sheets, grids = drivers.render_sample_sheets_sharded(G, ws, v, batch=9, shapes=True, shape_res=64, sampler_noise=noise)
    torch.cuda.current_stream().synchronize()
    assert sheets.shape == (S, *got[0][1].shape) and sorted(grids) == list(range(S))
    for i, sheet, sig in got:
        assert np.array_equal(sheets[i].numpy(), sheet) and np.array_equal(grids[i], sig), i


def _kernels(run, tmp_path):
    """Names of the library's kernels run() launches, in launch order, from a torch.profiler trace."""
    import json
    import re
    from torch.profiler import ProfilerActivity, profile
    x = torch.zeros(1, device=DEV)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(64):                    # a session can drop its first kernel records: these filler launches absorb that
            x.add_(1)
        torch.cuda.synchronize()
        run()
        torch.cuda.synchronize()
    trace = tmp_path / 'trace.json'
    prof.export_chrome_trace(str(trace))
    events = [e for e in json.loads(trace.read_text()).get('traceEvents', []) if e.get('cat') == 'kernel']
    if not events:
        pytest.skip('the trace recorded no kernel activity (CUPTI unavailable)')
    events.sort(key=lambda e: e['ts'])
    assert any('at::' in e['name'] for e in events[:64]), 'the filler launches were all dropped'
    return [e['name'] for e in events if re.search(OWN, e['name']) and 'at::' not in e['name']]


def test_one_backbone_pass_per_head(tiny, tmp_path):
    """Kernel launches of the driver over S = 4 seeds, 2 heads per call, with shapes: one caching synthesis call, one render_views call
    and one grid decode per head -- the backbones run once per call of B heads.  render_views launches no backbone kernel: its
    launches are those of synthesis minus at least the two backbones'.  The script's loop runs the backbones three times per seed."""
    from next3d_b200 import drivers
    cfg, G, v = tiny
    S, B = 4, 2
    ws = drivers.sample_sheet_ws(G, list(range(60, 60 + S)), truncation_psi=0.7)
    cams = drivers.sample_sheet_cameras(G)[0].to(DEV)
    eng = G._get_engine()
    passes, backbone = [], eng._backbone

    def counting(prefix, *a, **kw):
        passes.append((prefix, eng._N))
        return backbone(prefix, *a, **kw)
    eng._backbone = counting
    try:
        drv = _kernels(lambda: list(drivers.render_sample_sheets(G, ws, v, batch=3 * B, shapes=True, shape_res=64, seed=1)), tmp_path)
        assert sorted(passes) == sorted([('backbone.synthesis', B), ('texture_backbone.synthesis', B)] * (S // B)), passes
        syn = _kernels(lambda: G.synthesis(ws[:B], cams[:1].expand(B, -1), v.expand(B, -1, -1), noise_mode='const', cache_backbone=True,
                                           seed=1), tmp_path)
        bb = _kernels(lambda: (eng._backbone('texture_backbone.synthesis', cfg.plane_ch, 'const'),          # at the batch of syn
                               eng._backbone('backbone.synthesis', cfg.plane_ch * 3, 'const')), tmp_path)
        views = _kernels(lambda: G.render_views(cams[1:].repeat(B, 1), seed=2), tmp_path)
        grid = _kernels(lambda: eng.cached_sigma_grid(0, 64, torch.empty(64, 64, 64, device=DEV)), tmp_path)
        passes.clear()
        _script_sheets(G, [60], v, _noise(G, 1, 0))
        assert len(passes) == 6                                           # 3 yaws x 2 ws-only backbones for one seed
    finally:
        del eng._backbone
    assert len(grid) == 1 and len(bb) > 0
    assert len(drv) == (S // B) * (len(syn) + len(views)) + S * len(grid), (len(drv), len(syn), len(views), len(grid))
    assert len(views) <= len(syn) - len(bb), (len(views), len(syn), len(bb))


def test_cached_sigma_grid_refusals(tiny):
    from next3d_b200 import drivers
    _, G, v = tiny
    G.repack()                                                            # a rebuilt engine has nothing cached
    eng = G._get_engine()
    out = torch.empty(16, 16, 16, device=DEV)
    with pytest.raises(RuntimeError, match='needs cached planes'):
        eng.cached_sigma_grid(0, 16, out)
    ws = drivers.sample_sheet_ws(G, [1, 2], truncation_psi=0.7)
    cams = drivers.sample_sheet_cameras(G)[0].to(DEV)
    G.synthesis(ws, cams[:1].expand(2, -1), v.expand(2, -1, -1), noise_mode='const', cache_backbone=True, seed=0)
    with pytest.raises(RuntimeError, match='head 2, but the cache holds 2'):
        eng.cached_sigma_grid(2, 16, out)
    with pytest.raises(RuntimeError, match=r'float32 \[8\]\^3'):
        eng.cached_sigma_grid(1, 8, out)
    with pytest.raises(RuntimeError, match='is on cpu'):
        eng.cached_sigma_grid(1, 16, out.cpu())
    eng.cached_sigma_grid(1, 16, out)
    assert torch.equal(out.cpu(), torch.from_numpy(drivers.extract_sigma_grid(G, ws[1:], v, 16)))
