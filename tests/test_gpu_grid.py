"""GPU: grid videos.  The `views` entry points of the texture lookup and the plane blend against the old ones on repeated inputs;
synthesis with N = B * V images on a cache of B heads against plain synthesis of the repeated heads, eager and graphed; and the grid
drivers (render_grid_frames, reenact_grid_frames and their sharded twins) against a per-cell, per-frame synthesis loop laid out
as the scripts' layout_grid does (gen_videos_next3d.py:35-49, 128-171; reenact_avatar_next3d.py:56-70, 116-167)."""
import json

import numpy as np
import pytest
import torch

from tests.test_gpu_views import _backbone_launches, _clone, _generator, _inputs

pytestmark = pytest.mark.gpu
DEV = 'cuda'
KEYS = ('image', 'image_raw', 'image_depth')


def _layout_grid(img, grid_w, grid_h):
    """layout_grid of both scripts: [gh * gw, C, h, w] float -> [gh * h, gw * w, C] uint8 (numpy)."""
    _, channels, img_h, img_w = img.shape
    img = (img * 127.5 + 128).clamp(0, 255).to(torch.uint8)
    img = img.reshape(grid_h, grid_w, channels, img_h, img_w).permute(2, 0, 3, 1, 4)
    return img.reshape(channels, grid_h * img_h, grid_w * img_w).permute(1, 2, 0).cpu().numpy()


@pytest.fixture(scope='module')
def tiny():
    from next3d_b200 import config
    cfg = config.tiny_config(512)
    sd, G = _generator(cfg, 6)
    return cfg, G


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize('V', [1, 2, 3])
def test_views_kernels_equal_the_old_entry_points_on_repeated_inputs(V):
    from next3d_b200 import _lib as L
    from next3d_b200 import kernels as K
    g = torch.Generator().manual_seed(V)
    B, H, W, T, C, Fc = 2, 24, 20, 32, 32, 50
    N = B * V
    p2f = torch.randint(-1, Fc, (N * 4, H, W), generator=g, dtype=torch.int32).to(DEV)
    bary = torch.rand(N * 4, H, W, 3, generator=g)
    bary = (bary / bary.sum(-1, keepdim=True)).to(DEV)
    face_uv = (torch.rand(Fc, 3, 2, generator=g) * 2.2 - 1.1).to(DEV)
    tex = torch.randn(B, T, T, C, generator=g).to(DEV)
    mask = torch.rand(16, 16, generator=g).to(DEV)
    tp = [torch.full((3, N, H, W, C), float('nan'), device=DEV) for _ in range(2)]
    al = [torch.full((3, N, H, W), float('nan'), device=DEV) for _ in range(2)]
    rep = tex.repeat_interleave(V, 0)
    stream = torch.cuda.current_stream().cuda_stream
    L.check(L.lib.n3d_uv_sample(p2f.data_ptr(), bary.data_ptr(), face_uv.data_ptr(), rep.data_ptr(), mask.data_ptr(), N, H, W, T, T, C,
                                16, 16, tp[0].data_ptr(), al[0].data_ptr(), stream))
    K.uv_sample(p2f, bary, face_uv, tex, mask, tp[1], al[1], views=V)
    torch.cuda.synchronize()
    assert torch.equal(tp[0], tp[1]) and torch.equal(al[0].nan_to_num(7.0), al[1].nan_to_num(7.0))
    front = torch.randn(N, H, W, 32, generator=g).to(DEV)
    static = torch.randn(B, H, W, 96, generator=g).to(DEV)
    srep = static.repeat_interleave(V, 0)
    alpha = torch.rand(3, N, H, W, generator=g).to(DEV)
    out = [torch.full((N, 3, H, W, 32), float('nan'), device=DEV) for _ in range(2)]
    L.check(L.lib.n3d_blend_planes(front.data_ptr(), tp[0].data_ptr(), alpha.data_ptr(), srep.data_ptr(), N, H, W, out[0].data_ptr(), stream))
    K.blend_planes(front, tp[0], alpha, static, out[1], views=V)
    torch.cuda.synchronize()
    assert torch.equal(out[0], out[1])


# ------------------------------------------------------------------------------------------------ engine
def test_cached_heads_with_several_images_each(tiny):
    """B = 2 cached heads, V = 3 images each (own camera, mesh and sampler noise) == plain synthesis of the heads repeated, bit for
    bit, eager and graphed; the backbone launches are skipped."""
    cfg, G = tiny
    B, V = 2, 3
    N = B * V
    ws, c, v, noise = _inputs(cfg, G, N, 41)
    heads = ws[:B]
    rep = heads.repeat_interleave(V, 0)
    v = v + torch.randn(v.shape, generator=torch.Generator().manual_seed(2)).to(DEV) * 2e-3
    plain = _clone(G.synthesis(rep, c, v, noise_mode='const', sampler_noise=noise))
    eng = G._get_engine()
    n_plain = eng.launches
    bb = _backbone_launches(G, cfg)
    G.synthesis(heads, c[:B], v[:B], noise_mode='const', cache_backbone=True, seed=1)
    got = G.synthesis(rep, c, v, noise_mode='const', sampler_noise=noise, use_cached_backbone=True)
    for k in KEYS:
        assert torch.equal(got[k], plain[k]), k
    assert bb > 0 and eng.launches == n_plain - bb, (n_plain, eng.launches, bb)
    with pytest.raises(RuntimeError, match='batch 5.*batch 2'):
        G.synthesis(rep[:5], c[:5], v[:5], noise_mode='const', use_cached_backbone=True)
    with pytest.raises(RuntimeError, match='batch 6.*batch 2'):
        G.synthesis(rep, c, v, noise_mode='const', use_cached_backbone=True, cache_backbone=True)
    G.use_cuda_graph = True
    try:
        plain_g = _clone(G.synthesis(rep, c, v, noise_mode='const', seed=9))
        got_g = _clone(G.synthesis(rep, c, v, noise_mode='const', seed=9, use_cached_backbone=True))
        assert eng.launches == n_plain - bb
        # re-caching with another batch (B = 3, V = 2) at the same N: the reusing graph reads the new heads
        three = [0, 3, 5]                                              # heads 0, 1, 1
        G.synthesis(rep[three], c[three], v[three], noise_mode='const', cache_backbone=True, seed=1)
        plain3 = _clone(G.synthesis(rep[[0, 0, 3, 3, 5, 5]], c, v, noise_mode='const', seed=9))
        got3 = G.synthesis(rep[[0, 0, 3, 3, 5, 5]], c, v, noise_mode='const', seed=9, use_cached_backbone=True)
    finally:
        G.use_cuda_graph = False
    for k in KEYS:
        assert torch.equal(got_g[k], plain_g[k]), k
        assert torch.equal(got3[k], plain3[k]), k


# ------------------------------------------------------------------------------------------------ interpolation grid
def _grid_workload(cfg, G, grid, K_, w_frames):
    from next3d_b200 import drivers
    gw, gh = grid
    ws_grid = drivers.grid_keyframes(G, list(range(100, 100 + gw * gh * K_)), grid, truncation_psi=0.7)
    _, _, v, _ = _inputs(cfg, G, 1, 42)
    n = K_ * w_frames * gw * gh
    R = G.neural_rendering_resolution
    rk = G.rendering_kwargs
    g = torch.Generator().manual_seed(13)
    u_c = torch.rand(n, R * R, rk['depth_resolution'], 1, generator=g).to(DEV)
    u_f = torch.rand(n, R * R, rk['depth_resolution_importance'], generator=g).to(DEV)
    return ws_grid, v, (u_c, u_f)


def _grid_reference(G, ws_grid, v, w_frames, image_mode, noise):
    """gen_videos_next3d.py:128-171: one synthesis call per cell per frame, then layout_grid."""
    from next3d_b200 import drivers
    gh, gw, K_ = ws_grid.shape[:3]
    F = K_ * w_frames
    interp = [[drivers.interpolate_ws_device(ws_grid[yi, xi], w_frames) for xi in range(gw)] for yi in range(gh)]
    cams = drivers.orbit_camera_params(F, torch.tensor(G.rendering_kwargs['avg_camera_pivot']), G.rendering_kwargs['avg_camera_radius'])
    frames = []
    for f in range(F):
        imgs = []
        for yi in range(gh):
            for xi in range(gw):
                i = (f * gh + yi) * gw + xi
                img = G.synthesis(interp[yi][xi][f:f + 1], cams[f:f + 1].to(DEV), v, noise_mode='const',
                                  sampler_noise=(noise[0][i:i + 1], noise[1][i]))[image_mode][0]
                if image_mode == 'image_depth':
                    img = -img
                    img = (img - img.min()) / (img.max() - img.min()) * 2 - 1
                imgs.append(img)
        frames.append(_layout_grid(torch.stack(imgs), gw, gh))
    return frames


@pytest.mark.parametrize('image_mode', KEYS)
def test_render_grid_frames_equals_per_cell_loop(tiny, image_mode):
    """2x2 grid, 2 keyframes x 2 frames: 16 images in batches of 3 (frames split across batches, a ragged last batch)."""
    from next3d_b200 import drivers
    cfg, G = tiny
    grid, w_frames = (2, 2), 2
    ws_grid, v, noise = _grid_workload(cfg, G, grid, 2, w_frames)
    got = list(drivers.render_grid_frames(G, ws_grid, v, w_frames, batch=3, image_mode=image_mode, sampler_noise=noise))
    ref = _grid_reference(G, ws_grid, v, w_frames, image_mode, noise)
    assert len(got) == len(ref) == 4
    for f, (a, b) in enumerate(zip(got, ref)):
        assert a.shape[:2] == b.shape[:2] and a.shape[2] == 3, (a.shape, b.shape)
        assert np.array_equal(a, np.broadcast_to(b, a.shape)), f'frame {f}: max |diff| {np.abs(a.astype(int) - b.astype(int)).max()}'
    if image_mode == 'image':
        sharded = drivers.render_grid_frames_sharded(G, ws_grid, v, w_frames, batch=8, sampler_noise=noise)
        torch.cuda.current_stream().synchronize()
        assert sharded.shape == (4, *got[0].shape) and all(np.array_equal(sharded[f].numpy(), got[f]) for f in range(4))


def test_render_grid_frames_graph_path(tiny):
    from next3d_b200 import drivers
    cfg, G = tiny
    ws_grid, v, _ = _grid_workload(cfg, G, (3, 1), 1, 3)
    G.use_cuda_graph = True
    try:
        got = list(drivers.render_grid_frames(G, ws_grid, v, 3, batch=4, seed=5))
    finally:
        G.use_cuda_graph = False
    R = cfg.img_resolution
    assert len(got) == 3 and all(f.shape == (R, 3 * R, 3) and f.dtype == np.uint8 for f in got)
    assert np.abs(got[0][:, :R].astype(int) - got[0][:, R:2 * R].astype(int)).max() > 0


# ------------------------------------------------------------------------------------------------ reenactment grid
def _drive_root(tmp_path, cfg, G, n):
    """A driving directory: dataset.json, NNNN.png (seeded RGB photos, larger than the 512 crop), NNNN.obj and NNNN_kpt2d.txt (the
    demo mesh with jitter)."""
    from PIL import Image
    _, c, v, _ = _inputs(cfg, G, 1, 43)
    v = v.cpu()
    rng = np.random.RandomState(4)
    labels = []
    for k in range(n):
        name = f'{k:04d}'
        Image.fromarray(rng.randint(0, 256, (520, 530, 3), dtype=np.uint8)).save(tmp_path / f'{name}.png')
        vk = v[0].numpy() + rng.randn(*v[0].shape).astype(np.float32) * 1e-4
        (tmp_path / f'{name}.obj').write_text(''.join(f'v {float(a)!r} {float(b)!r} {float(c_)!r}\n' for a, b, c_ in vk[:5023]))
        (tmp_path / f'{name}_kpt2d.txt').write_text('\n'.join(f'{float(a)!r} {float(b)!r} {float(c_)!r}' for a, b, c_ in vk[5023:]) + '\n')
        cam = c[0].cpu().numpy().astype(np.float64)
        cam[3] += 0.01 * k
        labels.append([f'{name}.png', cam.tolist()])
    (tmp_path / 'dataset.json').write_text(json.dumps({'labels': labels}))
    return str(tmp_path)


def _reenact_reference(G, ws, root, noise):
    """reenact_avatar_next3d.py:125-167: per frame the photo, then one synthesis call per seed, then layout_grid (2x2)."""
    from PIL import Image
    from next3d_b200 import drivers, inputs
    sch = drivers.reenact_schedule(root, 100)
    S = ws.shape[0]
    frames = []
    for f, png in enumerate(sch['png_paths']):
        target_img = np.array(Image.open(png).crop((0, 0, 512, 512)))
        target_img = torch.tensor(target_img.transpose(2, 0, 1)).float().unsqueeze(0).to(DEV)
        target_img = target_img / 127.5 - 1.
        v = inputs.load_frame(sch['obj_paths'][f], sch['lms_paths'][f]).to(DEV)
        imgs = [target_img[0]]
        for s in range(S):
            i = f * S + s
            imgs.append(G.synthesis(ws[s:s + 1], sch['cams'][f:f + 1].to(DEV), v, noise_mode='const',
                                    sampler_noise=(noise[0][i:i + 1], noise[1][i]))['image'][0])
        frames.append(_layout_grid(torch.stack(imgs), 2, 2))
    return frames


def test_reenact_grid_frames_equals_per_seed_loop(tiny, tmp_path):
    """3 identities + the photo in a 2x2 grid, 5 frames in batches of 3 heads x 2 frames (a ragged last batch): the heads are cached
    once and every batch reuses them; frames equal the script's per-frame, per-seed loop pixel for pixel.  The sharded twin at
    world size 1 gives the same frames."""
    from next3d_b200 import drivers
    cfg, G = tiny
    root = _drive_root(tmp_path, cfg, G, 7)
    ws, _, _, _ = _inputs(cfg, G, 3, 44)
    S, F = 3, 5
    R = G.neural_rendering_resolution
    rk = G.rendering_kwargs
    g = torch.Generator().manual_seed(14)
    noise = (torch.rand(F * S, R * R, rk['depth_resolution'], 1, generator=g).to(DEV),
             torch.rand(F * S, R * R, rk['depth_resolution_importance'], generator=g).to(DEV))
    calls, synthesis = [], G.synthesis

    def recording(*a, **kw):
        calls.append((a[0].shape[0], kw.get('cache_backbone', False), kw.get('use_cached_backbone', False)))
        return synthesis(*a, **kw)
    G.synthesis = recording
    try:
        got = list(drivers.reenact_grid_frames(G, ws, root, 100, (2, 2), batch=6, sampler_noise=noise))
    finally:
        del G.synthesis
    assert calls == [(3, True, False)] + [(6, False, True)] * 3, calls
    ref = _reenact_reference(G, ws, root, noise)
    assert len(got) == len(ref) == F
    for f, (a, b) in enumerate(zip(got, ref)):
        assert a.shape == b.shape == (1024, 1024, 3)
        assert np.array_equal(a, b), f'frame {f}: max |diff| {np.abs(a.astype(int) - b.astype(int)).max()}'
    sharded = drivers.reenact_grid_frames_sharded(G, ws, root, 100, (2, 2), batch=6, sampler_noise=noise)
    torch.cuda.current_stream().synchronize()
    assert sharded.shape == (F, 1024, 1024, 3) and all(np.array_equal(sharded[f].numpy(), got[f]) for f in range(F))


def test_reenact_grid_frames_random_noise_runs_the_full_path(tiny, tmp_path):
    from next3d_b200 import drivers
    cfg, G = tiny
    root = _drive_root(tmp_path, cfg, G, 5)
    ws, _, _, _ = _inputs(cfg, G, 3, 45)
    calls, synthesis = [], G.synthesis

    def recording(*a, **kw):
        calls.append((a[0].shape[0], kw.get('cache_backbone', False), kw.get('use_cached_backbone', False)))
        return synthesis(*a, **kw)
    G.synthesis = recording
    try:
        got = list(drivers.reenact_grid_frames(G, ws, root, 100, (2, 2), batch=6, noise_mode='random', seed=3))
    finally:
        del G.synthesis
    assert calls == [(6, False, False)] * 2, calls
    assert len(got) == 3
    from PIL import Image
    sch = drivers.reenact_schedule(root, 100)
    for f, png in enumerate(sch['png_paths']):
        photo = torch.from_numpy(np.array(Image.open(png).crop((0, 0, 512, 512))))
        assert np.array_equal(got[f][:512, :512], drivers.photo_cell(photo, DEV).cpu().numpy())
        assert got[f][:512, 512:].std() > 0
