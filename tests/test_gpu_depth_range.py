"""GPU: one depth range per image (N3DRender.depth_range_per_image, n3d_depth_clamp_images, the `depth_range` keyword).  A batch of
N images in per-image mode gives each image the depth range and clamped depth of a launch of its own, and leaves rgb / depth / wsum
(and the normals path) bit-identical to the batch-global mode."""
import pytest
import torch

from tests.test_gpu_normals import _workload
from tests.test_gpu_render_long_rays import _dec

pytestmark = pytest.mark.gpu
DEV = 'cuda'


@pytest.fixture(scope='module')
def K():
    from next3d_b200 import kernels
    return kernels


def _outputs(N, M, per_image):
    nan = float('nan')
    mm = torch.tensor([float('inf'), float('-inf')], device=DEV)
    return [torch.full((N, M, 32), nan, device=DEV), torch.full((N, M), nan, device=DEV), torch.full((N, M), nan, device=DEV),
            mm.repeat(N, 1) if per_image else mm.clone()]


@pytest.mark.parametrize('D', [48, 96, 144])                 # the 16-, 32- and 64-lane layouts
@pytest.mark.parametrize('B,V', [(3, 1), (2, 3)])
def test_per_image_range_equals_one_launch_per_image(K, B, V, D):
    """Pair n and the clamped depth of image n == a flag-0 launch of image n alone (same injected uniforms), bit for bit; rgb,
    depth and wsum == the flag-0 launch of the whole batch; the batch-global pair is the min / max over the per-image pairs.
    res 13: ragged pixel blocks and groups that straddle CTAs in every layout."""
    N, res = B * V, 13
    M = res * res
    opts, planes, sd, c, u_c, u_f = _workload(N, res, D, D, 0)
    sets = planes[:B].permute(0, 1, 3, 4, 2).contiguous().to(DEV)
    cam, intr = c[:, :16].contiguous().to(DEV), c[:, 16:25].contiguous().to(DEV)
    u_c, u_f = u_c.to(DEV), u_f.to(DEV).view(N, M, D)
    dec = _dec(sd)
    glob, per = _outputs(N, M, False), _outputs(N, M, True)
    K.render_rays(sets, cam, intr, res, opts, dec, *glob, u_coarse=u_c, u_fine=u_f, views=V)
    K.render_rays(sets, cam, intr, res, opts, dec, *per, u_coarse=u_c, u_fine=u_f, views=V, depth_range_per_image=1)
    for x, y, name in zip(glob[:3], per[:3], ('rgb', 'depth', 'wsum')):
        assert torch.equal(x, y), name
    mm = per[3]
    assert mm.shape == (N, 2) and torch.equal(glob[3], torch.stack([mm[:, 0].min(), mm[:, 1].max()]))
    clamped = per[1].clone()
    K.depth_clamp_images(clamped, mm)
    for n in range(N):
        one = _outputs(1, M, False)
        K.render_rays(sets[n // V:n // V + 1], cam[n:n + 1], intr[n:n + 1], res, opts, dec, *one, u_coarse=u_c[n:n + 1],
                      u_fine=u_f[n].contiguous())
        assert torch.equal(one[3], mm[n]), (n, one[3], mm[n])
        assert torch.equal(one[1], per[1][n:n + 1]), n
        K.depth_clamp(one[1], one[3])
        assert torch.equal(one[1], clamped[n:n + 1]), n
    assert (mm[:, 0] < mm[:, 1]).all() and not torch.equal(mm[0], mm[-1])


@pytest.mark.parametrize('D', [48, 96, 144])
@pytest.mark.parametrize('B,V', [(3, 1), (1, 4)])
def test_per_image_range_through_normals_with_kernel_rng(K, B, V, D):
    """render_rays_normals in per-image mode with the in-kernel RNG: every output but the range == flag 0, and pair n == the min
    of the first and the max of the last sorted sample depth over image n's rays, read from the exported workspace."""
    N, res = B * V, 13
    M = res * res
    opts, planes, sd, c, _, _ = _workload(N, res, D, D, 0)
    sets = planes[:B].permute(0, 1, 3, 4, 2).contiguous().to(DEV)
    cam, intr = c[:, :16].contiguous().to(DEV), c[:, 16:25].contiguous().to(DEV)
    dec = _dec(sd)
    runs = []
    for per_image in (0, 1):
        out = _outputs(N, M, per_image)
        normal = torch.full((N, M, 3), float('nan'), device=DEV)
        ws = torch.full((K.normals_workspace_floats(N, res, opts),), float('nan'), device=DEV)
        K.render_rays_normals(sets, cam, intr, res, opts, dec, *out, normal, ws, seed=91, views=V, depth_range_per_image=per_image)
        runs.append(out + [normal, ws])
    for x, y, name in zip(runs[0][:3] + runs[0][4:], runs[1][:3] + runs[1][4:], ('rgb', 'depth', 'wsum', 'normal', 'workspace')):
        assert torch.equal(x.nan_to_num(123.0), y.nan_to_num(123.0)), name
    Dt = 2 * D
    samples = runs[1][5].view(N, M, 2 * Dt - 1)
    want = torch.stack([samples[:, :, 0].amin(1), samples[:, :, Dt - 1].amax(1)], 1)
    assert torch.equal(runs[1][3], want)
    assert torch.equal(runs[0][3], torch.stack([want[:, 0].min(), want[:, 1].max()]))


def test_generator_depth_range_keyword():
    """synthesis / render_views with depth_range='image' (eager and graphed): image and image_raw unchanged, image_depth of each
    image == a batch-1 call; the default is the batch-global range."""
    from next3d_b200 import config, weights
    from next3d_b200.triplane_next3d import TriPlaneGenerator
    cfg = config.tiny_config(512)
    G = TriPlaneGenerator.from_config(cfg, weights.make_state_dict(cfg, seed=6), device=DEV)
    N = 3
    z, cc, c, v = weights.demo_inputs(cfg, N, seed=8)
    ws = G.mapping(z.to(DEV), cc.to(DEV), truncation_psi=0.7, truncation_cutoff=14)
    c, v = c.to(DEV), v.to(DEV)
    u_c, u_f = (t.to(DEV) for t in weights.sampler_noise(cfg, N, seed=8))
    M = G.neural_rendering_resolution ** 2
    noise = (u_c, u_f)
    batch = {k: t.clone() for k, t in G.synthesis(ws, c, v, noise_mode='const', sampler_noise=noise).items()}
    per = {k: t.clone() for k, t in G.synthesis(ws, c, v, noise_mode='const', sampler_noise=noise, depth_range='image').items()}
    assert torch.equal(batch['image'], per['image']) and torch.equal(batch['image_raw'], per['image_raw'])
    for n in range(N):
        one = G.synthesis(ws[n:n + 1], c[n:n + 1], v[n:n + 1], noise_mode='const', sampler_noise=(u_c[n:n + 1], u_f[n * M:(n + 1) * M]))
        assert torch.equal(one['image_depth'], per['image_depth'][n:n + 1]), n
    with pytest.raises(ValueError, match='depth_range'):
        G.synthesis(ws, c, v, noise_mode='const', depth_range='frame')
    # render_views of one cached head, and the graph paths (the range is part of the graph key)
    G.synthesis(ws[:1], c[:1], v[:1], noise_mode='const', seed=1, cache_backbone=True)
    views = G.render_views(c, sampler_noise=noise, depth_range='image')['image_depth'].clone()
    for n in range(N):
        one = G.render_views(c[n:n + 1], sampler_noise=(u_c[n:n + 1], u_f[n * M:(n + 1) * M]))['image_depth']
        assert torch.equal(one, views[n:n + 1]), n
    eager = {r: G.render_views(c, seed=5, depth_range=r)['image_depth'].clone() for r in ('batch', 'image')}
    G.use_cuda_graph = True
    try:
        for r in ('batch', 'image', 'batch'):
            assert torch.equal(G.render_views(c, seed=5, depth_range=r)['image_depth'], eager[r]), r
        g_batch = G.synthesis(ws, c, v, noise_mode='const', seed=3)['image_depth'].clone()
        g_per = G.synthesis(ws, c, v, noise_mode='const', seed=3, depth_range='image')['image_depth'].clone()
    finally:
        G.use_cuda_graph = False
    assert torch.equal(g_batch, G.synthesis(ws, c, v, noise_mode='const', seed=3)['image_depth'])
    assert torch.equal(g_per, G.synthesis(ws, c, v, noise_mode='const', seed=3, depth_range='image')['image_depth'])
