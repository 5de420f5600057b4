"""GPU: surface normals (rendering option return_normal) -- n3d_render_rays_normals against the CPU oracle
(oracle.normals.render_normals, autograd through grid_sample and the decoder) and the generator's 'image_normal' output.

Normal metrics.  The direction of n_raw is ill-conditioned where |n_raw| is tiny, so the unit-normal error of a ray is weighted
by |n_raw_ref| / max |n_raw_ref| (weighted), and the plain unit-normal error is taken over the rays with |n_raw_ref| >= 1% of
the maximum (strong)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda'


@pytest.fixture(scope='module')
def K():
    from next3d_b200 import kernels
    return kernels


def _normal_errors(n, n_ref, n_raw_ref, keep=None):
    """-> (max weighted |dn|, max |dn| over the strong rays); n, n_ref [..., 3] unit normals, n_raw_ref [..., 3]; keep: rays compared."""
    dn = (n.double() - n_ref.double()).norm(dim=-1)
    mag = n_raw_ref.double().norm(dim=-1)
    keep = torch.ones_like(mag, dtype=torch.bool) if keep is None else keep
    weighted = (dn * mag / mag.max())[keep].max().item()
    strong = dn[keep & (mag >= 0.01 * mag.max())].max().item()
    return weighted, strong


def _check_against_oracle(sd, planes, o, d, opts, samples, normal, ref, tol_weighted=1e-4):
    """The exported samples against the oracle's sorted depths and final weights (fp32 rounding of the renderer), then the kernel's
    normals against the oracle evaluated on the kernel's own samples with the strict metrics, on every ray whose weighted samples
    stay clear of bilinear cell edges (oracle.normals.near_cell_edge: the density gradient jumps there, so the last-bit difference
    between the kernel's and the oracle's float formulation of a camera ray changes such a sample's normal by O(1)).  Against the
    oracle's own sampling the median ray must agree too.  ref = render_normals(..., return_samples=True)."""
    from oracle import normals as onr
    N, M, _ = normal.shape
    D = (samples.shape[-1] + 1) // 2
    t, w = samples[..., :D].cpu(), samples[..., D:].cpu()
    n_full, t_ref, w_ref = ref[3], ref[5], ref[6]
    assert (t - t_ref).abs().max().item() <= 1e-4, (t - t_ref).abs().max().item()
    assert (w - w_ref).abs().max().item() <= 1e-4, (w - w_ref).abs().max().item()
    n_ref, n_raw_ref = onr.composite_normals(sd, planes, o, d, opts, t, w)
    near = onr.near_cell_edge(planes, o, d, opts, t, w)
    weighted, strong = _normal_errors(normal.cpu(), n_ref, n_raw_ref, keep=~near)
    assert weighted <= tol_weighted and strong <= 1e-3, (weighted, strong, near.float().mean().item())
    assert near.float().mean().item() <= 0.25
    assert (normal.cpu().double() - n_full.double()).norm(dim=-1).median().item() <= 1e-4
    return n_raw_ref


def _workload(N, res, D, Df, ties):
    from next3d_b200 import config, weights
    cfg = config.tiny_config()
    opts = dict(cfg.rendering_kwargs, depth_resolution=D, depth_resolution_importance=Df)
    g = torch.Generator().manual_seed(47 + res)
    planes = torch.randn(N, 3, 32, 64, 64, generator=g)
    sd = {'decoder.net.0.weight': torch.randn(64, 32, generator=g), 'decoder.net.0.bias': torch.randn(64, generator=g) * 0.1,
          'decoder.net.2.weight': torch.randn(33, 64, generator=g), 'decoder.net.2.bias': torch.randn(33, generator=g) * 0.1}
    _, _, c, _ = weights.demo_inputs(cfg, N, seed=5)
    u_c = torch.rand(N, res * res, D, 1, generator=g)
    u_f = torch.rand(N * res * res, max(Df, 1), generator=g)
    if ties:
        u_f = torch.floor(u_f * 5) / 5 + 0.01
    return opts, planes, sd, c, u_c, u_f


# the shapes of test_gpu_kernels.py::test_render_rays: both lane layouts, ragged tiles, coarse-only, unequal resolutions, ties
@pytest.mark.parametrize('N,res,D,Df,ties', [(2, 32, 48, 48, 0), (1, 16, 96, 96, 0), (1, 24, 36, 36, 0), (1, 20, 48, 0, 0), (1, 16, 40, 24, 0),
                                             (2, 12, 12, 70, 0), (3, 64, 48, 48, 0), (1, 16, 48, 48, 1), (1, 12, 96, 96, 1), (1, 12, 96, 96, 0)])
def test_render_rays_normals_and_normal_pass(K, N, res, D, Df, ties):
    """render_rays_normals against render_rays (bit for bit) and the oracle; the normal pass alone (n3d_render_normals_pass) over the
    same workspace reproduces the normals exactly."""
    from oracle import normals as onr, renderer as orr
    opts, planes, sd, c, u_c, u_f = _workload(N, res, D, Df, ties)
    o, d = orr.ray_sampler(c[:, :16].reshape(-1, 4, 4), c[:, 16:25].reshape(-1, 3, 3), res)
    ref = onr.render_normals(sd, planes, o, d, opts, u_c, u_f, return_samples=True)
    dec = ((sd['decoder.net.0.weight'] / math.sqrt(32)).to(DEV).contiguous(), sd['decoder.net.0.bias'].to(DEV),
           (sd['decoder.net.2.weight'] / math.sqrt(64)).to(DEV).contiguous(), sd['decoder.net.2.bias'].to(DEV))
    pl = planes.permute(0, 1, 3, 4, 2).contiguous().to(DEV)
    cam, intr = c[:, :16].contiguous().to(DEV), c[:, 16:25].contiguous().to(DEV)
    M = res * res

    def outputs():
        return (torch.zeros(N, M, 32, device=DEV), torch.zeros(N, M, device=DEV), torch.zeros(N, M, device=DEV),
                torch.tensor([float('inf'), 0.0], device=DEV))

    for noise in (dict(u_coarse=u_c.to(DEV), u_fine=u_f.to(DEV)), dict(seed=123)):
        a, b = outputs(), outputs()
        K.render_rays(pl, cam, intr, res, opts, dec, *a, **noise)
        normal = torch.full((N, M, 3), float('nan'), device=DEV)
        work = torch.full((K.normals_workspace_floats(N, res, opts),), float('nan'), device=DEV)
        K.render_rays_normals(pl, cam, intr, res, opts, dec, *b, normal, work, **noise)
        for x, y, name in zip(a, b, ('rgb', 'depth', 'wsum', 'depth_minmax')):
            assert torch.equal(x, y), name
        if 'u_coarse' in noise:
            n_raw_ref = _check_against_oracle(sd, planes, o, d, opts, work.view(N, M, -1), normal, ref)
            # the normal pass alone (timing diagnostics) over the same workspace reproduces the normals
            alt = torch.full_like(normal, float('nan'))
            K.render_normals_pass(pl, cam, intr, res, opts, dec, alt, work)
            assert torch.equal(alt, normal)
        else:                                        # in-kernel RNG: unit length wherever the ray carries weight
            live = b[2] > 1e-3
            assert torch.isfinite(normal[live]).all()
            assert (normal[live].norm(dim=-1) - 1).abs().max().item() <= 1e-5


def test_render_rays_normals_rejects_a_short_workspace(K):
    opts, planes, sd, c, u_c, u_f = _workload(1, 8, 12, 12, 0)
    dec = tuple(t.to(DEV) for t in (sd['decoder.net.0.weight'], sd['decoder.net.0.bias'], sd['decoder.net.2.weight'], sd['decoder.net.2.bias']))
    rgb, depth, wsum = torch.zeros(1, 64, 32, device=DEV), torch.zeros(1, 64, device=DEV), torch.zeros(1, 64, device=DEV)
    normal = torch.zeros(1, 64, 3, device=DEV)
    assert K.normals_workspace_floats(1, 8, opts) == 64 * (2 * 24 - 1)
    with pytest.raises(RuntimeError, match='workspace'):
        K.render_rays_normals(planes.permute(0, 1, 3, 4, 2).contiguous().to(DEV), c[:, :16].contiguous().to(DEV), c[:, 16:25].contiguous().to(DEV),
                              8, opts, dec, rgb, depth, wsum, None, normal, torch.zeros(10, device=DEV), seed=1)


def test_generator_image_normal():
    """Flag on: image / image_raw / image_depth bit-identical to flag off; image_normal matches the oracle on the engine's own
    planes; graph replay == eager; toggling the flag re-captures the graph and adds the normal launch only while it is on."""
    from next3d_b200 import config, weights
    from next3d_b200.triplane_next3d import TriPlaneGenerator
    from oracle import normals as onr, renderer as orr
    cfg = config.tiny_config(512)
    sd = weights.make_state_dict(cfg, seed=2)
    G = TriPlaneGenerator.from_config(cfg, sd, device=DEV)
    N = 2
    z, c_cond, c_cam, v = weights.demo_inputs(cfg, N, seed=2)
    u_c, u_f = weights.sampler_noise(cfg, N, seed=2)
    ws = G.mapping(z.to(DEV), c_cond.to(DEV), truncation_psi=0.7, truncation_cutoff=14)
    kw = dict(noise_mode='const', sampler_noise=(u_c.to(DEV), u_f.to(DEV)))
    off = {k: t.clone() for k, t in G.synthesis(ws, c_cam.to(DEV), v.to(DEV), **kw).items()}
    launches_off = G._engine.launches
    assert 'image_normal' not in off
    G.rendering_kwargs['return_normal'] = True
    try:
        on = G.synthesis(ws, c_cam.to(DEV), v.to(DEV), return_intermediates=True, **kw)
        assert G._engine.launches == launches_off + 1
        for k in ('image', 'image_raw', 'image_depth'):
            assert torch.equal(on[k], off[k]), k
        R = cfg.neural_rendering_resolution
        n = on['image_normal']
        assert n.shape == (N, 3, R, R) and n.dtype == torch.float32
        planes = on['intermediates']['planes'].permute(0, 1, 4, 2, 3).cpu()
        o, d = orr.ray_sampler(c_cam[:, :16].reshape(-1, 4, 4), c_cam[:, 16:25].reshape(-1, 3, 3), R)
        sd_dec = {k: v_.float().cpu() for k, v_ in sd.items() if k.startswith('decoder.')}
        ref = onr.render_normals(sd_dec, planes, o, d, G.rendering_kwargs, u_c, u_f, return_samples=True)
        _check_against_oracle(sd_dec, planes, o, d, G.rendering_kwargs, on['intermediates']['normal_samples'],
                              n.permute(0, 2, 3, 1).reshape(N, R * R, 3), ref, tol_weighted=1e-3)
        # CUDA graph replay == eager (in-kernel RNG, same seed)
        eager = {k: t.clone() for k, t in G.synthesis(ws, c_cam.to(DEV), v.to(DEV), noise_mode='const', seed=7).items()}
        G.use_cuda_graph = True
        graphed = {k: t.clone() for k, t in G.synthesis(ws, c_cam.to(DEV), v.to(DEV), noise_mode='const', seed=7).items()}
        assert G._engine.launches == launches_off + 1
        assert set(graphed) == set(eager)
        for k in eager:
            assert torch.equal(graphed[k], eager[k]), k
    finally:
        G.rendering_kwargs['return_normal'] = False
    # flag off again: another graph, without the normal output or its launch
    plain = G.synthesis(ws, c_cam.to(DEV), v.to(DEV), noise_mode='const', seed=7)
    G.use_cuda_graph = False
    assert 'image_normal' not in plain and G._engine.launches == launches_off
    for k in ('image', 'image_raw', 'image_depth'):
        assert torch.equal(plain[k], graphed[k]), k
