"""CPU oracle of the normal path: ImportanceRenderer.normal_forward + MipRayMarcher2 with return_normal.
TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restates (fp32 torch on CPU):
  normal_forward        volumetric_rendering/renderer.py:271-355 (per-sample normal = -autograd grad of sigma w.r.t. the point)
  unify_samples         volumetric_rendering/renderer.py:164-182 (normals follow the depth sort)
  ray_march + normals   volumetric_rendering/ray_marcher.py:32-33, 61-64
The gradient is taken with torch.autograd.grad through grid_sample and the decoder, as the reference does, so it is independent of
the CUDA kernel's analytic formulation.  Sampling is exactly oracle.renderer.render's (same uniforms as arguments).
"""
import torch

from . import renderer as orr


def _model_with_normals(sd, planes, pts, opts):
    """pts [N,S,3] -> rgb [N,S,32], sigma [N,S,1], normal = -d sigma / d pts [N,S,3]."""
    pts = pts.detach().requires_grad_(True)
    with torch.enable_grad():
        rgb, sig = orr.run_model(sd, planes, pts, opts)
        grad = torch.autograd.grad(sig.sum(), pts)[0]
    return rgb.detach(), sig.detach(), -grad


def composite_normals(sd, planes, origins, dirs, opts, depths, weights):
    """Normals at given sorted samples: depths [N,M,D], final weights [N,M,D-1] (e.g. the ones the renderer used) ->
    normal [N,M,3] (unit length), normal_raw [N,M,3]."""
    N, M, D = depths.shape
    pts = (origins[:, :, None] + depths[..., None] * dirs[:, :, None]).reshape(N, -1, 3)
    _, _, nrm = _model_with_normals(sd, planes, pts, opts)
    nrm = nrm.reshape(N, M, D, 3)
    normal_raw = torch.sum(weights[..., None] * (nrm[:, :, :-1] + nrm[:, :, 1:]) / 2, -2) / weights.sum(-1, keepdim=True)
    return normal_raw / (torch.norm(normal_raw, dim=-1, keepdim=True) + 1e-7), normal_raw


def near_cell_edge(planes, origins, dirs, opts, depths, weights, tol=1e-6):
    """[N,M] True where a sample that carries weight lies within `tol` (world units) of a bilinear cell edge of some plane.  The
    density gradient jumps across a cell edge, so there a last-bit difference in the sample position (two float formulations of
    the same camera ray differ by a few ulps of the ~2.7-unit camera origin, ~2.4e-7 each) changes that sample's normal by O(1):
    such rays cannot be compared at fp32 precision.  The default, 1e-6, is about four such ulps."""
    N, M, D = depths.shape
    _, _, _, H, W = planes.shape
    scale = 2.0 / opts['box_warp']
    x = (origins[:, :, None] + depths[..., None] * dirs[:, :, None]) * scale
    coef = torch.zeros_like(depths)
    coef[..., :-1] += weights
    coef[..., 1:] += weights
    near = torch.zeros_like(depths, dtype=torch.bool)
    for a, b in orr._PLANE_COORDS:
        for axis, size in ((a, W), (b, H)):
            i = ((x[..., axis] + 1) * size - 1) / 2
            near |= (i - torch.round(i)).abs() < tol * scale * size / 2      # d i / d x = scale * size / 2 texels per world unit
    return (near & (coef > 0)).any(-1)


def render_normals(sd, planes, origins, dirs, opts, u_coarse, u_fine, return_samples=False):
    """-> rgb [N,M,32], depth [N,M,1], weight_sum [N,M,1], normal [N,M,3] (unit length), normal_raw [N,M,3] (before normalising).
    rgb / depth / weight_sum are oracle.renderer.render's.  return_samples: also the merged sorted depths [N,M,D] and the final
    weights [N,M,D-1] the composite used."""
    N, M, _ = origins.shape
    Dc = opts['depth_resolution']
    t0, t1 = float(opts['ray_start']), float(opts['ray_end'])
    depths_c = torch.linspace(t0, t1, Dc).reshape(1, 1, Dc, 1).repeat(N, M, 1, 1)
    depths_c = depths_c + u_coarse * ((t1 - t0) / (Dc - 1))
    pts = (origins[:, :, None] + depths_c * dirs[:, :, None]).reshape(N, -1, 3)
    rgb_c, sig_c, nrm_c = _model_with_normals(sd, planes, pts, opts)
    rgb_c, sig_c, nrm_c = rgb_c.reshape(N, M, Dc, -1), sig_c.reshape(N, M, Dc, 1), nrm_c.reshape(N, M, Dc, 3)
    Df = opts['depth_resolution_importance']
    if Df > 0:
        _, _, w = orr.ray_march(rgb_c, sig_c, depths_c, opts)
        depths_f = orr.sample_importance(depths_c, w, u_fine)
        pts = (origins[:, :, None] + depths_f * dirs[:, :, None]).reshape(N, -1, 3)
        rgb_f, sig_f, nrm_f = _model_with_normals(sd, planes, pts, opts)
        all_d = torch.cat([depths_c, depths_f], -2)
        all_c = torch.cat([rgb_c, rgb_f.reshape(N, M, Df, -1)], -2)
        all_s = torch.cat([sig_c, sig_f.reshape(N, M, Df, 1)], -2)
        all_n = torch.cat([nrm_c, nrm_f.reshape(N, M, Df, 3)], -2)
        _, idx = torch.sort(all_d, dim=-2, stable=True)
        all_d = torch.gather(all_d, -2, idx)
        all_c = torch.gather(all_c, -2, idx.expand(-1, -1, -1, all_c.shape[-1]))
        all_s = torch.gather(all_s, -2, idx)
        all_n = torch.gather(all_n, -2, idx.expand(-1, -1, -1, 3))
    else:
        all_d, all_c, all_s, all_n = depths_c, rgb_c, sig_c, nrm_c
    rgb, depth, w = orr.ray_march(all_c, all_s, all_d, opts)
    n_mid = (all_n[:, :, :-1] + all_n[:, :, 1:]) / 2
    normal_raw = torch.sum(w * n_mid, -2) / w.sum(2)
    normal = normal_raw / (torch.norm(normal_raw, dim=-1, keepdim=True) + 1e-7)
    if return_samples:
        return rgb, depth, w.sum(2), normal, normal_raw, all_d[..., 0], w[..., 0]
    return rgb, depth, w.sum(2), normal, normal_raw
