"""CPU oracle: ray generation, tri-plane sampling, MLP decode, importance sampling, compositing.
TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restates (fp32 torch on CPU):
  ray_sampler           volumetric_rendering/ray_sampler.py:24-63
  sample_from_planes    volumetric_rendering/renderer.py:30-72
  decoder               triplane_next3d.py:348-371 (OSGDecoder)
  ray_march             volumetric_rendering/ray_marcher.py:27-66 (MipRayMarcher2)
  render                volumetric_rendering/renderer.py:95-147, 184-268 (ImportanceRenderer, fixed ray_start/end)
The sampler's uniforms are ARGUMENTS (u_coarse [N,M,Dc,1], u_fine [N*M,Df]) instead of torch.rand calls
(renderer.py:205, :252) so the CUDA kernel and the reference can be fed identical noise.
"""
import torch
import torch.nn.functional as F

from . import ops


def ray_sampler(cam2world, intrinsics, res):
    N = cam2world.shape[0]
    cam = cam2world[:, :3, 3]
    fx, fy = intrinsics[:, 0, 0:1], intrinsics[:, 1, 1:2]
    cx, cy = intrinsics[:, 0, 2:3], intrinsics[:, 1, 2:3]
    sk = intrinsics[:, 0, 1:2]
    idx = torch.arange(res, dtype=cam2world.dtype)            # float32 in the reference; float64 for a high-precision evaluation
    centers = idx * (1.0 / res) + (0.5 / res)
    # ray m = i*res + j: x from column j, y from row i (ray_sampler.py:43-45: meshgrid 'ij', flip(0))
    y_cam = centers[:, None].expand(res, res).reshape(1, -1).expand(N, -1)
    x_cam = centers[None, :].expand(res, res).reshape(1, -1).expand(N, -1)
    z_cam = torch.ones(N, res * res, dtype=cam2world.dtype)
    x_lift = (x_cam - cx + cy * sk / fy - sk * y_cam / fy) / fx * z_cam
    y_lift = (y_cam - cy) / fy * z_cam
    pts = torch.stack([x_lift, y_lift, z_cam, torch.ones_like(z_cam)], -1)
    world = torch.bmm(cam2world, pts.permute(0, 2, 1)).permute(0, 2, 1)[:, :, :3]
    dirs = F.normalize(world - cam[:, None, :], dim=2)
    origins = cam[:, None, :].expand(-1, dirs.shape[1], -1).contiguous()
    return origins, dirs


# rows of the inverse plane-axis matrices, first two components (renderer.py:30-60):
# plane 0 <- (x, y), plane 1 <- (x, z), plane 2 <- (z, y)
_PLANE_COORDS = ((0, 1), (0, 2), (2, 1))


def sample_from_planes(planes, coords, box_warp):
    """planes [N,3,C,H,W], coords [N,S,3] -> features [N,3,S,C] (bilinear, zeros padding, align_corners=False)."""
    N, P, C, H, W = planes.shape
    coords = (2.0 / box_warp) * coords
    out = []
    for p, (a, b) in enumerate(_PLANE_COORDS):
        grid = torch.stack([coords[..., a], coords[..., b]], -1)[:, None]      # [N,1,S,2]
        f = F.grid_sample(planes[:, p], grid, mode='bilinear', padding_mode='zeros', align_corners=False)
        out.append(f[:, :, 0].permute(0, 2, 1))                                # [N,S,C]
    return torch.stack(out, 1)


def decoder(sd, feats):
    """feats [N,3,S,32] -> rgb [N,S,32], sigma [N,S,1]."""
    x = feats.mean(1)
    N, S, C = x.shape
    x = x.reshape(N * S, C)
    x = ops.fully_connected(x, sd['decoder.net.0.weight'], sd['decoder.net.0.bias'])
    x = F.softplus(x)
    x = ops.fully_connected(x, sd['decoder.net.2.weight'], sd['decoder.net.2.bias'])
    x = x.reshape(N, S, -1)
    rgb = torch.sigmoid(x[..., 1:]) * (1 + 2 * 0.001) - 0.001
    return rgb, x[..., 0:1]


def run_model(sd, planes, coords, opts):
    feats = sample_from_planes(planes, coords, opts['box_warp'])
    return decoder(sd, feats)


def ray_march(colors, densities, depths, opts):
    """[N,M,D,*] sorted along D -> composite rgb [N,M,C], depth [N,M,1], weights [N,M,D-1,1]."""
    deltas = depths[:, :, 1:] - depths[:, :, :-1]
    c_mid = (colors[:, :, :-1] + colors[:, :, 1:]) / 2
    s_mid = (densities[:, :, :-1] + densities[:, :, 1:]) / 2
    t_mid = (depths[:, :, :-1] + depths[:, :, 1:]) / 2
    assert opts['clamp_mode'] == 'softplus'
    s_mid = F.softplus(s_mid - 1)
    alpha = 1 - torch.exp(-(s_mid * deltas))
    shifted = torch.cat([torch.ones_like(alpha[:, :, :1]), 1 - alpha + 1e-10], -2)
    weights = alpha * torch.cumprod(shifted, -2)[:, :, :-1]
    rgb = torch.sum(weights * c_mid, -2)
    wsum = weights.sum(2)
    depth = torch.sum(weights * t_mid, -2) / wsum
    depth = torch.nan_to_num(depth, float('inf'))
    depth = torch.clamp(depth, torch.min(depths), torch.max(depths))           # batch-global range (ray_marcher.py:54)
    if opts.get('white_back', False):
        rgb = rgb + 1 - wsum
    return rgb * 2 - 1, depth, weights


def sample_pdf(bins, weights, u, eps=1e-5):
    n_w = weights.shape[1]
    weights = weights + eps
    pdf = weights / weights.sum(-1, keepdim=True)
    cdf = torch.cat([torch.zeros_like(pdf[:, :1]), torch.cumsum(pdf, -1)], -1)
    u = u.contiguous()
    inds = torch.searchsorted(cdf, u, right=True)
    below = (inds - 1).clamp_min(0)
    above = inds.clamp_max(n_w)
    cdf_b, cdf_a = torch.gather(cdf, 1, below), torch.gather(cdf, 1, above)
    bin_b, bin_a = torch.gather(bins, 1, below), torch.gather(bins, 1, above)
    denom = cdf_a - cdf_b
    denom = torch.where(denom < eps, torch.ones_like(denom), denom)
    return bin_b + (u - cdf_b) / denom * (bin_a - bin_b)


def sample_importance(z_vals, weights, u_fine):
    N, M, D, _ = z_vals.shape
    z = z_vals.reshape(N * M, D)
    w = weights.reshape(N * M, -1)
    w = F.max_pool1d(w[:, None].to(z.dtype), 2, 1, padding=1)
    w = F.avg_pool1d(w, 2, 1).squeeze(1)
    w = w + 0.01
    z_mid = 0.5 * (z[:, :-1] + z[:, 1:])
    return sample_pdf(z_mid, w[:, 1:-1], u_fine).reshape(N, M, u_fine.shape[1], 1)


def render(sd, planes, origins, dirs, opts, u_coarse, u_fine, return_depths=False):
    """-> rgb [N,M,32], depth [N,M,1], weight_sum [N,M,1] (+ the sorted sample depths [N,M,D] the composite used, with
    return_depths).  Runs in the dtype of its inputs: float32 is the reference's arithmetic, float64 a high-precision evaluation."""
    N, M, _ = origins.shape
    Dc = opts['depth_resolution']
    t0, t1 = float(opts['ray_start']), float(opts['ray_end'])
    assert not opts.get('disparity_space_sampling', False)
    depths_c = torch.linspace(t0, t1, Dc, dtype=origins.dtype).reshape(1, 1, Dc, 1).repeat(N, M, 1, 1)
    depths_c = depths_c + u_coarse * ((t1 - t0) / (Dc - 1))
    pts = (origins[:, :, None] + depths_c * dirs[:, :, None]).reshape(N, -1, 3)
    rgb_c, sig_c = run_model(sd, planes, pts, opts)
    rgb_c = rgb_c.reshape(N, M, Dc, -1)
    sig_c = sig_c.reshape(N, M, Dc, 1)
    Df = opts['depth_resolution_importance']
    if Df > 0:
        _, _, w = ray_march(rgb_c, sig_c, depths_c, opts)
        depths_f = sample_importance(depths_c, w, u_fine)
        pts = (origins[:, :, None] + depths_f * dirs[:, :, None]).reshape(N, -1, 3)
        rgb_f, sig_f = run_model(sd, planes, pts, opts)
        rgb_f = rgb_f.reshape(N, M, Df, -1)
        sig_f = sig_f.reshape(N, M, Df, 1)
        all_d = torch.cat([depths_c, depths_f], -2)
        all_c = torch.cat([rgb_c, rgb_f], -2)
        all_s = torch.cat([sig_c, sig_f], -2)
        _, idx = torch.sort(all_d, dim=-2, stable=True)
        all_d = torch.gather(all_d, -2, idx)
        all_c = torch.gather(all_c, -2, idx.expand(-1, -1, -1, all_c.shape[-1]))
        all_s = torch.gather(all_s, -2, idx)
        rgb, depth, w = ray_march(all_c, all_s, all_d, opts)
    else:
        all_d = depths_c
        rgb, depth, w = ray_march(rgb_c, sig_c, depths_c, opts)
    if return_depths:
        return rgb, depth, w.sum(2), all_d[..., 0]
    return rgb, depth, w.sum(2)
