"""CPU oracle: the whole generator forward (`TriPlaneGenerator.synthesis`) as fp32 torch on CPU.
TEST INFRASTRUCTURE, NOT PRODUCT CODE (see oracle/__init__.py).

Functional restatement over a flat state dict (names = the reference's state-dict names):
  mapping                networks_stylegan2.py:233-268 via triplane_next3d.py:111-115
  synthesis_layer        networks_stylegan2.py:311-330      torgb          :353-357
  synthesis_block        networks_stylegan2.py:544-588      backbone       :630-645
  styleunet              networks_stylegan2_styleunet.py:107-115, 198-207, 554-588
  rasterize              triplane_next3d.py:190-230 + volumetric_rendering/renderer.py:401-440, 505-547
  fill_mouth             volumetric_rendering/renderer.py:583-602
  gen_mouth_mask         triplane_next3d.py:330-344
  superresolution        superresolution.py:77-88 (4X), :279-290 (8XDC), SynthesisBlockNoUp :158-254
  synthesis              triplane_next3d.py:117-188
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from next3d_b200 import config as _config
from . import ops, renderer, rasterize as _rast


# ------------------------------------------------------------------------------------------ mapping

def mapping(sd, cfg, z, c, truncation_psi=1.0, truncation_cutoff=None, prefix='backbone.mapping', num_ws=28):
    rk = cfg.rendering_kwargs
    if rk['c_gen_conditioning_zero']:
        c = torch.zeros_like(c)
    c = c[:, :25] * rk.get('c_scale', 0)
    x = z.to(torch.float32)
    x = x * (x.square().mean(1, keepdim=True) + 1e-8).rsqrt()
    y = ops.fully_connected(c.to(torch.float32), sd[f'{prefix}.embed.weight'], sd[f'{prefix}.embed.bias'])
    y = y * (y.square().mean(1, keepdim=True) + 1e-8).rsqrt()
    x = torch.cat([x, y], 1)
    for i in range(2):
        x = ops.fully_connected(x, sd[f'{prefix}.fc{i}.weight'], sd[f'{prefix}.fc{i}.bias'], activation='lrelu',
                                lr_multiplier=0.01)
    x = x[:, None].repeat(1, num_ws, 1)
    if truncation_psi != 1:
        w_avg = sd[f'{prefix}.w_avg']
        if truncation_cutoff is None:
            x = w_avg.lerp(x, truncation_psi)
        else:
            x[:, :truncation_cutoff] = w_avg.lerp(x[:, :truncation_cutoff], truncation_psi)
    return x


# ------------------------------------------------------------------------------------------ StyleGAN2 blocks

def synthesis_layer(sd, p, x, w, up=1, noise_mode='const', clamp=None):
    """noise_mode: 'const', 'none', or a dict {layer name: [N,1,H,W] noise already multiplied by noise_strength} that stands for
    'random' with known draws (networks_stylegan2.py:318-319)."""
    styles = ops.fully_connected(w, sd[f'{p}.affine.weight'], sd[f'{p}.affine.bias'])
    noise = None
    if isinstance(noise_mode, dict):
        noise = noise_mode[p]
    elif noise_mode == 'const':
        noise = sd[f'{p}.noise_const'] * sd[f'{p}.noise_strength']
    elif noise_mode != 'none':
        raise ValueError('oracle supports noise_mode const/none or injected per-layer noise (random is not reproducible)')
    x = ops.modulated_conv2d(x, sd[f'{p}.weight'], styles, noise=noise, up=up, padding=1,
                             resample_filter=sd[f'{p}.resample_filter'], flip_weight=(up == 1))
    return ops.bias_act(x, sd[f'{p}.bias'], act='lrelu', clamp=clamp)


def torgb(sd, p, x, w, clamp=None):
    weight = sd[f'{p}.weight']
    styles = ops.fully_connected(w, sd[f'{p}.affine.weight'], sd[f'{p}.affine.bias'])
    styles = styles * (1.0 / math.sqrt(weight.shape[1] * weight.shape[2] ** 2))
    x = ops.modulated_conv2d(x, weight, styles, demodulate=False)
    return ops.bias_act(x, sd[f'{p}.bias'], clamp=clamp)


def synthesis_block(sd, p, x, img, ws, noise_mode='const', clamp=None, up=True, first=False):
    it = iter(ws.unbind(1))
    if first:
        x = sd[f'{p}.const'][None].repeat(ws.shape[0], 1, 1, 1)
    else:
        x = synthesis_layer(sd, f'{p}.conv0', x, next(it), up=2 if up else 1, noise_mode=noise_mode, clamp=clamp)
    x = synthesis_layer(sd, f'{p}.conv1', x, next(it), noise_mode=noise_mode, clamp=clamp)
    if img is not None and up:
        img = ops.upsample2d(img, sd[f'{p}.resample_filter'])
    y = torgb(sd, f'{p}.torgb', x, next(it), clamp=clamp)
    img = img + y if img is not None else y
    return x, img


def _split_ws(ws, resolutions):
    """ws.narrow(1, w_idx, num_conv + 1); w_idx += num_conv  (networks_stylegan2.py:634-639)."""
    out, idx = [], 0
    for res in resolutions:
        nconv = 1 if res == 4 else 2
        out.append(ws[:, idx: idx + nconv + 1])
        idx += nconv
    return out


def backbone(sd, cfg, prefix, ws, noise_mode='const'):
    res_list = _config.block_resolutions(cfg.plane_res)
    x = img = None
    for res, cur in zip(res_list, _split_ws(ws.to(torch.float32), res_list)):
        x, img = synthesis_block(sd, f'{prefix}.b{res}', x, img, cur, noise_mode=noise_mode, first=(res == 4))
    return img


def conv2d_layer(sd, p, x, k, activation='linear', down=1):
    w = sd[f'{p}.weight']
    w = w * (1.0 / math.sqrt(w.shape[1] * k * k))
    x = ops.conv2d_resample(x, w, f=sd[f'{p}.resample_filter'], down=down, padding=k // 2, flip_weight=True)
    return ops.bias_act(x, sd.get(f'{p}.bias'), act=activation)


def styleunet(sd, cfg, prefix, x_in, ws, in_size, final_size, num_cond_res, noise_mode='const'):
    res_list = _config.block_resolutions(cfg.plane_res)
    block_ws = _split_ws(ws.to(torch.float32), res_list)
    enc_res = _config.encoder_resolutions(in_size, final_size)
    cond_list, cond = [], None
    for i, res in enumerate(enc_res[:-1]):
        p = f'{prefix}.encoder.{i}'
        if res < in_size:
            x_in = ops.downsample2d(x_in, sd[f'{p}.resample_filter'])
        out = conv2d_layer(sd, f'{p}.fromrgb', x_in, 1)
        if cond is not None:
            out = out + cond
        out = conv2d_layer(sd, f'{p}.conv1', out, 3, activation='lrelu')
        cond = conv2d_layer(sd, f'{p}.conv2', out, 3, activation='lrelu', down=2)
        cond_list.append(cond)
    cond_list = cond_list[::-1]
    start = int(math.log2(final_size)) - 1
    x = img = None
    for index, (res, cur) in enumerate(zip(res_list[start:], block_ws[start:])):
        if 2 ** (index + int(math.log2(final_size))) < num_cond_res:
            if index == 0:
                x = conv2d_layer(sd, f'{prefix}.fusion.{index}', cond_list[index], 3)
            else:
                x = conv2d_layer(sd, f'{prefix}.fusion.{index}', torch.cat([x, cond_list[index]], 1), 3)
        x, img = synthesis_block(sd, f'{prefix}.b{res}', x, img, cur, noise_mode=noise_mode)
    return img


# ------------------------------------------------------------------------------------------ rasterization

VIEWS = ((0, 0, 0), (0, 90, 0), (0, -90, 0), (90, 0, 0))           # triplane_next3d.py:140-145


def angle2matrix(angles_deg):
    """[3] degrees -> [3,3]; fp32 sin/cos of angle*pi/180 (cos(90 deg) != 0 is reproduced, renderer.py:528-546)."""
    a = torch.tensor(angles_deg, dtype=torch.float32).reshape(1, 3) * np.pi / 180.
    s, c = torch.sin(a), torch.cos(a)
    cx, cy, cz = c[0, 0], c[0, 1], c[0, 2]
    sx, sy, sz = s[0, 0], s[0, 1], s[0, 2]
    return torch.stack([cz * cy, cz * sy * sx - sz * cx, cz * sy * cx + sz * sx,
                        sz * cy, sz * sy * sx + cz * cx, sz * sy * cx - cz * sx,
                        -sy, cy * sx, cy * cx]).reshape(3, 3)


def _bmm3_fma(p, R):
    """torch.bmm(p [N,P,3], R [N,3,3]) with the summation order written out: the reference's bmm (renderer.py:505-514 via
    triplane_next3d.py:197) leaves it to the BLAS; oneMKL's fp32 kernel evaluates K = 3 as the fused chain
    fma(p2, R2j, fma(p1, R1j, p0 * R0j)) (checked bit for bit in tests/test_oracle_vs_reference.py).  Each fma is emulated in
    float64, where the product of two float32 is exact, so the result does not depend on the BLAS of the machine running the
    oracle and the CUDA kernel can reproduce it exactly."""
    p64, R64 = p.double(), R.double()
    acc = (p64[:, :, 0:1] * R64[:, 0:1, :]).float()
    acc = (p64[:, :, 1:2] * R64[:, 1:2, :] + acc.double()).float()
    return (p64[:, :, 2:3] * R64[:, 2:3, :] + acc.double()).float()


def transform_view(points, view):
    """(v*[1,-1,1]) @ R + shift, *5, orth-proj with camera [1,0,0] (identity), negate y,z (triplane_next3d.py:194-205)."""
    p = points.clone()
    p[..., 1] *= -1
    R = angle2matrix(view)[None].expand(p.shape[0], -1, -1)
    p = (_bmm3_fma(p, R) + torch.tensor([[0, -0.01, -0.01]])) * torch.tensor([[5.0]])
    cam = torch.tensor([1., 0., 0.]).view(-1, 1, 3)
    p = torch.cat([p[:, :, :2] + cam[:, :, 1:], p[:, :, 2:]], 2) * cam[:, :, 0:1]
    p[:, :, 1:] = -p[:, :, 1:]
    return p


def rasterize_uv(verts_view, faces, face_uv, size=256):
    """Pytorch3dRasterizer.forward (renderer.py:401-440): -> [N,4,H,W] = bary-interpolated (u,v,1) + visibility,
    plus the raw pix_to_face index buffer [N,H,W] (int64) for bit-exact comparisons."""
    N = verts_view.shape[0]
    fixed = verts_view.clone()
    fixed[..., :2] = -fixed[..., :2]
    p2f, _, bary = _rast.rasterize_meshes(fixed.numpy(), faces.expand(N, -1, -1).numpy(), size, size)
    p2f = torch.from_numpy(p2f)
    bary = torch.from_numpy(bary)
    vis = (p2f > -1).float()
    attrs = face_uv.expand(N, -1, -1, -1).reshape(-1, 3, face_uv.shape[-1])
    idx = p2f.clamp_min(0)
    vals = (bary[..., None] * attrs[idx]).sum(-2)                       # [N,H,W,3]
    vals[p2f == -1] = 0
    return torch.cat([vals.permute(0, 3, 1, 2), vis[:, None]], 1), p2f


def fill_mouth(alpha):
    """[N,1,H,W] -> alpha with interior holes (pixels not reachable from the corner) set to 1."""
    masks = []
    for a in alpha:
        img = np.ascontiguousarray((a[0].numpy() * 255.).astype(np.float32))
        _rast.floodfill_(img, 0.0, 254.0, 255.0)
        masks.append(torch.from_numpy(img)[None] / 127.5 - 1)
    m = torch.stack(masks, 0)
    m = ((m * 2. - 1.) * -1. + 1.) / 2.
    return (alpha + m).clip(0, 1)


def rasterize(sd, v, lms, textures, uv_face_mask):
    N = v.shape[0]
    faces = sd['faces'][..., [0, 2, 1]]
    face_uv = sd['face_uvcoords'][:, :, [0, 2, 1]]
    rend, alphas, lm2d, p2fs = [], [], [], []
    for view in VIEWS:
        tv = transform_view(v, view)
        tv[:, :, 2] = tv[:, :, 2] + 10
        tl = transform_view(lms, view)[:, :, :2]
        r, p2f = rasterize_uv(tv, faces, face_uv)
        alpha = r[:, -1:]
        grid = r[:, :-1].permute(0, 2, 3, 1)[:, :, :, :2]
        mask = F.grid_sample(uv_face_mask.expand(N, -1, -1, -1), grid, align_corners=False)
        alpha = fill_mouth(mask * alpha)
        rend.append(F.grid_sample(textures, grid, align_corners=False))
        alphas.append(alpha)
        lm2d.append(tl)
        p2fs.append(p2f)
    side = rend[1] + rend[2]
    alpha_side = (alphas[1].bool() | alphas[1].bool()).float()          # sic: view 2 ignored (triplane_next3d.py:226)
    return [rend[0], side, rend[3]], [alphas[0], alpha_side, alphas[3]], lm2d, p2fs


def gen_mouth_mask(lms2d):
    lm = lms2d.clone().numpy()
    lm[..., 0] = lm[..., 0] * 128 + 128
    lm[..., 1] = lm[..., 1] * 128 + 128
    outer = lm[:, 48:60]
    avg = (outer[:, 0] + outer[:, 6]) * 0.5
    ups, bottoms = outer[..., 0].max(1, keepdims=True), outer[..., 0].min(1, keepdims=True)
    lefts, rights = outer[..., 1].min(1, keepdims=True), outer[..., 1].max(1, keepdims=True)
    side = (np.concatenate((ups - bottoms, rights - lefts), 1).max(1, keepdims=True) * 1.2).astype(int)
    return np.concatenate([(avg[:, 1:] - side // 2).astype(int), (avg[:, 1:] + side // 2).astype(int),
                           (avg[:, 0:1] - side // 2).astype(int), (avg[:, 0:1] + side // 2).astype(int)], 1)


# ------------------------------------------------------------------------------------------ superresolution

def superresolution(sd, cfg, rgb, x, ws):
    ws = ws[:, -1:, :].repeat(1, 3, 1)
    aa = cfg.rendering_kwargs['sr_antialias']
    if cfg.sr_module == '8XDC':
        need = x.shape[-1] != 128
    else:
        need = x.shape[-1] < 128
    if need:
        x = F.interpolate(x, size=(128, 128), mode='bilinear', align_corners=False, antialias=aa)
        rgb = F.interpolate(rgb, size=(128, 128), mode='bilinear', align_corners=False, antialias=aa)
    nm = cfg.rendering_kwargs['superresolution_noise_mode']
    # sr_num_fp16_res > 0 -> use_fp16 -> conv_clamp=256 even when executed in fp32; 0 -> no clamp (superresolution.py:271-276)
    clamp = cfg.sr_clamp
    x, rgb = synthesis_block(sd, 'superresolution.block0', x, rgb, ws, noise_mode=nm, clamp=clamp,
                             up=(cfg.sr_module == '8XDC'))
    x, rgb = synthesis_block(sd, 'superresolution.block1', x, rgb, ws, noise_mode=nm, clamp=clamp)
    return rgb


# ------------------------------------------------------------------------------------------ synthesis

def default_eye_mask():
    """The reference reads data/ffhq/uv_face_eye_mask.png (triplane_next3d.py:91), which is not shipped; every
    report in this repo uses a synthetic all-ones 256x256 mask instead."""
    return torch.ones(1, 1, 256, 256)


def synthesis(sd, cfg, ws, c, v, u_coarse, u_fine, noise_mode='const', neural_rendering_resolution=None,
              uv_face_mask=None, return_intermediates=False):
    uv_face_mask = default_eye_mask() if uv_face_mask is None else uv_face_mask
    R = neural_rendering_resolution or cfg.neural_rendering_resolution
    v, lms = v[:, :5023], v[:, 5023:]
    N = ws.shape[0]
    eg3d_ws, texture_ws = ws[:, :14], ws[:, 14:]
    cam2world = c[:, :16].view(-1, 4, 4)
    intrinsics = c[:, 16:25].view(-1, 3, 3)
    origins, dirs = renderer.ray_sampler(cam2world, intrinsics, R)

    textures = backbone(sd, cfg, 'texture_backbone.synthesis', texture_ws, noise_mode)
    rend, alphas, lm2d, p2f = rasterize(sd, v, lms, textures, uv_face_mask)

    front = rend[0]
    boxes = gen_mouth_mask(lm2d[0])
    crops = [front[i:i + 1, :, m[0]:m[1], m[2]:m[3]] for i, m in enumerate(boxes)]
    crops = torch.cat([F.interpolate(t, size=(64, 64), mode='bilinear', antialias=True) for t in crops], 0)
    mouth = styleunet(sd, cfg, 'mouth_backbone.synthesis', crops, eg3d_ws, 64, 4, 64, noise_mode)
    stitched = []
    for i, m in enumerate(boxes):
        d = front[i:i + 1].clone()
        side = int(m[1] - m[0])
        d[:, :, m[0]:m[1], m[2]:m[3]] = F.interpolate(mouth[i:i + 1], size=(side, side), mode='bilinear',
                                                      antialias=True)    # sic: (m1-m0) for both dims (:161)
        stitched.append(d)
    stitched = torch.cat(stitched, 0)
    blended_front = styleunet(sd, cfg, 'neural_blending.synthesis', stitched, eg3d_ws, 256, 32, 256, noise_mode)

    static = backbone(sd, cfg, 'backbone.synthesis', eg3d_ws, noise_mode)
    static = static.view(N, 3, 32, static.shape[-2], static.shape[-1])
    alpha = torch.cat(alphas, 1).unsqueeze(2)
    tex_planes = torch.cat((blended_front, rend[1], rend[2]), 1).view(*static.shape)
    planes = tex_planes * alpha + static * (1 - alpha)

    feat, depth, wsum = renderer.render(sd, planes, origins, dirs, cfg.rendering_kwargs, u_coarse, u_fine)
    feature_image = feat.permute(0, 2, 1).reshape(N, feat.shape[-1], R, R).contiguous()
    depth_image = depth.permute(0, 2, 1).reshape(N, 1, R, R)
    rgb_image = feature_image[:, :3]
    sr = superresolution(sd, cfg, rgb_image, feature_image, eg3d_ws)
    out = {'image': sr, 'image_raw': rgb_image, 'image_depth': depth_image}
    if return_intermediates:
        out.update(textures=textures, pix_to_face=torch.stack(p2f, 1), alphas=torch.cat(alphas, 1),
                   rendering_front=front, mouth_boxes=torch.from_numpy(boxes), mouth_crops=crops, mouth_plane=mouth,
                   stitched=stitched, blended_front=blended_front, static=static, planes=planes,
                   feature_image=feature_image, weights_sum=wsum)
    return out
