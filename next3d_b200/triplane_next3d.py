"""Drop-in `TriPlaneGenerator` for the reference's inference scripts (gen_samples_next3d.py:198-200,
gen_videos_next3d.py:104-105,155, reenact_avatar_next3d.py:123,164).

Mirrors training_avatar_texture/triplane_next3d.py:40-344:
  * constructor signature :41-53, attributes (`neural_rendering_resolution`, `rendering_kwargs`, `load_lms`, `fill_mouth`);
  * the module tree / parameter + buffer names of the reference (674 tensors, SURVEY.md section 8b), so that
    `load_state_dict(ref.state_dict())` and `misc.copy_params_and_buffers(G_ref, G_new, require_all=True)`
    (gen_samples_next3d.py:153-154) succeed;
  * `.mapping` :111-115, `.synthesis` :117-188 (same keyword arguments, same output dict), `.sample` / `.sample_mixed`
    :232-323, `.forward` :325-328.
Compute runs through next3d_b200.engine.Engine (hand-written sm_90a kernels); there is no CPU fallback: CPU inputs raise.
"""
import math

import torch

from . import config as _config
from . import weights as _weights
from .engine import Engine


class _Node(torch.nn.Module):
    """Plain container used to rebuild the reference's module tree from its parameter names."""


def _attach(root, dotted, tensor, as_param):
    parts = dotted.split('.')
    m = root
    for p in parts[:-1]:
        if p not in m._modules:
            m.add_module(p, _Node())
        m = m._modules[p]
    if as_param:
        m.register_parameter(parts[-1], torch.nn.Parameter(tensor, requires_grad=False))
    else:
        m.register_buffer(parts[-1], tensor)


_PARAM_KINDS = {'weight', 'bias', 'affine_bias', 'noise_strength', 'const'}


class TriPlaneGenerator(torch.nn.Module):
    def __init__(self, z_dim=512, c_dim=25, w_dim=512, img_resolution=512, img_channels=3, topology_path=None, sr_num_fp16_res=0,
                 mapping_kwargs={}, rendering_kwargs={}, sr_kwargs={}, **synthesis_kwargs):
        super().__init__()
        # legacy.load_network_pkl passes the pickled eye mask and topology buffers, so no file is read (private keywords)
        uv_face_mask = synthesis_kwargs.pop('_uv_face_mask', None)
        topo = synthesis_kwargs.pop('_topology_buffers', None)
        assert z_dim == 512 and w_dim == 512 and c_dim == 25 and img_channels == 3, 'only the FFHQ Next3D topology is supported'
        assert mapping_kwargs.get('num_layers', 2) == 2, 'MappingNetwork with num_layers=2 expected (train_next3d.py:369)'
        self.z_dim, self.c_dim, self.w_dim = z_dim, c_dim, w_dim
        self.img_resolution, self.img_channels = img_resolution, img_channels
        self.topology_path = topology_path
        rk = dict(_config.FFHQ_RENDERING_KWARGS)
        rk.update(rendering_kwargs)
        self.cfg = _config.GeneratorConfig(img_resolution=img_resolution,
                                           channel_base=synthesis_kwargs.get('channel_base', 32768),
                                           channel_max=synthesis_kwargs.get('channel_max', 512), rendering_kwargs=rk)
        self.rendering_kwargs = rk
        self.neural_rendering_resolution = 64
        self.load_lms = True
        self.fill_mouth = True
        self.sr_num_fp16_res = sr_num_fp16_res
        self._sr_precision = 'fp32'
        self.uv_face_mask = self._load_uv_face_mask() if uv_face_mask is None else uv_face_mask
        for name, shape, kind, _ in _config.param_spec(self.cfg):
            if kind == 'topology':
                topo = topo or _weights.topology_buffers(self._load_mesh(topology_path))
                _attach(self, name, topo[name].clone(), False)
            elif kind == 'filter':
                f = torch.tensor([1., 3., 3., 1.])
                f = torch.outer(f, f)
                _attach(self, name, f / f.sum(), False)
            else:
                _attach(self, name, torch.zeros(shape), kind in _PARAM_KINDS)
        self._engine = None
        self._engine_key = None
        self.use_cuda_graph = False      # opt-in: replay one captured CUDA graph per (batch, resolution) instead of ~200 launches

    @staticmethod
    def _load_uv_face_mask(path='data/ffhq/uv_face_eye_mask.png'):
        """Eye / face mask of the UV atlas (triplane_next3d.py:91-92: channel 0 of the PNG / 255, F.interpolate (nearest) to
        256^2).  Not part of the state dict and not shipped with the reference repo (SURVEY.md section 8c): when the file is
        absent an all-ones mask is used and a warning says so -- with a real checkpoint the alpha around the eyes then differs
        from the reference's.  Assigning `G.uv_face_mask = ...` later is honoured (it is part of the engine cache key)."""
        import os
        import warnings
        if os.path.isfile(path):
            try:
                import numpy as np
                from PIL import Image
                m = np.asarray(Image.open(path).convert('RGB'), dtype=np.float32)[:, :, 2] / 255.0   # cv2.imread is BGR: its channel 0 = blue
                return torch.nn.functional.interpolate(torch.from_numpy(m)[None, None].contiguous(), [256, 256])
            except Exception as e:                                                 # unreadable file: say so, keep going
                warnings.warn(f'next3d_b200: cannot read {path} ({e}); using an all-ones UV face mask')
        else:
            warnings.warn(f'next3d_b200: {path} not found; using an all-ones UV face mask (set G.uv_face_mask to the real one for '
                          f'checkpoint-faithful eyes)')
        return torch.ones(1, 1, 256, 256)

    @staticmethod
    def _load_mesh(topology_path):
        if topology_path is None or not str(topology_path).endswith('.obj'):
            return None
        import numpy as np
        v, vt, fv, ft = [], [], [], []
        with open(topology_path) as f:                                           # pytorch3d.io.load_obj subset (:79-82)
            for line in f:
                if line.startswith('v '):
                    v.append([float(x) for x in line.split()[1:4]])
                elif line.startswith('vt '):
                    vt.append([float(x) for x in line.split()[1:3]])
                elif line.startswith('f '):
                    toks = [t.split('/') for t in line.split()[1:4]]
                    fv.append([int(t[0]) - 1 for t in toks])
                    ft.append([int(t[1]) - 1 for t in toks])
        return dict(verts=np.asarray(v, np.float32), verts_uvs=np.asarray(vt, np.float32), faces=np.asarray(fv, np.int32),
                    uvfaces=np.asarray(ft, np.int32))

    # ------------------------------------------------------------------------------------------ construction helpers
    @classmethod
    def from_config(cls, cfg, state_dict=None, device='cuda'):
        G = cls(img_resolution=cfg.img_resolution, rendering_kwargs=cfg.rendering_kwargs, channel_base=cfg.channel_base,
                channel_max=cfg.channel_max, sr_num_fp16_res=cfg.sr_num_fp16_res)
        G.neural_rendering_resolution = cfg.neural_rendering_resolution
        if state_dict is not None:
            G.load_state_dict(state_dict)
        return G.eval().requires_grad_(False).to(device)

    @property
    def sr_precision(self):
        """Precision of the super-resolution head: 'fp32' (default: fp32-grade bf16x3 convolutions, the reference's CPU result) or
        'fp16' (opt-in, faster: fp16 activations and weights, one tensor-core product per k-step, fp32 accumulate -- the precision
        the reference gives its SR blocks on CUDA when sr_num_fp16_res > 0, superresolution.py:268-277, networks_stylegan2.py:547-549,
        but rounded at other points, so `image` is about 1e-3 of its range from either fp32 or the reference's fp16 answer and is
        not the latter; INTEGRATION.md section 1).  Only `image` depends on it; the next synthesis / render_views call runs in the new mode (graphs are captured per mode).  ValueError
        for any other value, and for 'fp16' with sr_num_fp16_res == 0 (the reference runs that SR head in fp32)."""
        return self._sr_precision

    @sr_precision.setter
    def sr_precision(self, mode):
        self._sr_precision = self._check_sr_precision(mode)

    def _check_sr_precision(self, mode):
        if mode not in ('fp32', 'fp16'):
            raise ValueError(f"sr_precision must be 'fp32' or 'fp16', got {mode!r}")
        if mode == 'fp16' and not self.sr_num_fp16_res > 0:
            raise ValueError("sr_precision='fp16' needs sr_num_fp16_res > 0: with sr_num_fp16_res == 0 the reference runs the "
                             "super-resolution head in fp32")
        return mode

    def repack(self):
        """Re-pack weights into the engine's layouts (call after changing parameters in place)."""
        self._engine = None

    def _state_version(self):
        """Changes whenever a parameter / buffer is written in place (load_state_dict, misc.copy_params_and_buffers, .copy_())."""
        return sum(t._version for t in self.state_dict(keep_vars=True).values())

    def _get_engine(self):
        dev = self.faces.device
        if dev.type != 'cuda':
            raise RuntimeError('next3d_b200.TriPlaneGenerator runs on CUDA (sm_90a) only: move the module with .to("cuda"); there is no '
                               'CPU fallback path')
        rk = self.rendering_kwargs
        # everything the packed engine bakes in: weights (version counter), the UV mask, pack-time rendering options
        key = (str(dev), self.img_resolution, self._state_version(), id(self.uv_face_mask), self.uv_face_mask._version,
               rk.get('superresolution_noise_mode', 'none'), self.sr_num_fp16_res)
        if self._engine is None or self._engine_key != key:
            import dataclasses
            cfg = dataclasses.replace(self.cfg, rendering_kwargs=rk, sr_num_fp16_res=self.sr_num_fp16_res)
            self._engine = Engine(cfg, self.state_dict(), device=dev, uv_face_mask=self.uv_face_mask)
            self._engine_key = key
        self._engine.rk = rk
        self._engine.sr_precision = self._check_sr_precision(self._sr_precision)     # sr_num_fp16_res may have changed since
        return self._engine

    # ------------------------------------------------------------------------------------------ reference API
    def mapping(self, z, c, truncation_psi=1, truncation_cutoff=None, update_emas=False):
        """backbone.mapping (MappingNetwork, networks_stylegan2.py:233-268) via triplane_next3d.py:111-115.  Tiny, once per
        latent, adjacent to (not inside) synthesis: plain PyTorch on the module's device."""
        rk = self.rendering_kwargs
        m = self.backbone.mapping
        if rk['c_gen_conditioning_zero']:
            c = torch.zeros_like(c)
        if z.is_cuda:                                   # one fused launch (n3d_mapping); the PyTorch lines below serve CPU tensors only
            from . import kernels as K
            tensors = dict(embed_w=m.embed.weight, embed_b=m.embed.bias, fc0_w=m.fc0.weight, fc0_b=m.fc0.bias, fc1_w=m.fc1.weight,
                           fc1_b=m.fc1.bias, w_avg=m.w_avg)
            for k, t in tensors.items():
                if t.device != z.device or t.dtype != torch.float32 or not t.is_contiguous():
                    raise RuntimeError(f'next3d_b200: mapping parameter {k} must be contiguous float32 on {z.device}')
            with torch.cuda.device(z.device):
                return K.mapping(z.to(torch.float32).contiguous(), c[:, :25].to(z.device, torch.float32).contiguous(), rk.get('c_scale', 0),
                                 tensors, truncation_psi, truncation_cutoff)
        c = c[:, :25] * rk.get('c_scale', 0)
        x = z.to(torch.float32)
        x = x * (x.square().mean(1, keepdim=True) + 1e-8).rsqrt()
        y = torch.addmm(m.embed.bias[None], c.to(torch.float32), (m.embed.weight * (1.0 / math.sqrt(self.c_dim))).t())
        y = y * (y.square().mean(1, keepdim=True) + 1e-8).rsqrt()
        x = torch.cat([x, y], 1)
        for fc in (m.fc0, m.fc1):
            w = fc.weight * (0.01 / math.sqrt(fc.weight.shape[1]))
            x = torch.nn.functional.leaky_relu(x.matmul(w.t()) + fc.bias * 0.01, 0.2) * math.sqrt(2)
        x = x[:, None].repeat(1, 28, 1)
        if truncation_psi != 1:
            if truncation_cutoff is None:
                x = m.w_avg.lerp(x, truncation_psi)
            else:
                x[:, :truncation_cutoff] = m.w_avg.lerp(x[:, :truncation_cutoff], truncation_psi)
        return x

    def synthesis(self, ws, c, v, neural_rendering_resolution=None, update_emas=False, cache_backbone=False, use_cached_backbone=False,
                  sampler_noise=None, seed=None, depth_range='batch', **synthesis_kwargs):
        """-> {'image': [N,3,R,R], 'image_raw': [N,3,r,r], 'image_depth': [N,1,r,r]} (triplane_next3d.py:117-188).
        Extra keyword `sampler_noise=(u_coarse [N,M,Dc,1], u_fine [N*M,Df])` injects the stratified / importance sampling
        uniforms (parity tests); by default the renderer draws them from an in-kernel counter RNG seeded per call.
        With `rendering_kwargs['return_normal']` set the output also holds 'image_normal' [N,3,r,r]: unit world-space normals
        -grad sigma composited like the colours (renderer.py:271-355, ray_marcher.py:61-64).
        `cache_backbone=True` also keeps this call's ws-only backbone outputs, blended planes, ws and noise_mode until the next caching
        call or a weight change; `use_cached_backbone=True` takes the two ws-only backbones from that cache and re-runs everything
        that depends on the mesh (triplane.py:120-128 of EG3D; no cache computes them), and `render_views` renders new cameras from
        the cached planes.  With B heads cached, use_cached_backbone takes N = B * V images (ws, c, v per image): image n takes its
        neural texture and static planes from head n // V, everything else is computed per image with the call's ws.  N not a
        multiple of B raises RuntimeError, and so does N != B when the call also sets cache_backbone.
        Extra keyword `depth_range`: 'batch' (default, the reference's semantics for a batched call) clamps every image's depth to the
        range of all the call's samples (ray_marcher.py:54); 'image' clamps each image to its own range, so 'image_depth' of a batch
        equals that of one call per image (the reference's scripts render one frame per call)."""
        neural_rendering_resolution = self._rendering_resolution(neural_rendering_resolution)
        noise_mode = synthesis_kwargs.get('noise_mode', 'random')
        seed = self._sampler_seed(seed, sampler_noise)
        eng = self._get_engine()
        flags = dict(cache_backbone=bool(cache_backbone), use_cached_backbone=bool(use_cached_backbone), depth_range=depth_range)
        if self.use_cuda_graph and sampler_noise is None and not synthesis_kwargs.get('return_intermediates', False):
            return eng.synthesis_graphed(ws, c, v, noise_mode=noise_mode, neural_rendering_resolution=neural_rendering_resolution, seed=seed,
                                         **flags)
        return eng.synthesis(ws, c, v, noise_mode=noise_mode, neural_rendering_resolution=neural_rendering_resolution,
                             sampler_noise=sampler_noise, seed=seed, return_intermediates=synthesis_kwargs.get('return_intermediates', False),
                             **flags)

    def render_views(self, c, neural_rendering_resolution=None, seed=None, sampler_noise=None, depth_range='batch'):
        """New camera views of the heads cached by `synthesis(..., cache_backbone=True)` with batch B, without regenerating them:
        c [N, 25] with N = B * V, view n belongs to head n // V -> the dict `synthesis` returns, for N images.  Renders the cached
        planes and runs super-resolution with the cached ws (the backbones' noise_mode is the caching call's; SR noise follows
        rendering_kwargs['superresolution_noise_mode']).  `depth_range` as in `synthesis`.  Raises RuntimeError when nothing is cached
        or B does not divide N."""
        neural_rendering_resolution = self._rendering_resolution(neural_rendering_resolution)
        seed = self._sampler_seed(seed, sampler_noise)
        eng = self._get_engine()
        if self.use_cuda_graph and sampler_noise is None:
            return eng.render_views_graphed(c, neural_rendering_resolution=neural_rendering_resolution, seed=seed, depth_range=depth_range)
        return eng.render_views(c, neural_rendering_resolution=neural_rendering_resolution, sampler_noise=sampler_noise, seed=seed,
                                depth_range=depth_range)

    def _rendering_resolution(self, r):
        if r is None:
            return self.neural_rendering_resolution
        self.neural_rendering_resolution = r
        return r

    @staticmethod
    def _sampler_seed(seed, sampler_noise):
        if seed is None:
            return int(torch.randint(0, 2 ** 31 - 1, (1,)).item()) if sampler_noise is None else 0
        return seed

    def sample_mixed(self, coordinates, directions, ws, v, truncation_psi=1, truncation_cutoff=None, update_emas=False, **synthesis_kwargs):
        """run_model on arbitrary points (triplane_next3d.py:278-323): -> {'rgb': [N,P,32], 'sigma': [N,P,1]}."""
        from . import kernels as K
        eng = self._get_engine()
        eng._on_device(coordinates=coordinates)
        planes = eng.compute_planes(ws, v, synthesis_kwargs.get('noise_mode', 'random'))
        N, P, _ = coordinates.shape
        sigma = torch.empty(N, P, device=planes.device)
        rgb = torch.empty(N, P, 32, device=planes.device)
        with torch.cuda.device(planes.device):
            K.sample_points(planes, coordinates.to(torch.float32).contiguous(), self.rendering_kwargs['box_warp'], eng.dec, sigma, rgb)
        return {'rgb': rgb, 'sigma': sigma[..., None]}

    def sample(self, coordinates, directions, z, c, v, truncation_psi=1, truncation_cutoff=None, update_emas=False, **synthesis_kwargs):
        ws = self.mapping(z, c, truncation_psi=truncation_psi, truncation_cutoff=truncation_cutoff, update_emas=update_emas)
        return self.sample_mixed(coordinates, directions, ws, v, **synthesis_kwargs)

    def forward(self, z, c, v, truncation_psi=1, truncation_cutoff=None, neural_rendering_resolution=None, update_emas=False,
                cache_backbone=False, use_cached_backbone=False, **synthesis_kwargs):
        ws = self.mapping(z, c, truncation_psi=truncation_psi, truncation_cutoff=truncation_cutoff, update_emas=update_emas)
        return self.synthesis(ws, c, v, update_emas=update_emas, neural_rendering_resolution=neural_rendering_resolution,
                              cache_backbone=cache_backbone, use_cached_backbone=use_cached_backbone, **synthesis_kwargs)
