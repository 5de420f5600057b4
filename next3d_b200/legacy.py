"""Load the reference's network pickles (`legacy.load_network_pkl`, reference legacy.py:24-61) without the reference tree.

The reference writes its networks with `torch_utils.persistence`: every persistent object is pickled as a call of
`torch_utils.persistence._reconstruct_persistent_obj(meta)`, and `meta` carries the source of the object's module, which the
reference's unpickler compiles and runs (persistence.py:181-205).  The unpickler here never does: it resolves every global through
an allowlist, turns persistent objects and the reference's other classes into inert records of their pickled state, and rebuilds
each generator as `next3d_b200.triplane_next3d.TriPlaneGenerator` from that state.  Pickled code is never run and no reference
package is imported.
"""
import collections
import io
import pickle

import numpy as np
import torch

from .triplane_next3d import TriPlaneGenerator

_REFERENCE_PACKAGES = ('training_avatar_texture', 'training', 'torch_utils', 'dnnlib')
_TOPOLOGY = ('dense_faces', 'faces', 'raw_uvcoords', 'uvcoords', 'uvfaces', 'face_uvcoords')
ORTH_SCALE = torch.tensor([[5.0]])                      # the projection raster.cu bakes in (triplane_next3d.py:105-106)
ORTH_SHIFT = torch.tensor([[0, -0.01, -0.01]])


class _Persistent:
    """A persistent reference object: its class name and pickled state (`meta['module_src']` is dropped unread)."""

    def __init__(self, class_name, state):
        self.class_name, self.state = class_name, state


class _Inert:
    """Any other class of the reference packages (e.g. ImportanceRenderer, RaySampler): keeps the pickled state, runs nothing."""

    def __init__(self, *args, **kwargs):
        self.state = {}

    def __setstate__(self, state):
        self.state = state if isinstance(state, dict) else {}


def _reconstruct_persistent_obj(meta):
    return _Persistent(meta.get('class_name'), meta.get('state'))


def _load_storage(b):
    return torch.load(io.BytesIO(b), map_location='cpu', weights_only=True)


def _numpy_multiarray():
    core = getattr(np, '_core', None) or np.core                 # numpy 2 renamed numpy.core to numpy._core
    return core.multiarray


_ALLOWED = {
    ('torch_utils.persistence', '_reconstruct_persistent_obj'): _reconstruct_persistent_obj,
    ('dnnlib.util', 'EasyDict'): dict,
    ('torch._utils', '_rebuild_tensor_v2'): torch._utils._rebuild_tensor_v2,
    ('torch._utils', '_rebuild_parameter'): torch._utils._rebuild_parameter,
    ('torch.storage', '_load_from_bytes'): _load_storage,
    ('collections', 'OrderedDict'): collections.OrderedDict,
    ('builtins', 'set'): set,                                    # pickle protocols < 4 write sets as calls of set()
    ('builtins', 'frozenset'): frozenset,
    ('numpy', 'dtype'): np.dtype,
    ('numpy', 'ndarray'): np.ndarray,
    ('torch', 'Size'): torch.Size,
    ('torch', 'device'): torch.device,
}
for _mod in ('numpy.core.multiarray', 'numpy._core.multiarray'):           # pickles from before and after numpy 2
    for _name in ('scalar', '_reconstruct'):
        _ALLOWED[(_mod, _name)] = getattr(_numpy_multiarray(), _name)


class _Unpickler(pickle.Unpickler):
    """Resolves globals through the allowlist above, torch.nn module classes, torch dtypes and inert stand-ins for the reference's
    classes; anything else raises pickle.UnpicklingError naming the global."""

    def find_class(self, module, name):
        if (module, name) in _ALLOWED:
            return _ALLOWED[(module, name)]
        if module.split('.')[0] in _REFERENCE_PACKAGES:
            return _Inert
        if module.startswith('torch.nn.modules.'):
            obj = getattr(getattr(torch.nn.modules, module.split('.')[3], None), name, None)
            if isinstance(obj, type) and issubclass(obj, torch.nn.Module):
                return obj
        if module == 'torch' and isinstance(getattr(torch, name, None), torch.dtype):
            return getattr(torch, name)
        raise pickle.UnpicklingError(f'next3d_b200.legacy: refusing to load global {module}.{name} from a network pickle')


def _fields(obj):
    if isinstance(obj, (_Persistent, _Inert)):
        return obj.state
    if isinstance(obj, torch.nn.Module):
        return obj.__dict__
    raise ValueError(f'unexpected {type(obj).__name__} in the module tree')


def _state_dict(obj, prefix='', out=None):
    """The reference module's state_dict() from its pickled fields: parameters, persistent buffers, then submodules, recursively."""
    out = {} if out is None else out
    f = _fields(obj)
    skip = f.get('_non_persistent_buffers_set') or set()
    for name, t in f.get('_parameters', {}).items():
        if t is not None:
            out[prefix + name] = t.detach()
    for name, t in f.get('_buffers', {}).items():
        if t is not None and name not in skip:
            out[prefix + name] = t
    for name, m in f.get('_modules', {}).items():
        if m is not None:
            _state_dict(m, f'{prefix}{name}.', out)
    return out


def _generator(key, node):
    """TriPlaneGenerator (CPU, eval, no grad) of the pickled reference generator `node`; ValueError naming the field when the pickle
    asks for something this implementation does not render."""
    if not isinstance(node, _Persistent) or node.class_name != 'TriPlaneGenerator':
        raise ValueError(f"{key}: class {getattr(node, 'class_name', type(node).__name__)!r} is not TriPlaneGenerator")
    st = node.state
    for field in ('load_lms', 'fill_mouth'):
        if st.get(field) is not True:
            raise ValueError(f'{key}.{field} is {st.get(field)!r}; only {field} = True is implemented')
    for field, want in (('orth_scale', ORTH_SCALE), ('orth_shift', ORTH_SHIFT)):
        got = st.get(field)
        if not torch.is_tensor(got) or not torch.equal(got.to(torch.float32), want):
            raise ValueError(f'{key}.{field} is {got!r}; the rasterizer implements {want.tolist()} only')
    mask = st.get('uv_face_mask')
    if not torch.is_tensor(mask) or tuple(mask.shape) != (1, 1, 256, 256):
        raise ValueError(f'{key}.uv_face_mask must be a [1, 1, 256, 256] tensor, got {getattr(mask, "shape", type(mask).__name__)}')
    sd = _state_dict(node)
    G = TriPlaneGenerator(*st['_init_args'], **st['_init_kwargs'], _uv_face_mask=mask.to(torch.float32).contiguous(),
                          _topology_buffers={k: sd[k] for k in _TOPOLOGY if k in sd})
    G.load_state_dict(sd, strict=True)
    G.init_args, G.init_kwargs = tuple(st['_init_args']), dict(st['_init_kwargs'])     # the scripts' --reload_modules path reads them
    G.neural_rendering_resolution = st['neural_rendering_resolution']
    G.rendering_kwargs = dict(st['rendering_kwargs'])
    return G.eval().requires_grad_(False)


def load_network_pkl(f, force_fp16=False):
    """Read a network pickle of the reference (an open binary file) -> dict as the reference's `legacy.load_network_pkl`:
    'G_ema' (and 'G' when present) as next3d_b200.triplane_next3d.TriPlaneGenerator on the CPU, eval and without gradients, ready
    for .to('cuda'); 'training_set_kwargs' as a plain dict (or None); 'D' and 'augment_pipe' are None, because discriminators and
    training are out of this project's scope.

    The generators keep the pickle's state dict, constructor arguments, `neural_rendering_resolution`, `rendering_kwargs` and UV
    eye mask `uv_face_mask` (the mask the reference's scripts render with by default); no file named by the pickle, such as
    `topology_path`, is opened.  No code stored in the pickle is run: a global outside the allowlist raises pickle.UnpicklingError.
    ValueError for `force_fp16=True` (fp16 backbones are not implemented) and for a generator this implementation would render
    differently: another class, load_lms or fill_mouth not True, another orth_scale / orth_shift."""
    if force_fp16:
        raise ValueError('force_fp16=True is not supported: the backbones run in fp32 only')
    data = _Unpickler(f).load()
    if not isinstance(data, dict) or 'G_ema' not in data:
        raise ValueError('not a network pickle: expected a dict with G_ema')
    out = {k: v for k, v in data.items() if k not in ('G', 'G_ema', 'D', 'augment_pipe')}
    converted = {}                                              # G and G_ema may be one pickled object
    for key in ('G', 'G_ema'):
        if data.get(key) is not None:
            node = data[key]
            if id(node) not in converted:
                converted[id(node)] = _generator(key, node)
            out[key] = converted[id(node)]
    out['D'] = out['augment_pipe'] = None
    tsk = out.get('training_set_kwargs')
    out['training_set_kwargs'] = None if tsk is None else dict(tsk)
    return out
