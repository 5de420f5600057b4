"""CPU: next3d_b200.legacy.load_network_pkl reads the reference's network pickles without the reference tree and runs no pickled
code, next3d_b200.mrc writes MRC2014 maps, and the standalone CLI refuses what it does not implement before loading a network.

Persistence-format pickles are written here without the reference: `_fake_reference` installs stand-in `torch_utils.persistence`
and `dnnlib.util` modules only while pickling, so the bytes name the same globals as a pickle the reference's own persistence code
writes (that case is checked against the real reference in test_reference_pickle_loads_without_reference)."""
import collections
import contextlib
import gzip
import io
import os
import pickle
import struct
import subprocess
import sys
import types
import warnings

import numpy as np
import pytest
import torch

from oracle import ref_shim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEMO = os.path.join(ROOT, 'tests', 'golden', 'demo')


# ------------------------------------------------------------------------------------------------ persistence-format pickles
@contextlib.contextmanager
def _fake_reference():
    """(reconstruct function, EasyDict class) registered as torch_utils.persistence._reconstruct_persistent_obj and
    dnnlib.util.EasyDict for the duration of the block; whatever those module names held before is restored."""
    names = ('torch_utils', 'torch_utils.persistence', 'dnnlib', 'dnnlib.util')
    saved = {n: sys.modules.get(n) for n in names}
    mods = {n: types.ModuleType(n) for n in names}

    def _reconstruct_persistent_obj(meta):
        raise AssertionError('only pickled here, never loaded')

    class EasyDict(dict):
        pass
    _reconstruct_persistent_obj.__module__ = 'torch_utils.persistence'
    _reconstruct_persistent_obj.__qualname__ = '_reconstruct_persistent_obj'
    EasyDict.__module__, EasyDict.__qualname__ = 'dnnlib.util', 'EasyDict'
    mods['torch_utils.persistence']._reconstruct_persistent_obj = _reconstruct_persistent_obj
    mods['dnnlib.util'].EasyDict = EasyDict
    sys.modules.update(mods)
    try:
        yield _reconstruct_persistent_obj, EasyDict
    finally:
        for n, m in saved.items():
            if m is None:
                sys.modules.pop(n, None)
            else:
                sys.modules[n] = m


class _PersistentNode:
    """Pickles as the reference's persistent objects do: _reconstruct_persistent_obj(meta) (persistence.py:120-128)."""

    def __init__(self, fn, class_name, state, module_src):
        self.fn, self.meta = fn, dict(type='class', version=6, module_src=module_src, class_name=class_name, state=state)

    def __reduce__(self):
        return self.fn, (self.meta,)


def _module_state(m, extra=None):
    return dict(training=False, _parameters=collections.OrderedDict(m._parameters), _buffers=collections.OrderedDict(m._buffers),
                _non_persistent_buffers_set=set(), _modules=collections.OrderedDict(), **(extra or {}))


def generator_fields(cfg, uv_face_mask, topology_path='data/demo/head_template.obj'):
    """The pickled attributes of a reference TriPlaneGenerator of config `cfg` (triplane_next3d.py:55-106) besides its module tree."""
    return dict(_init_args=(), _init_kwargs=dict(
        z_dim=512, c_dim=25, w_dim=512, img_resolution=cfg.img_resolution, img_channels=3, topology_path=topology_path,
        sr_num_fp16_res=cfg.sr_num_fp16_res, mapping_kwargs=dict(num_layers=2), rendering_kwargs=dict(cfg.rendering_kwargs),
        sr_kwargs=dict(channel_base=cfg.channel_base, channel_max=cfg.channel_max), num_fp16_res=0, conv_clamp=None,
        channel_base=cfg.channel_base, channel_max=cfg.channel_max),
        neural_rendering_resolution=cfg.neural_rendering_resolution, rendering_kwargs=dict(cfg.rendering_kwargs), _last_planes=None,
        load_lms=True, fill_mouth=True, uv_resolution=256, uv_face_mask=uv_face_mask, orth_scale=torch.tensor([[5.0]]),
        orth_shift=torch.tensor([[0, -0.01, -0.01]]))


def persistence_pickle(cfg, state_dict, fields, class_name='TriPlaneGenerator', module_src='', also=None):
    """Bytes of {'G': G, 'G_ema': G, 'D': None, 'training_set_kwargs': EasyDict(...)} in the reference's persistence format, G having
    the module tree and state dict of our TriPlaneGenerator (the reference's names) plus `fields`, every module persistent."""
    from next3d_b200.triplane_next3d import TriPlaneGenerator
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')                                    # the constructor's eye-mask fallback
        G = TriPlaneGenerator.from_config(cfg, state_dict, device='cpu')
    with _fake_reference() as (fn, EasyDict):
        def node(m, name, extra=None):
            st = _module_state(m, extra)
            for k, child in m._modules.items():
                st['_modules'][k] = node(child, type(child).__name__)
            return _PersistentNode(fn, name, st, module_src)
        top = node(G, class_name, fields)
        data = dict(G=top, G_ema=top, D=None, training_set_kwargs=EasyDict(class_name='training.dataset.ImageFolderDataset',
                                                                            resolution=cfg.img_resolution), **(also or {}))
        return pickle.dumps(data)


@pytest.fixture(scope='module')
def tiny():
    from next3d_b200 import config, weights
    cfg = config.tiny_config(512)
    sd = weights.make_state_dict(cfg, seed=3)
    mask = torch.rand(1, 1, 256, 256, generator=torch.Generator().manual_seed(5))
    return cfg, sd, mask


def _load(b, **kw):
    from next3d_b200 import legacy
    return legacy.load_network_pkl(io.BytesIO(b), **kw)


# ------------------------------------------------------------------------------------------------ against the reference
_CHILD = r'''
import importlib.abc, pickle, sys, warnings
BLOCKED = ('torch_utils', 'dnnlib', 'training_avatar_texture', 'training', 'pytorch3d', 'cv2')
class Block(importlib.abc.MetaPathFinder):
    def find_spec(self, name, path, target=None):
        if name.split('.')[0] in BLOCKED:
            raise ImportError(f'{name} is blocked')
sys.meta_path.insert(0, Block())
sys.path.insert(0, sys.argv[1])
import torch
from next3d_b200 import legacy
with warnings.catch_warnings(record=True) as caught:
    warnings.simplefilter('always')
    with open(sys.argv[2], 'rb') as f:
        d = legacy.load_network_pkl(f)
G = d['G_ema']
torch.save(dict(sd=G.state_dict(), init_args=G.init_args, init_kwargs=G.init_kwargs, nrr=G.neural_rendering_resolution,
                rk=G.rendering_kwargs, mask=G.uv_face_mask, same=d['G'] is G, cls=type(G).__module__ + '.' + type(G).__name__,
                D=d['D'], tsk=d['training_set_kwargs'], warnings=[str(w.message) for w in caught],
                imported=sorted(m for m in sys.modules if m.split('.')[0] in BLOCKED)), sys.argv[3])
'''


@pytest.mark.skipif(not ref_shim.available(), reason='reference tree not present')
def test_reference_pickle_loads_without_reference(tmp_path):
    """A pickle written by the reference's own persistence code (a tiny reference generator, never committed: it embeds the
    reference's source) loads in a process that cannot import any reference package, pytorch3d or cv2."""
    from next3d_b200 import config, weights
    cfg = config.tiny_config(512)
    G = ref_shim.build_reference_generator(cfg)
    G.load_state_dict(weights.make_state_dict(cfg, seed=4))
    G.uv_face_mask = torch.rand(1, 1, 256, 256, generator=torch.Generator().manual_seed(6))
    G.neural_rendering_resolution = 32
    pkl, out = tmp_path / 'ref.pkl', tmp_path / 'out.pt'
    pkl.write_bytes(pickle.dumps({'G': G, 'G_ema': G, 'D': None, 'training_set_kwargs': {'resolution': 512}}))
    subprocess.run([sys.executable, '-c', _CHILD, ROOT, str(pkl), str(out)], check=True, cwd=tmp_path)
    r = torch.load(out, weights_only=False)
    assert r['imported'] == [] and r['warnings'] == [], (r['imported'], r['warnings'])
    assert r['cls'] == 'next3d_b200.triplane_next3d.TriPlaneGenerator' and r['same'] and r['D'] is None
    assert r['tsk'] == {'resolution': 512} and type(r['tsk']) is dict
    want = G.state_dict()
    assert sorted(r['sd']) == sorted(want) and len(want) == 674
    for k, t in want.items():
        assert r['sd'][k].dtype == t.dtype and torch.equal(r['sd'][k], t), k
    assert r['init_args'] == tuple(G.init_args) and r['init_kwargs'] == dict(G.init_kwargs)
    assert r['nrr'] == 32 and r['rk'] == G.rendering_kwargs
    assert torch.equal(r['mask'], G.uv_face_mask)


# ------------------------------------------------------------------------------------------------ hand-built pickles
def test_hand_built_pickle_loads(tiny, tmp_path):
    """State dict, attributes and eye mask come from the pickle; the missing topology .obj it names is never opened; no warning."""
    cfg, sd, mask = tiny
    fields = generator_fields(cfg, mask, topology_path=str(tmp_path / 'missing.obj'))
    fields['neural_rendering_resolution'] = 128
    with warnings.catch_warnings():
        warnings.simplefilter('error')
        d = _load(persistence_pickle(cfg, sd, fields))
    G = d['G_ema']
    assert d['G'] is G and d['D'] is None and d['augment_pipe'] is None
    assert d['training_set_kwargs'] == {'class_name': 'training.dataset.ImageFolderDataset', 'resolution': 512}
    assert type(d['training_set_kwargs']) is dict
    got = G.state_dict()
    assert sorted(got) == sorted(sd)
    assert all(torch.equal(got[k], sd[k].to(got[k].dtype)) for k in sd)
    assert torch.equal(G.uv_face_mask, mask) and G.neural_rendering_resolution == 128
    assert G.rendering_kwargs == cfg.rendering_kwargs and G.init_kwargs == fields['_init_kwargs']
    assert not G.training and not any(p.requires_grad for p in G.parameters())


def test_module_source_is_never_run(tiny, tmp_path):
    cfg, sd, mask = tiny
    marker = tmp_path / 'ran'
    src = f'open({str(marker)!r}, "w").close()\nraise RuntimeError("module source executed")\n'
    d = _load(persistence_pickle(cfg, sd, generator_fields(cfg, mask), module_src=src))
    assert d['G_ema'] is not None and not marker.exists()


def _call_pickle(module, name, args):
    """Protocol-0 pickle bytes of the call module.name(*args)."""
    return f'c{module}\n{name}\n'.encode() + pickle.dumps(tuple(args), protocol=0)[:-1] + b'R.'


@pytest.mark.parametrize('module,name,arg', [
    ('builtins', 'eval', "__import__('pathlib').Path({m!r}).touch()"),
    ('os', 'system', 'touch {m}'),
    ('subprocess', 'Popen', ['touch', '{m}']),
])
def test_unsafe_globals_are_refused(tmp_path, module, name, arg):
    marker = str(tmp_path / 'called')
    arg = [a.format(m=marker) for a in arg] if isinstance(arg, list) else arg.format(m=marker)
    b = _call_pickle(module, name, [arg])
    with pytest.raises(pickle.UnpicklingError, match=rf'{module}\.{name}'):
        _load(b)
    assert not os.path.exists(marker)


@pytest.mark.parametrize('field,value', [
    ('load_lms', False), ('fill_mouth', False), ('orth_scale', torch.tensor([[4.0]])), ('orth_shift', torch.tensor([[0, 0.0, -0.01]])),
])
def test_unsupported_generators_are_refused(tiny, field, value):
    cfg, sd, mask = tiny
    fields = generator_fields(cfg, mask)
    fields[field] = value
    with pytest.raises(ValueError, match=field):
        _load(persistence_pickle(cfg, sd, fields))


def test_other_classes_and_force_fp16_are_refused(tiny):
    cfg, sd, mask = tiny
    with pytest.raises(ValueError, match='TriPlaneGenerator'):
        _load(persistence_pickle(cfg, sd, generator_fields(cfg, mask), class_name='TriPlaneGeneratorV2'))
    with pytest.raises(ValueError, match='force_fp16'):
        _load(persistence_pickle(cfg, sd, generator_fields(cfg, mask)), force_fp16=True)


# ------------------------------------------------------------------------------------------------ MRC2014 writer
def test_mrc_round_trip(tmp_path):
    from next3d_b200 import mrc
    data = np.random.RandomState(0).randn(4, 5, 6).astype(np.float32)
    path = tmp_path / 'grid.mrc'
    mrc.write_mrc(path, data)
    raw = path.read_bytes()
    assert len(raw) == 1024 + data.nbytes
    ints, floats = np.frombuffer(raw[:1024], '<i4'), np.frombuffer(raw[:1024], '<f4')
    assert tuple(ints[0:4]) == (6, 5, 4, 2) and tuple(ints[7:10]) == (6, 5, 4) and tuple(ints[16:19]) == (1, 2, 3)
    assert tuple(floats[10:13]) == (6.0, 5.0, 4.0) and tuple(floats[13:16]) == (90.0, 90.0, 90.0)
    d64 = data.astype(np.float64)
    assert tuple(floats[19:22]) == tuple(np.float32([d64.min(), d64.max(), d64.mean()])) and floats[54] == np.float32(d64.std())
    assert raw[208:212] == b'MAP ' and raw[212:214] == b'\x44\x44' and ints[27] == 20140
    assert struct.unpack('<i', raw[220:224])[0] == 0                                # no labels
    assert np.array_equal(np.frombuffer(raw[1024:], '<f4').reshape(4, 5, 6), data)


def test_mrc_reads_with_mrcfile(tmp_path):
    mrcfile = pytest.importorskip('mrcfile')
    if not hasattr(mrcfile, 'open'):                                              # a stand-in module installed by another test
        pytest.skip('mrcfile is not installed')
    from next3d_b200 import mrc
    data = np.random.RandomState(1).randn(3, 4, 5).astype(np.float32)
    mrc.write_mrc(tmp_path / 'grid.mrc', data)
    with mrcfile.open(tmp_path / 'grid.mrc', permissive=False) as m:
        assert np.array_equal(m.data, data) and m.header.mode == 2 and tuple(m.voxel_size.tolist()) == (1.0, 1.0, 1.0)


# ------------------------------------------------------------------------------------------------ CLI refusals
def _demo_args(tmp_path):
    obj, lms = tmp_path / 'demo.obj', tmp_path / 'demo_kpt2d.txt'
    obj.write_bytes(gzip.open(os.path.join(DEMO, 'demo.obj.gz')).read())
    lms.write_bytes(gzip.open(os.path.join(DEMO, 'demo_kpt2d.txt.gz')).read())
    return ['--obj_path', str(obj), '--lms_path', str(lms)]


@pytest.mark.parametrize('argv,match', [
    (['gen_samples', '--seeds', '0', '--outdir', 'o', '--shapes', 'True', '--shape-format', '.ply', '--lms_cond', 'True'], 'marching cubes'),
    (['gen_samples', '--seeds', '0', '--outdir', 'o'], 'lms_cond'),
    (['gen_videos', '--seeds', '0', '--outdir', 'o', '--cfg', 'AFHQ', '--lms_cond', 'True'], 'FFHQ'),
    (['gen_videos', '--seeds', '0', '--outdir', 'o', '--interpolate', 'False', '--grid', '2x1', '--lms_cond', 'True'], 'grid 1x1'),
    (['gen_videos', '--seeds', '0', '--outdir', 'o', '--lms_cond', 'True'], 'imageio'),
    (['reenact', '--seeds', '0', '--outdir', 'o', '--drive_root', 'd', '--lms_cond', 'True'], 'imageio'),
])
def test_cli_refuses_before_loading(tmp_path, monkeypatch, argv, match):
    """The refusals come before the network is opened: the --network file does not exist."""
    from next3d_b200.__main__ import main
    monkeypatch.setitem(sys.modules, 'imageio', None)                             # import imageio raises ImportError
    argv = argv + ['--network', str(tmp_path / 'missing.pkl')] + ([] if argv[0] == 'reenact' else _demo_args(tmp_path))
    with pytest.raises(SystemExit, match=match):
        main(argv)
