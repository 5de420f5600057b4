"""GPU: a generator loaded from a persistence-format network pickle (next3d_b200.legacy) renders bit-identically to the same weights
built with TriPlaneGenerator.from_config and the pickled eye mask, and the standalone CLI (python -m next3d_b200) writes the frames,
sheets and density grids of the drivers it runs."""
import io
import json
import sys
import types

import numpy as np
import pytest
import torch

from tests.test_legacy_cpu import _demo_args, generator_fields, persistence_pickle

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _mask(seed):
    return torch.rand(1, 1, 256, 256, generator=torch.Generator().manual_seed(seed))


def _load(path):
    from next3d_b200 import legacy
    with open(path, 'rb') as f:
        return legacy.load_network_pkl(f)['G_ema'].to(DEV)


@pytest.mark.parametrize('res', [512, 256])
def test_loaded_generator_matches_from_config(res):
    import warnings
    from next3d_b200 import config, legacy, weights
    from next3d_b200.triplane_next3d import TriPlaneGenerator
    cfg = config.tiny_config(res)
    sd = weights.make_state_dict(cfg, seed=7)
    mask = _mask(8)
    G = legacy.load_network_pkl(io.BytesIO(persistence_pickle(cfg, sd, generator_fields(cfg, mask))))['G_ema'].to(DEV)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')                                      # the all-ones eye-mask fallback of the constructor
        ref = TriPlaneGenerator.from_config(cfg, sd)
        ones = TriPlaneGenerator.from_config(cfg, sd)
    ref.uv_face_mask = mask.clone()
    ones.uv_face_mask = torch.ones(1, 1, 256, 256)
    z, c_cond, c_cam, v = weights.demo_inputs(cfg, 2, seed=1, device=DEV)
    noise = tuple(t.to(DEV) for t in weights.sampler_noise(cfg, 2, seed=1))

    def run(g):
        return g.synthesis(g.mapping(z, c_cond, truncation_psi=0.7), c_cam, v, noise_mode='const', sampler_noise=noise)
    got, want, all_ones = run(G), run(ref), run(ones)
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k].shape == want[k].shape and torch.equal(got[k], want[k]), k
    assert not torch.equal(got['image'], all_ones['image'])                 # the pickled (not an all-ones) mask is rendered


# ------------------------------------------------------------------------------------------------ the CLI
@pytest.fixture(scope='module')
def network(tmp_path_factory):
    from next3d_b200 import config, weights
    cfg = config.tiny_config(512)
    path = tmp_path_factory.mktemp('net') / 'tiny.pkl'
    path.write_bytes(persistence_pickle(cfg, weights.make_state_dict(cfg, seed=9), generator_fields(cfg, _mask(10))))
    return str(path)


class _Writer:
    def __init__(self, path, **kwargs):
        self.path, self.kwargs, self.frames, self.closed = path, kwargs, [], False

    def append_data(self, frame):
        self.frames.append(np.array(frame, copy=True))

    def close(self):
        self.closed = True


@pytest.fixture
def imageio(monkeypatch):
    """A stand-in imageio that records every writer and its frames."""
    mod = types.ModuleType('imageio')
    mod.writers = []

    def get_writer(path, **kwargs):
        mod.writers.append(_Writer(path, **kwargs))
        return mod.writers[-1]
    mod.get_writer = get_writer
    monkeypatch.setitem(sys.modules, 'imageio', mod)
    return mod


def _mesh(demo):
    from next3d_b200 import inputs
    return inputs.load_frame(demo[1], demo[3]).to(DEV)


def _assert_frames(got, want):
    assert len(got) == len(want) and len(want) > 0
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape and a.dtype == np.uint8 and np.array_equal(a, b), f'frame {i}'


def test_cli_gen_samples(network, tmp_path):
    from PIL import Image
    from next3d_b200 import drivers
    from next3d_b200.__main__ import main
    demo, out = _demo_args(tmp_path), tmp_path / 'out'
    main(['gen_samples', '--network', network, '--seeds', '3,5', '--outdir', str(out), '--shapes', 'True', '--shape-res', '64',
          '--lms_cond', 'True', *demo])
    G, v = _load(network), _mesh(demo)
    ws = drivers.sample_sheet_ws(G, [3, 5], 1, 14, 18)
    sheets = [s for _, s, _ in drivers.render_sample_sheets(G, ws, v, fov_deg=18, seed=0)]
    for i, seed in enumerate([3, 5]):
        assert np.array_equal(np.array(Image.open(out / f'seed{seed:04d}.png')), sheets[i]), seed
        raw = (out / f'seed{seed:04d}.mrc').read_bytes()
        assert tuple(np.frombuffer(raw[:16], '<i4')) == (64, 64, 64, 2)
        grid = drivers.extract_sigma_grid(G, ws[i:i + 1], v, 64)
        assert np.array_equal(np.frombuffer(raw[1024:], '<f4').reshape(64, 64, 64), grid), seed


def test_cli_gen_videos_grid(network, tmp_path, imageio):
    from next3d_b200 import drivers
    from next3d_b200.__main__ import main
    demo, out = _demo_args(tmp_path), tmp_path / 'out'
    main(['gen_videos', '--network', network, '--seeds', '0-3', '--grid', '2x1', '--w-frames', '2', '--outdir', str(out),
          '--lms_cond', 'True', *demo])
    (w,) = imageio.writers
    assert w.path == str(out / 'interpolation.mp4') and w.closed and w.kwargs['fps'] == 60
    G, v = _load(network), _mesh(demo)
    for k in ('depth_resolution', 'depth_resolution_importance'):                 # --sample_mult 2
        G.rendering_kwargs[k] *= 2
    ws = drivers.grid_keyframes(G, [0, 1, 2, 3], (2, 1), truncation_psi=1, truncation_cutoff=14)
    _assert_frames(w.frames, list(drivers.render_grid_frames(G, ws, v, 2, seed=0)))


def test_cli_gen_videos_orbit(network, tmp_path, imageio):
    from next3d_b200 import drivers
    from next3d_b200.__main__ import main
    demo, out = _demo_args(tmp_path), tmp_path / 'out'
    main(['gen_videos', '--network', network, '--seeds', '4', '--interpolate', 'False', '--w-frames', '3', '--sample_mult', '1',
          '--nrr', '32', '--image_mode', 'image_depth', '--outdir', str(out), '--lms_cond', 'True', *demo])
    (w,) = imageio.writers
    assert w.path == str(out / '4.mp4') and w.closed
    G, v = _load(network), _mesh(demo)
    G.neural_rendering_resolution = 32
    rk = G.rendering_kwargs
    ws = drivers.grid_keyframes(G, [4], (1, 1), truncation_psi=1, truncation_cutoff=14)[0, 0, :1]
    cams = drivers.orbit_camera_params(3, torch.tensor(rk['avg_camera_pivot']), rk['avg_camera_radius'])
    _assert_frames(w.frames, list(drivers.render_orbit(G, ws, cams, v, image_mode='image_depth', seed=0)))


def _drive_root(path, demo, n=5):
    """A driving directory from the demo mesh and landmarks: dataset.json, NNNN.png (seeded photos), NNNN.obj, NNNN_kpt2d.txt."""
    import shutil
    from PIL import Image
    from next3d_b200 import camera
    path.mkdir()
    rng = np.random.RandomState(2)
    intr = camera.fov_to_intrinsics(18.837).reshape(9)
    labels = []
    for k in range(n):
        name = f'{k:04d}'
        Image.fromarray(rng.randint(0, 256, (512, 512, 3), dtype=np.uint8)).save(path / f'{name}.png')
        shutil.copy(demo[1], path / f'{name}.obj')
        shutil.copy(demo[3], path / f'{name}_kpt2d.txt')
        pose = camera.look_at_pose(np.pi / 2 + 0.1 * k, np.pi / 2, torch.tensor([0, 0, 0.2]), 2.7)
        labels.append([f'{name}.png', torch.cat([pose.reshape(16), intr]).tolist()])
    (path / 'dataset.json').write_text(json.dumps({'labels': labels}))
    return str(path)


@pytest.mark.parametrize('fixed_camera', [False, True])
def test_cli_reenact(network, tmp_path, imageio, fixed_camera):
    from next3d_b200 import drivers
    from next3d_b200.__main__ import main
    demo, out = _demo_args(tmp_path), tmp_path / 'out'
    drive = _drive_root(tmp_path / 'drive', demo)
    main(['reenact', '--network', network, '--drive_root', drive, '--grid', '2x1', '--seeds', '6', '--outdir', str(out),
          '--num_frames', '3', '--fixed_camera', str(fixed_camera), '--lms_cond', 'True'])
    (w,) = imageio.writers
    assert w.path == str(out / 'reenact.mp4') and w.closed and w.kwargs['fps'] == 30
    G = _load(network)
    ws = drivers.sample_sheet_ws(G, [6], 1, 14, 18)
    fixed = drivers.sample_sheet_cameras(G, 18)[1] if fixed_camera else None
    _assert_frames(w.frames, list(drivers.reenact_grid_frames(G, ws, drive, 3, (2, 1), fixed_camera=fixed, seed=0)))
