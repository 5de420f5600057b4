"""GPU: the sm_90a PNG encoder (csrc/png.cu through next3d_b200.png) writes exactly the bytes of its numpy restatement
(tests/png_oracle.py, whose files decode to their pixels in tests/test_png_cpu.py) for the CPU suite's cases and for rendered
frames of the tiny generator, whatever the batch; and it refuses bad images."""
import numpy as np
import pytest
import torch

from tests import png_oracle as O
from tests.test_png_cpu import CONTENTS, SIZES, case_image

pytestmark = pytest.mark.gpu
DEV = 'cuda'


@pytest.mark.parametrize('H,W', SIZES, ids=[f'{h}x{w}' for h, w in SIZES])
def test_cases_equal_oracle(H, W):
    """All four contents of a size in one batch, then one at a time from numpy: the oracle's bytes both ways."""
    from next3d_b200.png import PngEncoder, encode_png
    imgs = np.stack([case_image(c, H, W) for c in CONTENTS])
    want = [O.encode(im) for im in imgs]
    assert encode_png(torch.from_numpy(imgs).to(DEV)) == want
    enc = PngEncoder(W, H, batch=1)
    got = []
    for im in imgs:
        got += enc.write(im)
    assert got + enc.flush() == want


@pytest.fixture(scope='module')
def rendered():
    from next3d_b200 import config, drivers, weights
    from tests.test_gpu_views import _generator
    cfg = config.tiny_config(512)
    _, G = _generator(cfg, 6)
    *_, v = weights.demo_inputs(cfg, 1, seed=0, device=DEV)
    rk = G.rendering_kwargs
    ws = drivers.grid_keyframes(G, [3], (1, 1), truncation_psi=0.7)[0, 0]
    cams = drivers.orbit_camera_params(6, torch.tensor(rk['avg_camera_pivot']), rk['avg_camera_radius'])
    return torch.stack([torch.as_tensor(f) for f in drivers.render_orbit(G, ws[:1], cams, v, seed=0)]).to(DEV)


@pytest.mark.parametrize('batch', [1, 3, 8])
def test_rendered_frames_equal_oracle(rendered, batch):
    """Rendered 512x512 frames as CUDA tensors, in batches that split the writes unevenly: the oracle's bytes in order."""
    from next3d_b200.png import PngEncoder
    frames = rendered
    want = [O.encode(f) for f in frames.cpu().numpy()]
    enc = PngEncoder(frames.shape[2], frames.shape[1], batch=batch)
    got = enc.write(frames[:2]) + enc.write(frames[2:5]) + enc.write(frames[5])
    assert got + enc.flush() == want


def test_refuses_bad_images():
    from next3d_b200.png import PngEncoder, encode_png
    enc = PngEncoder(8, 4)
    with pytest.raises(TypeError, match='uint8'):
        enc.write(np.zeros((4, 8, 3), np.float32))
    with pytest.raises(ValueError, match=r'shape \[N, 4, 8, 3\]'):
        enc.write(np.zeros((4, 8, 4), np.uint8))
    with pytest.raises(ValueError, match=r'shape \[N, 4, 8, 3\]'):
        enc.write(torch.zeros(2, 2, 4, 8, 3, dtype=torch.uint8))
    with pytest.raises(ValueError, match='positive dimensions'):
        PngEncoder(0, 4)
    with pytest.raises(ValueError, match='CUDA device'):
        PngEncoder(8, 4, device='cpu')
    with pytest.raises(ValueError, match=r'shape \[N, H, W, 3\]'):
        encode_png(np.zeros((2, 4, 8), np.uint8))
    assert enc.flush() == []


def test_rows_wider_than_one_stored_block():
    """2 x 22000 noise: each one-row stripe is 66001 filtered bytes, stored as two blocks."""
    from next3d_b200.png import encode_png
    img = case_image('noise', 2, 22000)
    info = {}
    want = O.encode(img, info)
    assert all(info['stored'])
    assert encode_png(torch.from_numpy(img).to(DEV)) == [want]


def test_device_without_index():
    """device='cuda' names the current device: frames on it are accepted."""
    from next3d_b200.png import PngEncoder
    img = case_image('gradient', 5, 7)
    enc = PngEncoder(7, 5, device='cuda')
    assert enc.write(torch.from_numpy(img).to('cuda:0')) + enc.flush() == [O.encode(img)]
