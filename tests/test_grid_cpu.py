"""CPU: the host side of the grid video drivers (--grid of gen_videos_next3d.py and reenact_avatar_next3d.py) against the
reference scripts' own code, whose results on these inputs are stored in tests/golden/reference_grid.npz
(tests.helpers.ReferenceVectors): keyframe seeds, the grid layout, the photo cell's arithmetic; the argument checks of the
drivers and of the `views` entry points; and the sharded gather loop on rectangular frames under gloo."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from next3d_b200 import drivers
from tests.helpers import ReferenceVectors, lib, refused
from tests.test_drivers_cpu import _reference_scripts

REF = ReferenceVectors('reference_grid')


class _Stop(Exception):
    pass


class _StubMapG(torch.nn.Module):
    """The attributes grid_keyframes and gen_interp_video read before rendering; mapping records its arguments and returns
    ws [n, 2, z_dim] = z (so the reshape to the grid can be checked), or stops the reference script right after its mapping call."""
    z_dim = 4
    img_resolution = 512

    def __init__(self, stop=False):
        super().__init__()
        self.p = torch.nn.Parameter(torch.zeros(1))
        self.rendering_kwargs = dict(avg_camera_pivot=[0, 0, 0.2], avg_camera_radius=2.7)
        self.stop, self.calls = stop, []

    def mapping(self, z, c, truncation_psi=1, truncation_cutoff=None):
        self.calls.append((z, c, truncation_psi, truncation_cutoff))
        if self.stop:
            raise _Stop
        return z.float()[:, None].repeat(1, 2, 1)


def _script_mapping_inputs(seeds, grid, num_keyframes, shuffle_seed):
    """(z, c) that gen_interp_video (gen_videos_next3d.py:77-104) hands to G.mapping."""
    G = _StubMapG(stop=True)
    with pytest.raises(_Stop):
        _reference_scripts()[1].gen_interp_video(G, 'unused.mp4', seeds, torch.zeros(1, 1, 3), shuffle_seed=shuffle_seed, grid_dims=grid,
                                                 num_keyframes=num_keyframes, psi=0.7, truncation_cutoff=14, device=torch.device('cpu'))
    z, c, _, _ = G.calls[0]
    return z, c


@pytest.mark.parametrize('case,seeds,grid,num_keyframes,shuffle_seed', [
    (0, [10720, 12374, 13393, 17099], (2, 2), None, None),
    (1, [1, 2, 3, 4, 5, 6], (3, 1), None, 7),
    (2, [5, 9, 11], (1, 2), 4, None),
    (3, [3, 1, 4, 1, 5], (2, 2), 3, 123),
])
def test_keyframe_seeds_and_cameras_match_the_script(case, seeds, grid, num_keyframes, shuffle_seed):
    G = _StubMapG()
    ws = drivers.grid_keyframes(G, seeds, grid, num_keyframes, shuffle_seed, truncation_psi=0.7, truncation_cutoff=14)
    z, c, psi, cutoff = G.calls[0]
    assert torch.equal(z, REF.get(f'z_{case}', lambda: _script_mapping_inputs(seeds, grid, num_keyframes, shuffle_seed)[0]))
    assert torch.equal(c, REF.get(f'c_{case}', lambda: _script_mapping_inputs(seeds, grid, num_keyframes, shuffle_seed)[1]))
    assert (psi, cutoff) == (0.7, 14)
    gw, gh = grid
    K = num_keyframes or len(seeds) // (gw * gh)
    assert ws.shape == (gh, gw, K, 2, G.z_dim)
    assert torch.equal(ws.reshape(-1, 2, G.z_dim)[:, 0], z.float())       # ws.reshape(grid_h, grid_w, num_keyframes, ...) (:106)


@pytest.mark.parametrize('grid', [(2, 2), (3, 1), (1, 3)])
def test_layout_equals_the_script_layout_grid(grid):
    """Cells converted to uint8 on their own and laid out after == layout_grid of the float cells, for two frames of seeded cells
    with values outside [-1, 1]; also when the cells arrive in batches that split frames."""
    gw, gh = grid
    cells = gw * gh
    g = torch.Generator().manual_seed(gw * 10 + gh)
    img = torch.randn(2 * cells, 3, 6, 5, generator=g) * 1.5
    got = drivers.layout_cells(drivers.to_uint8_hwc(img), gw, gh)
    assert got.shape == (2, gh * 6, gw * 5, 3)
    for f in range(2):
        ref = REF.get(f'layout_{gw}x{gh}_{f}', lambda: _reference_scripts()[1].layout_grid(img[f * cells:(f + 1) * cells], grid_w=gw,
                                                                                          grid_h=gh))
        assert np.array_equal(got[f].numpy(), ref.numpy())
    u8 = drivers.to_uint8_hwc(img)
    batches, b0 = [], 0
    for size in (3, 1, 2 * cells):                                        # ragged batches; the last is padded past the end
        part = u8[b0:b0 + size]
        n = part.shape[0]
        batches.append((torch.cat([part, part[-1:].expand(size - n, -1, -1, -1)]) if n < size else part, n))
        b0 += n
    whole = list(drivers._whole_frames(iter(batches), gw, gh))
    assert sum(nf for _, nf in whole) == 2 and torch.equal(torch.cat([fr for fr, _ in whole]), got)


def _script_photo_frame(photo):
    """The photo cell as reenact_avatar_next3d.py:133-135 computes it, through the reference's layout_grid (:56-70, :167)."""
    target_img = torch.tensor(photo.transpose(2, 0, 1)).float().unsqueeze(0)
    target_img = target_img / 127.5 - 1.
    return _reference_scripts()[1].layout_grid(target_img, grid_w=1, grid_h=1)


def test_photo_cell_arithmetic_is_the_script_s():
    photo = np.stack([np.arange(256, dtype=np.uint8).reshape(16, 16)] * 3, -1)
    photo[..., 1] = photo[..., 1][::-1]
    got = drivers.photo_cell(torch.from_numpy(photo), 'cpu')
    assert np.array_equal(got.numpy(), REF.get('photo_cell', lambda: _script_photo_frame(photo)).numpy())


def test_load_photo_crops_like_pil(tmp_path):
    from PIL import Image
    from next3d_b200 import inputs
    rng = np.random.RandomState(0)
    a = rng.randint(0, 256, (300, 520, 3), dtype=np.uint8)
    Image.fromarray(a).save(tmp_path / 'p.png')
    got = inputs.load_photo(str(tmp_path / 'p.png'))
    assert got.shape == (512, 512, 3) and got.dtype == torch.uint8
    assert np.array_equal(got[:300].numpy(), a[:, :512]) and not got[300:].any()      # PIL's crop past the edge reads 0
    Image.fromarray(a[..., 0]).save(tmp_path / 'gray.png')
    with pytest.raises(ValueError, match='RGB'):
        inputs.load_photo(str(tmp_path / 'gray.png'))


# ------------------------------------------------------------------------------------------------ argument checks
def test_grid_keyframes_refuses_seeds_not_divisible_by_the_grid():
    with pytest.raises(ValueError, match='divisible by grid'):
        drivers.grid_keyframes(_StubMapG(), [1, 2, 3], (2, 2))


@pytest.mark.parametrize('what', ['cells', 'resolution', 'pack'])
def test_reenact_grid_refuses(tmp_path, what):
    G = _StubMapG()
    ws = torch.zeros(3, 2, 4)
    root, grid = str(tmp_path), (2, 2)
    if what == 'cells':
        grid, match = (3, 1), 'grid 3x1 has 3 cells'
    elif what == 'resolution':
        G.img_resolution, match = 256, 'img_resolution 512'
    else:
        root, match = str(tmp_path / 'clip.n3dpack'), 'no driving photos'
    with pytest.raises(ValueError, match=match):
        list(drivers.reenact_grid_frames(G, ws, root, 10, grid))
    with pytest.raises(ValueError, match=match):
        drivers.reenact_grid_frames_sharded(G, ws, root, 10, grid, device='cpu')


@pytest.mark.parametrize('N,views', [(3, 2), (4, 0), (4, -1)])
def test_views_entry_points_refuse_bad_counts(N, views):
    L = lib()
    t = torch.zeros(4096)
    p = t.data_ptr()
    assert p % 16 == 0
    refused(L.lib.n3d_uv_sample_views(p, p, p, p, p, N, views, 4, 4, 4, 4, 32, 4, 4, p, p, None), 'not a multiple of views')
    refused(L.lib.n3d_blend_planes_views(p, p, p, p, N, views, 4, 4, p, None), 'not a multiple of views')


# ------------------------------------------------------------------------------------------------ sharded gather loop (gloo)
H, W = 3, 5                                                              # rectangular frames


def _frame(f):
    return (torch.arange(H * W * 3, dtype=torch.int64).reshape(H, W, 3) * 7 + f * 31).remainder(256).to(torch.uint8)


def _worker(rank, world, port, F, q):
    from next3d_b200 import distributed as D
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    D.init_from_env('gloo')
    plan = drivers.shard_plan(F, 2)

    def step(k, idx):
        return torch.stack([_frame(f) for f in idx])
    host = drivers._gather_frames(plan, step, H, W, 'cpu', None)
    if rank == 0:
        q.put(host.numpy())
    torch.distributed.destroy_process_group()


@pytest.mark.parametrize('F', [6, 5])                                   # equal shards (3 + 3), unequal (3 + 2)
def test_sharded_gather_rectangular_frames_gloo(F):
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, F, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = q.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert got.shape == (F, H, W, 3)
    for f in range(F):
        assert np.array_equal(got[f], _frame(f).numpy()), f
