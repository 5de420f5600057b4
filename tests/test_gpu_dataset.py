"""GPU: `python -m next3d_b200 gen_dataset` on the tiny generator.  Every image decodes to exactly the uint8 frame of a per-head
loop of synthesis / render_views with the same sampler seeds; labels, meshes, landmarks and heads.npz are written in the
reference's layout; and runs at world 2 and 3 (ranks sharing one GPU, one rank left without heads) write the tree of world 1,
byte for byte."""
import io
import json
import os

import numpy as np
import pytest
import torch
from PIL import Image

from tests.test_gpu_sharded_cli import _cli, inputs  # noqa: F401  (module fixture)

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _tree(d):
    out = {}
    for root, _, files in os.walk(d):
        for f in files:
            p = os.path.join(root, f)
            out[os.path.relpath(p, d)] = open(p, 'rb').read()
    return out


def _argv(net, demo, out, seeds, views=3, extra=()):
    return ['gen_dataset', '--network', net, '--outdir', out, '--lms_cond', 'True', '--seeds', seeds, '--views', str(views),
            '--batch', '2', *demo, *extra]


def test_images_equal_a_per_head_loop(inputs, tmp_path):
    from next3d_b200 import drivers, legacy
    from next3d_b200.__main__ import SAMPLER_SEED
    net, demo, _ = inputs
    out = str(tmp_path / 'o')
    _cli(_argv(net, demo, out, '0-2', views=3), 1)
    labels = json.load(open(os.path.join(out, 'images', 'dataset.json')))['labels']
    names = [drivers.dataset_image_name(i) for i in range(9)]
    assert [n for n, _ in labels] == names and all(len(c) == 25 for _, c in labels)
    heads = np.load(os.path.join(out, 'heads.npz'))
    assert list(heads['seed']) == [0, 1, 2] and list(heads['expression']) == [0, 0, 0] and heads['ws'].shape == (3, 28, 512)
    obj, lms = open(demo[1], 'rb').read(), open(demo[3], 'rb').read()
    for n in names:
        assert open(os.path.join(out, 'meshes', n.replace('png', 'obj')), 'rb').read() == obj
        assert open(os.path.join(out, 'lms', n.replace('png', 'txt')), 'rb').read() == lms
    # per head: seeds 2 c and 2 c + 1 of its call c, as the driver's calls draw them
    from next3d_b200 import inputs as I
    with open(net, 'rb') as f:
        G = legacy.load_network_pkl(f)['G_ema'].to(DEV)
    ws = drivers.sample_sheet_ws(G, [0, 1, 2])
    cams = drivers.dataset_cameras(G, [0, 1, 2], 3).to(DEV)
    v = I.load_frame(demo[1], demo[3]).to(DEV)
    with torch.no_grad():
        for h in range(3):
            c = h // 2
            # the call renders heads [2 c, 2 c + 1] (the last call repeats its head): render the same batch
            idx = [min(2 * c + j, 2) for j in range(2)]
            front = G.synthesis(ws[idx], cams[idx, 0], v.expand(2, -1, -1), noise_mode='const', cache_backbone=True,
                                seed=SAMPLER_SEED + 2 * c)['image']
            views = G.render_views(cams[idx, 1:].reshape(-1, 25), seed=SAMPLER_SEED + 2 * c + 1)['image']
            j = idx.index(h)
            want = drivers.to_uint8_hwc(torch.cat([front[j:j + 1], views[2 * j:2 * j + 2]])).cpu().numpy()
            for k in range(3):
                got = np.asarray(Image.open(os.path.join(out, 'images', names[3 * h + k])))
                np.testing.assert_array_equal(got, want[k], err_msg=f'head {h} view {k}')


@pytest.mark.parametrize('seeds', ['0-4', '0-1'])
def test_world_2_and_3_write_the_tree_of_world_1(inputs, tmp_path, seeds):
    """5 heads in calls of 2: ranks of 2 + 1 calls and 1 + 1 + 1 calls; 2 heads: one call, so ranks 1 and 2 own none."""
    net, demo, _ = inputs
    want = None
    for w in (1, 2, 3):
        out = str(tmp_path / f'w{w}')
        _cli(_argv(net, demo, out, seeds), w)
        got = _tree(out)
        assert got, f'world {w}: no output'
        if want is None:
            want = got
        else:
            assert sorted(got) == sorted(want), w
            for name in want:
                assert got[name] == want[name], f'world {w}: {name} differs'


def test_drive_root_expressions(inputs, tmp_path):
    """Two expressions per seed drawn from the driving frames: each image's mesh and landmarks are its driving frame's files."""
    from next3d_b200 import drivers
    net, _, drive = inputs
    out = str(tmp_path / 'o')
    _cli(['gen_dataset', '--network', net, '--outdir', out, '--lms_cond', 'True', '--seeds', '3-4', '--views', '2',
          '--drive_root', str(drive), '--expressions', '2'], 1)
    sched = drivers.reenact_schedule(str(drive), 1 << 30)
    heads = np.load(os.path.join(out, 'heads.npz'))
    seeds, ex = drivers.dataset_heads([3, 4], 2, len(sched['obj_paths']))
    assert list(heads['seed']) == seeds and list(heads['expression']) == ex
    for h, e in enumerate(ex):
        for v in range(2):
            n = drivers.dataset_image_name(2 * h + v)
            assert open(os.path.join(out, 'meshes', n.replace('png', 'obj')), 'rb').read() == open(sched['obj_paths'][e], 'rb').read()
            assert open(os.path.join(out, 'lms', n.replace('png', 'txt')), 'rb').read() == open(sched['lms_paths'][e], 'rb').read()
            Image.open(os.path.join(out, 'images', n)).load()
