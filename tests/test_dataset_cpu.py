"""CPU: the multi-view dataset driver and command.  The plan of each rank at world sizes 1-3 is the single-process run's calls
(batch, cache flags, sampler seeds) over whole calls; the frames of render_dataset on the recording stub generator equal a
per-head loop; heads, cameras, names and labels follow their seeded rules and the reference's dataset layout; and gen_dataset
refuses bad options before the network loads."""
import json
import os

import numpy as np
import pytest
import torch

from next3d_b200 import drivers
from tests.test_driver_calls_cpu import _StubG
from tests.test_sharded_video_cpu import _refuses


def _inputs(n_heads=7, V=3, M=2):
    torch.manual_seed(5)
    ws = torch.randn(n_heads, drivers.NUM_WS, 512)
    meshes = torch.randn(M, 11, 3)
    mesh_ids = [h % M for h in range(n_heads)]
    cams = drivers.dataset_cameras(_StubG(), list(range(n_heads)), V)
    return ws, meshes, mesh_ids, cams


@pytest.mark.parametrize('world', [1, 2, 3])
@pytest.mark.parametrize('n_heads,batch', [(7, 3), (2, 3), (6, 2)])
def test_rank_head_plans_are_the_single_process_run(world, n_heads, batch):
    ws, meshes, mesh_ids, cams = _inputs(n_heads)
    G1 = _StubG()
    single = [(h, f) for h, f in drivers.render_dataset(G1, ws, meshes, mesh_ids, cams, drivers.head_plan(n_heads, batch), seed=4)]
    calls = -(-n_heads // batch)
    assert [c[:5] for c in G1.calls] == [x for k in range(calls) for x in
                                         (('synthesis', batch, True, False, 4 + 2 * k), ('render_views', 2 * batch, False, False, 5 + 2 * k))]
    got, gcalls = [], []
    for r in range(world):
        G = _StubG()
        plan = drivers.head_plan(n_heads, batch, r, world)
        got += list(drivers.render_dataset(G, ws, meshes, mesh_ids, cams, plan, seed=4))
        gcalls += G.calls
    assert gcalls == G1.calls                                 # whole calls: no call runs twice
    assert [h for h, _ in got] == [h for h, _ in single] == list(range(0, n_heads, batch))
    assert all(torch.equal(a, b) for (_, a), (_, b) in zip(got, single))


def test_dataset_frames_equal_a_per_head_loop():
    ws, meshes, mesh_ids, cams = _inputs(5, V=3)
    frames = torch.cat([f for _, f in drivers.render_dataset(_StubG(), ws, meshes, mesh_ids, cams, drivers.head_plan(5, 2),
                                                             seed=None)])
    assert frames.shape == (15, 4, 4, 3) and frames.dtype == torch.uint8
    for h in range(5):
        G = _StubG()
        front = G.synthesis(ws[h:h + 1], cams[h, :1], meshes[mesh_ids[h]][None], noise_mode='const', cache_backbone=True)['image']
        views = G.render_views(cams[h, 1:])['image']
        want = drivers.to_uint8_hwc(torch.cat([front, views]))
        assert torch.equal(frames[3 * h:3 * h + 3], want), h


def test_heads_and_cameras_follow_their_seeded_rules():
    assert drivers.dataset_heads([3, 9]) == ([3, 9], [0, 0])
    seeds, ex = drivers.dataset_heads([3, 9], 2, 10)
    assert seeds == [3, 3, 9, 9]
    assert ex[:2] == sorted(np.random.RandomState([3, 0]).choice(10, 2, replace=False)) and ex[0] != ex[1]
    with pytest.raises(ValueError, match='expressions'):
        drivers.dataset_heads([1], 4, 3)
    G = _StubG()
    cams = drivers.dataset_cameras(G, [3, 9], 4, yaw_std=0.3, pitch_std=0.155, fov_deg=18.837)
    assert cams.shape == (2, 4, 25) and cams.dtype == torch.float32
    front = drivers.sample_sheet_cameras(G, 18.837)[1][0]
    assert torch.allclose(cams[0, 0], front) and torch.allclose(cams[1, 0], front)
    from next3d_b200 import camera
    n1, n2 = np.random.RandomState([9, 2]).randn(2)
    pose = camera.look_at_pose(np.pi / 2 + 0.3 * n1, np.pi / 2 + 0.155 * n2, torch.tensor([0, 0, 0.2]), 2.7).reshape(16)
    assert torch.allclose(cams[1, 2, :16], pose)
    assert torch.equal(drivers.dataset_cameras(G, [9], 4), drivers.dataset_cameras(G, [3, 9], 4)[1:])    # per seed, not per batch


def test_names_and_the_reference_mesh_mapping():
    assert drivers.dataset_image_name(0) == '00000/img00000000.png'
    assert drivers.dataset_image_name(12345) == '00012/img00012345.png'
    # dataset.py: mesh = os.path.join(mesh_path, fname.replace('png', 'obj')); lms = that .replace('meshes', 'lms').replace('obj', 'txt')
    root = '/data/out'
    fname = drivers.dataset_image_name(1234)
    mesh = os.path.join(root, 'meshes', fname.replace('png', 'obj'))
    assert mesh == '/data/out/meshes/00001/img00001234.obj'
    assert mesh.replace('meshes', 'lms').replace('obj', 'txt') == '/data/out/lms/00001/img00001234.txt'


@pytest.mark.parametrize('world', ['1', '2'])
@pytest.mark.parametrize('extra,match', [
    (['--views', '0'], 'views'),
    (['--drive_root', 'd', '--obj_path', 'a.obj', '--lms_path', 'a.txt'], 'not both'),
    (['--expressions', '2', '--obj_path', 'a.obj', '--lms_path', 'a.txt'], 'drive_root'),
    ([], 'obj_path'),
])
def test_cli_refuses_before_loading(tmp_path, monkeypatch, world, extra, match):
    from next3d_b200.__main__ import main
    for k in ('MASTER_ADDR', 'MASTER_PORT'):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv('WORLD_SIZE', world)
    monkeypatch.setenv('RANK', '0')
    with pytest.raises(SystemExit, match=match):
        main(['gen_dataset', '--seeds', '0', '--outdir', str(tmp_path / 'o'), '--lms_cond', 'True', '--network',
              str(tmp_path / 'missing.pkl'), *extra])
    assert not torch.distributed.is_initialized()
