"""GPU: the sm_90a H.264 encoder at its coding edges.  Every case of tests/test_h264_edges_cpu.py's table (the edge sequences at
2-sample crop remainders, one MB column of 66 rows, 65x33 MBs and the level-6.2 extremes of 1055 MBs along one side; every QP
0-51 in both streams; frame_num wraps; the free rate controller) through H264Writer gives the oracle's samples, IDR frames and
reconstruction planes bit for bit (under rate control, so the oracle's QP sequence), and so do rendered grid frames at 1024x1024
(64x64 MBs).  FFmpeg decodes the oracle's streams in the CPU file; cv2 is not needed here."""
import pytest
import torch

from tests import h264_oracle as O
from tests.test_gpu_h264 import DEV, STREAMS, assert_same, gpu_encode, oracle_encode
from tests.test_h264_edges_cpu import TABLE, case_id, edge_run, stream_args

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('case', TABLE, ids=case_id)
def test_gpu_edge_stream_equals_oracle(tmp_path, case):
    name, W, H, n, gop = case[:5]
    run = edge_run(case)
    got = gpu_encode(tmp_path / 'v.mp4', O.frames(name, W, H, n), W, H, gop, **stream_args(case))
    assert_same(got, (run[0], [i for i, x in enumerate(run[1]) if x], run[2]))


@pytest.fixture(scope='module')
def grid_frames():
    """4 rendered frames of a 2x2 grid of the tiny generator (1024x1024: 64x64 MBs, 2 keyframes per cell, 2 frames each)."""
    from next3d_b200 import config, drivers, weights
    from tests.test_gpu_views import _generator
    cfg = config.tiny_config(512)
    _, G = _generator(cfg, 6)
    *_, v = weights.demo_inputs(cfg, 1, seed=0, device=DEV)
    ws_grid = drivers.grid_keyframes(G, list(range(8)), (2, 2), truncation_psi=0.7)
    frames = list(drivers.render_grid_frames(G, ws_grid, v, 2, seed=0))
    del G
    torch.cuda.empty_cache()
    return frames


@pytest.mark.parametrize('stream', list(STREAMS))
def test_rendered_grid_frames_equal_oracle(tmp_path, grid_frames, stream):
    assert len(grid_frames) == 4 and grid_frames[0].shape == (1024, 1024, 3)
    got = gpu_encode(tmp_path / 'v.mp4', grid_frames, 1024, 1024, 60, fps=60, batch=4, **STREAMS[stream])
    assert_same(got, oracle_encode(grid_frames, 1024, 1024, 60, fps=60, **STREAMS[stream]))
