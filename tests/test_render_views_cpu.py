"""CPU: the `views` field of N3DRender (several camera views per plane set) is checked by n3d_render_rays / n3d_render_rays_normals
before anything reaches the device.  Every call carries ray_end < ray_start, which the library checks after `views` and the plane
size: a call whose views pass gets the ray-setup error, and nothing is launched either way."""
import ctypes as C

import pytest
import torch

from next3d_b200 import config

ENTRIES = ['n3d_render_rays', 'n3d_render_rays_normals']


def _call(entry, N, views, PH=4, PW=4):
    from next3d_b200 import _lib, kernels
    cfg = config.tiny_config()
    opts = dict(cfg.rendering_kwargs, ray_start=2.0, ray_end=1.0)
    planes = torch.zeros(1, 3, 4, 4, 32)
    cam, intr = torch.zeros(1, 16), torch.zeros(1, 9)
    dec = (torch.zeros(64, 32), torch.zeros(64), torch.zeros(33, 64), torch.zeros(33))
    out = torch.zeros(4 * 4 * 32)
    p = kernels._render_full_desc(planes, cam, intr, 4, opts, dec, out, out, out, None, None, None, 0, None)
    p.N, p.views, p.PH, p.PW = N, views, PH, PW          # only the checks read these: nothing is launched
    if entry == 'n3d_render_rays':
        rc = _lib.lib.n3d_render_rays(C.byref(p), None)
    else:
        rc = _lib.lib.n3d_render_rays_normals(C.byref(p), kernels.ptr(out), kernels.ptr(out), None)
    return rc, _lib.lib.n3d_last_error().decode()


@pytest.mark.parametrize('entry', ENTRIES)
@pytest.mark.parametrize('N,views', [(5, 2), (6, 4), (1, 2), (3, -1), (4, -4)])
def test_views_that_do_not_divide_n_or_are_negative_are_refused(entry, N, views):
    rc, msg = _call(entry, N, views)
    assert rc == -1 and f'views = {views}' in msg, (rc, msg)


@pytest.mark.parametrize('entry', ENTRIES)
@pytest.mark.parametrize('N,views', [(1, 0), (4, 1), (6, 3), (5, 5), (8, 8)])
def test_views_dividing_n_pass_the_check(entry, N, views):
    rc, msg = _call(entry, N, views)
    assert rc == -1 and 'bad ray setup' in msg, (rc, msg)


@pytest.mark.parametrize('entry', ENTRIES)
def test_plane_size_limit_counts_plane_sets(entry):
    """A 256^2 plane set is 25 MB, so 171 of them overflow 32-bit texel offsets; 240 views of 2 sets (or of 170) do not."""
    rc, msg = _call(entry, 171, 1, 256, 256)
    assert rc == -1 and '32-bit texel offsets' in msg, (rc, msg)
    for N, views in [(240, 120), (480, 240), (340, 2), (171, 171)]:
        rc, msg = _call(entry, N, views, 256, 256)
        assert rc == -1 and 'bad ray setup' in msg, (N, views, rc, msg)
    rc, msg = _call(entry, 342, 2, 256, 256)
    assert rc == -1 and '32-bit texel offsets' in msg, (rc, msg)


def test_sample_points_plane_size_limit():
    """n3d_sample_points reads N plane sets with the same 32-bit texel offsets: 171 sets at 256^2 are refused, 170 pass the size
    check (and are then refused for an rgb buffer that is not 8-byte aligned, which the library checks next, so nothing launches)."""
    from next3d_b200 import _lib
    planes = torch.zeros(3 * 4 * 4 * 32)
    dec = [torch.zeros(n) for n in (64 * 32, 64, 33 * 64, 33)]
    coords, sigma, rgb = torch.zeros(8 * 3), torch.zeros(8), torch.zeros(8 * 32 + 1)

    def call(N):
        rc = _lib.lib.n3d_sample_points(planes.data_ptr(), N, 256, 256, coords.data_ptr(), 8, 1.0, *(t.data_ptr() for t in dec),
                                        sigma.data_ptr(), rgb[1:].data_ptr(), None)
        return rc, _lib.lib.n3d_last_error().decode()

    rc, msg = call(171)
    assert rc == -1 and '32-bit texel offsets' in msg, (rc, msg)
    rc, msg = call(170)
    assert rc == -1 and 'rgb must be 8-byte aligned' in msg, (rc, msg)
