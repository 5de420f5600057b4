"""CPU: the gradient entry points (n3d_bias_act_grad, n3d_conv_wgrad, n3d_wgrad_operand) refuse bad arguments with
N3D_ERR_INVALID_ARG before any CUDA call."""
import ctypes as C

import pytest

from next3d_b200 import _lib

FAKE = 1 << 20            # a 16-byte aligned address that is never dereferenced: every call below fails its argument checks first


def _bias_act_grad(dy=FAKE, b=None, xref=FAKE, yref=FAKE, dyref=FAKE, dx=FAKE, dtype=0, numel=16, size_b=0, step_b=0, grad=1, act=3):
    return _lib.lib.n3d_bias_act_grad(dy, b, xref, yref, dyref, dx, dtype, numel, size_b, step_b, grad, act, 0.2, 1.0, -1.0, None)


@pytest.mark.parametrize('kw,what', [
    (dict(dy=None), b'null'), (dict(dx=None), b'null'), (dict(grad=0), b'grad mode'), (dict(grad=3), b'grad mode'),
    (dict(grad=2, act=3), b'grad mode'), (dict(act=0), b'act'), (dict(act=10), b'act'), (dict(dtype=2), b'dtype'),
    (dict(b=FAKE, size_b=0, step_b=1), b'bias'), (dict(act=9, xref=None), b'xref'), (dict(act=4, yref=None), b'yref'),
    (dict(grad=2, act=4, dyref=None), b'dyref')])
def test_bias_act_grad_refuses(kw, what):
    assert _bias_act_grad(**kw) == -1
    assert what in _lib.lib.n3d_last_error()


def _wgrad(**kw):
    p = _lib.ConvWgrad()
    p.a_hi = p.a_lo = p.b_hi = p.b_lo = p.dw = FAKE
    p.a_rows, p.a_cols, p.lda = 16, 128, 128
    p.b_rows, p.b_cols, p.ldb = 16, 128, 128
    p.G, p.M, p.N, p.T, p.K, p.splits = 1, 16, 16, 1, 128, 1
    for k, v in kw.items():
        setattr(p, k, v)
    return p


@pytest.mark.parametrize('kw,what', [
    (dict(a_hi=None), b'null'), (dict(dw=None), b'null'), (dict(N=12), b'multiple of 8'), (dict(G=0), b'bad sizes'),
    (dict(M=0), b'bad sizes'), (dict(T=0), b'taps'), (dict(T=10), b'taps'), (dict(K=100), b'multiple of 64'), (dict(K=0), b'multiple of 64'),
    (dict(lda=100), b'geometry'), (dict(b_cols=200), b'geometry'), (dict(a_rows=8), b'rows'), (dict(G=2), b'rows'),
    (dict(a_off=(_lib.I64 * 9)(4)), b'multiples of 8'), (dict(b_off=(_lib.I64 * 9)(-1)), b'multiples of 8'),
    (dict(b_row=(_lib.I32 * 9)(8)), b'rows'), (dict(a_row=(_lib.I32 * 9)(-8)), b'rows'), (dict(splits=0), b'slices'),
    (dict(splits=3), b'slices'), (dict(splits=2), b'workspace'), (dict(dw=FAKE + 4), b'aligned')])
def test_conv_wgrad_refuses(kw, what):
    assert _lib.lib.n3d_conv_wgrad(C.byref(_wgrad(**kw)), None) == -1
    assert what in _lib.lib.n3d_last_error()


def test_conv_wgrad_refuses_null_descriptor():
    assert _lib.lib.n3d_conv_wgrad(None, None) == -1


@pytest.mark.parametrize('args,what', [
    (dict(x=None), b'null'), (dict(s=3), b'bad sizes'), (dict(N=0), b'bad sizes'), (dict(ld=100), b'row stride'),
    (dict(ld=8), b'row stride'), (dict(hi=FAKE + 2), b'aligned')])
def test_wgrad_operand_refuses(args, what):
    a = dict(x=FAKE, N=1, C=4, H=8, W=8, s=1, pt=0, pl=0, PH=8, PW=8, ld=64, hi=FAKE, lo=FAKE)
    a.update(args)
    strides = (_lib.I64 * 4)(256, 64, 8, 1)
    rc = _lib.lib.n3d_wgrad_operand(a['x'], strides, a['N'], a['C'], a['H'], a['W'], a['s'], a['pt'], a['pl'], a['PH'], a['PW'], 0, a['ld'],
                                    a['hi'], a['lo'], None)
    assert rc == -1
    assert what in _lib.lib.n3d_last_error()
