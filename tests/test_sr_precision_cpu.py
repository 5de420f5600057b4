"""CPU: TriPlaneGenerator.sr_precision validation, the mode in the CUDA-graph keys, and the ctypes binding of the fp16 ABI additions
(N3DSplitOut.f16, N3DConvGemm.f16, n3d_modulate_f16, n3d_resize_aa_f16) against include/next3d_b200.h as a C compiler lays it out."""
import os
import re
import shutil
import subprocess
import types

import pytest

from next3d_b200 import config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _generator(sr_num_fp16_res):
    from next3d_b200.triplane_next3d import TriPlaneGenerator
    cfg = config.tiny_config(512)
    cfg.sr_num_fp16_res = sr_num_fp16_res
    return TriPlaneGenerator.from_config(cfg, device='cpu')


def test_sr_precision_attribute():
    G = _generator(4)
    assert G.sr_precision == 'fp32'
    G.sr_precision = 'fp16'
    assert G.sr_precision == 'fp16'
    G.sr_precision = 'fp32'
    for bad in ('bf16', 'FP16', None, 16):
        with pytest.raises(ValueError):
            G.sr_precision = bad
    assert G.sr_precision == 'fp32'


def test_fp16_needs_sr_num_fp16_res():
    G = _generator(0)
    with pytest.raises(ValueError, match='sr_num_fp16_res'):
        G.sr_precision = 'fp16'
    assert G.sr_precision == 'fp32'
    G4 = _generator(4)
    G4.sr_precision = 'fp16'
    G4.sr_num_fp16_res = 0                   # changed afterwards: the next call refuses (before any device work)
    with pytest.raises(ValueError, match='sr_num_fp16_res'):
        G4._check_sr_precision(G4.sr_precision)


def test_graph_keys_include_the_mode():
    """A graph captured in one mode is never replayed in the other: the mode is part of every graph key (_render_key)."""
    from next3d_b200.engine import Engine
    rk = config.FFHQ_RENDERING_KWARGS
    k32 = Engine._render_key(types.SimpleNamespace(rk=rk, sr_precision='fp32'), 64)
    k16 = Engine._render_key(types.SimpleNamespace(rk=rk, sr_precision='fp16'), 64)
    assert k32 != k16 and k32[:-1] == k16[:-1]


def _header_params(name):
    src = re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'next3d_b200.h')).read(), flags=re.S)
    m = re.search(r'\b' + name + r'\s*\(([^)]*)\)', src)
    return [a.strip() for a in m.group(1).split(',')]


@pytest.mark.parametrize('name', ['n3d_modulate_f16', 'n3d_resize_aa_f16'])
def test_f16_entry_points_bound_with_the_header_arity(name):
    from next3d_b200 import _lib
    assert name in _lib.EXPORTS
    assert len(_lib._SIGNATURES[name][0]) == len(_header_params(name))
    assert hasattr(_lib.lib, name)


def test_struct_layout_matches_the_header(tmp_path):
    """sizeof / offsetof of the structs that gained an f16 field, from the C compiler, equal the ctypes binding's."""
    import ctypes
    from next3d_b200 import _lib
    cc = shutil.which('cc') or shutil.which('gcc')
    if cc is None:
        pytest.skip('no C compiler')
    prog = tmp_path / 'layout.c'
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "next3d_b200.h"\nint main(void) {\n'
                    '  printf("%zu %zu %zu %zu %zu\\n", sizeof(N3DSplitOut), offsetof(N3DSplitOut, f16), sizeof(N3DConvGemm),\n'
                    '         offsetof(N3DConvGemm, f16), offsetof(N3DConvGemm, out));\n  return 0;\n}\n')
    exe = tmp_path / 'layout'
    subprocess.check_call([cc, '-I', os.path.join(ROOT, 'include'), str(prog), '-o', str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    want = [ctypes.sizeof(_lib.SplitOut), _lib.SplitOut.f16.offset, ctypes.sizeof(_lib.ConvGemm), _lib.ConvGemm.f16.offset,
            _lib.ConvGemm.out.offset]
    assert got == want
