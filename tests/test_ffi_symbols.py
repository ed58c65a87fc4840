"""The C-ABI library loads and exports every symbol include/deephar_b200.h declares
(no compute calls: there is no GPU in the CPU test run)."""
import ctypes
import os
import re

from deephar_b200 import _ffi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, 'include', 'deephar_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(dh_[a-z0-9_]+)\s*\(', src)))


def test_library_exports_all_declared_symbols():
    names = _declared()
    assert len(names) >= 15
    lib = ctypes.CDLL(_ffi.LIB_PATH)
    for n in names:
        assert hasattr(lib, n), 'missing export %s' % n


def test_binding_covers_header():
    assert sorted(_ffi.SIGNATURES) == _declared()


def test_version_and_error_string():
    lib = _ffi.lib()
    assert lib.dh_version() >= 100
    assert isinstance(lib.dh_last_error(), bytes)


def test_no_gpu_fails_loudly():
    import pytest
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    from deephar_b200 import reception
    m = reception.build((64, 64, 3), 16, 2, num_blocks=1).init_synthetic_weights()
    import numpy as np
    with pytest.raises(_ffi.DeepharB200Error):
        m.predict(np.zeros((1, 64, 64, 3), np.float32))
    h = ctypes.c_void_p()
    assert lib_rc(h) != 0


def lib_rc(h):
    return _ffi.lib().dh_ctx_create(ctypes.byref(h), 0)


def test_header_is_plain_c_and_struct_layouts_match_ctypes():
    """The boundary is a C ABI: the header must compile as C99 (no C++, no torch types), and the ctypes mirrors in
    _ffi.py must have the compiler's struct sizes."""
    import shutil
    import subprocess
    import tempfile
    import pytest
    gcc = shutil.which('gcc')
    if gcc is None:
        pytest.skip('no gcc')
    hdr = os.path.join(ROOT, 'include', 'deephar_b200.h')
    subprocess.check_call([gcc, '-fsyntax-only', '-x', 'c', '-std=c99', '-Wall', '-Werror', hdr])
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, 's.c')
        open(src, 'w').write('#include <stdio.h>\n#include "deephar_b200.h"\nint main(void) { printf("%zu %zu %zu %zu %zu\\n", '
                             'sizeof(dh_view), sizeof(dh_conv_desc), sizeof(dh_packed_w), sizeof(dh_frame_src), '
                             'sizeof(dh_conv_plan_info)); return 0; }\n')
        exe = os.path.join(d, 's')
        subprocess.check_call([gcc, '-std=c99', '-I', os.path.join(ROOT, 'include'), src, '-o', exe])
        sizes = [int(v) for v in subprocess.check_output([exe]).split()]
    assert sizes == [ctypes.sizeof(_ffi.dh_view), ctypes.sizeof(_ffi.dh_conv_desc), ctypes.sizeof(_ffi.dh_packed_w),
                     ctypes.sizeof(_ffi.dh_frame_src), ctypes.sizeof(_ffi.dh_conv_plan_info)]
