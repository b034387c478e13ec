"""CPU-side checks of the C ABI: the library builds, loads, and exports every symbol include/sipmask_b200.h declares."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from sipmask_b200 import _lib, build
    path = build.build()
    assert os.path.exists(path)
    lib = ctypes.CDLL(path)
    header = open(os.path.join(ROOT, 'include', 'sipmask_b200.h')).read()
    declared = sorted(set(re.findall(r'\b(smb_[a-z0-9_]+)\s*\(', header)))
    assert declared, 'no declarations parsed'
    for name in declared:
        assert hasattr(lib, name), 'missing export %s' % name
    assert sorted(declared) == sorted(_lib.SYMBOLS)
    assert lib.smb_version() >= 100


def test_conv_plan_info_layout_and_null_arguments():
    """ConvPlanInfo lays out smb_conv_plan_info_t's fields in the header's order, and smb_conv_plan_info refuses null
    pointers (no device needed)."""
    from sipmask_b200 import _lib, build
    header = open(os.path.join(ROOT, 'include', 'sipmask_b200.h')).read()
    body = re.search(r'typedef struct \{([^}]*)\} smb_conv_plan_info_t;', header).group(1)
    fields = []
    for decl in body.split(';'):
        decl = decl.strip()
        if decl:
            assert decl.startswith('int '), decl
            fields += [re.match(r'(\w+)', f.strip()).group(1) for f in decl[4:].split(',')]
    assert [f[0] for f in _lib.ConvPlanInfo._fields_] == fields
    n = int(re.search(r'#define SMB_CONV_MAX_LEVELS (\d+)', header).group(1))
    assert _lib.CONV_MAX_LEVELS == n
    arrays = [f for f in fields if '%s[SMB_CONV_MAX_LEVELS]' % f in body]
    assert ctypes.sizeof(_lib.ConvPlanInfo) == 4 * (len(fields) - len(arrays) + n * len(arrays))
    lib = ctypes.CDLL(build.build())
    lib.smb_last_error.restype = ctypes.c_char_p
    info = _lib.ConvPlanInfo()
    assert lib.smb_conv_plan_info(None, ctypes.byref(info)) == -1
    assert b'smb_conv_plan_info' in lib.smb_last_error()


def test_ops_fail_loudly_without_cuda():
    import torch
    from sipmask_b200 import ops, _lib
    if torch.cuda.is_available():
        pytest.skip('CUDA present')
    with pytest.raises(_lib.SmbError):
        ops.crop_split(torch.zeros(4, 4, 4, 1), torch.zeros(1, 4))
    with pytest.raises(_lib.SmbError):
        ops.nms(torch.zeros(3, 5), 0.5)
    with pytest.raises(_lib.SmbError):
        ops.mask_assemble(torch.zeros(32, 4, 4), torch.zeros(1, 128), torch.zeros(1, 4), 0.5)


def test_sass_contains_hopper_instructions():
    """The conv kernel must be real wgmma / TMA code: warpgroup MMAs (HGMMA) fed by tensor-memory-accelerator loads."""
    import shutil
    import subprocess
    from sipmask_b200 import build
    if shutil.which('cuobjdump') is None:
        pytest.skip('cuobjdump not available')
    sass = subprocess.run(['cuobjdump', '-sass', build.LIB], capture_output=True, text=True).stdout
    for mnemonic in ('HGMMA', 'UTMALDG', 'WARPGROUP.ARRIVE'):
        assert mnemonic in sass, mnemonic
