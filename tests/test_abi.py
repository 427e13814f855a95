"""CPU: the C-ABI shared library loads, exports every symbol include/opengenie_b200.h declares, validates
its arguments without touching a GPU, and the Python side refuses to run without CUDA (no fallback)."""
import ctypes
import os
import subprocess

import pytest
import torch

from open_genie_b200 import _lib


def test_library_exports_every_declared_symbol():
    protos = _lib.PROTOTYPES
    assert len(protos) >= 28 and 'og_conv3d_fwd' in protos and 'og_lfq_fwd' in protos
    lib = _lib.load()
    for name in protos:
        assert hasattr(lib, name), f'{name} declared in the header but not exported by the library'
    assert lib.og_abi_version() >= 1 and lib.og_compiled_sm() == 90
    out = subprocess.run(['nm', '-D', '--defined-only', _lib.LIB_PATH], capture_output=True, text=True).stdout
    exported = {ln.split()[-1] for ln in out.splitlines() if ' T ' in ln and ln.split()[-1].startswith('og_')}
    assert exported == set(protos), exported ^ set(protos)      # no undeclared entry points either


def test_argument_validation_returns_status_codes_not_crashes():
    lib = _lib.load()
    # null pointers / bad channel counts are rejected before any CUDA call
    rc = lib.og_conv3d_fwd(None, 64, 3, 3, 3, 1, 1, 1, None, 0, None, 1728, None, None, None, None, 0, 1, 2, 8, 8, 64,
                           None, 0, None, None)
    assert rc == -1 and b'null pointer' in lib.og_last_error()
    buf = ctypes.create_string_buffer(64)
    p = ctypes.addressof(buf)
    rc = lib.og_conv3d_fwd(p, 48, 3, 3, 3, 1, 1, 1, None, 0, p, 1296, None, None, None, p, 0, 1, 2, 8, 8, 64, None, 0,
                           None, None)
    assert rc == -1 and b'multiple of 64' in lib.og_last_error()
    rc = lib.og_conv3d_wgrad(p, 64, p, 72, p, 72, 1, 1, 1, 0, 0, 0, 1, 1, 8, 8, None, 0, None)
    assert rc == -1
    rc = lib.og_lfq_fwd(p, 18, 4, 25, 100.0, 0, .25, .1, 1., None, None, 0, p, None, None, None)
    assert rc == -1 and b'codebook_dim' in lib.og_last_error()
    assert lib.og_lfq_workspace_bytes(16, 25) == 0 and lib.og_lfq_workspace_bytes(16, 18) > 0
    with pytest.raises(RuntimeError, match='og_gn_stats failed'):
        _lib.call('og_gn_stats', None, 1, 1, 8, 1, None, None)


def test_no_cpu_fallback_in_the_product():
    import open_genie_b200 as og
    from oracle import fixtures as fx
    tok = og.VideoTokenizer(fx.MINI_ENC, fx.MINI_DEC, d_codebook=6, gan_loss_weight=0, perc_loss_weight=0)
    with pytest.raises(RuntimeError, match='no CPU path'):
        tok.tokenize(torch.zeros(fx.MINI_VIDEO_SHAPE))
    from open_genie_b200.module.quantization import LookupFreeQuantization
    with pytest.raises(RuntimeError, match='no CPU path'):
        LookupFreeQuantization(4, input_dim=4)(torch.zeros(1, 3, 4))
    # and nothing under open_genie_b200/ imports the oracle
    root = os.path.dirname(_lib._HERE)
    for dp, _, fs in os.walk(os.path.join(root, 'open_genie_b200')):
        for f in fs:
            if f.endswith('.py'):
                src = open(os.path.join(dp, f)).read()
                assert 'import oracle' not in src and 'from oracle' not in src, f
