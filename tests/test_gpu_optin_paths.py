"""The opt-in kernel paths read their switches once per process, so they are exercised by re-running the relevant parity
tests in a child process with the switch set: conv3d split-K variants (in-kernel finish, single atomic slab) and the
dynamic tile scheduler against the convolution / tokenizer tests."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONV_TESTS = ['tests/test_gpu_layers.py', 'tests/test_gpu_tokenizer.py']


def _rerun(tests, switch):
    name, _, value = switch.partition('=')
    env = dict(os.environ, **{name: value})
    r = subprocess.run([sys.executable, '-m', 'pytest', *tests, '-m', 'gpu', '-q', '-x', '-p', 'no:cacheprovider'], cwd=ROOT,
                       env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]


@pytest.mark.gpu
@pytest.mark.parametrize('switch', ['OG_SPLITK_FUSED=1', 'OG_IGEMM_DYNAMIC=1', 'OG_SPLITK_SLABS=0'])
def test_conv_parity_with_optin_switch(switch):
    _rerun(CONV_TESTS, switch)

