"""CPU: the reference's two CUDA ops as built by oracle/build_ref_ops.py (`build()` runs it).

  * both binaries exist under oracle/_ref/, each carries an sm_90a cubin, and oracle/ref_ops.py
    imports them without a GPU, exposing the reference's entry points;
  * the package's upfirdn2d output size follows the reference's C arithmetic, including the
    signals shorter than the kernel where C truncation and Python's floor disagree.
The GPU comparison of the ops themselves is tests/test_gpu_reference_ops.py.
"""
import os
import subprocess

import pytest

from oracle import build_ref_ops, ref_ops


def test_reference_op_binaries_exist_after_build():
    paths = build_ref_ops.build()          # a no-op when they are fresh (or the checkout absent)
    assert sorted(paths) == sorted(ref_ops.NAMES)
    for name in ref_ops.NAMES:
        assert paths[name] == ref_ops.path(name)
        assert os.path.getsize(ref_ops.path(name)) > 0


@pytest.mark.parametrize('name', ['rwref_upfirdn2d', 'rwref_fused_bias_act'])
def test_reference_op_binary_carries_an_sm90a_cubin(name):
    from rewriting_b200 import build as rw_build
    cuobjdump = os.path.join(os.path.dirname(rw_build.find_nvcc()), 'cuobjdump')
    out = subprocess.run([cuobjdump, '--list-elf', ref_ops.path(name)], stdout=subprocess.PIPE,
                         stderr=subprocess.STDOUT, text=True, check=True).stdout
    elfs = [ln for ln in out.splitlines() if '.cubin' in ln]
    assert elfs and all('sm_90a' in ln for ln in elfs), out


def test_reference_ops_import_without_a_gpu():
    upfirdn2d_op, fused = ref_ops.load()
    assert callable(upfirdn2d_op.upfirdn2d) and callable(fused.fused_bias_act)
    assert 'upfirdn2d (CUDA)' in upfirdn2d_op.upfirdn2d.__doc__
    assert 'fused bias act (CUDA)' in fused.fused_bias_act.__doc__
    assert ref_ops.load()[0] is upfirdn2d_op          # loaded once


def _c_div(a, b):
    """C's `/` on ints: truncation toward zero."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def test_upfirdn2d_output_length_is_the_references_c_arithmetic():
    from rewriting_b200 import ops
    for down in (1, 2, 3):
        for n in range(-3 * down, 40):
            # upfirdn2d_kernel.cu: out = (in*up + pad0 + pad1 - k + down) / down
            assert ops._upfirdn2d_out_len(n, down) == _c_div(n + down, down), (n, down)
            if n >= -down:
                assert ops._upfirdn2d_out_len(n, down) == n // down + 1
    # in_h = 1, a 4-tap kernel, no pad, down 2: the reference returns 0 rows (floor gave -1)
    assert ops._upfirdn2d_out_len(1 - 4, 2) == 0
