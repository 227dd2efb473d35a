"""TEST INFRASTRUCTURE ONLY — the reference's two CUDA ops, as built by oracle/build_ref_ops.py.

`load()` imports `oracle/_ref/rwref_upfirdn2d.so` and `oracle/_ref/rwref_fused_bias_act.so` by
file path and returns them as (upfirdn2d_op, fused): the same pybind11 entry points the reference
calls, `upfirdn2d_op.upfirdn2d(input, kernel, up_x, up_y, down_x, down_y, pad_x0, pad_x1, pad_y0,
pad_y1)` and `fused.fused_bias_act(input, bias, refer, act, grad, alpha, scale)`.  It never reads
a reference checkout, so it works wherever the binaries were carried; a missing or unloadable
binary raises (importing needs torch, not a GPU).
"""
import importlib.machinery
import importlib.util
import os

import torch  # noqa: F401  (the extensions resolve libc10 / libtorch from the loaded torch)

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, '_ref')
NAMES = ('rwref_upfirdn2d', 'rwref_fused_bias_act')

_MODS = {}


def path(name):
    return os.path.join(REF_DIR, name + '.so')


def _import(name):
    mod = _MODS.get(name)
    if mod is None:
        p = path(name)
        if not os.path.exists(p):
            raise ImportError('%s is not built: run oracle/build_ref_ops.py (build() does)' % p)
        loader = importlib.machinery.ExtensionFileLoader(name, p)
        spec = importlib.util.spec_from_file_location(name, p, loader=loader)
        mod = importlib.util.module_from_spec(spec)
        loader.exec_module(mod)
        _MODS[name] = mod
    return mod


def load():
    """(upfirdn2d_op, fused): the reference's modules of the same names."""
    return _import('rwref_upfirdn2d'), _import('rwref_fused_bias_act')
