"""TEST INFRASTRUCTURE ONLY — builds the reference's two CUDA ops for sm_90a into oracle/_ref/.

The reference (davidbau/rewriting) JIT-builds `utils/stylegan2/op/upfirdn2d.cpp` +
`upfirdn2d_kernel.cu` and `fused_bias_act.cpp` + `fused_bias_act_kernel.cu` with
`torch.utils.cpp_extension.load` on first import.  This recipe compiles the same, unmodified
sources in place from a reference checkout (nothing is copied, patched or vendored), under the
module names `rwref_upfirdn2d` and `rwref_fused_bias_act`, and keeps only the two `.so` files:

    oracle/_ref/rwref_upfirdn2d.so
    oracle/_ref/rwref_fused_bias_act.so

`oracle/_ref/` is git-ignored; the binaries stand in for the reference's GPU ops wherever the
checkout is absent (`oracle/ref_ops.py` loads them by path; tests/test_gpu_reference_ops.py
compares the package's kernels with them).  nvcc cross-compiles sm_90a without a GPU.

    python oracle/build_ref_ops.py [--force]

The checkout is found at $RW_REFERENCE_ROOT, else at `oracle.ref_shim.REFERENCE_ROOT`.  Without
it, existing binaries are kept as they are; without either, `build()` raises.
"""
import os
import shutil
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle.ref_shim import REFERENCE_ROOT    # noqa: E402

OUT_DIR = os.path.join(HERE, '_ref')

# module name -> (sources under utils/stylegan2/op of the reference)
OPS = {
    'rwref_upfirdn2d': ('upfirdn2d.cpp', 'upfirdn2d_kernel.cu'),
    'rwref_fused_bias_act': ('fused_bias_act.cpp', 'fused_bias_act_kernel.cu'),
}


def reference_root():
    return os.environ.get('RW_REFERENCE_ROOT') or REFERENCE_ROOT


def artefact(name):
    return os.path.join(OUT_DIR, name + '.so')


def _sources(root, name):
    return [os.path.join(root, 'utils', 'stylegan2', 'op', f) for f in OPS[name]]


def _stale(root, name):
    so = artefact(name)
    if not os.path.exists(so):
        return True
    t = os.path.getmtime(so)
    return any(os.path.getmtime(s) > t for s in _sources(root, name))


def build(force=False, verbose=False):
    """Compile both ops into oracle/_ref/ (when missing or older than their sources).  Returns
    {module name: .so path}."""
    root = reference_root()
    have_ref = all(os.path.exists(s) for n in OPS for s in _sources(root, n))
    have_so = all(os.path.exists(artefact(n)) for n in OPS)
    if not have_ref:
        if have_so:
            return {n: artefact(n) for n in OPS}
        raise RuntimeError(
            'the reference CUDA ops are neither built (%s) nor buildable: no reference checkout '
            'with utils/stylegan2/op/*.cu at %r (set RW_REFERENCE_ROOT)' % (OUT_DIR, root))
    todo = [n for n in OPS if force or _stale(root, n)]
    if not todo:
        return {n: artefact(n) for n in OPS}
    from torch.utils import cpp_extension
    os.makedirs(OUT_DIR, exist_ok=True)
    env_keep = {k: os.environ.get(k) for k in ('TORCH_CUDA_ARCH_LIST', 'MAX_JOBS')}
    os.environ['TORCH_CUDA_ARCH_LIST'] = '9.0a'          # sm_90a cubin, as the package's library
    os.environ.setdefault('MAX_JOBS', '4')
    try:
        for name in todo:
            with tempfile.TemporaryDirectory(prefix=name + '_') as bdir:
                so = cpp_extension.load(name, sources=_sources(root, name), build_directory=bdir,
                                        verbose=verbose, is_python_module=False)
                tmp = artefact(name) + '.tmp'
                shutil.copyfile(so, tmp)
                os.replace(tmp, artefact(name))
    finally:
        for k, v in env_keep.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    return {n: artefact(n) for n in OPS}


if __name__ == '__main__':
    for n, p in build(force='--force' in sys.argv, verbose='-v' in sys.argv).items():
        print(n, p)
