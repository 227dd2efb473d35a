"""Build librw_b200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

The library is plain `extern "C"` (include/rewriting_b200.h); it is loaded with
ctypes by rewriting_b200._cabi.  Nothing here links against torch.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'librw_b200.so')
SOURCES = ['api.cu', 'conv_tc.cu', 'upconv_tc.cu', 'gram_tc.cu', 'simt.cu', 'bwd.cu', 'rewrite.cu',
           'insert_wide.cu', 'proggan.cu', 'vgg.cu', 'lpips.cu', 'gen_bwd.cu',
           'seg.cu', 'dissect.cu', 'faceparse.cu']
NVCC_FLAGS = [
    '-gencode', 'arch=compute_90a,code=sm_90a',
    '-lineinfo', '-O3', '-std=c++17',
    '-Xcompiler', '-fPIC',
    '-cudart', 'shared',
]


def find_nvcc():
    for cand in (os.environ.get('NVCC'), shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError('nvcc not found (needed to build librw_b200.so)')


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    deps.append(os.path.join(HERE, '..', 'include', 'rewriting_b200.h'))
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force=False, verbose=False):
    """Compile every .cu of the package into librw_b200.so. Returns the path."""
    if not force and not needs_build():
        return LIB
    nvcc = find_nvcc()
    objs = []
    objdir = os.path.join(HERE, 'build')
    os.makedirs(objdir, exist_ok=True)
    procs = []
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace('.cu', '.o'))
        cmd = [nvcc, '-c', os.path.join(CSRC, src), '-o', obj] + NVCC_FLAGS
        if verbose:
            cmd += ['-Xptxas', '-v']
            print(' '.join(cmd), flush=True)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE,
                                            stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, pr in procs:
        out, _ = pr.communicate()
        if pr.returncode != 0:
            failed = True
            sys.stderr.write('nvcc failed for %s:\n%s\n' % (src, out))
        elif verbose and out:
            print(out)
    if failed:
        raise RuntimeError('nvcc compilation failed')
    cmd = [nvcc, '-shared', '-o', LIB] + objs + ['-cudart', 'shared',
                                                  '-gencode', 'arch=compute_90a,code=sm_90a']
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError('link failed:\n' + r.stdout)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
