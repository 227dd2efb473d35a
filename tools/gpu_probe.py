"""GPU bring-up probe for the tensor-core kernels.

Each case runs in its own subprocess (a trapped kernel poisons the CUDA
context) with a timeout, and prints one JSON line.  This pins, on hardware, the
UMMA descriptor conventions the kernels rely on — in particular the MN-major
LBO/SBO assignment of the col-GEMM — before the full test-suite is trusted.

    python tools/gpu_probe.py            # all cases
    python tools/gpu_probe.py rowgemm    # one case, in-process
"""
import ctypes
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def _split(cabi, x):
    import torch
    hi = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    lo = torch.empty_like(hi)
    cabi.call('rw_split_rows', _ptr(x), x.numel(), _ptr(hi), _ptr(lo), None)
    return hi, lo


def case_rowgemm(rows, K, N):
    import torch
    from rewriting_b200 import _cabi
    torch.manual_seed(0)
    a = torch.randn(rows, K, device='cuda')
    w = torch.randn(N, K, device='cuda')
    ahi, alo = _split(_cabi, a)
    whi, wlo = _split(_cabi, w)
    out = torch.full((rows, N), float('nan'), device='cuda')
    _cabi.call('rw_debug_rowgemm', _ptr(ahi), _ptr(alo), _ptr(whi), _ptr(wlo), rows, K, N,
               _ptr(out), None)
    torch.cuda.synchronize()
    ref = a.double().cpu() @ w.double().cpu().t()
    err = (out.double().cpu() - ref).abs().max().item()
    # single-pass bf16 would give ~1e-1 here; the 3-term split ~1e-4
    return dict(case='rowgemm', rows=rows, K=K, N=N, max_abs_err=err,
                ref_absmax=ref.abs().max().item(), ok=bool(err < 2e-3))


def case_colgemm(rows, Cm, Cn, lbo, sbo):
    import torch
    from rewriting_b200 import _cabi
    torch.manual_seed(1)
    a = torch.randn(rows, Cm, device='cuda')
    b = torch.randn(rows, Cn, device='cuda')
    ahi, alo = _split(_cabi, a)
    bhi, blo = _split(_cabi, b)
    out = torch.full((Cm, Cn), float('nan'), device='cuda')
    lib = _cabi.load()
    nbytes = lib.rw_gram_workspace_bytes(Cm, Cn, rows, 1)
    ws = torch.empty(max(nbytes, 4) // 4 + 16, device='cuda')
    _cabi.call('rw_debug_colgemm', _ptr(ahi), _ptr(alo), _ptr(bhi), _ptr(blo), rows, Cm, Cn,
               lbo, sbo, _ptr(out), _ptr(ws), ws.numel() * 4, None)
    torch.cuda.synchronize()
    ref = a.double().cpu().t() @ b.double().cpu()
    err = (out.double().cpu() - ref).abs().max().item()
    return dict(case='colgemm', rows=rows, Cm=Cm, Cn=Cn, lbo=lbo, sbo=sbo, max_abs_err=err,
                ref_absmax=ref.abs().max().item(), ok=bool(err < 5e-3))


CASES = {
    'rowgemm_small': lambda: case_rowgemm(300, 128, 128),
    'rowgemm_big': lambda: case_rowgemm(5000, 512, 256),
    'colgemm_a': lambda: case_colgemm(1000, 128, 256, 8192, 1024),
    'colgemm_b': lambda: case_colgemm(1000, 128, 256, 1024, 8192),
    'colgemm_big': lambda: case_colgemm(20000, 512, 512, 0, 0),
}


def main():
    if len(sys.argv) > 1:
        name = sys.argv[1]
        try:
            res = CASES[name]()
        except Exception as e:  # noqa: BLE001
            res = dict(case=name, ok=False, error='%s: %s' % (type(e).__name__, e))
        res['name'] = name
        print('PROBE ' + json.dumps(res), flush=True)
        return
    results = []
    for name in CASES:
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), name],
                               capture_output=True, text=True, timeout=180)
            lines = [l for l in r.stdout.splitlines() if l.startswith('PROBE ')]
            if lines:
                results.append(json.loads(lines[-1][6:]))
            else:
                results.append(dict(name=name, ok=False, rc=r.returncode,
                                    stderr=r.stderr[-600:], stdout=r.stdout[-300:]))
        except subprocess.TimeoutExpired:
            results.append(dict(name=name, ok=False, error='timeout'))
        print(json.dumps(results[-1]), flush=True)
    os.makedirs('gpurun_out', exist_ok=True)
    with open('gpurun_out/probe.json', 'w') as f:
        json.dump(results, f, indent=1)


if __name__ == '__main__':
    main()
