"""Records the reference's outputs on the seeded host-helper cases of oracle/host_cases.py into
tests/golden/host_helpers.npz (tests/test_host_vs_reference.py compares this package with them).
Needs a checkout of the reference (see oracle/ref_shim.py)."""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import host_cases                                # noqa: E402
from oracle.ref_shim import load_reference                   # noqa: E402

if __name__ == '__main__':
    ref = load_reference()
    from utils.sampler import FixedSubsetSampler              # the reference's, after the shim
    impl = types.SimpleNamespace(zdataset=ref.zdataset, renormalize=ref.renormalize,
                                 ganrewrite=ref.ganrewrite, nethook=ref.nethook,
                                 FixedSubsetSampler=FixedSubsetSampler)
    out = host_cases.fingerprints(host_cases.run(impl))
    np.savez_compressed(os.path.join(ROOT, 'tests', 'golden', 'host_helpers.npz'), **out)
    print('%d cases' % len(out))
