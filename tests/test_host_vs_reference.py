"""CPU: the device-independent host helpers of this package (zdataset, renormalize, the
rewriter's crop / paste geometry, zca_from_cov, nethook subsequence / InstrumentedModel,
FixedSubsetSampler) against what the reference computed on the same seeded cases
(oracle/host_cases.py; recorded by oracle/make_golden_host.py into tests/golden/host_helpers.npz)."""
import os
import types

import numpy as np
import torch

from oracle import host_cases

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'host_helpers.npz')


def test_host_helpers_equal_the_reference():
    from rewriting_b200.rewrite import ganrewrite
    from rewriting_b200.utils import nethook, renormalize, zdataset
    from rewriting_b200.utils.sampler import FixedSubsetSampler
    impl = types.SimpleNamespace(zdataset=zdataset, renormalize=renormalize, ganrewrite=ganrewrite,
                                 nethook=nethook, FixedSubsetSampler=FixedSubsetSampler)
    got = host_cases.fingerprints(host_cases.run(impl))
    want = dict(np.load(GOLD))
    assert sorted(got) == sorted(want)
    for name, w in want.items():
        g = got[name]
        assert g.shape == w.shape, name
        if w.dtype.kind in 'US':
            assert str(g) == str(w), name
        else:
            np.testing.assert_array_equal(g, w, err_msg=name)      # bit-identical on every check
    assert len(want) >= 19


def test_subsequence_shares_weights_and_instrumented_model_close_restores():
    """the two checks that concern this package's objects only"""
    from rewriting_b200.utils import nethook
    x = torch.randn(5, 6, generator=torch.Generator().manual_seed(0))
    for kw in host_cases.SUBSEQ_CASES:
        m = host_cases.toy()
        s = nethook.subsequence(m, share_weights=True, **kw)
        ids = {id(p) for p in m.parameters()}
        assert all(id(p) in ids for p in s.parameters())
    m = host_cases.toy()
    im = nethook.InstrumentedModel(m)
    im.retain_layers(['b.b1', ('d', 'out')])
    im.edit_layer('b.b1', ablation=0.5, replacement=torch.randn(5, 6))
    im(x)
    im.close()
    assert torch.equal(m(x).detach(), host_cases.toy()(x).detach())
