"""CPU: the row criterion of `oracle/trajectory_check.py` on the float32 oracle against itself.

Two float32 runs of `sg2_oracle.insert_loop` from keys k and k·(1 + 2⁻²¹), and the float64 shadow's
own W against the float32 oracle, must pass `check_rows` with the shadow recorded on k; wrong
oracle variants (lr × 1.001 in one row, the final projection onto span(d) dropped) must fail it.
The rank-32 `low_rank_gradient` case of seed 12 (the one `tests/test_gpu_persistent_paths.py`
once skipped) is where a row does part: one output of row 102 sits at the leaky-ReLU kink at
step 2, and the float32 and float64 loops end 0.11 apart on that row."""
import pytest
import torch

from oracle import sg2_oracle as orc
from oracle import trajectory_check as tc

CIN, NITER, LR = 128, 10, 0.05


def _case(cout, B, h, w, rank, seed):
    """The random case of test_gpu_persistent_paths._insert_case (styled target, goal + 1)."""
    g = torch.Generator().manual_seed(seed)
    style = torch.randn(B, CIN, generator=g) * 0.5 + 1
    k = style[:, :, None, None] * torch.randn(B, CIN, h, w, generator=g)
    W0 = torch.randn(cout, CIN, 3, 3, generator=g)
    bias = torch.randn(cout, generator=g)
    g = torch.Generator().manual_seed(seed)
    q, _ = torch.linalg.qr(torch.randn(CIN, rank, generator=g))
    d = q.t().contiguous()
    with torch.no_grad():
        target = orc.target_forward(k, style, W0[None], 0.37, bias) + 1.0
    return dict(k=k, style=style, W0=W0, bias=bias, d=d, target=target, lrg=rank > 2)


def _oracle(c, k=None, lr=LR, low_rank_insert=True):
    return orc.insert_loop(c['W0'][None], c['k'] if k is None else k, c['style'], c['target'],
                           0.37, c['bias'], c['d'], NITER, piter=10, lr=lr,
                           low_rank_gradient=c['lrg'], low_rank_insert=low_rank_insert)[0]


def _shadow(c):
    B, _, h, w = c['k'].shape
    return tc.shadow('styled', c['W0'], c['k'], c['style'], c['target'], c['d'], NITER, LR,
                     low_rank_gradient=c['lrg'], noise=orc.noise_table(B, h * w), noise_w=0.37,
                     bias=c['bias'], device='cpu')


@pytest.fixture(scope='module')
def cases():
    out = {}
    for name, args in (('rank32_seed12', (534, 1, 5, 6, 32, 12)),
                       ('rank2', (64, 1, 8, 10, 2, 3))):
        c = _case(*args)
        c['W'] = _oracle(c)
        c['rec'] = _shadow(c)
        out[name] = c
    return out


@pytest.mark.parametrize('name', ['rank32_seed12', 'rank2'])
def test_oracle_against_itself_passes(cases, name):
    c = cases[name]
    rec = c['rec']
    Wp = _oracle(c, k=c['k'] * (1 + 2 ** -21))
    tc.check_rows(Wp, c['W'], rec, what='keys (1 + 2^-21)')
    parted = tc.check_rows(rec.W, c['W'], rec, what='float64 shadow')
    if name == 'rank32_seed12':
        # not vacuous: the float64 and float32 loops part on one row, at a certified decision
        assert list(parted) == [102], parted
        err, (step, kind, margin, _), _ = parted[102]
        assert err > 0.05 and kind == 'kink' and step == 2 and margin < tc.TAU / 8, parted


def test_criterion_refuses_wrong_oracles(cases):
    c = cases['rank2']
    rec = c['rec']
    cert = rec.certified()
    assert not cert.all()
    o = int((~cert).nonzero()[0, 0])
    W = c['W'].clone()
    W[o] = _oracle(c, lr=LR * 1.001)[o]                # lr x 1.001 in one uncertified row
    with pytest.raises(AssertionError, match='without a decision within tau'):
        tc.check_rows(W, c['W'], rec)
    W = _oracle(c, low_rank_insert=False)               # the projection onto span(d) dropped
    with pytest.raises(AssertionError, match='without a decision within tau'):
        tc.check_rows(W, c['W'], rec)
    W = c['W'].clone()
    W[o, 0, 0, 0] = float('nan')
    with pytest.raises(AssertionError):
        tc.check_rows(W, c['W'], rec)


def test_ill_conditioned_case_excuses_nothing(cases):
    """With more certified rows than the cap, a certified row is held to 1e-4 like any other."""
    c = cases['rank2']
    rec = tc.shadow('styled', c['W0'], c['k'], c['style'], c['target'], c['d'], NITER, LR,
                    noise=orc.noise_table(1, 80), noise_w=0.37, bias=c['bias'], tau=1.0,
                    device='cpu')
    assert rec.certified().all()
    W = c['W'].clone()
    W[5] = _oracle(c, lr=LR * 1.001)[5]
    with pytest.raises(AssertionError, match='none excused'):
        tc.check_rows(W, c['W'], rec)
