"""Host-side routing of linear_insert (no GPU): the Λ-mode twins of the fused insert kernels are
bound, and a key crop takes the same route as the projected edit except where the Λ state no
longer fits next to rw_insert_loop's crop in shared memory."""
import ctypes
import os

import numpy as np

from rewriting_b200 import _cabi
from rewriting_b200.rewrite import ganrewrite
from conftest import GOLD

route = ganrewrite.fused_insert_kernel


def _linear(B, Cin, Cout, h, w):
    return route(B, Cin, Cout, h, w, linear=True)


def test_new_symbols_are_exported():
    lib = _cabi.load()
    for name in ('rw_linear_insert_loop', 'rw_linear_insert_loop_wide'):
        assert name in _cabi.SIGNATURES
        assert getattr(lib, name) is not None
    # rw_linear_insert_args: size_t struct_size + 5 pointers
    assert ctypes.sizeof(_cabi.LinearInsertArgs) == 6 * 8
    # the projected edit's struct is unchanged
    assert [f for f, _ in _cabi.InsertArgs._fields_][-4:] == [
        'one_minus_beta1', 'one_minus_beta2', 'beta1_exact', 'beta2_exact']


SHAPES = [
    (1, 512, 512, 8, 9),      # config 4 (hat_on_horse_ears.json, layer 8)
    (1, 512, 512, 16, 16), (4, 512, 512, 20, 16), (1, 512, 256, 6, 5),
    (1, 512, 512, 32, 32), (1, 512, 512, 12, 24), (1, 512, 512, 10, 17),
    (1, 128, 128, 24, 40), (1, 128, 128, 32, 64), (2, 512, 512, 10, 20),
    (5, 512, 512, 8, 8), (1, 48, 48, 32, 32), (1, 1024, 512, 32, 32), (1, 64, 64, 32, 32),
    (1, 512, 512, 64, 64), (4, 512, 512, 40, 16), (1, 256, 256, 128, 128),
    (4, 512, 512, 64, 64), (1, 128, 128, 64, 64),
]


def test_linear_route_matches_the_projected_route():
    for f in ('config4_hat.npz', 'sg2_layer8.npz'):
        gold = np.load(os.path.join(GOLD, f))
        B, Cin, h, w = gold['goal_in_fmap'].shape
        assert _linear(B, Cin, gold['goal_out_fmap'].shape[1], h, w) == 'rw_linear_insert_loop'
    for shape in SHAPES:
        r, rl = route(*shape), _linear(*shape)
        assert (rl is None) == (r is None), shape
        if r is not None:
            assert rl == r.replace('rw_', 'rw_linear_', 1), shape
    assert route(1, 512, 512, 32, 32) == 'rw_insert_loop_wide'
    assert _linear(1, 512, 512, 32, 32) == 'rw_linear_insert_loop_wide'
    assert _linear(1, 512, 512, 8, 9) == 'rw_linear_insert_loop'


def test_lambda_state_moves_the_largest_small_crops_to_autograd():
    # a 16-column crop one row past the Λ-mode limit: it fits rw_insert_loop's 225 KB of shared
    # memory, but not together with the 13.5 KB of Λ state.  Crops that large are far past the
    # wide kernel's WIDE_MAX_WORK, so linear_insert runs them through autograd.
    small_limit = (225 * 1024 // 4 - 8 * 512 * 9 - 1440) // 8           # largest B*h*w at Cin 512
    lin_limit = (225 * 1024 // 4 - 8 * 512 * 9 - 1440 - 3 * 4 * 32 * 9) // 8
    assert lin_limit < small_limit
    h = lin_limit // 16 + 1
    assert h * 16 <= small_limit
    assert route(1, 512, 512, h, 16) == 'rw_insert_loop'
    assert _linear(1, 512, 512, h, 16) is None
    assert ganrewrite.wide_insert_work(1, 512, h, 16) > ganrewrite.WIDE_MAX_WORK
    assert _linear(1, 512, 512, lin_limit // 16, 16) == 'rw_linear_insert_loop'
