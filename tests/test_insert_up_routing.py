"""CPU: which loop an odd (upsampling) layer's edit runs on, for the shapes of the 256^2 generator
(ganrewrite.fused_insert_up_kernel, UP_MAX_WORK from tools/bench_insert_up.py, DESIGN.md §6)."""
import pytest
import torch

from rewriting_b200.rewrite import ganrewrite as g

UP, LINEAR_UP = 'rw_insert_loop_up', 'rw_linear_insert_loop_up'

# (layer, Cin, Cout) of the odd layers of the 256^2 generator and their key maps
ODD = {3: (512, 512, 4), 5: (512, 512, 8), 7: (512, 512, 16), 9: (512, 512, 32),
       11: (512, 256, 64), 13: (256, 128, 128)}
# the hat request's tight crop (7 x 9 at layer 9) scaled to each odd layer, as benchmarked
HAT = {3: (1, 2), 5: (2, 3), 7: (4, 5), 9: (7, 9), 11: (14, 18), 13: (28, 36)}


@pytest.mark.parametrize('layer', sorted(ODD))
def test_tight_crops_at_every_odd_layer_take_the_up_kernel(layer):
    cin, cout, _ = ODD[layer]
    h, w = HAT[layer]
    assert g.fused_insert_up_kernel(1, cin, cout, h, w) == UP
    assert g.fused_insert_up_kernel(1, cin, cout, h, w, linear=True) == LINEAR_UP


def test_whole_maps():
    assert g.fused_insert_up_kernel(1, 512, 512, 16, 16) == UP            # layer 7
    assert g.fused_insert_up_kernel(1, 512, 512, 32, 32) == UP            # layer 9, at the limit
    assert g.up_insert_work(1, 512, 32, 32) == g.UP_MAX_WORK
    assert g.fused_insert_up_kernel(1, 512, 256, 64, 64) is None          # layer 11
    assert g.fused_insert_up_kernel(1, 256, 128, 128, 128) is None        # layer 13


def test_keys_past_the_measured_limit_stay_on_autograd():
    assert g.fused_insert_up_kernel(1, 256, 128, 48, 64) is None          # measured slower
    assert g.up_insert_work(1, 256, 48, 64) > g.UP_MAX_WORK
    assert g.fused_insert_up_kernel(1, 512, 512, 33, 32) is None
    assert g.fused_insert_up_kernel(2, 512, 512, 32, 32) is None
    assert g.fused_insert_up_kernel(2, 512, 512, 16, 16) == UP


def test_batch_channels_and_rank_limits():
    assert g.fused_insert_up_kernel(4, 512, 512, 7, 9) == UP
    assert g.fused_insert_up_kernel(5, 512, 512, 7, 9) is None
    assert g.fused_insert_up_kernel(1, 64, 64, 7, 9) is None              # layers 15+: Cin < 128
    assert g.fused_insert_up_kernel(1, 528, 512, 7, 9) is None
    # rank > 32 is refused before the target model is looked at
    assert g.SeqStyleGanRewriter._fused_up_plan(None, {}, None, torch.zeros(33, 512)) is None
    assert g.SeqStyleGanRewriter._fused_up_plan(None, {}, None, None) is None


def test_even_layer_routing_is_unchanged():
    assert g.fused_insert_kernel(1, 512, 512, 8, 9) == 'rw_insert_loop'
    assert g.WIDE_MAX_WORK == 512 * 32 * 32
