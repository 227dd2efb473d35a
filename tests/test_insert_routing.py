"""Host-side routing of the insert loop (no GPU): which fused kernel, if any, a key crop takes."""
import os

import numpy as np

from rewriting_b200.rewrite import ganrewrite
from conftest import GOLD

route = ganrewrite.fused_insert_kernel


def test_small_crops_keep_the_shared_memory_kernel():
    # the crops of the config-4 edit (hat_on_horse_ears.json at layer 8) and of the layer-8 goldens
    for f in ('config4_hat.npz', 'sg2_layer8.npz'):
        gold = np.load(os.path.join(GOLD, f))
        B, Cin, h, w = gold['goal_in_fmap'].shape
        assert w <= 16
        assert route(B, Cin, gold['goal_out_fmap'].shape[1], h, w) == 'rw_insert_loop'
    assert route(1, 512, 512, 16, 16) == 'rw_insert_loop'
    assert route(4, 512, 512, 20, 16) == 'rw_insert_loop'        # 1280 pixels, 225 KB of smem
    assert route(1, 512, 256, 6, 5) == 'rw_insert_loop'          # ProgGAN layer 6 golden


def test_wide_keys_take_the_wide_kernel():
    assert route(1, 512, 512, 32, 32) == 'rw_insert_loop_wide'   # whole layer-8 map
    assert route(1, 512, 512, 12, 24) == 'rw_insert_loop_wide'
    assert route(1, 512, 512, 10, 17) == 'rw_insert_loop_wide'
    assert route(1, 128, 128, 24, 40) == 'rw_insert_loop_wide'
    assert route(1, 128, 128, 32, 64) == 'rw_insert_loop_wide'   # layer-14 crop of DESIGN.md §6
    assert route(2, 512, 512, 10, 20) == 'rw_insert_loop_wide'


def test_keys_outside_both_kernels_stay_on_autograd():
    assert route(5, 512, 512, 8, 8) is None                      # B > 4
    assert route(1, 48, 48, 32, 32) is None                      # Cin % 32 != 0
    assert route(1, 1024, 512, 32, 32) is None                   # weight rows exceed smem
    assert route(1, 64, 64, 32, 32) is None                      # below the wide kernel's Cin
    # past the measured crossover the tensor-core autograd loop is faster
    assert route(1, 512, 512, 64, 64) is None                    # whole layer-10 map
    assert route(4, 512, 512, 40, 16) is None                    # t and g overflow the smem
    assert route(1, 256, 256, 128, 128) is None                  # whole layer-12 map
    assert route(4, 512, 512, 64, 64) is None
    assert ganrewrite.WIDE_MAX_WORK < 4 * 512 * 64 * 64
    # below 256 input channels the weight gradient leaves warps idle: counted as 256
    assert route(1, 128, 128, 64, 64) is None
    assert ganrewrite.wide_insert_work(1, 128, 32, 64) == ganrewrite.wide_insert_work(1, 256, 32, 64)
