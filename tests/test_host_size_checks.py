"""CPU: the ProgGAN pixel-norm / nearest-2x forwards and the noise injection refuse every size < 1
on its own, before anything is launched.  A check on the product of the sizes alone lets sign-paired
negatives through (B = -2, H = -4 gives B·H·W > 0), and the kernels then index below their
buffers.  The refusal needs no device: the pointers here are never dereferenced."""
import ctypes

import pytest

BAD_ARG = -1
P = ctypes.c_void_p(1 << 20)        # non-null and 8-byte aligned; never read or written


def _status(name, *args):
    from rewriting_b200 import _cabi
    return getattr(_cabi.load(), name)(*args)


PAIRED = [  # sizes whose product is positive while two of them are negative
    ('rw_pixel_norm_nchw', (P, -2, 8, -4, 4, 0, P, None)),
    ('rw_pixel_norm_nchw', (P, -2, 8, 4, -4, 1, P, None)),
    ('rw_pixel_norm_nchw', (P, 2, 8, -4, -4, 0, P, None)),
    ('rw_pixel_norm_nchw', (P, 2, -8, -4, 4, 0, P, None)),
    ('rw_nearest_up2', (P, -16, -4, 4, P, None)),
    ('rw_nearest_up2', (P, 16, -4, -4, P, None)),
    ('rw_nearest_up2', (P, -16, 4, -4, P, None)),
    ('rw_add_noise', (P, P, 16, P, -2, -8, 16, P, None)),
    ('rw_add_noise', (P, P, 16, P, 2, -8, -16, P, None)),
    ('rw_add_noise', (P, P, 16, P, -2, 8, -16, P, None)),
]


@pytest.mark.parametrize('name,args', PAIRED, ids=['%s-%d' % (n, i) for i, (n, _) in enumerate(PAIRED)])
def test_sign_paired_negative_sizes_are_refused(name, args):
    assert _status(name, *args) == BAD_ARG
