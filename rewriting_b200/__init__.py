"""rewriting_b200 — Hopper-native (H100) hot path of davidbau/rewriting.

Layout: `csrc/` (CUDA kernels + C-ABI, built into librw_b200.so), `ops` (torch-facing
wrappers / autograd), `utils/` and `rewrite/` (host-side mirror of the reference's operator,
module, statistics and rewriter APIs), `dist` (z-batch sharding).

`install_aliases()` registers the package's `utils` and `rewrite` sub-packages under the
reference's top-level import names so notebooks written against the reference
(`from utils.stylegan2 import load_seq_stylegan`, `from rewrite import ganrewrite`) run
unchanged.
"""
import sys

__version__ = '0.1.0'


def install_aliases(reference_root=None):
    """Register `utils` / `rewrite` as the reference's top-level package names.

    With `reference_root` (or $REWRITING_REFERENCE_ROOT) pointing at a checkout of
    davidbau/rewriting, modules this package does not provide — the notebook UI
    (`rewrite/rewriteapp.py`, `utils/labwidget.py`, `paintwidget.py`, `show.py`) — are looked up
    in the checkout AFTER this package's own directories, so `from rewrite import ganrewrite,
    rewriteapp` gives this package's rewriter and the reference's device-independent UI."""
    import os
    from . import utils as _utils, rewrite as _rewrite
    from .utils import (imgviz, nethook, pbar, quickdissect, renormalize, runningstats, segmenter,
                        tally, upsample, zdataset, stylegan2)
    from .rewrite import ganrewrite
    sys.modules.setdefault('utils', _utils)
    sys.modules.setdefault('rewrite', _rewrite)
    for name, mod in [('imgviz', imgviz), ('nethook', nethook), ('pbar', pbar),
                      ('quickdissect', quickdissect), ('renormalize', renormalize),
                      ('runningstats', runningstats), ('segmenter', segmenter), ('tally', tally),
                      ('upsample', upsample), ('zdataset', zdataset),
                      ('stylegan2', stylegan2)]:
        sys.modules.setdefault('utils.' + name, mod)
    sys.modules.setdefault('rewrite.ganrewrite', ganrewrite)
    reference_root = reference_root or os.environ.get('REWRITING_REFERENCE_ROOT')
    if reference_root:
        for pkg, sub in ((_utils, 'utils'), (_rewrite, 'rewrite')):
            extra = os.path.join(reference_root, sub)
            if os.path.isdir(extra) and extra not in pkg.__path__:
                pkg.__path__.append(extra)
