"""Mirror of iw3/backward_warp.py:96-121 (apply_divergence_grid_sample)."""
import torch
from .. import _lib
from ._common import VIEWS, COMPOSE_NONE, prep


def apply_divergence_grid_sample(c, depth, divergence, convergence, synthetic_view="both", compose=COMPOSE_NONE):
    """c: B,3,H,W float; depth: B,1,h,w float (any resolution) -> (left_eye, right_eye).

    One fused sm_90a kernel (csrc/warp_backward.cu) replaces make_grid +
    F.interpolate(grid) + 2x F.grid_sample + clamp.  ``compose`` (extension) selects a
    fused SBS (returns B,3,H,2W) or dubois-anaglyph (B,3,H,W) epilogue instead.  ``convergence`` is a float or a B,1,1,1
    tensor (one value per frame, as the auto-convergence estimator returns it).
    """
    assert synthetic_view in {"both", "right", "left"}      # backward_warp.py:97
    c = prep(c, "c")
    depth = prep(depth, "depth")
    B, _, H, W = c.shape
    _, _, h, w = depth.shape
    if compose == COMPOSE_NONE:
        left, right = torch.empty_like(c), torch.empty_like(c)
    else:
        left = torch.empty((B, 3, H, 2 * W if compose == 1 else W), device=c.device, dtype=torch.float32)
        right = None
    with torch.cuda.device(c.device):
        if torch.is_tensor(convergence):
            # per-frame convergence (auto-convergence): B,1,1,1, one value per frame
            conv = prep(convergence, "convergence").reshape(-1)
            assert conv.numel() == B, "convergence tensor must hold one value per frame"
            _lib.check(_lib.lib().nb200_backward_warp_conv(
                _lib.ptr(c), _lib.ptr(depth), B, H, W, h, w, float(divergence), _lib.ptr(conv),
                VIEWS[synthetic_view], compose, _lib.ptr(left), _lib.ptr(right), _lib.stream_ptr(c.device)))
        else:
            _lib.check(_lib.lib().nb200_backward_warp(
                _lib.ptr(c), _lib.ptr(depth), B, H, W, h, w, float(divergence), float(convergence),
                VIEWS[synthetic_view], compose, _lib.ptr(left), _lib.ptr(right), _lib.stream_ptr(c.device)))
    return (left, right) if compose == COMPOSE_NONE else left
