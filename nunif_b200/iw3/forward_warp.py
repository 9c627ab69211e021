"""Mirror of iw3/forward_warp.py:246-256 (apply_divergence_forward_warp)."""
import torch
from .. import _lib
from ._common import VIEWS, COMPOSE_NONE, prep


def apply_divergence_forward_warp(c, depth, divergence, convergence, method=None,
                                  synthetic_view="both", return_mask=False, inconsistent_shift=False,
                                  width_base=True, compose=COMPOSE_NONE):
    """Depth-ordered bilinear forward warp (+ hole fill when method == "forward_fill").

    Row-parallel sm_90a kernel (csrc/warp_forward.cu); semantics follow
    depth_order_bilinear_forward_warp (forward_warp.py:140-243) including the
    100-iteration caps.  ``inconsistent_shift=True`` (a debugging variant of the
    reference, forward_warp.py:34-37) is not on the hot path and is rejected.
    """
    assert synthetic_view in {"both", "right", "left"}      # forward_warp.py:145
    if inconsistent_shift:
        raise NotImplementedError("inconsistent_shift=True is not supported by the H100 forward warp")
    c = prep(c, "c")
    depth = prep(depth, "depth")
    B, _, H, W = c.shape
    _, _, h, w = depth.shape
    fill = 1 if method == "forward_fill" else 0
    dev = c.device
    if compose == COMPOSE_NONE:
        left, right = torch.empty_like(c), torch.empty_like(c)
    else:
        left, right = torch.empty((B, 3, H, 2 * W), device=dev, dtype=torch.float32), None
    lm = rm = None
    if return_mask:
        lm = torch.zeros((B, 1, H, W), device=dev, dtype=torch.float32)
        rm = torch.zeros((B, 1, H, W), device=dev, dtype=torch.float32)
    ws_bytes = _lib.lib().nb200_forward_warp_workspace(B, H, W, h, w)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev) if ws_bytes else None
    with torch.cuda.device(dev):
        if torch.is_tensor(convergence):
            # per-frame convergence (auto-convergence): B,1,1,1, one value per frame
            conv = prep(convergence, "convergence").reshape(-1)
            assert conv.numel() == B, "convergence tensor must hold one value per frame"
            fn, cv = _lib.lib().nb200_forward_warp_conv, _lib.ptr(conv)
        else:
            fn, cv = _lib.lib().nb200_forward_warp, float(convergence)
        _lib.check(fn(
            _lib.ptr(c), _lib.ptr(depth), B, H, W, h, w, float(divergence), cv, fill,
            VIEWS[synthetic_view], 1 if width_base else 0, compose, _lib.ptr(left), _lib.ptr(right),
            _lib.ptr(lm if synthetic_view != "right" else None), _lib.ptr(rm if synthetic_view != "left" else None),
            _lib.ptr(ws), _lib.stream_ptr(dev)))
    if compose != COMPOSE_NONE:
        return left
    if return_mask:
        # forward_warp.py:229,243: the non-synthesised eye has no mask
        return left, right, (lm if synthetic_view != "right" else None), (rm if synthetic_view != "left" else None)
    return left, right
