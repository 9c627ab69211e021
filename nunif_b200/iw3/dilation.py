"""Mirror of iw3/dilation.py:5-27,67-98,115-152."""
import torch
from .. import _lib
from ._common import prep


def edge_dilation_parse(edge_dilation):
    """dilation.py:5-22 (same accepted types and ValueError)."""
    if isinstance(edge_dilation, (list, tuple)):
        if len(edge_dilation) == 0:
            x = y = 0
        elif len(edge_dilation) == 1:
            x = y = edge_dilation[0]
        else:
            x, y = edge_dilation[0], edge_dilation[1]
    elif isinstance(edge_dilation, int):
        x = y = edge_dilation
    elif edge_dilation is None:
        x = y = 0
    else:
        raise ValueError(f"Unsupported edge_dilation type {type(edge_dilation)}. "
                         "Supported types: int, list, tuple.")
    return x, y


def edge_dilation_is_enabled(edge_dilation):
    """dilation.py:25-27."""
    x, y = edge_dilation_parse(edge_dilation)
    return x != 0 or y != 0


@torch.inference_mode()
def dilate_edge(x, n):
    """x: B,1,h,w float CUDA tensor; n: int or [x_iter, y_iter] -> new tensor."""
    x_iter, y_iter = edge_dilation_parse(n)
    x = prep(x, "x")
    assert x.ndim == 4                                       # dilation.py:102
    B, _, h, w = x.shape
    out = torch.empty_like(x)
    lib = _lib.lib()
    ws = torch.empty(lib.nb200_dilate_edge_workspace(B, h, w), dtype=torch.uint8, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(lib.nb200_dilate_edge(_lib.ptr(x), B, h, w, int(x_iter), int(y_iter), _lib.ptr(out),
                                         _lib.ptr(ws), _lib.stream_ptr(x.device)))
    return out


def _mask_op(mask, **kw):
    from .forward_inpaint import inpaint_mask
    return inpaint_mask(mask, **kw)


def mask_closing(mask, kernel_size=3, n_iter=2):
    """dilation.py:145-152 (3x3, 2 iterations): closing of a B,1,h,w mask, OR the input, as float."""
    assert kernel_size == 3 and n_iter == 2, "the engine implements mask_closing's defaults"
    return _mask_op(mask.float(), binarize=False, closing=True)


def dilate_outer(mask, n_iter, base_width=None):
    """dilation.py:67-82: runs grow n pixels to the right, n = max(round(W / base_width * n_iter), 1)."""
    if n_iter <= 0:
        return mask
    return _mask_op(mask.float(), binarize=False, closing=False, outer_dilation=n_iter, base_width=base_width).to(mask.dtype)


def dilate_inner(mask, n_iter, base_width=None):
    """dilation.py:85-98: runs grow n pixels to the left."""
    if n_iter <= 0:
        return mask
    return _mask_op(mask.float(), binarize=False, closing=False, inner_dilation=n_iter, base_width=base_width).to(mask.dtype)
