"""Mirror of iw3's learned stereo warps: the `sbs.row_flow_v3` (iw3/models/row_flow_v3.py) and `sbs.row_flow_v2`
(iw3/models/row_flow_v2.py) models in delta_output mode, and their drivers apply_divergence_nn_LR / apply_divergence_nn_delta /
apply_divergence_nn_symmetric (iw3/backward_warp.py:124-232,344-379), loaded by load_row_flow_model
(iw3/stereo_model_factory.py:98-113).

The v3 delta network runs as wgmma GEMMs + the kernels in csrc/rowflow_kernels.cu, the v2 network is one fused kernel
(csrc/rowflow_v2.cu); the warp is the fused grid-sample kernel (csrc/warp_backward.cu, nb200_backward_warp_delta and its
_f16 / _sym forms).  steps > 1 (iterative re-warping of the depth, :205-226) and preserve_screen_border (:33-47) run the same
kernels once per step.
"""
import os
import torch
from .. import _lib
from . import _common
from .base_depth_model import HUB_MODEL_DIR

class MLBW:
    """Packed `sbs.mlbw` (iw3/models/mlbw.py; methods mlbw_l2 / mlbw_l4 and their `s` variants, and mask_mlbw_l2 with
    hole_mask=True) in delta_output mode: ``model(x)`` with x = B,3,h,w returns ``(delta B,L,h,w, layer_weight B,L,h,w)``, and for
    a hole_mask model also the hole logits B,1,h,w (_forward_delta_only, :232-240, without the y interleave)."""
    name = "sbs.mlbw"
    symmetric = False
    delta_output = True

    def __init__(self, state_dict, device="cuda:0"):
        self.device = _lib.cuda_device(device)
        self._h = _lib.Model("MLBW", state_dict, self.device)
        self.num_layers = int(_lib.lib().nb200_mlbw_num_layers(self._h))
        self.hole_mask = bool(_lib.lib().nb200_mlbw_has_hole_mask(self._h))

    def __call__(self, x):
        _lib.require_cuda(x, "x")
        assert x.ndim == 4 and x.shape[1] == 3
        B, _, h, w = x.shape
        xf = x.float().contiguous()
        delta = torch.empty((B, self.num_layers, h, w), dtype=torch.float32, device=x.device)
        lw = torch.empty_like(delta)
        if self.hole_mask:
            logits = torch.empty((B, 1, h, w), dtype=torch.float32, device=x.device)
            with torch.cuda.device(x.device):
                _lib.check(_lib.lib().nb200_mlbw_delta_hole(self._h, _lib.ptr(xf), B, h, w, _lib.ptr(delta), _lib.ptr(lw), _lib.ptr(logits),
                                                            _lib.stream_ptr(x.device)))
            return delta, lw, logits
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().nb200_mlbw_delta(self._h, _lib.ptr(xf), B, h, w, _lib.ptr(delta), _lib.ptr(lw), _lib.stream_ptr(x.device)))
        return delta, lw


class RowFlowV3:
    """Packed `sbs.row_flow_v3`; ``model(x)`` with x = B,3,h,w (depth, divergence feature, convergence feature) returns the
    delta B,2,h,w (x component, zero y component) like the reference with ``delta_output=True`` (row_flow_v3.py:111-116).
    ``symmetric=True`` is the row_flow_v3_sym checkpoint: apply_divergence_nn_LR then warps both eyes from one delta."""
    name = "sbs.row_flow_v3"
    symmetric = False
    delta_output = True
    _kind, _entry = "ROW_FLOW_V3", "nb200_row_flow_delta"

    def __init__(self, state_dict, device="cuda:0", symmetric=False):
        self.device = _lib.cuda_device(device)
        self.symmetric = bool(symmetric)
        self._h = _lib.Model(self._kind, state_dict, self.device)

    def delta_x(self, x):
        _lib.require_cuda(x, "x")
        assert x.ndim == 4 and x.shape[1] == 3
        B, _, h, w = x.shape
        xf = x.float().contiguous()
        out = torch.empty((B, 1, h, w), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check(getattr(_lib.lib(), self._entry)(self._h, _lib.ptr(xf), B, h, w, _lib.ptr(out), _lib.stream_ptr(x.device)))
        return out

    def __call__(self, x):
        d = self.delta_x(x)
        return torch.cat([d, torch.zeros_like(d)], dim=1)


class RowFlowV2(RowFlowV3):
    """Packed `sbs.row_flow_v2` (row_flow_v2.py:10-86), the same surface as RowFlowV3.  Its delta is the fp16 autocast output
    (_forward_delta_only does not cast it to fp32, :80-86), returned as fp32 holding fp16 values; ``delta_f16`` tells the drivers
    that the reference's ``delta * delta_scale`` is then an fp16 product."""
    name = "sbs.row_flow_v2"
    delta_f16 = True
    _kind, _entry = "ROW_FLOW_V2", "nb200_row_flow_v2_delta"

    def __init__(self, state_dict, device="cuda:0"):
        super().__init__(state_dict, device)


def make_divergence_feature_value(divergence, convergence, image_width):
    """iw3/backward_warp.py:8-15."""
    divergence_pix = divergence * 0.5 * 0.01 * image_width
    return divergence_pix / 32.0, (-divergence_pix * convergence) / 32.0


def _warp_delta(c, delta, delta_scale, f16=False):
    """backward_warp(c, grid, delta, delta_scale); ``f16``: delta holds fp16 values and the product is an fp16 op."""
    B, _, H, W = c.shape
    h, w = delta.shape[-2:]
    out = torch.empty_like(c)
    fn = _lib.lib().nb200_backward_warp_delta_f16 if f16 else _lib.lib().nb200_backward_warp_delta
    with torch.cuda.device(c.device):
        _lib.check(fn(_lib.ptr(c), _lib.ptr(delta), B, H, W, h, w, float(delta_scale), _lib.ptr(out), _lib.stream_ptr(c.device)))
    return out


def make_input(depth, divergence, convergence, preserve_screen_border=False, image_width=None):
    """make_input_tensor(None, depth, ...) for a batch (iw3/backward_warp.py:18-63): depth, divergence feature, convergence
    feature; with preserve_screen_border the two features fade linearly to zero over `border_pix` columns at both edges.
    ``image_width`` is the base width of the feature values: max(H, W) in apply_divergence_nn_delta (the default), W in
    apply_divergence_nn_symmetric.  ``convergence`` is a float or a B,1,1,1 tensor (one value per frame)."""
    B, _, H, W = depth.shape
    base = max(H, W) if image_width is None else image_width
    dv, cv = make_divergence_feature_value(divergence, convergence, base)
    df = torch.full_like(depth, dv)
    if torch.is_tensor(cv):
        # a B,1,1,1 convergence tensor: (-divergence_pix * c) / 32 per frame in fp32, expanded over the map (:24-25)
        cf = cv.to(device=depth.device, dtype=depth.dtype).reshape(B, 1, 1, 1).expand_as(depth).clone()
    else:
        cf = torch.full_like(depth, cv)
    if preserve_screen_border:
        bp = round(divergence * 0.75 * 0.01 * base * (W / base))                               # :36
        if bp > 0:
            wl = torch.linspace(0.0, 1.0, bp, device=depth.device)
            wr = torch.linspace(1.0, 0.0, bp, device=depth.device)
            for f in (df, cf):
                f[..., :bp] = wl * f[..., :bp]
                f[..., -bp:] = wr * f[..., -bp:]
    return torch.cat([depth, df, cf], dim=1)


def apply_divergence_nn_delta(model, c, depth, divergence, convergence, steps, shift, preserve_screen_border=False, enable_amp=True):
    """iw3/backward_warp.py:185-232."""
    steps = 1 if steps is None else int(steps)
    assert steps >= 1
    if not enable_amp:
        raise NotImplementedError("nunif_b200 implements the reference's CUDA autocast (fp16) forward only")
    _lib.require_cuda(c, "c")
    _lib.require_cuda(depth, "depth")
    c, depth = c.float().contiguous(), depth.float().contiguous()
    if shift > 0:
        c, depth = torch.flip(c, (3,)), torch.flip(depth, (3,))
    B, _, H, W = depth.shape
    delta_scale = 1.0 / (W // 2 - 1)                                                           # :201
    f16 = getattr(model, "delta_f16", False)
    depth_warp, deltas = depth, []
    for j in range(steps):
        deltas.append(model.delta_x(make_input(depth_warp, divergence / steps, convergence, preserve_screen_border)))
        if j + 1 < steps:
            # backward_warp(depth_warp, grid, delta, delta_scale) :220-221 (the warp kernel takes 3-channel frames)
            depth_warp = _warp_delta(depth_warp.expand(-1, 3, -1, -1).contiguous(), deltas[-1], delta_scale, f16)[:, :1].contiguous()
    z = c
    for delta in deltas:                                                                       # :223-226
        z = _warp_delta(z, delta, delta_scale, f16)
    return torch.flip(z, (3,)) if shift > 0 else z


MASK_MLBW_THRESHOLD = 0.15   # iw3/mlbw_inpaint.py:18, and the hole fill of backward_warp.py:334-338


def postprocess_hole_mask(mask_logits, target_size, threshold, inner_dilation=0, outer_dilation=0, mirror=False):
    """iw3/backward_warp.py:382-393: closing of the hole logits (3x3, one iteration), the align-corners bilinear resize to
    target_size, sigmoid > threshold, dilate_inner and dilate_outer with base_width = the logits' width -> a B,1,H,W float mask of
    0 / 1.  ``mirror=True`` gives what forward_left computes on the flipped logits (iw3/mlbw_inpaint.py:28-34), flipped back.

    Two launches: nb200_hole_mask (closing, resize, threshold), then the row-run dilation of nb200_inpaint_mask.  The reference
    dilates inner before outer; OR-shifts to the left and to the right commute (an OR over [x - outer, x + inner] of the row, zero
    outside it, either way), so the one-pass run dilation gives the same mask."""
    from .forward_inpaint import inpaint_mask
    mask_logits = _common.prep(mask_logits, "mask_logits")
    assert mask_logits.ndim == 4 and mask_logits.shape[1] == 1
    B, _, h, w = mask_logits.shape
    H, W = (int(v) for v in target_size)
    mask = torch.empty((B, 1, H, W), dtype=torch.float32, device=mask_logits.device)
    with torch.cuda.device(mask_logits.device):
        _lib.check(_lib.lib().nb200_hole_mask(_lib.ptr(mask_logits), B, h, w, H, W, float(threshold), int(bool(mirror)), _lib.ptr(mask),
                                              _lib.stream_ptr(mask_logits.device)))
    if inner_dilation <= 0 and outer_dilation <= 0:
        return mask
    return inpaint_mask(mask, inner_dilation=inner_dilation, outer_dilation=outer_dilation, base_width=w, mirror=mirror,
                        binarize=True, closing=False)


def apply_divergence_nn_delta_weight(model, c, depth, divergence, convergence, steps, shift, preserve_screen_border=False, enable_amp=True,
                                     return_mask=False):
    """iw3/backward_warp.py:262-341 for sbs.mlbw: every flow layer warps the frame, the warps are blended with the
    (antialias-bilinear resized) layer weights.  ``steps`` is ignored by the reference for this model.  A hole_mask model
    (mask_mlbw_l2) also predicts hole logits at depth resolution: ``return_mask=True`` returns ``(z, logits)`` (flipped back with
    the frame for shift > 0), otherwise the holes are blacked out, z * (1 - postprocess_hole_mask(logits, (H, W), 0.15))."""
    if not enable_amp:
        raise NotImplementedError("nunif_b200 implements the reference's CUDA autocast (fp16) forward only")
    _lib.require_cuda(c, "c")
    _lib.require_cuda(depth, "depth")
    c, depth = c.float().contiguous(), depth.float().contiguous()
    if shift > 0:
        c, depth = torch.flip(c, (3,)), torch.flip(depth, (3,))
    B, _, H, W = depth.shape
    out = model(make_input(depth, divergence, convergence, preserve_screen_border))
    delta, lw = out[:2]
    logits = out[2] if getattr(model, "hole_mask", False) else None
    if c.shape[2:] != lw.shape[2:]:                                                            # :296-298
        L = lw.shape[1]
        lw_full = torch.empty((B, L, c.shape[2], c.shape[3]), dtype=torch.float32, device=c.device)
        with torch.cuda.device(c.device):
            _lib.check(_lib.lib().nb200_depth_resize_aa(_lib.ptr(lw.contiguous()), B * L, H, W, c.shape[2], c.shape[3], _lib.ptr(lw_full),
                                                        _lib.stream_ptr(c.device)))
        lw = lw_full
    delta_scale = 1.0 / (W // 2 - 1)
    z = torch.zeros_like(c)
    for i in range(model.num_layers):                                                          # :304-309
        z += _warp_delta(c, delta[:, i:i + 1].contiguous(), delta_scale) * lw[:, i:i + 1]
    z = z.clamp_(0, 1)
    if shift > 0:
        z = torch.flip(z, (3,))
        if logits is not None:
            logits = torch.flip(logits, (3,))
    if return_mask:
        return z, logits
    if logits is not None:                                                                     # :332-339
        z = z * (1 - postprocess_hole_mask(logits, c.shape[-2:], MASK_MLBW_THRESHOLD))
    return z


def apply_divergence_nn(model, c, depth, divergence, convergence, steps, shift, preserve_screen_border=False, enable_amp=True):
    """iw3/backward_warp.py:163-182."""
    fn = apply_divergence_nn_delta_weight if getattr(model, "name", "") == "sbs.mlbw" else apply_divergence_nn_delta
    return fn(model, c, depth, divergence, convergence, steps, shift, preserve_screen_border=preserve_screen_border, enable_amp=enable_amp)


def apply_divergence_nn_symmetric(model, c, depth, divergence, convergence, synthetic_view, enable_amp=True):
    """iw3/backward_warp.py:344-379: one delta from the feature values at base width W (the depth width, not max(H, W)), no flip,
    and both eyes warped from it with opposite signs in one launch (nb200_backward_warp_delta_sym).  The eye a single view does
    not synthesise is a copy of c.  There is no steps / preserve_screen_border here, as in the reference."""
    assert synthetic_view in {"both", "right", "left"}
    assert model.symmetric
    if not enable_amp:
        raise NotImplementedError("nunif_b200 implements the reference's CUDA autocast (fp16) forward only")
    _lib.require_cuda(c, "c")
    _lib.require_cuda(depth, "depth")
    c, depth = c.float().contiguous(), depth.float().contiguous()
    B, _, H, W = depth.shape
    if synthetic_view != "both":
        divergence = divergence * 2                                                             # :352-353
    delta = model.delta_x(make_input(depth, divergence, convergence, image_width=W))           # :359-365
    delta_scale = 1.0 / (W // 2 - 1)                                                           # :367
    left, right = torch.empty_like(c), torch.empty_like(c)
    Bc, _, Hc, Wc = c.shape
    with torch.cuda.device(c.device):
        _lib.check(_lib.lib().nb200_backward_warp_delta_sym(_lib.ptr(c), _lib.ptr(delta), Bc, Hc, Wc, H, W, delta_scale,
                                                            int(synthetic_view != "right"), int(synthetic_view != "left"),
                                                            _lib.ptr(left), _lib.ptr(right), _lib.stream_ptr(c.device)))
    return left, right


def apply_divergence_nn_LR(model, c, depth, divergence, convergence, steps=None, synthetic_view="both",
                           preserve_screen_border=False, enable_amp=True):
    """iw3/backward_warp.py:124-160: the symmetric models (row_flow_v3_sym) through apply_divergence_nn_symmetric, the others
    (sbs.row_flow_v3, sbs.row_flow_v2, sbs.mlbw) one eye at a time."""
    assert synthetic_view in {"both", "right", "left"}
    if getattr(model, "symmetric", False):                                                     # :133-136
        return apply_divergence_nn_symmetric(model, c, depth, divergence, convergence, synthetic_view=synthetic_view,
                                             enable_amp=enable_amp)
    kw = dict(steps=steps, preserve_screen_border=preserve_screen_border, enable_amp=enable_amp)
    if synthetic_view == "both":
        return (apply_divergence_nn(model, c, depth, divergence, convergence, shift=-1, **kw),
                apply_divergence_nn(model, c, depth, divergence, convergence, shift=1, **kw))
    if synthetic_view == "right":
        return c, apply_divergence_nn(model, c, depth, divergence * 2, convergence, shift=1, **kw)
    return apply_divergence_nn(model, c, depth, divergence * 2, convergence, shift=-1, **kw), c


# load_row_flow_model (iw3/stereo_model_factory.py:98-113): method -> (model class, symmetric, release checkpoint,
# iw3/stereo_model_factory.py:12-14)
ROW_FLOW_METHODS = {
    "row_flow": (RowFlowV3, False, "iw3_row_flow_v3_20250627.pth"),
    "row_flow_v3": (RowFlowV3, False, "iw3_row_flow_v3_20250627.pth"),
    "row_flow_sym": (RowFlowV3, True, "iw3_row_flow_v3_sym_20250628.pth"),
    "row_flow_v3_sym": (RowFlowV3, True, "iw3_row_flow_v3_sym_20250628.pth"),
    "row_flow_v2": (RowFlowV2, False, "iw3_row_flow_v2_20240130.pth"),
}


def load_row_flow_model(method, device="cuda:0", path=None):
    """The side model of ``--method row_flow*``.  ``path`` defaults to HUB_MODEL_DIR/checkpoints/<release file>; the engine
    never downloads it.  The checkpoint is a nunif checkpoint ({"name", "state_dict"}) whose name must match the method's
    model."""
    if method not in ROW_FLOW_METHODS:
        raise ValueError(method)
    cls, symmetric, ckpt = ROW_FLOW_METHODS[method]
    path = path if path is not None else os.path.join(HUB_MODEL_DIR, "checkpoints", ckpt)
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path}: the {cls.name} checkpoint of --method {method} is missing (the engine does not download models)")
    data = torch.load(path, map_location="cpu", weights_only=True)
    name = data.get("name") if isinstance(data, dict) else None
    if name != cls.name:
        raise ValueError(f"{path}: checkpoint model name is {name!r}, expected {cls.name!r}")
    if cls is RowFlowV3:
        return cls(data["state_dict"], device, symmetric=symmetric)
    return cls(data["state_dict"], device)
