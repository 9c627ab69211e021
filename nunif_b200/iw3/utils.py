"""The stereo dispatcher of iw3 under its reference name and signature: ``apply_divergence(depth, im, args, side_model)``
(iw3/utils.py:292-391) and the single-image driver ``process_image`` (iw3/utils.py:505-545, without the file / autocrop
layers, which stay in the reference's host code).

``args`` is the reference's argparse namespace; the fields read here are the ones the reference reads on this path:
``method, mapper, convergence, divergence, synthetic_view, warp_steps, preserve_screen_border, stereo_width, disable_amp,
mask_inner_dilation, mask_outer_dilation, inpaint_max_width, state["convergence_model"]``.  ``mapper`` is any name of
iw3/mapper.py; build it from ``--foreground-scale`` / ``--mapper-type`` with ``resolve_mapper_name`` as iw3/utils.py:2341-2344
does.  A convergence model must be the
engine's ``ConvergenceEstimator`` (``--convergence-mode sod_v1``).  Anything the engine does not implement raises ``NotImplementedError`` - never a silent
fallback."""
import torch

from .. import _lib
from ._common import prep
from .backward_warp import apply_divergence_grid_sample
from .forward_warp import apply_divergence_forward_warp
from .depth_scaler import depth_mapper
from .row_flow import apply_divergence_nn_LR
from .postprocess import postprocess_image
from .convergence_estimator import ConvergenceEstimator

_WARP = {"grid_sample": "backward", "backward": "backward", "forward": "forward", "forward_fill": "forward"}


def _arg(args, name, default=None):
    return getattr(args, name, default)


def resize_depth_aa(depth, height, width):
    """F.interpolate(depth, size=(height, width), mode="bilinear", align_corners=True, antialias=True) for a B,1,h,w
    depth map (nb200_depth_resize_aa)."""
    d = prep(depth, "depth")
    B, C, h, w = d.shape
    out = torch.empty((B, C, height, width), dtype=torch.float32, device=d.device)
    with torch.cuda.device(d.device):
        _lib.check(_lib.lib().nb200_depth_resize_aa(_lib.ptr(d), B * C, h, w, height, width, _lib.ptr(out), _lib.stream_ptr(d.device)))
    return out


def apply_divergence(depth, im, args, side_model, reset_pts=None):
    """depth: normalised [0, 1] depth CHW / BCHW, im: the frame(s) with the same batch layout -> (left_eye, right_eye)."""
    batched = depth.ndim == 4
    if not batched:
        depth, im = depth.unsqueeze(0), im.unsqueeze(0)
    state = _arg(args, "state", None) or {}
    convergence_model = state.get("convergence_model")
    if convergence_model is not None and not isinstance(convergence_model, ConvergenceEstimator):
        raise NotImplementedError("auto-convergence needs the engine's estimator in args.state['convergence_model'] "
                                  f"(nunif_b200.iw3.ConvergenceEstimator), got {type(convergence_model).__name__}")
    if not _arg(args, "disable_amp", False) is False:
        raise NotImplementedError("--disable-amp (fp32 side model) is not implemented: the engine runs the CUDA autocast numerics")
    if convergence_model is not None:
        # --convergence-mode sod_v1 (:303-307): a B,1,1,1 convergence per frame, mapped like the depth
        convergence = depth_mapper(convergence_model(im, depth, reset_pts=reset_pts), args.mapper)
    else:
        convergence = args.convergence
    depth = depth_mapper(depth, args.mapper)                                    # get_mapper(args.mapper)(depth), :313
    method = args.method
    if method == "NULL":
        eyes = (im.clone(), im.clone())
    elif _WARP.get(method) == "backward":
        eyes = apply_divergence_grid_sample(im, depth, args.divergence, convergence=convergence,
                                            synthetic_view=args.synthetic_view)
    elif _WARP.get(method) == "forward":
        eyes = apply_divergence_forward_warp(im, depth, args.divergence, convergence=convergence, method=method,
                                             synthetic_view=args.synthetic_view, width_base=False)
    elif method == "forward_inpaint":
        # side_model.infer per frame (:333-367); image mode returns no delayed frames (flush() -> (None, None))
        if side_model is None:
            raise ValueError("method forward_inpaint needs side_model (nunif_b200.iw3.ForwardInpaint)")
        eyes = side_model.infer(im, depth, args.divergence, convergence, synthetic_view=args.synthetic_view,
                                inner_dilation=_arg(args, "mask_inner_dilation", 0), outer_dilation=_arg(args, "mask_outer_dilation", 0),
                                max_width=_arg(args, "inpaint_max_width", None), enable_amp=True)
    elif method == "mlbw_l2_inpaint":
        # the same per-frame side_model.infer as forward_inpaint (:333-367), with preserve_screen_border passed through
        if side_model is None:
            raise NotImplementedError("method mlbw_l2_inpaint needs side_model: the H100 engine does not build the reference's "
                                      "MLBWInpaint implicitly (pass nunif_b200.iw3.MLBWInpaint)")
        eyes = side_model.infer(im, depth, args.divergence, convergence, preserve_screen_border=_arg(args, "preserve_screen_border", False),
                                synthetic_view=args.synthetic_view, inner_dilation=_arg(args, "mask_inner_dilation", 0),
                                outer_dilation=_arg(args, "mask_outer_dilation", 0), max_width=_arg(args, "inpaint_max_width", None),
                                enable_amp=True)
    else:
        # the learned warps (row_flow*, mlbw*): apply_divergence_nn_LR with args.side_model (:363-385)
        if _arg(args, "stereo_width", None) is not None:
            # --stereo-width (:370-379): the warp runs at this width, with the frame's aspect ratio (not the depth's)
            H, W = im.shape[2:]
            stereo_width = min(W, args.stereo_width)
            if depth.shape[3] != stereo_width:
                depth = resize_depth_aa(depth, int(H * (stereo_width / W)), stereo_width).clamp_(0, 1)
        if side_model is None:
            raise ValueError(f"method {method} needs side_model")
        eyes = apply_divergence_nn_LR(side_model, im, depth, args.divergence, convergence, _arg(args, "warp_steps", None),
                                      synthetic_view=args.synthetic_view,
                                      preserve_screen_border=_arg(args, "preserve_screen_border", False), enable_amp=True)
    left_eye, right_eye = eyes
    if not batched:
        left_eye, right_eye = left_eye.squeeze(0), right_eye.squeeze(0)
    return left_eye, right_eye


def process_image(x, args, depth_model, side_model):
    """iw3/utils.py:505-545 for a CHW float frame already on the GPU (no autocrop / rgbd / debug branches)."""
    assert depth_model.get_ema_buffer_size() == 1
    with torch.inference_mode():
        depth = depth_model.infer(x, tta=_arg(args, "tta", False), low_vram=_arg(args, "low_vram", False),
                                  enable_amp=not _arg(args, "disable_amp", False),
                                  edge_dilation=_arg(args, "edge_dilation", 2), depth_aa=_arg(args, "depth_aa", False))
        depth = depth_model.minmax_normalize_chw(depth)
        left_eye, right_eye = apply_divergence(depth, x, args, side_model)
        return postprocess_image(left_eye, right_eye, args)
