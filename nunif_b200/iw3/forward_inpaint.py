"""iw3's `forward_inpaint` stereo method in image mode (iw3/forward_inpaint.py:18-40,69-103,235-297): the forward warp leaves
holes behind foreground edges, and the `inpaint.light_inpaint_v1` network (iw3/models/light_inpaint_v1.py) paints them.

The warp is csrc/warp_forward.cu, the mask chain and the network are csrc/inpaint_kernels.cu + the wgmma GEMM
(csrc/inpaint_model.cu).  Video mode (`light_video_inpaint_v1`, a 12-frame queue) is not implemented and raises.
"""
import contextlib
import os
import torch

from .. import _lib
from ._common import prep
from .base_depth_model import HUB_MODEL_DIR
from .forward_warp import apply_divergence_forward_warp

MODEL_NAME = "inpaint.light_inpaint_v1"
CHECKPOINT = "iw3_light_inpaint_v1_20250919.pth"   # iw3/inpaint_utils.py:45


def default_checkpoint():
    """HUB_MODEL_DIR/checkpoints/<release file> (iw3/hub_dir.py, torch.hub's layout); the engine never downloads it."""
    return os.path.join(HUB_MODEL_DIR, "checkpoints", CHECKPOINT)


def load_state_dict(path):
    """A nunif checkpoint (nunif/models/utils.py save_model): {"name": ..., "state_dict": ...}."""
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path}: the {MODEL_NAME} checkpoint is missing (the engine does not download models)")
    data = torch.load(path, map_location="cpu", weights_only=True)
    name = data.get("name") if isinstance(data, dict) else None
    if name != MODEL_NAME:
        raise ValueError(f"{path}: checkpoint model name is {name!r}, expected {MODEL_NAME!r}")
    return data["state_dict"]


class LightInpaintV1:
    """Packed `inpaint.light_inpaint_v1`.  ``infer(x, mask, mirror=False)`` is LightInpaintV1.infer(x, mask)
    (light_inpaint_v1.py:102-154) for x B,3,H,W and a binary mask B,1,H,W; ``mirror=True`` runs it on the flipped frame and
    mask and flips the result back, as forward_left does."""
    name = MODEL_NAME

    def __init__(self, state_dict=None, device="cuda:0"):
        self.device = _lib.cuda_device(device)
        if state_dict is None or isinstance(state_dict, (str, os.PathLike)):
            state_dict = load_state_dict(state_dict if state_dict is not None else default_checkpoint())
        self._h = _lib.Model("LIGHT_INPAINT_V1", state_dict, self.device)

    def infer(self, x, mask, mirror=False):
        x, mask = prep(x, "x"), prep(mask, "mask")
        assert x.ndim == 4 and x.shape[1] == 3 and mask.shape == (x.shape[0], 1, *x.shape[2:])
        B, _, H, W = x.shape
        out = torch.empty_like(x)
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().nb200_light_inpaint(self._h, _lib.ptr(x), _lib.ptr(mask), B, H, W, 1 if mirror else 0,
                                                      _lib.ptr(out), _lib.stream_ptr(x.device)))
        return out


def inpaint_mask(mask, inner_dilation=0, outer_dilation=0, base_width=None, mirror=False, binarize=True, closing=True):
    """forward_right's mask chain (forward_inpaint.py:18-25): mask > 0, mask_closing, dilate_outer, dilate_inner; with
    ``mirror`` forward_left's (:28-40) on the flipped mask, flipped back.  One row-tiled pass (csrc/inpaint_kernels.cu)."""
    mask = prep(mask, "mask")
    B, _, H, W = mask.shape
    out = torch.empty_like(mask)
    with torch.cuda.device(mask.device):
        _lib.check(_lib.lib().nb200_inpaint_mask(_lib.ptr(mask), B, H, W, int(binarize), int(closing), int(outer_dilation),
                                                 int(inner_dilation), int(base_width or 0), int(mirror), _lib.ptr(out),
                                                 _lib.stream_ptr(mask.device)))
    return out


def resize_max_width(x, max_width):
    """forward_inpaint.py:74-81: frames wider than max_width are resized (antialiased bilinear) to an even size."""
    if max_width is None or x.shape[-1] <= max_width:
        return x
    if max_width % 2 != 0:
        max_width += 1
    new_h = int((max_width / x.shape[-1]) * x.shape[-2])
    if new_h % 2 != 0:
        new_h += 1
    x = prep(x, "x")
    B, _, H, W = x.shape
    out = torch.empty((B, 3, new_h, max_width), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().nb200_resize_bilinear_aa(_lib.ptr(x), B, H, W, new_h, max_width, _lib.ptr(out),
                                                       _lib.stream_ptr(x.device)))
    return out


class ForwardInpaint:
    """The side model of `--method forward_inpaint` with the reference's surface (forward_inpaint.py:235-297), image mode only.
    Every frame of a batch is processed in one call; the result equals the reference's per-frame loop
    (iw3/utils.py:333-367)."""

    def __init__(self, model=None, device="cuda:0"):
        self.device = torch.device(device)
        self.model = model if isinstance(model, LightInpaintV1) else LightInpaintV1(model, device=self.device)
        self.mode = "image"

    def set_mode(self, mode):
        assert mode in {"video", "image"}
        if mode == "video":
            raise NotImplementedError("forward_inpaint video mode (light_video_inpaint_v1) is not implemented by the H100 engine")
        self.mode = mode

    def reset(self):
        pass

    def flush(self, enable_amp=True):
        return None, None

    def compile(self):
        pass

    def clear_compiled_model(self):
        pass

    def compile_context(self, enabled=True):
        return contextlib.nullcontext()

    def _eye(self, eye, mask, mirror, kw):
        return self.model.infer(eye, inpaint_mask(mask, mirror=mirror, **kw), mirror=mirror)

    @torch.inference_mode()
    def infer(self, x, depth, divergence, convergence, synthetic_view="both", inner_dilation=0, outer_dilation=0, max_width=None,
              enable_amp=True, **_kwargs):
        """ForwardInpaintImage.forward (forward_inpaint.py:69-103): x B,3,H,W, depth B,1,h,w -> (left_eye, right_eye)."""
        if not enable_amp:
            raise NotImplementedError("nunif_b200 implements the reference's CUDA autocast (fp16) forward only")
        assert synthetic_view in {"both", "right", "left"}
        x = resize_max_width(prep(x, "x"), max_width)
        left, right, lm, rm = apply_divergence_forward_warp(x, depth, divergence, convergence, synthetic_view=synthetic_view,
                                                            return_mask=True, width_base=False)
        kw = dict(inner_dilation=inner_dilation, outer_dilation=outer_dilation, base_width=depth.shape[-1])
        if synthetic_view in ("both", "left"):
            left = self._eye(left, lm, True, kw)
        if synthetic_view in ("both", "right"):
            right = self._eye(right, rm, False, kw)
        return left, right
