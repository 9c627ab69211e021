"""iw3's `mlbw_l2_inpaint` stereo method in image mode (iw3/mlbw_inpaint.py:18-151,296-360): the hole-mask MLBW warp
(`sbs.mask_mlbw_l2`, iw3/models/mlbw.py) places the pixels and predicts where it leaves holes, and `inpaint.light_inpaint_v1` paints
them.

The warp network and the hole head are csrc/mlbw.cu + the wgmma GEMM, the hole mask is nb200_hole_mask + the row-run dilation of
nb200_inpaint_mask, and the inpainting network is forward_inpaint's LightInpaintV1.  Video mode (`light_video_inpaint_v1`, a
12-frame queue) is not implemented and raises.
"""
import contextlib
import os
import torch

from ._common import prep
from .base_depth_model import HUB_MODEL_DIR
from .forward_inpaint import LightInpaintV1, resize_max_width
from .row_flow import MLBW, MASK_MLBW_THRESHOLD, apply_divergence_nn_delta_weight, postprocess_hole_mask

MASK_MLBW_NAME = "sbs.mlbw"
MASK_MLBW_CHECKPOINT = "iw3_mask_mlbw_l2_d1_20250903.pth"   # iw3/inpaint_utils.py:15,91-96


def default_mask_mlbw_checkpoint():
    """HUB_MODEL_DIR/checkpoints/<release file> (torch.hub's layout); the engine never downloads it."""
    return os.path.join(HUB_MODEL_DIR, "checkpoints", MASK_MLBW_CHECKPOINT)


def load_mask_mlbw_state_dict(path):
    """The mask-MLBW nunif checkpoint: {"name": "sbs.mlbw", "kwargs": {..., "hole_mask": True}, "state_dict": ...}."""
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path}: the mask_mlbw_l2 checkpoint is missing (the engine does not download models)")
    data = torch.load(path, map_location="cpu", weights_only=True)
    name = data.get("name") if isinstance(data, dict) else None
    if name != MASK_MLBW_NAME:
        raise ValueError(f"{path}: checkpoint model name is {name!r}, expected {MASK_MLBW_NAME!r}")
    if not (data.get("kwargs") or {}).get("hole_mask", False):
        raise ValueError(f"{path}: {MASK_MLBW_NAME} checkpoint without kwargs['hole_mask']: not a mask_mlbw model")
    return data["state_dict"]


class MLBWInpaint:
    """The side model of `--method mlbw_l2_inpaint` with the reference's surface (mlbw_inpaint.py:296-360), image mode only.
    ``model``: a LightInpaintV1, its state_dict or a checkpoint path; ``mask_mlbw``: an MLBW with a hole head, its state_dict or a
    checkpoint path.  None means the release checkpoint under HUB_MODEL_DIR/checkpoints.  Every frame of a batch is processed in
    one call; the result equals the reference's per-frame loop (iw3/utils.py:333-367)."""

    def __init__(self, model=None, mask_mlbw=None, device="cuda:0"):
        self.device = torch.device(device)
        self.model = model if isinstance(model, LightInpaintV1) else LightInpaintV1(model, device=self.device)
        if not isinstance(mask_mlbw, MLBW):
            if mask_mlbw is None or isinstance(mask_mlbw, (str, os.PathLike)):
                mask_mlbw = load_mask_mlbw_state_dict(mask_mlbw if mask_mlbw is not None else default_mask_mlbw_checkpoint())
            mask_mlbw = MLBW(mask_mlbw, device=self.device)
        if not mask_mlbw.hole_mask:
            raise ValueError("mask_mlbw must be an sbs.mlbw with a hole_mask head (mask_mlbw_l2)")
        self.mask_mlbw = mask_mlbw
        self.mode = "image"

    def set_mode(self, mode):
        assert mode in {"video", "image"}
        if mode == "video":
            raise NotImplementedError("mlbw_l2_inpaint video mode (light_video_inpaint_v1) is not implemented by the H100 engine")
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

    def _warp(self, x, depth, divergence, convergence, shift, preserve_screen_border):
        return apply_divergence_nn_delta_weight(self.mask_mlbw, x, depth, divergence, convergence, 1, shift,
                                                preserve_screen_border=preserve_screen_border, return_mask=True)

    def _eye(self, eye, logits, mirror, inner_dilation, outer_dilation):
        # forward_right / forward_left (mlbw_inpaint.py:21-34); mirror replaces forward_left's flips of the eye, the logits and the result
        mask = postprocess_hole_mask(logits, eye.shape[-2:], MASK_MLBW_THRESHOLD, inner_dilation, outer_dilation, mirror=mirror)
        return self.model.infer(eye, mask, mirror=mirror)

    @torch.inference_mode()
    def infer(self, x, depth, divergence, convergence, preserve_screen_border=False, synthetic_view="both", inner_dilation=0,
              outer_dilation=0, max_width=None, enable_amp=True, **_kwargs):
        """MLBWInpaintImage.forward (mlbw_inpaint.py:112-151): x B,3,H,W, depth B,1,h,w -> (left_eye, right_eye)."""
        if not enable_amp:
            raise NotImplementedError("nunif_b200 implements the reference's CUDA autocast (fp16) forward only")
        assert synthetic_view in {"both", "right", "left"}
        x = resize_max_width(prep(x, "x"), max_width)
        left = right = x
        # apply_divergence (:37-72): a single synthetic view takes the whole divergence
        div = divergence if synthetic_view == "both" else divergence * 2
        if synthetic_view in ("both", "left"):
            left, lm = self._warp(x, depth, div, convergence, -1, preserve_screen_border)
            left = self._eye(left, lm, True, inner_dilation, outer_dilation)
        if synthetic_view in ("both", "right"):
            right, rm = self._warp(x, depth, div, convergence, 1, preserve_screen_border)
            right = self._eye(right, rm, False, inner_dilation, outer_dilation)
        return left, right
