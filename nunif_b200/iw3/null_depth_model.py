"""Mirror of iw3/null_depth_model.py, iw3's ``--depth-model NULL``: the weight-free "dummy depth model for performance
benchmark".  Its depth is the frame bilinearly resized to R x R and averaged over the channels, so the stereo stage after
it (warps, learned warps, inpainting, postprocess) can be run and timed without a depth network.

``NullDepthNet(resolution)(x)`` is the reference's ``NullDepth.forward`` (:17-21), ``F.interpolate(x, (R, R),
mode="bilinear")`` then ``x.mean(dim=1, keepdim=True)`` with R = ``resolution`` or 392, as one fused kernel
(``nb200_null_depth``, csrc/null_depth.cu) whose arithmetic is that of ATen's CUDA kernels.  ``NullDepthModel`` has the
reference's surface with one deliberate difference: ``multi_gpu_supported`` is False, as for every engine depth model (one
process owns one GPU, DESIGN.md section 6), where the reference returns True.
"""
import torch

from .. import _lib
from .base_depth_model import BaseDepthModel
from .dilation import dilate_edge, edge_dilation_is_enabled

DEFAULT_RESOLUTION = 392     # null_depth_model.py:13-14; not rounded to a multiple of 14


class NullDepthNet:
    """``net(x)``: x B,3,H,W fp32 CUDA -> B,1,R,R fp32 on ``x.device``.  There are no weights, so it runs on whichever GPU
    holds ``x``."""

    def __init__(self, resolution=None):
        self.resolution = DEFAULT_RESOLUTION if resolution is None else int(resolution)
        if self.resolution <= 0:
            raise ValueError(f"resolution must be positive, got {resolution}")

    def __call__(self, x):
        _lib.require_cuda(x, "x")
        if x.ndim != 4 or x.shape[1] != 3:
            raise ValueError(f"expected B,3,H,W frames, got {tuple(x.shape)}")
        if x.dtype != torch.float32:
            raise TypeError(f"the NULL depth kernel takes float32 frames, got {x.dtype}")
        B, _, H, W = x.shape
        R = self.resolution
        x = x.contiguous()
        out = torch.empty((B, 1, R, R), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().nb200_null_depth(_lib.ptr(x), B, H, W, R, _lib.ptr(out), _lib.stream_ptr(x.device)))
        return out


class NullDepthModel(BaseDepthModel):
    """iw3/null_depth_model.py:24-79 on the engine: the BaseDepthModel surface (load / infer / EMA normaliser) with nothing
    to load."""

    def __init__(self, model_type="NULL"):
        super().__init__(model_type)

    def load_model(self, model_type, resolution=None, device=None, **kwargs):
        return NullDepthNet(resolution)

    @torch.inference_mode()
    def infer(self, x, tta=False, low_vram=False, enable_amp=True, edge_dilation=0, **kwargs):
        """null_depth_model.py:31-49.  x: 3,H,W or B,3,H,W -> 1,R,R or B,1,R,R.  The network is run once also with
        ``tta=True``: the reference's ``(m(x) + m(x)) * 0.5`` equals ``m(x)`` bit for bit in fp32.  ``enable_amp`` and
        ``low_vram`` change nothing; the reference's model is fp32 either way."""
        batch = x.ndim != 3
        if not batch:
            x = x.unsqueeze(0)
        x = self.model(x)
        if edge_dilation_is_enabled(edge_dilation):
            x = dilate_edge(x, edge_dilation)           # not inverted: is_metric() is False
        if not batch:
            x = x.squeeze(0)
        return x

    @classmethod
    def get_name(cls):
        return "NullDepth"

    @classmethod
    def supported(cls, model_type):
        return model_type == "NULL"

    @classmethod
    def get_model_path(cls, model_type):
        return None

    @classmethod
    def has_checkpoint_file(cls, model_type):
        return cls.supported(model_type)

    def is_metric(self):
        return False

    def is_video_supported(self):
        return True

    @classmethod
    def force_update(cls):
        pass                                            # nothing to download
