"""iw3's auto-convergence (``--convergence-mode sod_v1``): the `iw3.sod_v1` salient-object network (iw3/models/sod_v1.py, a
U^2-Net-p, nunif/utils/u2netp.py) and ``ConvergenceEstimator`` (iw3/convergence_estimator.py) under their reference names.

The network runs as the sm_90a kernels of csrc/sod.cu; the position rule (mask, two quantiles, branch, clamp) and the EMA
run on the device as well, so a call makes no host synchronisation (the reference syncs on ``numel() == 0`` and
``q_range < 1e-6``)."""
import ctypes
import os
import torch
from .. import _lib
from ._common import prep
from .base_depth_model import HUB_MODEL_DIR

SOD_SIZE = 192             # SODV1's i2i_in_size
SOD_NAMES = ("iw3.sod_v1", "iw3.dsod_v1")
SOD_CHECKPOINT = "iw3_sod_v1_20260125.pth"   # the file name of convergence_estimator.py's SOD_URL


class SODV1:
    """Packed `iw3.sod_v1` (in eval mode after ``.fuse()``).  ``infer(rgb, depth)`` returns ``(saliency, depth_192)`` like
    SODV1.infer under CUDA autocast: saliency B,1,192,192 (fp32 tensor holding the fp16 sigmoid), depth_192 the fp32 bilinear
    resize of depth."""
    name = "iw3.sod_v1"

    def __init__(self, state_dict, device="cuda:0"):
        self.device = _lib.cuda_device(device)
        self._h = _lib.Model("SOD_V1", state_dict, self.device)

    def infer(self, rgb, depth):
        rgb = prep(rgb, "rgb")
        depth = prep(depth, "depth")
        assert rgb.ndim == 4 and rgb.shape[1] == 3 and depth.ndim == 4 and depth.shape[1] == 1
        assert rgb.shape[0] == depth.shape[0]
        B, _, H, W = rgb.shape
        h, w = depth.shape[-2:]
        sal = torch.empty((B, 1, SOD_SIZE, SOD_SIZE), dtype=torch.float32, device=rgb.device)
        d192 = torch.empty_like(sal)
        with torch.cuda.device(rgb.device):
            _lib.check(_lib.lib().nb200_sod_forward(self._h, _lib.ptr(rgb), B, H, W, _lib.ptr(depth), h, w, _lib.ptr(sal),
                                                    _lib.ptr(d192), _lib.stream_ptr(rgb.device)))
        return sal, d192


def depth_position_from_ratio(saliency_map, depth, pos):
    """ConvergenceEstimator.depth_position_from_ratio (convergence_estimator.py:33-58) in one kernel: B,1,h,w saliency and
    depth -> B,1,1,1 fp32.  The quantiles equal torch.quantile bit for bit."""
    s = prep(saliency_map, "saliency_map")
    d = prep(depth, "depth")
    B = d.shape[0]
    n = d[0].numel()
    assert s.shape[0] == B and s[0].numel() == n
    out = torch.empty((B, 1, 1, 1), dtype=torch.float32, device=d.device)
    with torch.cuda.device(d.device):
        _lib.check(_lib.lib().nb200_sod_position(_lib.ptr(s), _lib.ptr(d), B, n, float(pos), _lib.ptr(out), _lib.stream_ptr(d.device)))
    return out


def load_sod_state_dict(path=None):
    """The state_dict of the release checkpoint: HUB_MODEL_DIR/checkpoints/iw3_sod_v1_20260125.pth by default.  The engine
    never downloads it; the checkpoint's model name must be iw3.sod_v1 (or its alias iw3.dsod_v1)."""
    path = path if path is not None else os.path.join(HUB_MODEL_DIR, "checkpoints", SOD_CHECKPOINT)
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path}: the iw3.sod_v1 checkpoint of --convergence-mode sod_v1 is missing "
                                "(the engine does not download models)")
    data = torch.load(path, map_location="cpu", weights_only=True)
    name = data.get("name") if isinstance(data, dict) else None
    if name not in SOD_NAMES:
        raise ValueError(f"{path}: checkpoint model name is {name!r}, expected one of {SOD_NAMES}")
    return data["state_dict"]


class ConvergenceEstimator:
    """iw3/convergence_estimator.py:11-81 with the reference's signature.  ``compile`` is accepted and ignored.  ``path``
    overrides the checkpoint location and ``state_dict`` skips the file (e.g. seeded weights); ``load_state_dict`` replaces
    the weights later."""

    def __init__(self, convergence, device_id, enable_ema=False, decay=0.9, compile=False, path=None, state_dict=None):
        self.device = torch.device("cuda", device_id) if isinstance(device_id, int) else torch.device(device_id)
        self.convergence = convergence
        self.enable_ema = enable_ema
        self.decay = decay
        self.model = SODV1(state_dict if state_dict is not None else load_sod_state_dict(path), self.device)
        self._ema = torch.zeros(2, dtype=torch.float32, device=self.device)   # {ema, has_value}, never read by the host

    def load_state_dict(self, state_dict):
        self.model = SODV1(state_dict, self.device)
        return self

    def reset(self, enable_ema=None, decay=None):
        if enable_ema is not None:
            self.enable_ema = enable_ema
        if decay is not None:
            self.decay = decay
        self._ema.zero_()

    @staticmethod
    def depth_position_from_ratio(saliency_map, depth, pos):
        return depth_position_from_ratio(saliency_map, depth, pos)

    @torch.inference_mode()
    def __call__(self, rgb, depth, reset_pts=None):
        rgb = rgb.to(self.device)
        depth = depth.to(self.device)
        saliency, depth_scaled = self.model.infer(rgb, depth)
        z_pos = depth_position_from_ratio(saliency, depth_scaled, self.convergence)
        if not self.enable_ema:
            return z_pos
        B = z_pos.shape[0]
        resets = None
        if reset_pts is not None:
            resets = (ctypes.c_int * B)(*[1 if r else 0 for r in reset_pts])
        out = torch.empty_like(z_pos)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().nb200_sod_ema(_lib.ptr(self._ema), _lib.ptr(z_pos), B, resets, float(self.decay), _lib.ptr(out),
                                                _lib.stream_ptr(self.device)))
        return out
