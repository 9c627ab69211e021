"""Mirror of `iw3.depth_aa` (iw3/models/depth_aa.py:30-87): the learned anti-aliasing filter batch_infer applies to the
Depth-Anything output when ``depth_aa`` is set (iw3/depth_anything_model.py:153-154, :190-194).

The Linears / 1x1 / 3x3 convolutions run on the wgmma GEMM, everything else in csrc/depth_aa.cu (nb200_depth_aa)."""
import torch
from .. import _lib


class DepthAA:
    """Packed `iw3.depth_aa`.  ``model(x)`` = DepthAA.forward in eval mode (clamped), ``model.infer(x)`` = DepthAA.infer."""
    name = "iw3.depth_aa"

    def __init__(self, state_dict, device="cuda:0"):
        self.device = _lib.cuda_device(device)
        self._h = _lib.Model("DEPTH_AA", state_dict, self.device)

    def _run(self, x, mode):
        _lib.require_cuda(x, "x")
        assert x.ndim == 4 and x.shape[1] == 1, "depth_aa expects B,1,H,W"
        if x.device != self.device:
            raise ValueError(f"input on {x.device} but the model lives on {self.device}")
        B, _, H, W = x.shape
        xf = x.float().contiguous()
        out = torch.empty_like(xf)
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().nb200_depth_aa(self._h, _lib.ptr(xf), B, H, W, mode, _lib.ptr(out), _lib.stream_ptr(x.device)))
        return out

    def __call__(self, x, clamp=None):
        """DepthAA.forward (:57-87): eval mode clamps unless ``clamp=False``."""
        return self._run(x, 0 if (clamp is None or clamp) else 2)

    forward = __call__

    def infer(self, x):
        """DepthAA.infer (:46-55): normalise by the min / max of the whole tensor, filter, de-normalise."""
        return self._run(x, 1)
