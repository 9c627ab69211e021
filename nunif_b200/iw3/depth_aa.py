"""Mirror of `iw3.depth_aa` (iw3/models/depth_aa.py:30-87): the learned anti-aliasing filter batch_infer applies to the
Depth-Anything output when ``depth_aa`` is set (iw3/depth_anything_model.py:153-154, :190-194).

The Linears / 1x1 / 3x3 convolutions run on the wgmma GEMM, everything else in csrc/depth_aa.cu (nb200_depth_aa)."""
import ctypes
import torch
from .. import _lib

KIND_DEPTH_AA = 10     # NB200_MODEL_DEPTH_AA


class DepthAA:
    """Packed `iw3.depth_aa`.  ``model(x)`` = DepthAA.forward in eval mode (clamped), ``model.infer(x)`` = DepthAA.infer."""
    name = "iw3.depth_aa"

    def __init__(self, state_dict, device="cuda:0"):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("nunif_b200 models live on a CUDA (sm_90) device; there is no CPU path")
        items = [(k, v.detach().to("cpu", torch.float32).contiguous()) for k, v in state_dict.items()]
        n = len(items)
        names = (ctypes.c_char_p * n)(*[k.encode() for k, _ in items])
        datas = (ctypes.c_void_p * n)(*[v.data_ptr() for _, v in items])
        numels = (ctypes.c_int64 * n)(*[v.numel() for _, v in items])
        h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().nb200_model_create(KIND_DEPTH_AA, n, names, datas, numels, 0, ctypes.byref(h)))
        self._h = h

    def __del__(self):
        try:
            if self._h:
                _lib.lib().nb200_model_destroy(self._h)
                self._h = None
        except Exception:
            pass

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
