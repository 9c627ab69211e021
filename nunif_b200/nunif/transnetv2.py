"""TransNetV2 (nunif/utils/transnetv2.py), the shot-boundary network behind iw3's ``--scene-detect``, under its reference
name.  The network runs as the sm_90a kernels of csrc/transnet.cu and the wgmma GEMM; there is no CPU path."""
import os
import torch
from .. import _lib
from ..iw3.base_depth_model import HUB_MODEL_DIR

FRAME_SHAPE = (3, 27, 48)
CHECKPOINT = "transnetv2-pytorch-weights.pth"   # the file name of TransNetV2.load's URL


def checkpoint_path():
    """Where torch.hub's load_state_dict_from_url caches the release weights when iw3 runs under TorchHubDir(HUB_MODEL_DIR)."""
    return os.path.join(HUB_MODEL_DIR, "checkpoints", CHECKPOINT)


class TransNetV2:
    """Packed TransNetV2 with the default configuration (F=16, L=3, S=2, D=1024) in eval mode.  ``model(x)`` takes x
    [T,3,27,48] (one window) or [B,T,3,27,48] float and returns ``(one_hot [B,T,1], {"many_hot": [B,T,1]})`` fp32 logits like
    TransNetV2.forward; every window is padded in time on its own, as in the reference."""

    def __init__(self, state_dict, device="cuda:0"):
        self.device = _lib.cuda_device(device)
        self._h = _lib.Model("TRANSNET_V2", state_dict, self.device)

    @classmethod
    def load(cls, device="cuda:0", path=None):
        """The release weights from HUB_MODEL_DIR/checkpoints/transnetv2-pytorch-weights.pth (or ``path``); never downloaded."""
        path = path if path is not None else checkpoint_path()
        if not os.path.exists(path):
            raise FileNotFoundError(f"{path}: the TransNetV2 checkpoint of --scene-detect is missing "
                                    "(the engine does not download models)")
        return cls(torch.load(path, map_location="cpu", weights_only=True), device)

    def eval(self):
        return self

    def __call__(self, inputs):
        assert torch.is_tensor(inputs) and inputs.dtype in {torch.float32, torch.float16}
        if inputs.ndim == 4 and tuple(inputs.shape[1:]) == FRAME_SHAPE:
            inputs = inputs.unsqueeze(0)
        else:
            assert inputs.ndim == 5 and tuple(inputs.shape[2:]) == FRAME_SHAPE, "incorrect input type and/or shape"
        _lib.require_cuda(inputs, "inputs")
        x = inputs.to(self.device, torch.float32).contiguous()
        B, T = x.shape[:2]
        one_hot = torch.empty((B, T, 1), dtype=torch.float32, device=self.device)
        many_hot = torch.empty_like(one_hot)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().nb200_transnetv2_forward(self._h, _lib.ptr(x), B, T, _lib.ptr(one_hot), _lib.ptr(many_hot),
                                                           _lib.stream_ptr(self.device)))
        return one_hot, {"many_hot": many_hot}
