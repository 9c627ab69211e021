"""Mirror of iw3/zoedepth_model.py for ZoeD_Any_N / ZoeD_Any_K, iw3's default depth model, on the H100 engine.

The reference builds these through torch.hub ("nagadomi/Depth-Anything_iw3:main", DepthAnythingMetricDepth, model_type
"indoor" / "outdoor", zoedepth_model.py:154-170): ZoeDepth's metric bins head over a Depth-Anything V1 ViT-L/14 encoder and
DPT head, with ``prep_mod = 14`` and network heights 392 (landscape) / 518 (portrait) (:190-199).  Here the same checkpoints
(upstream key names ``core.core.pretrained.*``, ``core.core.depth_head.*``, ``conv2``, ``seed_bin_regressor``, ...) are packed into
the native container (csrc/zoe_model.cu) and run by ``nb200_zoedepth_forward``.  ZoeD_Any_N has the "softplus" bins head of
ZoeD_N; ZoeD_Any_K the "normed" one (bins bounded to [1e-3, 80], sorted at the last level).  Loading, ``batch_infer`` and
``infer`` are ZoeDepthModel's (the reference uses one class for all ZoeDepth checkpoints).
"""
from os import path
from .. import _lib
from .base_depth_model import HUB_MODEL_DIR
from .zoedepth_model import ZoeDepthModel, ZoeDepthNet

_KIND_KEYS = {"ZoeD_Any_N": "ZOEDEPTH_ANY_N", "ZoeD_Any_K": "ZOEDEPTH_ANY_K"}   # model type -> _lib.MODEL_KINDS key
KINDS = {t: _lib.MODEL_KINDS[k] for t, k in _KIND_KEYS.items()}

MODEL_FILES = {   # zoedepth_model.py:17-19
    "ZoeD_Any_N": path.join(HUB_MODEL_DIR, "checkpoints", "depth_anything_metric_depth_indoor.pt"),
    "ZoeD_Any_K": path.join(HUB_MODEL_DIR, "checkpoints", "depth_anything_metric_depth_outdoor.pt"),
}


class ZoeDepthAnythingNet(ZoeDepthNet):
    """The packed network: ``net(x)`` == ``ZoeDepth.forward(x)['metric_depth']`` of the Depth-Anything metric model
    (x: B,3,H,W normalised (x - 0.5) / 0.5, H,W % 14 == 0 -> B,1,H,W metric depth).  The checkpoint must match
    ``model_type``: an indoor checkpoint packed as ZoeD_Any_K (or the reverse) is refused at load."""

    def __init__(self, state_dict, device="cuda:0", model_type="ZoeD_Any_N"):
        if model_type not in KINDS:
            raise ValueError(f"model_type: choose from {list(KINDS)}")
        super().__init__(state_dict, device, kind=_KIND_KEYS[model_type])
        self.model_type = model_type
        self.prep_mod = 14                      # zoedepth_model.py:190-199
        self.prep_h_height = 392
        self.prep_v_height = 518


class ZoeDepthAnythingModel(ZoeDepthModel):
    """iw3's ZoeDepthModel("ZoeD_Any_N" | "ZoeD_Any_K") on the engine: the full BaseDepthModel surface (load / infer / EMA
    normaliser), the reference's signatures."""
    MODEL_FILES = MODEL_FILES

    def __init__(self, model_type="ZoeD_Any_N"):
        super().__init__(model_type)

    @classmethod
    def multi_gpu_supported(cls, model_type):
        return False                            # zoedepth_model.py:235-236

    def _wrap(self, state_dict, resolution, device):
        net = ZoeDepthAnythingNet(state_dict, device, self.model_type)
        if resolution is not None:              # :192-196
            if resolution % net.prep_mod != 0:
                resolution += net.prep_mod - resolution % net.prep_mod
            net.prep_h_height = net.prep_v_height = resolution
        return net
