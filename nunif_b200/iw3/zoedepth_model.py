"""Mirror of iw3/zoedepth_model.py (ZoeDepthModel / batch_infer, lines 89-233) for the ZoeD_N metric depth network on the
H100 engine.

The reference obtains the network from torch.hub ("nagadomi/ZoeDepth_iw3:main", ZoeD_N, config_mode="infer",
zoedepth_model.py:151-157) and removes its internal resize/normalise (`model.core.prep = lambda x: x`, :169); here the
same checkpoint (ZoeD_M12_N.pt, upstream key names `core.core.pretrained.*`, `core.core.scratch.*`, `conv2`,
`seed_bin_regressor`, ...) is packed into the native container (csrc/zoe_model.cu) and run as wgmma GEMMs + the
kernels in csrc/depth_kernels.cu / zoe_kernels.cu.  ``infer`` keeps the reference's signature and output convention:
B,1,h,w (or 1,h,w) float32 on ``x.device`` = the NEGATED metric depth of the unpadded frame (larger = nearer).

Not built: ZoeD_K / ZoeD_NK (two bin heads + the patch-transformer domain classifier) - `supported()` says so and the
constructor raises.  The Depth-Anything-metric checkpoints ZoeD_Any_N / ZoeD_Any_K run through ZoeDepthAnythingModel
(zoedepth_any_model.py), a subclass that shares this class's loading and ``infer``.
"""
from os import path
import torch
from .. import _lib
from .base_depth_model import BaseDepthModel, HUB_MODEL_DIR
from .zoedepth_preprocess import batch_preprocess
from .dilation import dilate_edge, edge_dilation_is_enabled

MODEL_FILES = {   # zoedepth_model.py:12-19 (the one checkpoint the engine implements)
    "ZoeD_N": path.join(HUB_MODEL_DIR, "checkpoints", "ZoeD_M12_N.pt"),
}


def _strip_checkpoint(ckpt):
    """ZoeD_M12_N.pt is saved as {"model": state_dict, ...} by the upstream trainer; accept either form."""
    if isinstance(ckpt, dict) and "model" in ckpt and isinstance(ckpt["model"], dict):
        return ckpt["model"]
    return ckpt


class ZoeDepthNet:
    """The packed network: ``net(x)`` == ``ZoeDepth.forward(x)['metric_depth']`` (x: B,3,H,W normalised, H,W % 32 == 0
    -> B,1,H,W metric depth)."""

    def __init__(self, state_dict, device="cuda:0", kind="ZOEDEPTH_N"):
        self.device = _lib.cuda_device(device)
        self._h = _lib.Model(kind, {k: v for k, v in _strip_checkpoint(state_dict).items() if torch.is_tensor(v)}, self.device)
        self.metric_depth = True
        self.prep_mod = 32                      # zoedepth_model.py:172-180
        self.prep_h_height = 384
        self.prep_v_height = 512

    def __call__(self, x):
        _lib.require_cuda(x, "x")
        assert x.ndim == 4 and x.shape[1] == 3
        if x.device != self.device:
            raise RuntimeError(f"input on {x.device}, model on {self.device}")
        B, _, H, W = x.shape
        xf = x.float().contiguous()
        out = torch.empty((B, 1, H, W), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().nb200_zoedepth_forward(self._h, _lib.ptr(xf), B, H, W, _lib.ptr(out), _lib.stream_ptr(x.device)))
        return out


@torch.inference_mode()
def batch_infer(model, im, flip_aug=True, low_vram=False, enable_amp=False, output_device="cpu", device=None,
                edge_dilation=0, **kwargs):
    """zoedepth_model.py:89-148.  ``enable_amp`` is accepted for signature parity: the engine always runs the reference's
    CUDA numerics (fp16 autocast); ``low_vram`` only changes the reference's batching."""
    device = device if device is not None else model.device
    assert torch.is_tensor(im) and im.ndim in (3, 4)
    batch = im.ndim == 4
    x = (im if batch else im.unsqueeze(0)).to(device)
    x, pad_h, pad_w = batch_preprocess(x, h_height=model.prep_h_height, v_height=model.prep_v_height,
                                       ensure_multiple_of=model.prep_mod)
    if flip_aug:
        x = torch.cat([x, torch.flip(x, dims=[3])], dim=0)          # :108-111
    out = torch.nan_to_num(model(x))                                # _forward :23-27
    out = out[:, :, pad_h:out.shape[2] - pad_h, pad_w:out.shape[3] - pad_w]
    if edge_dilation_is_enabled(edge_dilation):
        out = dilate_edge(-out, edge_dilation)                      # :125-127 (dilate_edge works on "larger = nearer")
    else:
        out = -out
    if flip_aug:
        n = out.shape[0] // 2
        z = (out[:n] + torch.flip(out[n:], dims=[3])) * 0.5         # :132-139
    else:
        z = out
    if not batch:
        z = z.squeeze(0)
    return z.to(output_device)


class ZoeDepthModel(BaseDepthModel):
    """iw3/zoedepth_model.py:151-233 on the engine: the full BaseDepthModel surface (load / infer / EMA normaliser)."""
    MODEL_FILES = MODEL_FILES

    def __init__(self, model_type="ZoeD_N"):
        if not self.supported(model_type):
            hint = " (ZoeD_Any_N / ZoeD_Any_K: use ZoeDepthAnythingModel or create_depth_model)" if model_type.startswith("ZoeD_Any") else ""
            raise ValueError(f"{type(self).__name__} implements {sorted(self.MODEL_FILES)}; ZoeD_K / ZoeD_NK are not built{hint}")
        super().__init__(model_type)

    @classmethod
    def get_name(cls):
        return "ZoeDepth"

    @classmethod
    def supported(cls, model_type):
        return model_type in cls.MODEL_FILES

    @classmethod
    def get_model_path(cls, model_type):
        return cls.MODEL_FILES[model_type]

    def is_metric(self):
        return True

    def _wrap(self, state_dict, resolution, device):
        net = ZoeDepthNet(state_dict, device)
        if resolution is not None:                                   # :173-177
            if resolution % net.prep_mod != 0:
                resolution += net.prep_mod - resolution % net.prep_mod
            net.prep_h_height = net.prep_v_height = resolution
        return net

    def load_model(self, model_type, resolution=None, device=None):
        """The reference builds the module through torch.hub and lets it download its weights (:153-157); here the same
        checkpoint file is read from ``get_model_path(model_type)``."""
        ckpt = self.get_model_path(model_type)
        if not path.exists(ckpt):
            raise FileNotFoundError(f"{ckpt} not found (nunif_b200 does not download checkpoints)")
        return self._wrap(torch.load(ckpt, map_location="cpu", weights_only=True), resolution, device)

    def load_state_dict(self, state_dict, gpu=0, resolution=None):
        """``load`` from an in-memory state_dict with the upstream key names (tests, bench: seeded weights)."""
        from .base_depth_model import _device_of
        self.device = _device_of(gpu)
        self.model = self._wrap(state_dict, resolution, self.device)
        return self

    def infer(self, x, tta=False, low_vram=False, enable_amp=True, edge_dilation=0, **kwargs):
        """zoedepth_model.py:203-213."""
        if not enable_amp:
            raise NotImplementedError("nunif_b200 implements the reference's CUDA autocast (fp16) forward only")
        if not torch.is_tensor(x):
            import numpy as np
            x = torch.from_numpy(np.asarray(x, dtype=np.uint8).copy()).permute(2, 0, 1).float().div_(255.0).to(self.device)
        _lib.require_cuda(x, "x")
        return batch_infer(self.model, x, flip_aug=tta, low_vram=low_vram, enable_amp=enable_amp, output_device=x.device,
                           device=x.device, edge_dilation=edge_dilation)

    def infer_raw(self, *args, **kwargs):
        return batch_infer(self.model, *args, **kwargs)
