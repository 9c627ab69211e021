"""Mirror of iw3/depth_anything_model.py (DepthAnythingModel / batch_infer, lines 113-253) for the
Depth-Anything-V2 (Any_V2_S/B/L) and V1 (Any_S/B/L) relative-depth networks on the H100 engine.

The reference obtains the network from torch.hub ("nagadomi/Depth-Anything_iw3:main", DepthAnything(encoder="v2_vits"),
depth_anything_model.py:223-230); here the same checkpoint (upstream key names ``pretrained.*`` / ``depth_head.*``) is
packed into the native container (csrc/depth_model.inl) and run as wgmma GEMMs + the kernels in
csrc/depth_kernels.cu.  ``infer`` keeps the reference's signature and output convention: depth B,1,h,w (or 1,h,w)
float32 on ``x.device``, larger = nearer.
"""
import ctypes
from os import path
import torch
from .. import _lib
from .base_depth_model import BaseDepthModel, HUB_MODEL_DIR
from .depth_anything_preprocess import batch_preprocess
from .dilation import dilate_edge, edge_dilation_is_enabled

# NB200_MODEL_DEPTH_ANYTHING_V2_{S,B,L}, NB200_MODEL_DEPTH_ANYTHING_V1_{S,B,L}; model types as in iw3/depth_anything_model.py
# NAME_MAP.  V1 is the same network with the hooks on the last four blocks.
KINDS = {"vits": 6, "vitb": 8, "vitl": 9}
V1_KINDS = {"vits": 20, "vitb": 21, "vitl": 22}
ENCODER_OF = {"Any_V2_S": "vits", "Any_V2_B": "vitb", "Any_V2_L": "vitl", "Any_S": "vits", "Any_B": "vitb", "Any_L": "vitl"}
V1_MODELS = {"Any_S", "Any_B", "Any_L"}
AA_SUPPORTED_MODELS = {"Any_V2_S", "Any_V2_B", "Any_V2_L"}   # depth_anything_model.py:61-65


class DepthAnythingNet:
    """The packed network: ``net(x)`` == ``DepthAnythingV2.forward`` (or the V1 ``DepthAnything.forward`` with ``v1=True``)
    (x: B,3,H,W normalised, H,W % 14 == 0 -> B,H,W)."""

    def __init__(self, state_dict, device="cuda:0", encoder="vits", v1=False):
        if encoder not in KINDS:
            raise ValueError(f"encoder: choose from {list(KINDS)}")
        self.encoder = encoder
        self.v1 = v1
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
            _lib.check(_lib.lib().nb200_model_create((V1_KINDS if v1 else KINDS)[encoder], n, names, datas, numels, 0, ctypes.byref(h)))
        self._h = h
        self.metric_depth = False
        self.prep_lower_bound = 392

    def __del__(self):
        try:
            if self._h:
                _lib.lib().nb200_model_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def __call__(self, x):
        _lib.require_cuda(x, "x")
        assert x.ndim == 4 and x.shape[1] == 3
        if x.device != self.device:
            raise RuntimeError(f"input is on {x.device} but the model's packed weights live on {self.device}")
        B, _, H, W = x.shape
        xf = x.float().contiguous()
        out = torch.empty((B, H, W), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().nb200_depth_anything_forward(self._h, _lib.ptr(xf), B, H, W, _lib.ptr(out), _lib.stream_ptr(x.device)))
        return out


@torch.inference_mode()
def batch_infer(model, im, flip_aug=True, low_vram=False, enable_amp=False, output_device="cpu", device=None,
                edge_dilation=2, depth_aa=None, limit_resolution=False, **kwargs):
    """depth_anything_model.py:122-182.  ``enable_amp`` is accepted for signature parity: the engine always runs the
    reference's CUDA numerics (fp16 autocast).  ``depth_aa``: a packed `iw3.depth_aa` (nunif_b200.iw3.depth_aa.DepthAA) or
    None (:153-154)."""
    device = device if device is not None else model.device
    assert torch.is_tensor(im) and im.ndim in (3, 4)
    batch = im.ndim == 4
    x = (im if batch else im.unsqueeze(0)).to(device)
    x = batch_preprocess(x, model.prep_lower_bound, limit_resolution=limit_resolution)
    if flip_aug:
        x = torch.cat([x, torch.flip(x, dims=[3])], dim=0)           # :140-142 (low_vram only changes the batching)
    out = torch.nan_to_num(model(x).unsqueeze(1))                    # _forward :113-119
    if depth_aa is not None:
        out = depth_aa.infer(out)                                    # :153-154
    if edge_dilation_is_enabled(edge_dilation):
        out = dilate_edge(out, edge_dilation) if not model.metric_depth else -dilate_edge(-out, edge_dilation)
    if model.metric_depth:
        out = -out
    if flip_aug:
        n = out.shape[0] // 2
        z = (out[:n] + torch.flip(out[n:], dims=[3])) * 0.5          # :163-171
    else:
        z = out
    if not batch:
        z = z.squeeze(0)
    return z.to(output_device)


MODEL_FILES = {   # depth_anything_model.py:37-42 (the relative-depth V1 and V2 checkpoints)
    "Any_S": path.join(HUB_MODEL_DIR, "checkpoints", "depth_anything_vits14.pth"),
    "Any_B": path.join(HUB_MODEL_DIR, "checkpoints", "depth_anything_vitb14.pth"),
    "Any_L": path.join(HUB_MODEL_DIR, "checkpoints", "depth_anything_vitl14.pth"),
    "Any_V2_S": path.join(HUB_MODEL_DIR, "checkpoints", "depth_anything_v2_vits.pth"),
    "Any_V2_B": path.join(HUB_MODEL_DIR, "checkpoints", "depth_anything_v2_vitb.pth"),
    "Any_V2_L": path.join(HUB_MODEL_DIR, "checkpoints", "depth_anything_v2_vitl.pth"),
}


class DepthAnythingModel(BaseDepthModel):
    """iw3/depth_anything_model.py:185-281 on the engine: the full BaseDepthModel surface (load / infer / EMA normaliser)."""

    def __init__(self, model_type="Any_V2_S"):
        if model_type not in ENCODER_OF:
            raise ValueError(f"the H100 engine implements {list(ENCODER_OF)} (Depth-Anything V1 / V2 relative-depth models)")
        super().__init__(model_type)

    @classmethod
    def get_name(cls):
        return "DepthAnything"

    @classmethod
    def supported(cls, model_type):
        return model_type in ENCODER_OF

    @classmethod
    def get_model_path(cls, model_type):
        return MODEL_FILES[model_type]

    def is_metric(self):
        return False

    def _wrap(self, state_dict, resolution, device):
        net = DepthAnythingNet(state_dict, device, encoder=ENCODER_OF[self.model_type], v1=self.model_type in V1_MODELS)
        lb = resolution or 392                                        # :232-235 (GUI 512 -> 518)
        if lb % 14 != 0:
            lb += 14 - lb % 14
        net.prep_lower_bound = lb
        return net

    def load_model(self, model_type, resolution=None, device=None):
        """The reference builds the module through torch.hub and lets it download its weights (:186-238); here the same
        checkpoint file is read from ``get_model_path(model_type)``."""
        ckpt = self.get_model_path(model_type)
        if not path.exists(ckpt):
            raise FileNotFoundError(f"{ckpt} not found (nunif_b200 does not download checkpoints)")
        return self._wrap(torch.load(ckpt, map_location="cpu", weights_only=True), resolution, device)

    def load_state_dict(self, state_dict, gpu=0, resolution=None, limit_resolution=False):
        """``load`` from an in-memory state_dict with the upstream key names (tests, bench: seeded weights)."""
        from .base_depth_model import _device_of
        self.device = _device_of(gpu)
        self.limit_resolution = limit_resolution
        self.model = self._wrap(state_dict, resolution, self.device)
        return self

    def infer(self, x, tta=False, low_vram=False, enable_amp=True, edge_dilation=0, depth_aa=False, **kwargs):
        """depth_anything_model.py:241-253.  The V1 models have no depth_aa (:190-194): ``depth_aa=True`` runs without it."""
        depth_aa = depth_aa and self.model_type in AA_SUPPORTED_MODELS
        if not enable_amp:
            raise NotImplementedError("nunif_b200 implements the reference's CUDA autocast (fp16) forward only")
        if not torch.is_tensor(x):
            import numpy as np
            x = torch.from_numpy(np.asarray(x, dtype=np.uint8).copy()).permute(2, 0, 1).float().div_(255.0).to(self.device)
        _lib.require_cuda(x, "x")
        if depth_aa and getattr(self, "depth_aa", None) is None:
            raise RuntimeError("depth_aa=True needs the iw3.depth_aa weights: call load_depth_aa(state_dict) first (the reference "
                               "downloads iw3_depth_aa_20250530.pth in load(), :190-192; nunif_b200 does not download)")
        return batch_infer(self.model, x, flip_aug=tta, low_vram=low_vram, enable_amp=enable_amp, output_device=x.device,
                           device=x.device, edge_dilation=edge_dilation, depth_aa=self.depth_aa if depth_aa else None,
                           limit_resolution=self.limit_resolution)

    depth_aa = None

    def load_depth_aa(self, state_dict):
        """The learned anti-aliasing filter the reference attaches in load() (:190-194); ``state_dict`` with the keys of
        `iw3.depth_aa` (the ``state_dict`` entry of iw3_depth_aa_20250530.pth).  Only the V2 models take it."""
        if self.model_type not in AA_SUPPORTED_MODELS:
            raise ValueError(f"depth_aa is attached to {sorted(AA_SUPPORTED_MODELS)} only (depth_anything_model.py:61-65), not {self.model_type}")
        from .depth_aa import DepthAA
        self.depth_aa = DepthAA(state_dict, self.device)
        return self
