"""Model containers with the reference's I2IBaseModel contract
(nunif/models/model.py:65-86) backed by the sm_90a engine.

A container owns a packed fp16 weight blob on ONE device, created from a
state_dict with the reference's key names (strict, like load_state_dict).
"""
import ctypes
import torch
from .. import _lib

KINDS = {
    "waifu2x.upcunet": 1, "waifu2x.cunet": 2,
    "waifu2x.swin_unet_1x": 3, "waifu2x.swin_unet_2x": 4, "waifu2x.swin_unet_4x": 5,
    "waifu2x.upconv_7": 13, "waifu2x.vgg_7": 14,
}


def _cunet_validator(size):            # waifu2x/models/cunet.py:124-125
    return size % 4 == 0


def _swin_validator(size):             # waifu2x/models/swin_unet.py:202-205
    return size > 16 and (size - 16) % 12 == 0 and (size - 16) % 16 == 0


def _any_size_validator(size):         # upconv_7 / vgg_7 register no validator (nunif/models/model.py:51-62)
    return True


def _validator_for(name):
    if "cunet" in name:
        return _cunet_validator
    if name in ("waifu2x.upconv_7", "waifu2x.vgg_7"):
        return _any_size_validator
    return _swin_validator


class B200I2IModel:
    """Drop-in for an ``I2IBaseModel`` instance in eval mode."""

    def __init__(self, name, state_dict, device="cuda:0", no_clip=False, _handle=None, _downscale=1, _parent=None):
        if name not in KINDS:
            raise ValueError(f"Unknown model name: {name}")          # nunif/models/register.py:22-28
        self.name = name
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("nunif_b200 models live on a CUDA (sm_90) device; there is no CPU path")
        self._downscale = _downscale
        self._parent = _parent  # keeps the shared handle alive (to_2x(shared=True))
        self.training = False
        self.i2i_in_channels = 3
        self.i2i_default_tile_size = 256                              # model.py:69
        self.i2i_default_batch_size = 4
        self._validator = _validator_for(name)
        lib = _lib.lib()
        if _handle is not None:
            self._h = _handle
            self._own = False
        else:
            items = [(k, v.detach().to("cpu", torch.float32).contiguous()) for k, v in state_dict.items()]
            n = len(items)
            names = (ctypes.c_char_p * n)(*[k.encode() for k, _ in items])
            datas = (ctypes.c_void_p * n)(*[v.data_ptr() for _, v in items])
            numels = (ctypes.c_int64 * n)(*[v.numel() for _, v in items])
            h = ctypes.c_void_p()
            with torch.cuda.device(self.device):
                _lib.check(lib.nb200_model_create(KINDS[name], n, names, datas, numels, 1 if no_clip else 0, ctypes.byref(h)))
            self._h = h
            self._own = True
        s, o, b = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        _lib.check(lib.nb200_model_info(self._h, ctypes.byref(s), ctypes.byref(o), ctypes.byref(b)))
        if _downscale == 1:
            self.i2i_scale, self.i2i_offset = s.value, o.value
            self.i2i_blend_size = b.value if b.value > 0 else None   # cunet passes blend_size=None
        else:                                                          # swin_unet.py:345-350
            self.i2i_scale, self.i2i_offset, self.i2i_blend_size = 4 // _downscale, 32 // _downscale, 4 * _downscale

    def __del__(self):
        try:
            if getattr(self, "_own", False) and self._h:
                _lib.lib().nb200_model_destroy(self._h)
                self._h = None
        except Exception:
            pass

    # ---- I2IBaseModel surface
    def find_valid_tile_size(self, base_tile_size):
        """model.py:51-62,82-86."""
        if base_tile_size is None:
            base_tile_size = self.i2i_default_tile_size
        t = int(base_tile_size)
        while t > 0:
            if self._validator(t):
                return t
            t -= 1
        raise ValueError(f"Could not find valid tile size: tile_size={base_tile_size}")

    def get_device(self):
        return self.device

    def eval(self):
        return self

    def to_2x(self, shared=True):
        """SwinUNet4x.to_2x (swin_unet.py:289-295): same weights + bicubic-AA /2."""
        if self.name != "waifu2x.swin_unet_4x":
            raise AttributeError("to_2x is defined for waifu2x.swin_unet_4x only")
        return B200I2IModel(self.name, None, self.device, _handle=self._h, _downscale=2, _parent=self)

    def to_1x(self, shared=True):
        if self.name != "waifu2x.swin_unet_4x":
            raise AttributeError("to_1x is defined for waifu2x.swin_unet_4x only")
        return B200I2IModel(self.name, None, self.device, _handle=self._h, _downscale=4, _parent=self)

    def weight_blob(self):
        """(device_ptr, nbytes) of the packed weights, for the one-time NCCL broadcast."""
        p, n = ctypes.c_void_p(), ctypes.c_size_t()
        _lib.check(_lib.lib().nb200_model_weight_blob(self._h, ctypes.byref(p), ctypes.byref(n)))
        return p.value, n.value

    @torch.no_grad()
    def __call__(self, x):
        """model(minibatch): x B,3,T,T float/half in [0,1] on self.device -> B,3,S,S in the dtype the reference returns under CUDA
        autocast: fp16 for the native models, fp32 for the 4x-derived 2x / 1x models (they resize ``z.float()``)."""
        _lib.require_cuda(x, "x")
        if x.device != self.device:
            raise RuntimeError(f"input is on {x.device} but the model's packed weights live on {self.device}")
        assert x.ndim == 4 and x.shape[1] == 3 and x.shape[2] == x.shape[3]
        B, _, T, _ = x.shape
        xh = torch.zeros((B, T, T, 8), device=x.device, dtype=torch.float16)
        xh[..., :3] = x.permute(0, 2, 3, 1)
        S = T * self.i2i_scale - 2 * self.i2i_offset
        z = torch.empty((B, 3, S, S), device=x.device, dtype=torch.float16 if self._downscale == 1 else torch.float32)
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().nb200_model_forward(self._h, _lib.ptr(xh), B, T, self._downscale, _lib.ptr(z),
                                                      _lib.stream_ptr(x.device)))
        return z


NOT_BUILT = {   # registered by the reference (waifu2x/models/swin_unet.py:306-336,390-394) but outside this engine: loud, not "unknown"
    "waifu2x.swin_unet_8x": "SwinUNet8x (scale_factor 8 variant, no released weights)",
    "waifu2x.swin_unet_4xl": "swin_unet_4xl (base_dim 192 + LayerNormNoBias variant, no released weights)",
}


def create_model(name, state_dict, device="cuda:0", **kwargs):
    """nunif.models.create_model + load_state_dict (register.py:52-63, utils.py:57-58).  ``kwargs`` are the constructor
    arguments a checkpoint carries (`load_model` passes `data["kwargs"]`): the ones that change the arithmetic and are not
    built raise instead of being ignored."""
    if name in NOT_BUILT:
        raise NotImplementedError(f"{name}: {NOT_BUILT[name]} is not implemented by nunif_b200")
    if kwargs.get("pre_antialias"):
        raise NotImplementedError("pre_antialias=True (swin_unet.py:252-258,281-282: bicubic x2 up / down of every tile before the "
                                  "network) is not implemented by nunif_b200")
    if kwargs.get("layer_norm") or kwargs.get("base_dim", 96) != 96:
        raise NotImplementedError("swin_unet variants with layer_norm=True / base_dim != 96 are not implemented by nunif_b200")
    for k in ("in_channels", "out_channels"):
        if kwargs.get(k, 3) != 3:
            raise NotImplementedError(f"{k}={kwargs[k]}: the engine implements the released 3-channel models")
    no_clip = bool(kwargs.get("no_clip", False))
    if name == "waifu2x.swin_unet_downscaled":
        # SwinUNetDownscaled (swin_unet.py:339-387): the 4x network (same `unet.*` keys) + antialiased bicubic /2 or /4
        f = int(kwargs.get("downscale_factor", 2))
        if f not in (2, 4):
            raise AssertionError("downscale_factor must be 2 or 4")                      # :344
        base = B200I2IModel("waifu2x.swin_unet_4x", state_dict, device=device, no_clip=no_clip)
        return base.to_2x() if f == 2 else base.to_1x()
    return B200I2IModel(name, state_dict, device=device, no_clip=no_clip)


def load_model(model_path, device="cuda:0", weights_only=True):
    """nunif.models.load_model (utils.py:42-74): reads the reference's .pth dict
    {nunif_model, name, kwargs, state_dict, ...} -> (model, meta)."""
    data = torch.load(model_path, map_location="cpu", weights_only=weights_only)
    if "nunif_model" not in data:
        raise ValueError(f"{model_path} is not a nunif model")       # utils.py:72-73
    kwargs = dict(data.get("kwargs", {}))
    model = create_model(data["name"], data["state_dict"], device=device, **kwargs)
    data.pop("state_dict")
    return model, data
