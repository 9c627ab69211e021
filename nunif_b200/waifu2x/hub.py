"""`waifu2x` hub entry for the H100 engine: the same public surface as the reference's
``Waifu2xImageModel`` / ``waifu2x()`` factory (waifu2x/hub.py:31-175), built as a thin adapter.

Design (not a transcription): the reference class mixes mode bookkeeping, device plumbing and three input
front-ends in one class body.  Here

* ``_ModeTable``   owns the method aliases and the (method, noise_level) validation rules (hub.py:60-69,151-163),
* ``_decode`` / ``_encode``   are the only places that know about PIL (hub.py:105-120, nunif/utils/pil_io.py:218-253),
* ``Waifu2xImageModel``   is a small facade: every ``infer*`` funnels into ``_run`` -> ``Waifu2x.convert``.

Engine restrictions are loud, never silent: models live on one sm_90 device (``cpu()`` raises), the forward is the
reference's CUDA autocast numerics (``amp=False`` / ``float()`` raise), nothing is downloaded.
"""
import os
from os import path

import torch

from .utils import Waifu2x

MODEL_DIR = os.environ.get("NUNIF_B200_MODEL_DIR",
                           path.join(os.environ.get("NUNIF_HOME", path.expanduser("~/.nunif")), "waifu2x", "pretrained_models"))

_ARCH_STYLES = (("swin_unet", ("art", "art_scan", "photo")), ("cunet", ("art",)), ("upconv_7", ("art", "photo")))
NO_4X_MODELS = {"cunet/art", "upconv_7/art", "upconv_7/photo"}
METHODS = ["noise", "scale", "noise_scale", "scale2x", "noise_scale2x", "scale4x", "noise_scale4x"]


def _types(model_dir):
    """model_type -> checkpoint directory; bare style names mean swin_unet (hub.py:10-18)."""
    table = {}
    for arch, styles in _ARCH_STYLES:
        for style in styles:
            table[f"{arch}/{style}"] = path.join(model_dir, arch, style)
            if arch == "swin_unet":
                table[style] = table[f"{arch}/{style}"]
    return table


MODEL_TYPES = _types(MODEL_DIR)


class _ModeTable:
    """Method aliases and the rules tying a method to a noise level."""
    ALIASES = {"scale2x": "scale", "noise_scale2x": "noise_scale"}
    DENOISING = {"scale": "noise_scale", "scale4x": "noise_scale4x"}      # plain upscale + noise_level >= 0
    NEEDS_NOISE = {"noise", "noise_scale", "noise_scale4x"}
    ONLY_4X = {"scale4x", "noise_scale4x"}

    @classmethod
    def canonical(cls, method, noise_level):
        if method is None:
            return None
        method = cls.ALIASES.get(method, method)
        if noise_level is not None and noise_level >= 0:
            method = cls.DENOISING.get(method, method)
        return method

    @classmethod
    def check(cls, model_type, method, noise_level):
        if method in cls.ONLY_4X and model_type in NO_4X_MODELS:
            raise ValueError(f"method: {model_type} does not support {method}")
        if method in cls.NEEDS_NOISE and noise_level not in {0, 1, 2, 3}:
            raise ValueError("noise_level: choose from (0, 1, 2, 3)")


def _decode(pil_image, keep_alpha):
    """PIL image -> (rgb 3xHxW, alpha 1xHxW or None) float in [0, 1] (pil_io.to_tensor semantics)."""
    import numpy as np
    with_alpha = keep_alpha and pil_image.mode in ("RGBA", "LA")
    pixels = np.asarray(pil_image.convert("RGBA" if with_alpha else "RGB"), dtype=np.uint8)
    chw = torch.from_numpy(pixels.copy()).permute(2, 0, 1).to(torch.float32) / 255.0
    return chw[:3], (chw[3:4] if with_alpha else None)


def _encode(rgb, alpha):
    """(rgb, alpha) tensors -> PIL image, quantised like pil_io.to_image (clamp(round(x * 255)))."""
    from PIL import Image
    planes = rgb if alpha is None else torch.cat([rgb, alpha.to(rgb.device)], dim=0)
    q = (planes.float() * 255.0).round_().clamp_(0, 255).to(torch.uint8)
    return Image.fromarray(q.permute(1, 2, 0).cpu().numpy(), mode="RGB" if alpha is None else "RGBA")


class Waifu2xImageModel():
    def __init__(self, model_type, method=None, noise_level=-1, device_ids=[-1], tile_size=None, batch_size=None,
                 keep_alpha=True, amp=True, model_dir=None):
        types = _types(model_dir) if model_dir else MODEL_TYPES
        if model_type not in types:
            raise ValueError(f"model_type: choose from {list(types.keys())}")
        if method is not None and method not in METHODS:
            raise ValueError(f"method: choose from {METHODS}")
        if not amp:
            raise NotImplementedError("nunif_b200 implements the reference's CUDA autocast (fp16) forward only: amp=False is not available")
        self.model_type, self.keep_alpha, self.amp = model_type, keep_alpha, True
        self.tile_size, self.batch_size = tile_size, batch_size
        self.method = self.noise_level = None
        self.ctx = Waifu2x(types[model_type], device_ids)
        if method is None:
            self.ctx.load_model_all(load_4x=model_type not in NO_4X_MODELS)
        else:
            canon = _ModeTable.canonical(method, noise_level)
            _ModeTable.check(model_type, canon, noise_level)
            self.ctx.load_model(canon, noise_level)
            self.method, self.noise_level = canon, noise_level

    # ---- mode
    normalize_method = staticmethod(_ModeTable.canonical)

    def set_mode(self, method, noise_level=-1):
        canon = _ModeTable.canonical(method, noise_level)
        _ModeTable.check(self.model_type, canon, noise_level)
        self.method, self.noise_level = canon, noise_level

    # ---- device / precision plumbing (delegated; unsupported requests raise in Waifu2x)
    def _delegate(self, name, *args):
        getattr(self.ctx, name)(*args)
        return self

    def compile(self):
        return self._delegate("compile")

    def to(self, device):
        return self._delegate("to", device)

    def cuda(self):
        return self._delegate("to", "cuda")

    def cpu(self):
        return self._delegate("to", "cpu")

    def half(self):
        return self._delegate("half")

    def float(self):
        return self._delegate("float")

    is_half = property(lambda self: self.ctx.is_half)
    device = property(lambda self: self.ctx.device)

    # ---- inference
    def _run(self, rgb, alpha, tta, output_type, overrides):
        noise_level = overrides.get("noise_level", self.noise_level)
        method = _ModeTable.canonical(overrides.get("method", self.method), -1 if noise_level is None else noise_level)
        if method is None:
            raise ValueError("method is None. Call `model.set_mode(method, noise_level)` or use method and noise_level kwargs")
        with torch.inference_mode():
            rgb, alpha = self.ctx.convert(rgb, alpha, method, noise_level, tile_size=self.tile_size,
                                          batch_size=self.batch_size, tta=tta, enable_amp=True)
        return (rgb, alpha) if output_type == "tensor" else _encode(rgb, alpha)

    def infer_tensor(self, rgb, alpha=None, tta=False, output_type="pil", **kwargs):
        return self._run(rgb, alpha, tta, output_type, kwargs)

    def infer_pil(self, pil_image, tta=False, output_type="pil", **kwargs):
        rgb, alpha = _decode(pil_image, self.keep_alpha)
        cast = (lambda t: t.to(self.device).half()) if self.is_half else (lambda t: t.to(self.device))
        return self._run(cast(rgb), None if alpha is None else cast(alpha), tta, output_type, kwargs)

    def infer_file(self, filepath, tta=False, output_type="pil", **kwargs):
        from PIL import Image
        with Image.open(filepath) as im:
            im.load()
            return self.infer_pil(im, tta=tta, output_type=output_type, **kwargs)

    def infer(self, x, tta=False, output_type="pil", **kwargs):
        if torch.is_tensor(x):
            return self.infer_tensor(x, tta=tta, output_type=output_type, **kwargs)
        if isinstance(x, (str, os.PathLike)):
            return self.infer_file(x, tta=tta, output_type=output_type, **kwargs)
        if type(x).__module__.startswith("PIL."):
            return self.infer_pil(x, tta=tta, output_type=output_type, **kwargs)
        raise ValueError("Unsupported input format")

    __call__ = infer

    def convert(self, input_filepath, output_filepath, tta=False, format="png", **kwargs):
        self.infer_file(input_filepath, tta=tta, **kwargs).save(output_filepath, format=format)


def waifu2x(model_type="art", method=None, noise_level=-1, device_ids=[-1], tile_size=None, batch_size=None,
            keep_alpha=True, amp=True, **kwargs):
    """The torch.hub entry point (waifu2x/hub.py:166-175) minus the network download: checkpoints must already be in
    ``model_dir`` / ``MODEL_DIR``."""
    return Waifu2xImageModel(model_type=model_type, method=method, noise_level=noise_level, device_ids=device_ids,
                             tile_size=tile_size, batch_size=batch_size, keep_alpha=keep_alpha, amp=amp,
                             model_dir=kwargs.get("model_dir"))
