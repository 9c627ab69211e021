"""Mirror of waifu2x/utils.py:42-297 (class Waifu2x): model slots per method/noise level,
load_model (2x/1x derived from 4x), render, convert."""
from os import path
import torch
from ..nunif.models import load_model
from ..nunif.render import tiled_render
from ..nunif.alpha import AlphaBorderPadding
from ..nunif.tta import tta_split, tta_merge
import torch.nn.functional as F
from .. import _lib


def _require_amp(enable_amp):
    if not enable_amp:
        raise NotImplementedError("nunif_b200 implements the reference's CUDA autocast (fp16) forward only; "
                                  "enable_amp=False (fp32 forward) is not implemented")


class Waifu2x():
    def __init__(self, model_dir, gpus):
        self.scale_model = None
        self.scale4x_model = None
        self.noise_models = [None] * 4
        self.noise_scale_models = [None] * 4
        self.noise_scale4x_models = [None] * 4
        self.alpha_pad = AlphaBorderPadding()
        # nunif/device.py:12-32 create_device: gpus[0] < 0 means CPU in the reference; this engine is CUDA-only
        gpu = gpus[0] if isinstance(gpus, (list, tuple)) else gpus
        if isinstance(gpu, int) and gpu < 0:
            gpu = 0
        self.device = torch.device(f"cuda:{gpu}") if isinstance(gpu, int) else torch.device(gpu)
        if self.device.type != "cuda":
            raise RuntimeError("nunif_b200.waifu2x runs on CUDA (sm_90) only")
        self.gpus = gpus
        self.model_dir = model_dir
        self.is_half = False

    def compile(self):
        """waifu2x/utils.py:49-58 wraps the modules in torch.compile; this engine's kernels are compiled ahead of time
        (nvcc, sm_90a), so there is nothing left to do - same results either way, as in the reference."""
        return self

    def _loaded_models(self):
        slots = [self.scale_model, self.scale4x_model, *self.noise_models, *self.noise_scale_models, *self.noise_scale4x_models]
        return [m for m in slots if m is not None]

    @torch.inference_mode()
    def warmup(self, tile_size=None, batch_size=None, enable_amp=True):
        """waifu2x/utils.py:60-83: one forward per loaded model and batch size, which here sizes the workspaces, sets the
        per-device kernel attributes and loads the cubins before the first real frame."""
        _require_amp(enable_amp)
        for model in self._loaded_models():
            t = model.i2i_default_tile_size if tile_size is None else model.find_valid_tile_size(tile_size)
            n = model.i2i_default_batch_size if batch_size is None else batch_size
            for bs in range(n, 0, -1):
                model(torch.zeros((bs, 3, t, t), device=self.device, dtype=torch.float16 if self.is_half else torch.float32))
        torch.cuda.synchronize(self.device)
        return self

    def to(self, device):
        """The packed weights live on the device they were created on (one process per GPU); only a no-op move is possible."""
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("nunif_b200 models cannot be moved to the CPU")
        if device.index is not None and device != self.device and self._loaded_models():
            raise RuntimeError(f"nunif_b200 models are bound to {self.device}; create a Waifu2x(gpus=[{device.index}]) instead")
        if device.index is not None:
            self.device = device
        return self

    def half(self):
        """Reference: weights and inputs in fp16 (utils.py:90-93).  The engine's storage is fp16 already; this only
        switches the tensors handed to / returned by ``model(x)`` and ``infer_pil`` to fp16."""
        self.is_half = True
        return self

    def float(self):
        """Reference default state: fp32 weights run under CUDA autocast (nunif/device.py:58-71) - the numerics this engine
        implements.  (An fp32 *forward*, ``enable_amp=False``, is not implemented and raises.)"""
        self.is_half = False
        return self

    def load_model_by_name(self, filename):
        return load_model(path.join(self.model_dir, filename), device=self.device, weights_only=True)[0]

    def has_model_file(self, filename):
        return path.exists(path.join(self.model_dir, filename))

    # method -> (checkpoint file pattern, method whose 4x model the 2x/1x variant is derived from, derivation)
    # (waifu2x/utils.py:128-176: the released swin_unet directories only ship 4x checkpoints; 2x and 1x are the
    #  4x network followed by an antialiased bicubic downscale, swin_unet.py:289-303)
    _CHECKPOINTS = {
        "scale4x": ("scale4x.pth", None, None),
        "scale": ("scale2x.pth", "scale4x", "to_2x"),
        "noise_scale4x": ("noise{n}_scale4x.pth", None, None),
        "noise_scale": ("noise{n}_scale2x.pth", "noise_scale4x", "to_2x"),
        "noise": ("noise{n}.pth", "noise_scale4x", "to_1x"),
    }

    def _slot(self, method, noise_level, value=None):
        per_level = {"noise": self.noise_models, "noise_scale": self.noise_scale_models,
                     "noise_scale4x": self.noise_scale4x_models}.get(method)
        if value is None:
            return per_level[noise_level] if per_level is not None else getattr(self, method + "_model")
        if per_level is not None:
            per_level[noise_level] = value
        else:
            setattr(self, method + "_model", value)
        return value

    def _load_model(self, method, noise_level):
        """waifu2x/utils.py:128-176, table-driven."""
        if method not in self._CHECKPOINTS:
            raise ValueError(method)
        if self._slot(method, noise_level) is not None:
            return
        pattern, base, derive = self._CHECKPOINTS[method]
        filename = pattern.format(n=noise_level)
        if self.has_model_file(filename):
            self._slot(method, noise_level, self.load_model_by_name(filename))
        elif base is None:
            raise FileNotFoundError(f"{filename} not found in {self.model_dir}")
        else:
            self._load_model(base, noise_level)
            self._slot(method, noise_level, getattr(self._slot(base, noise_level), derive)())

    def load_model(self, method, noise_level):
        """waifu2x/utils.py:178-199: also keeps the plain scale model next to a noise_scale one (alpha channel pass)."""
        assert (method in ("scale", "noise_scale", "noise", "scale4x", "noise_scale4x"))
        assert (method in {"scale", "scale4x"} or 0 <= noise_level and noise_level < 4)
        self._load_model(method, noise_level)
        companion = {"noise_scale4x": "scale4x", "noise_scale": "scale"}.get(method)
        if companion is not None:
            try:
                self._load_model(companion, -1)
            except FileNotFoundError:
                pass

    def load_model_all(self, load_4x=True):
        """waifu2x/utils.py:201-216."""
        order = (["scale4x", "noise_scale4x"] if load_4x else []) + ["scale", "noise_scale", "noise"]
        for method in order:
            for noise_level in ([-1] if method in {"scale", "scale4x"} else range(4)):
                self._load_model(method, noise_level)

    def _model(self, method, noise_level):
        return self._slot(method, noise_level)

    @torch.inference_mode()
    def render(self, x, method, noise_level, tile_size=None, batch_size=None, enable_amp=True):
        """waifu2x/utils.py:218-241.  (Reference default ``enable_amp=False``; the only implemented mode here is True.)"""
        _require_amp(enable_amp)
        assert (method in ("scale", "noise_scale", "noise", "scale4x", "noise_scale4x"))
        assert (method in {"scale", "scale4x"} or 0 <= noise_level and noise_level < 4)
        return tiled_render(x, self._model(method, noise_level), tile_size=tile_size, batch_size=batch_size,
                            enable_amp=enable_amp)

    def convert(self, x, alpha, method, noise_level, tile_size=None, batch_size=None,
                tta=False, enable_amp=True, output_device="cpu"):
        """waifu2x/utils.py:255-297.  (Reference default ``enable_amp=False``; the only implemented mode here is True.)"""
        _require_amp(enable_amp)
        assert (not torch.is_grad_enabled())
        assert (x.shape[0] == 3)
        assert (alpha is None or alpha.shape[0] == 1 and alpha.shape[1:] == x.shape[1:])
        assert (method in ("scale", "scale4x", "noise_scale", "noise_scale4x", "noise"))
        assert (method in {"scale", "scale4x"} or 0 <= noise_level and noise_level < 4)
        x = x.to(self.device)
        blank_alpha = True
        if alpha is not None:
            # check all 1 alpha channel (waifu2x/utils.py:266-268)
            blank_alpha = bool(torch.equal(alpha, torch.ones(alpha.shape, device=alpha.device, dtype=alpha.dtype)))
        if alpha is not None and not blank_alpha:
            alpha = alpha.to(self.device)
            x = self.alpha_pad(x, alpha, self._model(method, noise_level).i2i_offset)       # :269-271
        if tta:
            rgb = tta_merge([self.render(xx, method, noise_level, tile_size, batch_size, enable_amp)
                             for xx in tta_split(x)])                                         # :272-275
        else:
            rgb = self.render(x, method, noise_level, tile_size, batch_size, enable_amp)
        rgb = rgb.to(output_device)
        if alpha is not None and method in ("scale", "noise_scale", "scale4x", "noise_scale4x"):
            s = 4 if method in {"scale4x", "noise_scale4x"} else 2
            if not blank_alpha:
                model = self.scale4x_model if method in {"scale4x", "noise_scale4x"} else self.scale_model
                if model is not None:
                    # second render pass on the alpha plane (:282-287)
                    alpha = alpha.expand(3, alpha.shape[1], alpha.shape[2])
                    alpha = tiled_render(alpha, model, tile_size=tile_size, batch_size=batch_size,
                                         enable_amp=enable_amp).mean(0, keepdim=True)
                else:
                    alpha = F.interpolate(alpha.unsqueeze(0), scale_factor=s, mode="bilinear").squeeze(0)   # :288-291
            else:
                # all-ones alpha: the nearest upscale of ones is ones (:292-294)
                alpha = torch.ones((1, alpha.shape[1] * s, alpha.shape[2] * s), dtype=alpha.dtype, device=output_device)
            alpha = alpha.to(output_device)
        return rgb, alpha
