"""The ``BaseDepthModel`` contract of iw3 (iw3/base_depth_model.py:30-194) for engine-backed depth models.

``iw3.utils`` drives every depth model through this surface - ``load`` / ``loaded`` / ``compile_context`` (:41-45,
:97-132), ``infer``, the EMA look-ahead normaliser controls (:152-174) and ``minmax_normalize[_chw]`` /
``flush_minmax_normalize`` (:176-194) - e.g. ``process_image`` (iw3/utils.py:505-545) calls
``get_ema_buffer_size() -> infer() -> minmax_normalize_chw()``.  Differences that are deliberate and loud:

* the network is compiled ahead of time for sm_90a, so ``compile`` / ``compile_context`` have nothing to do;
* one process owns one GPU (DESIGN.md section 6): a list of several GPUs raises instead of building the reference's
  ``DeviceSwitchInference`` thread pool;
* checkpoints are read from disk only (``force_update`` would need the network and raises).
"""
import contextlib
import os
from os import path

import torch

from .depth_scaler import EMAMinMaxScaler

HUB_MODEL_DIR = os.environ.get(
    "NUNIF_B200_IW3_HUB_DIR",
    path.join(os.environ.get("NUNIF_HOME", path.expanduser("~/.nunif")), "iw3", "pretrained_models", "hub"))


def _device_of(gpu):
    """nunif.device.create_device for the one case the engine supports: a single CUDA ordinal."""
    if isinstance(gpu, (list, tuple)):
        if len(gpu) != 1:
            raise ValueError("nunif_b200 runs one process per GPU (torchrun); pass a single device id, "
                             "not the DeviceSwitchInference list form")
        gpu = gpu[0]
    if isinstance(gpu, torch.device):
        device = gpu
    elif isinstance(gpu, str):
        device = torch.device(gpu)
    else:
        if int(gpu) < 0:
            raise RuntimeError("nunif_b200 depth models need a CUDA (sm_90) device; there is no CPU path")
        device = torch.device("cuda", int(gpu))
    if device.type != "cuda":
        raise RuntimeError("nunif_b200 depth models need a CUDA (sm_90) device; there is no CPU path")
    return device


class BaseDepthModel:
    def __init__(self, model_type):
        self.device = None
        self.model = None
        self.model_type = model_type
        self.scaler = self.create_depth_scaler()
        self.limit_resolution = False

    # ---- to be provided by the concrete model (the reference's abstract methods, :47-95,148-150)
    @classmethod
    def get_name(cls):
        raise NotImplementedError

    @classmethod
    def supported(cls, model_type):
        raise NotImplementedError

    @classmethod
    def get_model_path(cls, model_type):
        raise NotImplementedError

    @classmethod
    def has_checkpoint_file(cls, model_type):
        return path.exists(cls.get_model_path(model_type))

    @classmethod
    def multi_gpu_supported(cls, model_type):
        return False

    @classmethod
    def force_update(cls):
        raise RuntimeError("nunif_b200 never downloads: place the checkpoint at get_model_path(model_type)")

    force_update_hub = staticmethod(lambda github, model: BaseDepthModel.force_update())

    def is_metric(self):
        raise NotImplementedError

    def load_model(self, model_type, resolution, device):
        raise NotImplementedError

    def infer(self, x, **kwargs):
        raise NotImplementedError

    # ---- lifecycle
    def create_depth_scaler(self):
        return EMAMinMaxScaler(decay=0, buffer_size=1)          # :37-39, may be overridden

    def load(self, gpu=0, resolution=None, limit_resolution=False, **kwargs):
        self.device = _device_of(gpu)
        self.limit_resolution = limit_resolution
        self.model = self.load_model(self.model_type, resolution=resolution, device=self.device, **kwargs)
        return self

    def loaded(self):
        return self.model is not None

    def get_model(self):
        return self.model

    def is_image_supported(self):
        return True

    def is_video_supported(self):
        return True

    def compile(self):
        """Nothing to do: the kernels are compiled ahead of time (the reference wraps the module in torch.compile, :137-146)."""

    def clear_compiled_model(self):
        pass

    def compile_context(self, enabled=True):
        return contextlib.nullcontext()

    # ---- stateful normaliser controls (:152-174)
    def enable_ema(self, decay, buffer_size=None):
        self.scaler.reset(decay=decay, buffer_size=buffer_size)

    def get_ema_state(self):
        return self.scaler.decay, self.scaler.buffer_size

    def disable_ema(self):
        self.scaler.reset(decay=0, buffer_size=1)

    def reset_ema(self, decay=None, buffer_size=None):
        self.scaler.reset(decay=decay, buffer_size=buffer_size)

    def reset_state(self):
        pass

    def reset(self):
        self.reset_ema()
        self.reset_state()

    def get_ema_buffer_size(self):
        return self.scaler.buffer_size

    # ---- normalisation (:176-194)
    def minmax_normalize_chw(self, depth, return_minmax=False):
        return self.scaler(depth, return_minmax=return_minmax)

    def flush_minmax_normalize(self, return_minmax=False):
        return self.scaler.flush(return_minmax=return_minmax)

    def minmax_normalize(self, depth, reset_ema=None):
        assert depth.ndim == 4
        flags = [False] * depth.shape[0] if reset_ema is None else list(reset_ema)
        assert len(flags) == depth.shape[0]
        out = []
        for frame, scene_end in zip(depth, flags):
            y = self.minmax_normalize_chw(frame)
            if y is not None:
                out.append(y)
            if scene_end:
                out.extend(self.flush_minmax_normalize())
                self.reset_ema()
        return out

    # ---- depth image files (:196-249): host-side PNG I/O, 16-bit like the reference.  The device path: save a uint16
    # map from depth_io.export_depth_u16; load_depth(..., device=) decodes on the GPU (depth_io.import_depth).
    @staticmethod
    def save_normalized_depth(depth, file_path, png_info={}, min_depth_value=None, max_depth_value=None):
        """``depth``: normalised fp32 (1,h,w), quantised here as the reference does, or the uint16 (h,w) map of
        ``export_depth_u16``, written as is."""
        from PIL import Image
        from PIL.PngImagePlugin import PngInfo
        info = dict(png_info)
        if min_depth_value is not None:
            info["iw3_min_depth_value"] = float(min_depth_value)
        if max_depth_value is not None:
            info["iw3_max_depth_value"] = float(max_depth_value)
        meta = PngInfo()
        for k, v in info.items():
            meta.add_text(k, str(v))
        if depth.dtype == torch.uint16:
            px = depth.cpu().numpy()
        else:
            px = (0xffff * torch.clamp(depth, 0, 1)).to(torch.uint16).squeeze(0).cpu().numpy()
        Image.fromarray(px).save(file_path, pnginfo=meta)

    @staticmethod
    def load_depth(file_path, device=None):
        """-> (depth (1,H,W) fp32, PNG text + filename).  With ``device`` the decoded map is uploaded as is and
        converted there (nb200_depth_import); without, on the host."""
        import numpy as np
        from PIL import Image
        with Image.open(file_path) as im:
            text = dict(getattr(im, "text", {}))
            arr = np.asarray(im)
        lo = hi = None
        try:
            lo, hi = float(text["iw3_min_depth_value"]), float(text["iw3_max_depth_value"])
        except (KeyError, ValueError, TypeError):
            lo = hi = None
        text["filename"] = file_path
        if device is not None:
            from .depth_io import import_depth
            return import_depth(arr, device, (lo, hi) if lo is not None else None), text
        depth = torch.from_numpy(arr.astype(np.float32))
        depth = depth.unsqueeze(0) if depth.ndim == 2 else depth.permute(2, 0, 1)
        if arr.dtype != np.float32:
            depth = torch.clamp(depth / 0xffff, 0, 1)
        if depth.shape[0] != 1:
            depth = depth.mean(dim=0, keepdim=True)
        if lo is not None and hi is not None:
            depth = depth * (hi - lo) + lo
        return depth, text
