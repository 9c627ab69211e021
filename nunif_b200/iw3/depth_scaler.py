"""Mirror of iw3/depth_scaler.py: the stateless per-frame normaliser (:4-17, with the disparity mapper of
iw3/mapper.py, nunif_b200/iw3/mapper.py, fused into the same pass) and the stateful ``EMAMinMaxScaler`` (:64-142) whose min/max ring and EMA
values live on the device (csrc/ema_scaler.cu) - no host synchronisation per frame."""
import ctypes
import torch
from .. import _lib
from ._common import prep
from .mapper import descriptor, apply_mapper


def minmax_normalize(depth, mapper="none", return_minmax=False):
    """depth: B,1,h,w (or 1,h,w): per-frame (x-min)/(max-min) clamp[0,1], then get_mapper(mapper) (any name of
    iw3/mapper.py, blends and chains included) in the same pass.  No host sync (the reference's ``if scale > 0``
    syncs)."""
    squeeze = depth.ndim == 3
    d = prep(depth.unsqueeze(0) if squeeze else depth, "depth")
    desc = descriptor(mapper)
    B = d.shape[0]
    n = d[0].numel()
    out = torch.empty_like(d)
    mm = torch.empty((B, 2), device=d.device, dtype=torch.float32) if return_minmax else None
    with torch.cuda.device(d.device):
        _lib.check(_lib.lib().nb200_minmax_mapper(_lib.ptr(d), B, n, ctypes.byref(desc), _lib.ptr(out), _lib.ptr(mm),
                                                  _lib.stream_ptr(d.device)))
    out = out[0] if squeeze else out
    return (out, mm) if return_minmax else out


def depth_mapper(depth, mapper="none"):
    """iw3/mapper.py get_mapper(mapper)(depth) for any mapper name; an identity mapper returns ``depth`` itself."""
    return apply_mapper(depth, descriptor(mapper))


class EMAMinMaxScaler:
    """depth_scaler.py:64-142.  ``scaler(frame)`` queues the frame and returns the oldest queued frame normalised with the
    EMA of the look-ahead ring's amin/amax - or ``None`` while the ring fills (:98-103).  ``min_value`` / ``max_value`` are
    0-dim DEVICE tensors (views of the scaler state), never read on the host.

      SimpleMinMaxScaler: decay=0, buffer_size=1;  IncrementalEMAScaler: decay=0.75, buffer_size=1;
      WindowEMAScaler: decay=0.9, buffer_size=30   (:65-67)
    """
    _MODES = {"minmax": 0, "max": 1}

    def __init__(self, decay=0, buffer_size=1, mode="minmax"):
        assert mode in self._MODES
        assert buffer_size > 0
        self.mode = mode
        self._h = None
        self._device = None
        self.frame_queue = []
        self.decay, self.buffer_size = float(decay), int(buffer_size)
        self._filled_once = False

    def __del__(self):
        try:
            if self._h:
                _lib.lib().nb200_ema_scaler_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def _handle(self, device):
        if self._h is None or self._device != device:
            if self._h is not None:
                _lib.lib().nb200_ema_scaler_destroy(self._h)
            h = ctypes.c_void_p()
            with torch.cuda.device(device):
                _lib.check(_lib.lib().nb200_ema_scaler_create(self.buffer_size, self.decay, self._MODES[self.mode], ctypes.byref(h)))
            self._h, self._device = h, device
        return self._h

    def reset(self, decay=None, buffer_size=None, **kwargs):
        """:76-86 (the frame queue is dropped, like the reference)."""
        if decay is not None:
            self.decay = float(decay)
        if buffer_size is not None:
            self.buffer_size = int(buffer_size)
        self.frame_queue = []
        self._filled_once = False
        if self._h is not None:
            with torch.cuda.device(self._device):
                _lib.check(_lib.lib().nb200_ema_scaler_reset(self._h, self.decay, self.buffer_size))

    def _normalize(self, frame, from_ring, return_minmax):
        out = torch.empty_like(frame)
        mm = torch.empty(2, device=frame.device, dtype=torch.float32) if return_minmax else None
        with torch.cuda.device(frame.device):
            _lib.check(_lib.lib().nb200_ema_scaler_normalize(self._h, _lib.ptr(frame), frame.numel(), 1 if from_ring else 0, -1.0,
                                                             _lib.ptr(out), _lib.ptr(mm), _lib.stream_ptr(frame.device)))
        return (out, mm[0], mm[1]) if return_minmax else out

    def __call__(self, frame, return_minmax=False):
        return self.update(frame, return_minmax=return_minmax)

    def update(self, frame, return_minmax=False):
        frame = prep(frame, "frame")
        h = self._handle(frame.device)
        self.frame_queue.append(frame)
        filled = ctypes.c_int(0)
        with torch.cuda.device(frame.device):
            _lib.check(_lib.lib().nb200_ema_scaler_update(h, _lib.ptr(frame), frame.numel(), ctypes.byref(filled),
                                                          _lib.stream_ptr(frame.device)))
        if not filled.value:
            return (None, None, None) if return_minmax else None
        self._filled_once = True
        return self._normalize(self.frame_queue.pop(0), False, return_minmax)

    def flush(self, return_minmax=False):
        """:122-142: the queued frames with the last EMA values (or the ring's amin/amax if none exists yet)."""
        if not self.frame_queue:
            self.reset()
            return []
        frames = [self._normalize(f, not self._filled_once, return_minmax) for f in self.frame_queue]
        self.reset()
        return frames
