"""Frame scheduling for video callbacks: the role of ``FrameCallbackPool`` (nunif/utils/video.py:1622-1757) and of the
per-thread CUDA streams iw3 wraps around it (iw3/utils.py:709-831), re-designed for one process per GPU.

The reference overlaps host<->device copies with compute by running the batch callback on a thread pool (one stream per
thread) and converting frames with blocking ``to_tensor`` / ``to_frame`` calls.  Here the overlap comes from the hardware
queues directly - no threads, no locks, deterministic ticket order:

    slot ring (depth R, default 3), each slot = pinned uint8 input batch + device uint8 batch + pinned uint8 output batch
    copy-in stream   H2D of slot k+1 ...........  |  under
    compute stream   uint8->float (csrc/frame_ops.cu), frame_callback(batch BCHW float) , float->uint8   of slot k
    copy-out stream  D2H of slot k-1 ...........  |  under

``pipeline(frame)`` queues one HWC uint8 (or uint16) frame and returns the list of finished frames that are next in
submission order (possibly empty) - the calling convention of ``FrameCallbackPool.__call__``; ``pipeline(None)`` /
``finish()`` drains.  ``frame_callback(batch)`` receives B,3,H,W float32 in [0,1] on the GPU and returns B',3,H',W' float
(B' may differ from B: models with look-ahead buffers emit later), exactly what the reference's batch callbacks do.

``hdr2sdr`` is the reference's HDR input stage (video.py:309-416, applied by input_reformatter :1025-1041 when
``use_hdr2sdr`` holds): PQ / HLG BT.2020 rgb48 frames tone-mapped to BT.709 / BT.601 SDR by csrc/hdr2sdr.cu.
``FrameBatchPipeline(..., hdr2sdr=(color_trc, output_colorspace))`` runs it as the uint16 -> float conversion of each batch.

``FrameBatchPipeline(..., grain=(strength, speed[, seed]))`` is waifu2x's video film grain (waifu2x/ui_utils.py:167-175):
the float -> uint8 / uint16 conversion of each callback output becomes the fused temporal grain + quantise kernel
(csrc/rgb_noise.cu), whose noise buffer stays on the device and advances over the emitted frames in ticket order.
"""
import ctypes

import torch

from .. import _lib
from ..iw3.frames import hwc_to_chw_float, chw_float_to_hwc
from .rgb_noise import TemporalGrain

COLORSPACE_BT2020 = 9
COLOR_TRC_SMPTE2084 = 16            # PQ (HDR10)
COLOR_TRC_ARIB_STD_B67 = 18         # HLG
_HDR2SDR_TARGETS = {"bt709", "bt709-tv", "bt709-pc", "bt601", "bt601-tv", "bt601-pc"}
_SDR_COLORSPACE = {"bt709": 0, "bt601": 1}   # NB200_SDR_BT709 / NB200_SDR_BT601


def use_hdr2sdr(frame_colorspace, color_trc, target_colorspace):
    """The condition of input_reformatter (video.py:1026-1029): a BT.2020 frame of a PQ or HLG stream, written out as
    BT.709 / BT.601 (``target_colorspace`` with or without its -tv / -pc suffix)."""
    return (frame_colorspace == COLORSPACE_BT2020 and color_trc in {COLOR_TRC_SMPTE2084, COLOR_TRC_ARIB_STD_B67}
            and target_colorspace in _HDR2SDR_TARGETS)


def _check_hdr2sdr_args(color_trc, output_colorspace, output="uint16"):
    if color_trc not in (COLOR_TRC_SMPTE2084, COLOR_TRC_ARIB_STD_B67):
        raise ValueError(f"color_trc must be {COLOR_TRC_SMPTE2084} (PQ) or {COLOR_TRC_ARIB_STD_B67} (HLG), got {color_trc!r}")
    if output_colorspace not in _SDR_COLORSPACE:
        raise ValueError(f"output_colorspace must be 'bt709' or 'bt601', got {output_colorspace!r}")
    if output not in ("uint16", "float"):
        raise ValueError(f"output must be 'uint16' or 'float', got {output!r}")


def hdr2sdr(x, color_trc, output_colorspace, pq_exposure=110.0, pq_white_point=5.0, hlg_exposure=1.2, hlg_white_point=0.8,
            hlg_saturation_gain=0.9, output="uint16", device=None):
    """nunif/utils/video.py:309-416 on rgb48 frames: x uint16 HWC or BHWC, full range, BT.2020 with the PQ (color_trc 16)
    or HLG (18) transfer, moved to ``device`` (default: x's device, which must be a GPU).

    output="uint16": the tone-mapped rgb48 frame(s) hdr2sdr returns, same shape as x.
    output="float":  that frame / 65535 as float32 CHW / BCHW - the frame ``to_tensor`` / ``hwc_to_chw_float`` would make of
                     it, without the intermediate uint16 frame."""
    _check_hdr2sdr_args(color_trc, output_colorspace, output)
    if not torch.is_tensor(x) or x.dtype != torch.uint16:
        raise ValueError("hdr2sdr expects a uint16 (rgb48) tensor")
    if x.ndim not in (3, 4) or x.shape[-1] != 3:
        raise ValueError(f"hdr2sdr expects HWC or BHWC frames with 3 channels, got shape {tuple(x.shape)}")
    dev = torch.device(device) if device is not None else x.device
    if dev.type != "cuda":
        raise ValueError("hdr2sdr runs on a CUDA (sm_90) device: pass device= a GPU or a CUDA tensor")
    xc = x.to(dev).contiguous()
    B = 1 if x.ndim == 3 else x.shape[0]
    H, W = x.shape[-3], x.shape[-2]
    if output == "float":
        out = torch.empty((B, 3, H, W), dtype=torch.float32, device=xc.device)
    else:
        out = torch.empty((B, H, W, 3), dtype=torch.uint16, device=xc.device)
    params = (ctypes.c_double * 5)(pq_exposure, pq_white_point, hlg_exposure, hlg_white_point, hlg_saturation_gain)
    with torch.cuda.device(xc.device):
        _lib.check(_lib.lib().nb200_hdr2sdr(_lib.ptr(xc), B, H, W, int(color_trc), _SDR_COLORSPACE[output_colorspace], params,
                                            int(output == "float"), _lib.ptr(out), _lib.stream_ptr(xc.device)))
    return out[0] if x.ndim == 3 else out


class _Slot:
    __slots__ = ("h_in", "d_in", "h_out", "n", "n_out", "ready", "done", "out_shape", "direct")

    def __init__(self):
        self.h_in = self.d_in = self.h_out = None
        self.n = self.n_out = 0
        self.direct = 0          # bit i: frame i of the batch being filled was copied straight from the caller's pinned memory
        self.ready = torch.cuda.Event()
        self.done = torch.cuda.Event()
        self.out_shape = None


class FrameBatchPipeline:
    def __init__(self, frame_callback, batch_size, device="cuda:0", depth=3, use_16bit=False, copy_output=True, hdr2sdr=None,
                 grain=None):
        assert batch_size > 0 and depth >= 2
        # (strength, speed[, seed]): add temporal film grain to every emitted frame as it is converted for the encoder
        if grain is not None:
            if len(grain) not in (2, 3):
                raise ValueError("grain must be (strength, speed) or (strength, speed, seed)")
            grain = TemporalGrain(*grain)
        self.grain = grain
        # (color_trc, output_colorspace): tone-map each uint16 batch to SDR (hdr2sdr(..., output="float")) in place of the
        # plain uint16 -> float conversion, so the callback receives SDR frames
        if hdr2sdr is not None:
            if not use_16bit:
                raise ValueError("hdr2sdr needs use_16bit=True (rgb48 frames)")
            color_trc, output_colorspace = hdr2sdr
            _check_hdr2sdr_args(color_trc, output_colorspace)
            hdr2sdr = (color_trc, output_colorspace)
        self.hdr2sdr = hdr2sdr
        self.frame_callback = frame_callback
        self.batch_size = int(batch_size)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("FrameBatchPipeline runs on a CUDA (sm_90) device")
        self.dtype = torch.uint16 if use_16bit else torch.uint8
        self.bits = 16 if use_16bit else 8
        self.slots = [_Slot() for _ in range(depth)]
        self.s_in = torch.cuda.Stream(self.device)
        self.s_out = torch.cuda.Stream(self.device)
        self.head = 0            # slot being filled
        self.inflight = []       # slot indices in submission (ticket) order
        self.fill = 0
        self.submitted = self.returned = 0
        # False: returned frames are VIEWS of the slot's pinned output batch, valid until `depth` more batches have been submitted
        # (an encoder that consumes each frame immediately saves one host memcpy per frame)
        self.copy_output = copy_output

    # ---- host side
    def _slot_buffers(self, slot, frame):
        shape = (self.batch_size,) + tuple(frame.shape)
        if slot.h_in is None or tuple(slot.h_in.shape) != shape:
            slot.h_in = torch.empty(shape, dtype=self.dtype).pin_memory()
            slot.d_in = torch.empty(shape, dtype=self.dtype, device=self.device)

    def __call__(self, frame):
        if frame is None:
            return self.finish()
        frame = torch.as_tensor(frame)
        assert frame.ndim == 3 and frame.shape[2] == 3 and frame.dtype == self.dtype, "HWC uint8/uint16 frame expected"
        slot = self.slots[self.head]
        if self.fill > 0 and tuple(frame.shape) != tuple(slot.h_in.shape[1:]):
            # the frame size changed inside a batch: submit the frames of the old size as a partial batch
            self._launch(slot, self.fill)
            slot = self.slots[self.head]
        if self.fill == 0:
            if self.head in self.inflight:           # ring is full: the oldest ticket must be returned first
                out = self._collect(block=True)
            else:
                out = []
            self._slot_buffers(slot, frame)
        else:
            out = []
        if frame.is_pinned() and frame.is_contiguous():
            # zero-copy submit: the frame's own page-locked memory is the DMA source (a decoder writing into pinned buffers, the
            # bench); the caller must not overwrite it before the batch it belongs to has been launched
            with torch.cuda.stream(self.s_in):
                slot.d_in[self.fill].copy_(frame, non_blocking=True)
            slot.direct |= 1 << self.fill
        else:
            slot.h_in[self.fill].copy_(frame)        # host memcpy into the pinned batch (pageable source, e.g. a PyAV ndarray)
        self.fill += 1
        if self.fill == self.batch_size:
            self._launch(slot, self.fill)
        return out + self._collect(block=False)

    def _launch(self, slot, n):
        comp = torch.cuda.current_stream(self.device)
        with torch.cuda.stream(self.s_in):
            if slot.direct == 0:
                slot.d_in[:n].copy_(slot.h_in[:n], non_blocking=True)
            else:
                for i in range(n):                   # frames staged on the host go now; the pinned ones are already in flight
                    if not (slot.direct >> i) & 1:
                        slot.d_in[i].copy_(slot.h_in[i], non_blocking=True)
            slot.ready.record(self.s_in)
        slot.direct = 0
        comp.wait_event(slot.ready)
        with torch.inference_mode():
            if self.hdr2sdr is None:
                x = hwc_to_chw_float(slot.d_in[:n])
            else:
                x = hdr2sdr(slot.d_in[:n], *self.hdr2sdr, output="float")
            y = self.frame_callback(x)
            if y is not None and y.numel() > 0:
                if self.grain is None:
                    u = chw_float_to_hwc(y, use_16bit=self.bits == 16)
                else:
                    u = self.grain(y, dtype=self.dtype)
                slot.n_out = u.shape[0]
                if slot.h_out is None or tuple(slot.h_out.shape[1:]) != tuple(u.shape[1:]) or slot.h_out.shape[0] < u.shape[0]:
                    slot.h_out = torch.empty((max(u.shape[0], self.batch_size),) + tuple(u.shape[1:]), dtype=self.dtype).pin_memory()
                ev = torch.cuda.Event()
                ev.record(comp)
                self.s_out.wait_event(ev)
                with torch.cuda.stream(self.s_out):
                    slot.h_out[:slot.n_out].copy_(u, non_blocking=True)
                    u.record_stream(self.s_out)
                    slot.done.record(self.s_out)
            else:
                slot.n_out = 0
                slot.done.record(comp)
        slot.n = n
        self.inflight.append(self.head)
        self.submitted += 1
        self.head = (self.head + 1) % len(self.slots)
        self.fill = 0

    def _collect(self, block):
        out = []
        while self.inflight:
            slot = self.slots[self.inflight[0]]
            if not block and not slot.done.query():
                break
            slot.done.synchronize()
            out += [slot.h_out[i].clone() if self.copy_output else slot.h_out[i] for i in range(slot.n_out)]
            self.inflight.pop(0)
            self.returned += 1
            block = False
        return out

    def finish(self):
        """Submit the partial batch and return every remaining frame in order (FrameCallbackPool.finish)."""
        if self.fill > 0:
            self._launch(self.slots[self.head], self.fill)
        out = []
        while self.inflight:
            out += self._collect(block=True)
        return out
