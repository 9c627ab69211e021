"""SBD.detect_boundary (nunif/utils/shot_boundary_detection.py:20-111): the frames at which a shot ends, found by TransNetV2
over overlapping windows.

The caller decodes the video at 48x27 (the reference's ``scale=48:27:flags=bilinear``) and passes the frames with their pts;
decoding, ``max_fps``, start/end time and the stop events are not part of this module.  The windowing is the reference's,
step for step (``WindowQueue``): batches of ``padding_size`` frames as FrameCallbackPool delivers them, a short last batch
padded with its last frame, ``padding_size`` copies of the first frame in front, one window whenever ``window_size //
padding_size`` chunks are queued (predictions ``[padding_size:-padding_size]`` kept, the oldest chunks dropped), then chunks of
the last frame until the last kept pts is the last frame's.  Windows are assembled on the device, several ready windows share
one forward (each is computed on its own), and the predictions stay on the device until the one host synchronisation at
the end, where the reference synchronises once per window."""
import numpy as np
import torch

from ..iw3.frames import hwc_to_chw_float
from .transnetv2 import TransNetV2

WINDOW_BATCH = 8   # ready windows that share one forward


class WindowQueue:
    """The chunk queue of detect_boundary over arbitrary per-frame items (device frames, or frame indices for planning).
    ``push(items, pts)`` takes one FrameCallbackPool batch (at most ``padding_size`` frames) and ``finish()`` the end of the
    stream; both return the windows that became ready, as (items, pts) lists of ``window_size``."""

    def __init__(self, window_size=100, padding_size=25):
        assert (window_size % padding_size == 0 and
                window_size // padding_size >= 3)  # pad1 + frames + pad2
        self.window_size, self.padding_size = window_size, padding_size
        self.chunks = []
        self.first = True
        self.frame_count = 0
        self.last_kept_pts = None

    def _ready(self):
        if len(self.chunks) != self.window_size // self.padding_size:
            return []
        items = [x for c, _ in self.chunks for x in c]
        pts = [p for _, c in self.chunks for p in c]
        self.last_kept_pts = pts[self.window_size - self.padding_size - 1]
        del self.chunks[:(self.window_size - self.padding_size * 2) // self.padding_size]
        return [(items, pts)]

    def push(self, items, pts):
        assert 0 < len(items) == len(pts) <= self.padding_size
        self.frame_count += len(items)
        n = self.padding_size - len(items)
        items, pts = list(items) + [items[-1]] * n, list(pts) + [pts[-1]] * n
        if self.first:
            self.first = False
            self.chunks.append(([items[0]] * self.padding_size, [pts[0]] * self.padding_size))
        self.chunks.append((items, pts))
        return self._ready()

    def finish(self):
        if self.frame_count == 0:
            raise ValueError("detect_boundary: no frames")
        last_item, last_pts = self.chunks[-1][0][-1], self.chunks[-1][1][-1]
        out = []
        while self.last_kept_pts is None or self.last_kept_pts != last_pts:
            self.chunks.append(([last_item] * self.padding_size, [last_pts] * self.padding_size))
            out += self._ready()
        return out


def window_plan(pts, window_size=100, padding_size=25):
    """The windows detect_boundary runs for a stream of frames with these pts, as lists of frame indices, and the
    frame count the kept predictions are cut to."""
    q = WindowQueue(window_size, padding_size)
    windows = []
    for s in range(0, len(pts), padding_size):
        idx = list(range(s, min(s + padding_size, len(pts))))
        windows += [w for w, _ in q.push(idx, [pts[i] for i in idx])]
    windows += [w for w, _ in q.finish()]
    return windows, q.frame_count


def _to_device(batch, device):
    x = torch.stack([torch.as_tensor(np.ascontiguousarray(f)) if not torch.is_tensor(f) else f for f in batch])
    if not x.is_cuda:
        x = x.pin_memory().to(device, non_blocking=True)
    return hwc_to_chw_float(x.to(device))


def _predict(frames, device, window_size, padding_size, model):
    """Every frame's boundary probability (a device tensor, cut to the frame count) and the pts of the kept predictions;
    no host synchronisation."""
    q = WindowQueue(window_size, padding_size)
    ready, preds, kept_pts = [], [], []

    def run(windows):
        if not windows:
            return
        x = torch.stack([torch.stack(items) for items, _ in windows])
        with torch.inference_mode():
            one_hot, _ = model(x)
        preds.append(torch.sigmoid(one_hot.flatten(1))[:, padding_size:-padding_size].flatten())
        kept_pts.extend(p for _, pts in windows for p in pts[padding_size:-padding_size])

    def queue(windows):
        ready.extend(windows)
        if len(ready) >= WINDOW_BATCH:
            run(ready)
            ready.clear()

    batch, batch_pts = [], []
    for frame, pts in frames:
        batch.append(frame)
        batch_pts.append(int(pts))
        if len(batch) == padding_size:
            queue(q.push(list(_to_device(batch, device)), batch_pts))
            batch, batch_pts = [], []
    if batch:
        queue(q.push(list(_to_device(batch, device)), batch_pts))
    queue(q.finish())
    run(ready)
    n = q.frame_count
    return torch.cat(preds)[:n], kept_pts[:n]


def detect_boundary(frames, device="cuda:0", window_size=100, padding_size=25, threshold=0.5, model=None):
    """``frames``: iterable of (frame, pts), frame an HWC uint8 / uint16 27x48 image (numpy or torch).  Returns the set of pts
    whose shot-boundary probability exceeds ``threshold`` (the pts is the END of a segment).  ``model`` defaults to
    TransNetV2.load(device)."""
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("detect_boundary runs TransNetV2 on a CUDA (sm_90) device; there is no CPU path")
    model = model if model is not None else TransNetV2.load(device)
    prob, pts = _predict(frames, device, window_size, padding_size, model)
    hit = (prob > threshold).cpu().tolist()
    return set(p for p, h in zip(pts, hit) if h)
