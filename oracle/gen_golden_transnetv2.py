"""Generate tests/golden/transnetv2.npz by running the REAL reference (nagadomi/nunif, a checkout given by --reference or
$NUNIF_REFERENCE, imported read-only) on the CPU in fp32:
    python oracle/gen_golden_transnetv2.py --reference PATH/TO/nunif

TransNetV2 is the reference module loaded with synth.transnetv2_state_dict(0) (strict; TransNetV2.load is replaced so
nothing is downloaded).  detect_boundary is the reference function: PyAV is not installed, so nunif.utils.video is imported
over a stand-in `av` module that covers only its import, and VU.hook_frame is replaced by a feeder that pushes the seeded
frames (synth.shot_sequence, pts = 1001 * i + 7) through the real FrameCallbackPool and finishes it as hook_frame does.
Frames are stored as checksums (per-frame sums of the HWC integers); the tests regenerate them.
  win{01,255}_{one,many}     the logits [100] of one window (sequence WIN_SEED) at [0, 1] and at 0..255 scale
  len{L}_sum                 per-frame checksums of the length-L sequence (seed L) for L in LENGTHS
  len{L}_win_pts, _win_prob  pts [K][100] of every window detect_boundary ran and its sigmoid(one_hot) [K][100]
  len{L}_set                 the returned segment pts, sorted
  u16_*                      the same for a uint16 sequence of U16_LEN frames (seed U16_SEED)
  keys                       the state_dict key names of TransNetV2()
"""
import argparse
import enum
import os
import sys
import tempfile
import types
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nunif_b200 import synth  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "transnetv2.npz")
LENGTHS = (1, 24, 25, 26, 50, 75, 100, 101, 137, 260)
WIN_SEED = 500
U16_SEED, U16_LEN = 501, 137


def pts_of(n):
    return [1001 * i + 7 for i in range(n)]


def install_av_stub():
    """The part of PyAV nunif.utils.video touches at import time."""
    av = types.ModuleType("av")
    av.__version__ = "14.0.0"
    av.codecs_available = set()
    video = types.ModuleType("av.video")
    reformatter = types.ModuleType("av.video.reformatter")
    reformatter.ColorRange = enum.IntEnum("ColorRange", {"UNSPECIFIED": 0, "MPEG": 1, "JPEG": 2})
    reformatter.Colorspace = enum.IntEnum("Colorspace", {"ITU709": 1, "ITU601": 5})
    av.video, video.reformatter = video, reformatter
    sys.modules.update({"av": av, "av.video": video, "av.video.reformatter": reformatter})


class FakeFrame:
    def __init__(self, arr, pts):
        self.arr, self.pts = arr, pts
        bits = 16 if arr.dtype == np.uint16 else 8
        self.format = types.SimpleNamespace(components=[types.SimpleNamespace(bits=bits)])

    def to_ndarray(self, format):
        assert format == ("rgb48le" if self.arr.dtype == np.uint16 else "rgb24")
        return self.arr.copy()


def main():
    install_av_stub()
    import nunif.utils.video as VU
    import nunif.utils.shot_boundary_detection as SBD
    from nunif.utils.transnetv2 import TransNetV2

    sd = synth.transnetv2_state_dict(0)
    model = TransNetV2().eval()
    assert list(model.state_dict().keys()) == synth.transnetv2_keys()
    model.load_state_dict(sd, strict=True)
    TransNetV2.load = lambda self, map_location="cpu": (self.load_state_dict(sd, strict=True), self)[1]

    sequences = {}

    def feeder(video_file, callback_pool, **kwargs):
        for arr, p in sequences[video_file]:
            callback_pool(FakeFrame(arr, p))
        callback_pool(None)

    VU.hook_frame = feeder
    calls = []
    forward = TransNetV2.forward

    def recording_forward(self, x):
        out = forward(self, x)
        calls.append((x.clone(), torch.sigmoid(out[0]).flatten().clone()))
        return out

    TransNetV2.forward = recording_forward

    out = {"keys": np.array(synth.transnetv2_keys())}
    x = torch.from_numpy(synth.shot_sequence(WIN_SEED, 100)).permute(0, 3, 1, 2).float()
    for tag, xs in (("01", x / 255), ("255", x)):
        one, extra = forward(model, xs)
        out[f"win{tag}_one"], out[f"win{tag}_many"] = one.flatten(), extra["many_hot"].flatten()
    out["win_sum"] = x.flatten(1).sum(1).long()

    margin = []
    cases = [(f"len{n}", synth.shot_sequence(n, n)) for n in LENGTHS] + [("u16", synth.shot_sequence(U16_SEED, U16_LEN, True))]
    for tag, arr in cases:
        n = arr.shape[0]
        pts = pts_of(n)
        sequences[tag] = list(zip(arr, pts))
        scale = 65535.0 if arr.dtype == np.uint16 else 255.0
        lookup = {torch.from_numpy(a.astype(np.float32)).permute(2, 0, 1).div(scale).numpy().tobytes(): p for a, p in zip(arr, pts)}
        assert len(lookup) == n, "frames must be distinct to recover the window pts"
        calls.clear()
        seg = SBD.detect_boundary(tag, device="cpu")
        win_pts = [[lookup[f.contiguous().numpy().tobytes()] for f in xw] for xw, _ in calls]
        probs = torch.stack([p for _, p in calls])
        kept = probs[:, 25:75].flatten()[:n]
        margin.append(float((kept - 0.5).abs().min()))
        frac = float((kept > 0.5).float().mean())
        print(f"{tag}: {n} frames, {len(calls)} windows, {len(seg)} boundaries ({frac:.2f} of frames), min |p - 0.5| {margin[-1]:.2e}")
        out[f"{tag}_sum"] = arr.reshape(n, -1).astype(np.int64).sum(1)
        out[f"{tag}_win_pts"] = np.array(win_pts, dtype=np.int64)
        out[f"{tag}_win_prob"] = probs
        out[f"{tag}_set"] = np.array(sorted(seg), dtype=np.int64)
    print(f"smallest |p - 0.5| over all sequences: {min(margin):.3e}")
    np.savez_compressed(OUT, **{k: (v.numpy() if torch.is_tensor(v) else np.asarray(v)) for k, v in out.items()})
    print("wrote", OUT, os.path.getsize(OUT) // 1024, "KiB")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=os.environ.get("NUNIF_REFERENCE"), help="checkout of nagadomi/nunif")
    args = ap.parse_args()
    if not args.reference:
        ap.error("give the reference checkout with --reference or $NUNIF_REFERENCE")
    # the reference creates its home directory on import; keep it out of the (read-only) reference tree
    os.environ.setdefault("NUNIF_HOME", tempfile.mkdtemp(prefix="nunif_home_"))
    sys.path.insert(0, os.path.abspath(args.reference))
    torch.set_grad_enabled(False)
    torch.manual_seed(0)
    main()
