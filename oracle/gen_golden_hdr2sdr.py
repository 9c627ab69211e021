"""Generate tests/golden/hdr2sdr.npz by running the REAL reference nunif/utils/video.py:309-416 ``hdr2sdr`` on the CPU, in
fp32, on oracle/hdr2sdr.py golden_inputs() under every CONFIGS entry.

PyAV is not needed: a stand-in `av` module covers what nunif.utils.video touches at import and what hdr2sdr touches
(ColorRange / Colorspace members, VideoFrame.from_ndarray, which here returns a frame object holding the array), and the
input "frame" is an object whose to_ndarray returns the fixed rgb48 array.

Run from the repository root, as a module:
    PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=<nunif checkout> python -m oracle.gen_golden_hdr2sdr

  in/<frame>/checksum, in/<frame>/corner   oracle.hdr2sdr.input_checksum and the top-left 4 x 4 pixels of the input
  out/<config>/{gray,edges}/delta          the uint16 [H][W][3] rgb48 frame hdr2sdr returned, as int32 [H*W][3] raster deltas
  out/<config>/perm/sha256, sample         its SHA-256 and its pixels at oracle.hdr2sdr.perm_sample_index()
                                           (oracle.hdr2sdr.encode_output / reference_output)
"""
import enum
import os
import sys
import types

import numpy as np
import torch

from oracle import hdr2sdr as ohs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "hdr2sdr.npz")


def install_av_stub():
    av = types.ModuleType("av")
    av.__version__ = "14.0.0"
    av.codecs_available = set()
    av.time_base = 1000000
    video = types.ModuleType("av.video")
    reformatter = types.ModuleType("av.video.reformatter")
    frame = types.ModuleType("av.video.frame")
    reformatter.ColorRange = enum.IntEnum("ColorRange", {"UNSPECIFIED": 0, "MPEG": 1, "JPEG": 2})
    reformatter.Colorspace = enum.IntEnum("Colorspace", {"ITU709": 1, "ITU601": 5})

    class VideoFrame:
        @staticmethod
        def from_ndarray(array, format):
            assert format == "rgb48le" and array.dtype == np.uint16
            f = VideoFrame()
            f.array = array.copy()
            return f

    frame.VideoFrame = VideoFrame
    av.video, video.reformatter, video.frame = video, reformatter, frame
    sys.modules.update({"av": av, "av.video": video, "av.video.reformatter": reformatter, "av.video.frame": frame})


class FakeFrame:
    """The rgb48 frame of a BT.2020 stream, as to_ndarray(format="rgb48le", dst_color_range=JPEG) returns it."""
    colorspace = 9
    color_range = 2
    pts = dts = opaque = None
    time_base = None

    def __init__(self, arr):
        self.arr = arr

    def to_ndarray(self, format, src_color_range=None, dst_color_range=None):
        assert format == "rgb48le"
        return self.arr.copy()


def main():
    install_av_stub()
    import nunif.utils.video as VU
    torch.set_num_threads(1)
    frames = ohs.golden_inputs()
    out = {}
    for name, x in frames.items():
        out[f"in/{name}/checksum"] = np.int64(ohs.input_checksum(x))
        out[f"in/{name}/corner"] = x[:4, :4].numpy()
    for cname, trc, cs, kw in ohs.CONFIGS:
        for name, x in frames.items():
            y = VU.hdr2sdr(FakeFrame(x.numpy()), trc, cs, device="cpu", **kw)
            for k, v in ohs.encode_output(name, y.array).items():
                out[f"out/{cname}/{name}/{k}"] = v
            assert np.array_equal(y.array, ohs.hdr2sdr(x, trc, cs, **kw).numpy()), (cname, name)
    for config in ohs.CONFIGS:
        for name, x in frames.items():
            y = VU.hdr2sdr(FakeFrame(x.numpy()), *config[1:3], device="cpu", **config[3]).array
            assert np.array_equal(ohs.reference_output(out, config, name, x), y), (config[0], name)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
