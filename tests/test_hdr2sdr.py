"""CPU: the hdr2sdr oracle (oracle/hdr2sdr.py) against the real reference's output (tests/golden/hdr2sdr.npz, made by
oracle/gen_golden_hdr2sdr.py from nunif/utils/video.py:309-416), the use_hdr2sdr condition (video.py:1026-1029), and the
argument checks of the engine's hdr2sdr and FrameBatchPipeline(hdr2sdr=...), which refuse before touching a device."""
import numpy as np
import pytest
import torch

from oracle import hdr2sdr as ohs
from tests.util import load_golden


@pytest.fixture(scope="module")
def golden():
    return load_golden("hdr2sdr")


@pytest.fixture(scope="module")
def inputs(golden):
    frames = ohs.golden_inputs()
    for name, x in frames.items():
        assert ohs.input_checksum(x) == int(golden[f"in/{name}/checksum"]), f"{name}: regenerated input drifted"
        assert np.array_equal(x[:4, :4].numpy(), golden[f"in/{name}/corner"]), name
    return frames


@pytest.mark.parametrize("config", ohs.CONFIGS, ids=[c[0] for c in ohs.CONFIGS])
def test_oracle_matches_reference_bit_exact(config, golden, inputs):
    cname, trc, cs, kw = config
    for name, x in inputs.items():
        got = ohs.hdr2sdr(x, trc, cs, **kw).numpy()
        if name in ohs.FULL_FRAMES:
            assert np.array_equal(got, ohs.reference_output(golden, config, name, x)), (cname, name)
        else:
            key = f"out/{cname}/{name}/"
            assert np.array_equal(got.reshape(-1, 3)[ohs.perm_sample_index()], golden[key + "sample"]), (cname, name)
            assert np.array_equal(ohs.digest(got), golden[key + "sha256"]), (cname, name)


def _reference_condition(frame_colorspace, color_trc, target_colorspace):
    # video.py:1026-1029, verbatim but for the names
    return (frame_colorspace == 9 and
            color_trc in {16, 18} and
            target_colorspace in {"bt709", "bt709-tv", "bt709-pc",
                                  "bt601", "bt601-tv", "bt601-pc"})


def test_use_hdr2sdr_truth_table():
    from nunif_b200.nunif.video import use_hdr2sdr
    n_true = 0
    for fcs in (0, 1, 2, 5, 6, 7, 8, 9, 10):
        for trc in (1, 2, 6, 8, 13, 14, 15, 16, 17, 18):
            for target in ("bt709", "bt709-tv", "bt709-pc", "bt601", "bt601-tv", "bt601-pc", "bt2020", "bt2020-tv", "auto",
                           "bt709-xx", "BT709", "", None):
                want = _reference_condition(fcs, trc, target)
                assert use_hdr2sdr(fcs, trc, target) == want, (fcs, trc, target)
                n_true += want
    assert n_true == 2 * 6


def test_hdr2sdr_rejects_bad_arguments_before_the_device():
    from nunif_b200.nunif.video import hdr2sdr
    x = torch.zeros(4, 6, 3, dtype=torch.uint16)
    bad = [
        dict(x=x.to(torch.uint8)),
        dict(x=x.float()),
        dict(x=x.numpy()),
        dict(x=x[..., :2]),
        dict(x=x[0]),
        dict(x=x.reshape(1, 1, 4, 6, 3)),
        dict(color_trc=1),
        dict(color_trc=17),
        dict(output_colorspace="bt2020"),
        dict(output_colorspace="bt709-tv"),
        dict(output="uint8"),
        dict(device="cpu"),
        dict(),                                   # a CPU tensor and no device: nowhere to run
    ]
    for kw in bad:
        args = dict(x=x, color_trc=16, output_colorspace="bt709")
        args.update(kw)
        with pytest.raises(ValueError):
            hdr2sdr(args.pop("x"), args.pop("color_trc"), args.pop("output_colorspace"), **args)


def test_pipeline_hdr2sdr_option_is_checked():
    from nunif_b200.nunif.video import FrameBatchPipeline
    with pytest.raises(ValueError, match="use_16bit"):
        FrameBatchPipeline(lambda x: x, 2, hdr2sdr=(16, "bt709"))
    with pytest.raises(ValueError):
        FrameBatchPipeline(lambda x: x, 2, use_16bit=True, hdr2sdr=(1, "bt709"))
    with pytest.raises(ValueError):
        FrameBatchPipeline(lambda x: x, 2, use_16bit=True, hdr2sdr=(18, "bt2020"))
