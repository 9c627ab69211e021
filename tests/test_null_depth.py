"""CPU checks of iw3's NULL depth model: the oracle against the golden of the real reference (tests/golden/null_depth.npz),
the host contract of NullDepthModel (iw3/null_depth_model.py:24-79) and its routing through create_depth_model, none of
which may touch CUDA, and the argument checks of nb200_null_depth."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import null_depth as ond
from tests.util import load_golden

G = load_golden("null_depth")


@pytest.mark.parametrize("spec", ond.CASES, ids=[c[0] for c in ond.CASES])
def test_oracle_matches_reference_golden(spec):
    case = spec[0]
    x = ond.frames(spec)
    assert float(x.double().sum()) == float(G[f"{case}/input_sum"])
    assert np.array_equal(x[..., :8, :8].numpy(), G[f"{case}/input_corner"])
    R = spec[4] or 392
    for tta, dil in ond.VARIANTS:
        key = f"{case}/t{tta}_d{dil}"
        y = ond.infer(x.clone(), spec[4], bool(tta), dil)
        assert tuple(y.shape) == tuple(G[f"{key}/shape"]) == (spec[1], 1, R, R), key
        assert np.array_equal(ond.digest(y.numpy()), G[f"{key}/sha256"]), key
        for i, c in enumerate(ond.crops(y)):
            assert np.array_equal(c.numpy(), G[f"{key}/crop{i}"]), (key, i)


def test_tta_is_the_plain_forward_and_chw_squeezes():
    """(m(x) + m(x)) * 0.5 == m(x) in fp32, which lets the engine run the kernel once under tta; CHW in -> 1,R,R out."""
    x = ond.frames(ond.CASES[3])
    assert torch.equal(ond.infer(x, 64, tta=True), ond.infer(x, 64, tta=False))
    assert ond.infer(x[0], 64).shape == (1, 64, 64)
    assert torch.equal(ond.infer(x[0], 64), ond.infer(x, 64)[0])


@pytest.fixture
def no_cuda(monkeypatch):
    from nunif_b200 import _lib

    def refuse(*a, **k):
        raise AssertionError("the NULL model's host surface must make no CUDA call")
    monkeypatch.setattr(_lib, "lib", refuse)


def test_host_contract(no_cuda):
    from nunif_b200.iw3 import BaseDepthModel, NullDepthModel, NullDepthNet
    m = NullDepthModel("NULL")
    assert isinstance(m, BaseDepthModel) and m.model_type == "NULL" and not m.loaded()
    assert NullDepthModel.get_name() == "NullDepth"
    assert NullDepthModel.supported("NULL") and not NullDepthModel.supported("Any_V2_S") and not NullDepthModel.supported("null")
    assert NullDepthModel.get_model_path("NULL") is None
    assert NullDepthModel.has_checkpoint_file("NULL") is True and NullDepthModel.has_checkpoint_file("Any_V2_S") is False
    assert not m.is_metric() and m.is_video_supported() and m.is_image_supported()
    assert NullDepthModel.multi_gpu_supported("NULL") is False       # the engine's single-GPU policy; the reference says True
    NullDepthModel.force_update()                                     # nothing to download: a no-op, not an error
    assert m.get_ema_buffer_size() == 1
    # load needs no weights and no device work; R is the resolution as given, 392 by default, not rounded to 14
    for res, want in ((None, 392), (518, 518), (512, 512), (500, 500), (1, 1)):
        mm = NullDepthModel("NULL").load(gpu=0, resolution=res)
        assert mm.loaded() and isinstance(mm.get_model(), NullDepthNet) and mm.get_model().resolution == want
        assert mm.device == torch.device("cuda", 0)
    with pytest.raises(ValueError):
        NullDepthNet(0)
    with pytest.raises(RuntimeError, match="CUDA"):
        NullDepthModel("NULL").load(gpu=-1)                             # the engine has no CPU path
    with pytest.raises(ValueError):
        NullDepthModel("NULL").load(gpu=[0, 1])
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        m.load(gpu=0).infer(torch.rand(1, 3, 8, 8))


def test_create_depth_model_routes_null(no_cuda):
    from nunif_b200.iw3 import NullDepthModel, create_depth_model
    from nunif_b200.iw3.depth_model_factory import NOT_BUILT
    assert "NULL" not in NOT_BUILT
    m = create_depth_model("NULL")
    assert type(m) is NullDepthModel and m.model_type == "NULL"
    m.load(gpu=0, resolution=518)
    assert m.get_model().resolution == 518


def test_header_declares_null_depth():
    from nunif_b200 import _lib
    from tests.test_abi import declared_symbols
    assert "nb200_null_depth" in declared_symbols() and "nb200_null_depth" in _lib.SIGNATURES


def test_null_depth_refuses_bad_arguments():
    """The checks run before anything touches the device, so they hold without a GPU."""
    from nunif_b200 import build, _lib
    build.build()
    lib = _lib.lib()
    buf = ctypes.create_string_buffer(64)
    x, out = ctypes.c_void_p(ctypes.addressof(buf)), ctypes.c_void_p(ctypes.addressof(buf) + 32)
    for args, msg in (((None, 1, 8, 8, 4, out), "null pointer"), ((x, 1, 8, 8, 4, None), "null pointer"),
                      ((x, 0, 8, 8, 4, out), "bad shape"), ((x, 1, 0, 8, 4, out), "bad shape"),
                      ((x, 1, 8, -1, 4, out), "bad shape"), ((x, 1, 8, 8, 0, out), "bad shape"),
                      ((x, 1, 8, 8, 4, x), "alias")):
        assert lib.nb200_null_depth(*args, None) != 0, args
        assert msg in lib.nb200_last_error().decode(), (args, lib.nb200_last_error())
