"""CPU: the film-grain oracle (oracle/rgb_noise.py) against the real reference's output (tests/golden/rgb_noise.npz, made by
oracle/gen_golden_rgb_noise.py from nunif/utils/rgb_noise.py), the half-resolution nearest rule against F.interpolate, the
numpy restatement of the engine's Philox4x32-10 against published known answers, and the engine's argument checks, which
refuse before any CUDA call."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import rgb_noise as orn
from tests.util import load_golden


@pytest.fixture(scope="module")
def golden():
    return load_golden("rgb_noise")


def ulp_diff(a, b):
    """|a - b| in fp32 ulps (both finite, same sign region)."""
    ia = np.asarray(a, np.float32).view(np.int32).astype(np.int64)
    ib = np.asarray(b, np.float32).view(np.int32).astype(np.int64)
    return np.abs(ia - ib)


@pytest.mark.parametrize("case", orn.NOISE_CASES, ids=[c[0] for c in orn.NOISE_CASES])
def test_oracle_noise_matches_reference_bit_exact(case, golden):
    name, shape, level, seed = case
    torch.manual_seed(seed)
    n = orn.rgb_noise_like(torch.zeros(shape), level).numpy()
    if name in orn.FULL_NOISE:
        assert np.array_equal(orn.digest(n), golden[f"noise/{name}/sha256"]), name
        for i, (sy, sx) in enumerate(orn.CROPS):
            assert np.array_equal(n[..., sy, sx], golden[f"noise/{name}/crop{i}"]), (name, i)
    else:
        assert np.array_equal(n, golden[f"noise/{name}"]), name


def test_oracle_apply_matches_reference(golden):
    for i, (name, shape) in enumerate(orn.APPLY_CASES):
        rgb = orn.golden_rgb(shape, 100 + i)
        noise = torch.from_numpy(golden[f"apply/{name}/noise"])
        for pname, kw in orn.PARAMS.items():
            got = orn.apply_rgb_noise(rgb.clone(), noise.clone(), **kw).numpy()
            want = golden[f"apply/{name}/{pname}"]
            assert int(ulp_diff(got, want).max()) <= 1, (name, pname)


def test_oracle_temporal_matches_reference(golden):
    buf = None
    for t, shape in enumerate(orn.TEMPORAL_SHAPES):
        rgb = orn.golden_rgb(shape, 300 + t)
        torch.manual_seed(400 + t)
        noise = orn.rgb_noise_like(rgb)
        assert np.array_equal(noise.numpy(), golden[f"temporal/noise{t}"]), t
        buf = orn.temporal_step(buf, noise, orn.TEMPORAL_SPEED)
        assert np.array_equal(buf.numpy(), golden[f"temporal/buffer{t}"]), t
        y = orn.apply_rgb_noise(rgb, buf, strength=orn.TEMPORAL_STRENGTH)
        assert int(ulp_diff(y.numpy(), golden[f"temporal/out{t}"]).max()) <= 1, t
        assert np.array_equal(orn.from_tensor(y, 8).numpy(), golden[f"temporal/u8_{t}"]), t
        assert np.array_equal(orn.from_tensor(y, 16).numpy(), golden[f"temporal/u16_{t}"]), t


def test_nearest_rule_matches_interpolate():
    """The index rule the oracle and the kernel use is F.interpolate(mode="nearest", size=...) for every H, W in 2..40."""
    for H in range(2, 41):
        for W in range(2, 41):
            src = torch.arange((H // 2) * (W // 2), dtype=torch.float32).view(1, 1, H // 2, W // 2)
            want = F.interpolate(src, size=(H, W), mode="nearest")[0, 0].long().numpy()
            iy, ix = orn.nearest_index(H, H // 2), orn.nearest_index(W, W // 2)
            assert np.array_equal(iy[:, None] * (W // 2) + ix[None, :], want), (H, W)
    assert orn.nearest_index(5, 2).tolist() == [0, 0, 0, 1, 1]      # not d // 2


def test_philox_known_answers():
    """Random123's known-answer vectors for Philox4x32-10 (kat_vectors)."""
    cases = [
        ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
        ((0xFFFFFFFF,) * 4, (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
        ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
         (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
    ]
    for ctr, key, want in cases:
        got = orn.philox4x32_10(*ctr, *key)
        assert tuple(int(v) for v in got) == want, ctr


def test_engine_noise_restatement_is_standard_normal():
    n = orn.engine_noise(123, 0, 1, (3, 200, 300)).ravel()
    assert abs(n.mean()) < 5 / np.sqrt(n.size) and abs(n.var() - 1) < 5 * np.sqrt(2 / n.size)


@pytest.fixture(scope="module")
def lib():
    from nunif_b200 import build, _lib
    build.build()
    return _lib.lib()


def test_level2_refusal_before_cuda(lib):
    """H or W < 2 at level 2 has an empty half-resolution field (the reference fails on it); the engine refuses it in Python
    and in the C entry points, with dummy host pointers, before any CUDA call."""
    from nunif_b200.nunif.rgb_noise import rgb_noise_like, apply_rgb_noise_like
    for shape in ((3, 1, 5), (3, 5, 1), (2, 3, 1, 1)):
        with pytest.raises(ValueError, match="level 2"):
            rgb_noise_like(torch.zeros(shape))
    with pytest.raises(ValueError, match="level 2"):
        apply_rgb_noise_like(torch.zeros(3, 1, 8), seed=1)
    d, o = ctypes.create_string_buffer(256), ctypes.create_string_buffer(256)
    params = (ctypes.c_double * 4)(0.2, 2.2, 0.8, 0.5)
    assert lib.nb200_rgb_noise(1, 0, 2, 1, 3, 1, 5, d, None) != 0
    assert b"level 2 needs" in lib.nb200_last_error()
    assert lib.nb200_apply_rgb_noise(d, 1, 3, 5, 1, None, 1, 0, 2, None, 0, params, 1, 0, o, None) != 0
    assert b"level 2 needs" in lib.nb200_last_error()
    assert lib.nb200_rgb_noise(1, 0, 3, 1, 3, 4, 4, d, None) != 0
    assert b"level must be 1 or 2" in lib.nb200_last_error()
    bad = (ctypes.c_double * 4)(0.2, 2.2, 1.5, 0.5)
    assert lib.nb200_apply_rgb_noise(d, 1, 3, 4, 4, d, 1, 0, 2, None, 0, bad, 1, 0, o, None) != 0
    assert b"light_decay_strength" in lib.nb200_last_error()
    assert lib.nb200_apply_rgb_noise(d, 1, 4, 4, 4, d, 1, 0, 2, None, 0, params, 1, 8, o, None) != 0
    assert b"3 channels" in lib.nb200_last_error()


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback(lib):
    from nunif_b200.nunif.rgb_noise import rgb_noise_like, apply_rgb_noise
    with pytest.raises(RuntimeError, match="CUDA"):
        rgb_noise_like(torch.zeros(3, 8, 8))
    with pytest.raises(RuntimeError, match="CUDA"):
        apply_rgb_noise(torch.zeros(3, 8, 8), torch.zeros(3, 8, 8))
    d = ctypes.create_string_buffer(256)
    assert lib.nb200_rgb_noise(1, 0, 2, 1, 3, 4, 4, d, None) != 0      # a launch without a device fails loudly


def test_argument_checks():
    from nunif_b200.nunif.rgb_noise import apply_rgb_noise, rgb_noise_like
    from nunif_b200.nunif.video import FrameBatchPipeline
    with pytest.raises(ValueError, match="level"):
        rgb_noise_like(torch.zeros(3, 8, 8), level=3)
    with pytest.raises(ValueError, match="offset"):
        rgb_noise_like(torch.zeros(3, 8, 8), offset=2 ** 32)
    with pytest.raises(ValueError, match="light_decay_strength"):
        apply_rgb_noise(torch.zeros(3, 8, 8), torch.zeros(3, 8, 8), light_decay_strength=1.5)
    with pytest.raises(ValueError, match="gamma"):
        apply_rgb_noise(torch.zeros(3, 8, 8), torch.zeros(3, 8, 8), gamma=0.0)
    with pytest.raises(ValueError, match="noise shape"):
        apply_rgb_noise(torch.zeros(3, 8, 8), torch.zeros(3, 8, 9))
    with pytest.raises(ValueError, match="grain"):
        FrameBatchPipeline(lambda x: x, 2, device="cpu", grain=(0.2,))


def test_seed_follows_torch_manual_seed():
    from nunif_b200.nunif.rgb_noise import draw_seed
    torch.manual_seed(5)
    a = draw_seed()
    torch.manual_seed(5)
    assert draw_seed() == a and 0 <= a < 2 ** 63
