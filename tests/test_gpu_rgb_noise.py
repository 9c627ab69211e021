"""GPU: waifu2x's film grain (csrc/rgb_noise.cu).

* The noise field against its numpy restatement (oracle.rgb_noise.engine_noise: same Philox counters, Box-Muller in
  float64) and its statistics: level 2 mean, variance 0.5, correlation 0.5 inside a half-resolution cell and 0 across
  cells, channels, frames and calls; level 1 against N(0, 1) by a KS test.  Same (seed, offset): same bits.
* apply_rgb_noise against the reference's op sequence on CUDA (oracle.rgb_noise.apply_rgb_noise on the GPU) given the same
  noise: float within 2 fp32 ulp; uint8 / uint16 equal except where the float lies within 2 ulp of a rounding boundary.
* FrameBatchPipeline(grain=...) against a sequential loop of the reference's recurrence fed the regenerated noise, and the
  stationary variance of its buffer; grain=None unchanged; the waifu2x image and video compositions."""
import types

import numpy as np
import pytest
import torch

from oracle import rgb_noise as orn
from tests.util import load_golden, log_metric

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def ulps(a, b):
    a, b = a.float().contiguous(), b.float().contiguous()
    return (a.view(torch.int32).long() - b.view(torch.int32).long()).abs()


def check_float(got, want, tag, max_ulp=2):
    d = ulps(got.to(DEV), want.to(DEV))
    log_metric("rgb_noise_apply_vs_cuda_oracle", case=tag, samples=d.numel(), differ=int((d > 0).sum()), max_ulp=int(d.max()))
    assert int(d.max()) <= max_ulp, f"{tag}: {int(d.max())} ulp"


def check_quantised(got, want_f, bits, tag):
    """got (.., H, W, 3) uint against from_tensor of the reference's float want_f (.., 3, H, W): equal, or off by one code
    where want_f * scale lies within 2 ulp (of want_f, scaled) of a rounding boundary."""
    scale = 65535.0 if bits == 16 else 255.0
    y = want_f.to(DEV).float().movedim(-3, -1).contiguous()
    v = y * scale
    want = v.round()
    ulp = torch.nextafter(y, torch.full_like(y, float("inf"))) - y
    near = ((v - v.floor()) - 0.5).abs() <= 2 * ulp * scale + torch.nextafter(v, torch.full_like(v, float("inf"))) - v
    d = (got.to(DEV).float() - want).abs()
    ok = (d == 0) | (near & (d <= 1))
    log_metric("rgb_noise_quantised_vs_cuda_oracle", case=tag, bits=bits, differ=int((d > 0).sum()), near=int(near.sum()))
    assert bool(ok.all()), f"{tag}: {int((~ok).sum())} codes off beyond the rounding-boundary allowance"


# ---- noise

@pytest.mark.parametrize("shape,level", [((3, 5, 7), 2), ((3, 5, 7), 1), ((2, 3, 7, 5), 2), ((3, 2, 3), 2), ((3, 33, 17), 2),
                                         ((1, 64, 96), 2), ((3, 1081, 1919), 2)])
def test_noise_matches_counter_restatement(shape, level):
    from nunif_b200.nunif.rgb_noise import rgb_noise_like
    seed, offset = 0x1234_5678_9ABC_DEF0, 77
    got = rgb_noise_like(torch.zeros(shape, device=DEV), level, seed=seed, offset=offset).double().cpu().numpy()
    want = orn.engine_noise(seed, offset, level, shape)
    err = np.abs(got - want) / (1 + np.abs(want))
    assert err.max() < 4e-6, (shape, level, err.max())


def test_noise_reproducible_and_offset_changes_field():
    from nunif_b200.nunif.rgb_noise import rgb_noise_like
    base = torch.zeros(3, 270, 481, device=DEV)
    a = rgb_noise_like(base, seed=5, offset=3)
    assert torch.equal(a, rgb_noise_like(base, seed=5, offset=3))
    b = rgb_noise_like(base, seed=5, offset=4)
    c = rgb_noise_like(base, seed=6, offset=3)
    assert float((a == b).float().mean()) < 1e-3 and float((a == c).float().mean()) < 1e-3
    torch.manual_seed(1)
    d = rgb_noise_like(base)
    torch.manual_seed(1)
    assert torch.equal(d, rgb_noise_like(base))


def _corr(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    a, b = a - a.mean(), b - b.mean()
    return float((a * b).sum() / (a.norm() * b.norm())), a.numel()


def test_noise_statistics_level2():
    from nunif_b200.nunif.rgb_noise import rgb_noise_like
    n = rgb_noise_like(torch.zeros(2, 3, 1080, 1920, device=DEV), seed=99, offset=0)
    N = n.numel()
    assert N >= 8_000_000
    x = n.double()
    # a half-resolution cell of 4 pixels shares 0.5 * h: Var(sum of a cell) = 4 * 0.25 + (4 * 0.5)^2 = 5, 1.25 per pixel
    mean, var = float(x.mean()), float(x.var())
    assert abs(mean) < 5 * np.sqrt(1.25 / N), mean
    assert abs(var - 0.5) < 5 * 0.5 * np.sqrt(2 / (N / 4)), var
    pairs = {
        "cell_x": (n[..., :, 0::2], n[..., :, 1::2], 0.5),
        "cell_y": (n[..., 0::2, :], n[..., 1::2, :], 0.5),
        "across_cells_x": (n[..., :, 1:-1:2], n[..., :, 2::2], 0.0),
        "across_cells_y": (n[..., 1:-1:2, :], n[..., 2::2, :], 0.0),
        "channels": (n[:, 0], n[:, 1], 0.0),
        "frames": (n[0], n[1], 0.0),
        "calls": (n[0], rgb_noise_like(torch.zeros(3, 1080, 1920, device=DEV), seed=99, offset=1), 0.0),
    }
    for name, (a, b, want) in pairs.items():
        r, k = _corr(a, b)
        log_metric("rgb_noise_corr", pair=name, corr=f"{r:.5f}", n=k)
        assert abs(r - want) < 5 * 2 / np.sqrt(k), (name, r)
    log_metric("rgb_noise_level2", mean=f"{mean:.3e}", var=f"{var:.6f}", n=N)


def test_noise_level1_ks():
    from scipy import stats
    from nunif_b200.nunif.rgb_noise import rgb_noise_like
    n = rgb_noise_like(torch.zeros(3, 1024, 1024, device=DEV), level=1, seed=3).double().cpu().numpy().ravel()
    p = stats.kstest(n, "norm").pvalue
    log_metric("rgb_noise_level1_ks", n=n.size, p=f"{p:.4f}")
    assert p > 1e-3, p


# ---- apply

def _inputs(shape, seed):
    g = torch.Generator().manual_seed(seed)
    rgb = orn.golden_rgb(shape, seed).to(DEV)
    noise = (torch.randn(shape, generator=g) * 2).to(DEV)
    return rgb, noise


def _apply_both(rgb, noise, kw, tag):
    from nunif_b200.nunif.rgb_noise import apply_rgb_noise
    want = orn.apply_rgb_noise(rgb.clone(), noise.clone(), **kw)
    check_float(apply_rgb_noise(rgb, noise, **kw), want, tag)
    for bits, dt in ((8, torch.uint8), (16, torch.uint16)):
        if rgb.shape[-3] == 3:
            check_quantised(apply_rgb_noise(rgb, noise, dtype=dt, **kw), want, bits, tag)


@pytest.mark.parametrize("pname", list(orn.PARAMS))
def test_apply_parity_odd_sizes_every_params(pname):
    kw = orn.PARAMS[pname]
    for shape in ((3, 301, 517), (2, 3, 37, 53), (1, 9, 11)):
        rgb, noise = _inputs(shape, 5)
        _apply_both(rgb, noise, kw, f"{pname}/{shape}")


def test_apply_parity_golden():
    g = load_golden("rgb_noise")
    for i, (name, shape) in enumerate(orn.APPLY_CASES):
        rgb = orn.golden_rgb(shape, 100 + i).to(DEV)
        noise = torch.from_numpy(g[f"apply/{name}/noise"]).to(DEV)
        for pname, kw in orn.PARAMS.items():
            _apply_both(rgb, noise, kw, f"golden/{name}/{pname}")


@pytest.mark.parametrize("pname", ["default", "g2_lds03"])
def test_apply_parity_4k(pname):
    rgb, noise = _inputs((3, 2160, 3840), 8)
    _apply_both(rgb, noise, orn.PARAMS[pname], f"4k/{pname}")


def test_fused_generation_equals_given_noise():
    """apply_rgb_noise_like generates in the kernel exactly the field rgb_noise_like returns."""
    from nunif_b200.nunif.rgb_noise import rgb_noise_like, apply_rgb_noise, apply_rgb_noise_like
    rgb, _ = _inputs((3, 123, 77), 9)
    for level in (1, 2):
        noise = rgb_noise_like(rgb, level, seed=42, offset=6)
        assert torch.equal(apply_rgb_noise_like(rgb, 0.3, level, seed=42, offset=6), apply_rgb_noise(rgb, noise, 0.3))


# ---- temporal: the pipeline's grain stage

def _frames(n, shapes, bits, seed):
    g = torch.Generator().manual_seed(seed)
    dt = torch.uint16 if bits == 16 else torch.uint8
    hi = 65536 if bits == 16 else 256
    return [torch.randint(0, hi, shapes[t] + (3,), generator=g, dtype=torch.int32).to(dt) for t in range(n)]


def _reference_video(frames, bits, convert, strength, speed, seed):
    """ui_utils.py:150-178, frame by frame, with the noise rgb_noise_like(seed, offset=t) regenerates."""
    from nunif_b200.iw3.frames import hwc_to_chw_float
    from nunif_b200.nunif.rgb_noise import rgb_noise_like
    buf, outs = None, []
    for t, f in enumerate(frames):
        x = hwc_to_chw_float(f.to(DEV))                          # what the pipeline hands its callback
        y = convert(x)
        buf = orn.temporal_step(buf, rgb_noise_like(y, seed=seed, offset=t), speed)
        outs.append(orn.apply_rgb_noise(y, buf, strength=strength))
    return outs, buf


@pytest.mark.parametrize("bits", [8, 16])
def test_pipeline_grain_matches_sequential_reference(bits):
    from nunif_b200.nunif.video import FrameBatchPipeline
    seed = 1234
    shapes = [(72, 128)] * 11 + [(90, 160)] * 12                  # resolution change at frame 11
    frames = _frames(23, shapes, bits, 3)
    pipe = FrameBatchPipeline(lambda x: x, 4, device=DEV, depth=3, use_16bit=bits == 16, grain=(0.2, 0.8, seed))
    got = []
    for f in frames:
        got += pipe(f)
    got += pipe.finish()
    assert len(got) == 23
    want, buf = _reference_video(frames, bits, lambda x: x, 0.2, 0.8, seed)
    for t, (u, y) in enumerate(zip(got, want)):
        check_quantised(u, y, bits, f"pipeline/{bits}/frame{t}")
    assert torch.equal(pipe.grain.buffer, buf)                    # the buffer recurrence is bit-exact


def test_grain_buffer_stationary_variance():
    from nunif_b200.nunif.rgb_noise import TemporalGrain
    s = 0.8
    grain = TemporalGrain(0.2, s, seed=77)
    x = torch.full((4, 3, 540, 960), 0.5, device=DEV)
    for _ in range(4):
        grain(x)
    b = grain.buffer.double()
    want = s / (2 - s) * 0.5
    # each buffer value is Gaussian; the half-resolution cells make neighbours correlated, so count N / 4 samples
    tol = 5 * want * np.sqrt(2 / (b.numel() / 4))
    log_metric("rgb_noise_buffer_var", var=f"{float(b.var()):.6f}", want=f"{want:.6f}")
    assert abs(float(b.var()) - want) < tol and abs(float(b.mean())) < 5 * np.sqrt(1.25 / b.numel())


def test_pipeline_without_grain_unchanged():
    from nunif_b200.iw3.frames import hwc_to_chw_float, chw_float_to_hwc
    from nunif_b200.nunif.video import FrameBatchPipeline
    frames = _frames(7, [(40, 64)] * 7, 8, 4)
    cb = lambda x: (x * 0.75 + 0.1).clamp(0, 1)                  # noqa: E731
    pipe = FrameBatchPipeline(cb, 3, device=DEV)
    got = []
    for f in frames:
        got += pipe(f)
    got += pipe.finish()
    for f, u in zip(frames, got):
        assert torch.equal(u, chw_float_to_hwc(cb(hwc_to_chw_float(f.to(DEV)))).cpu())


# ---- waifu2x ui_utils compositions

class _StubCtx:
    """Stands in for Waifu2x: a deterministic per-pixel 'conversion' that keeps values in [0, 1]."""

    def convert(self, x, alpha, method, noise_level, tile_size=None, batch_size=None, tta=False, enable_amp=True,
                output_device="cpu"):
        return (x * 0.8 + 0.1).to(output_device), alpha


def _args(**kw):
    a = dict(rotate_left=False, rotate_right=False, method="scale", noise_level=0, tile_size=64, batch_size=1, tta=False,
             disable_amp=False, grain=True, grain_strength=0.3, grain_speed=0.6, state={"device": torch.device(DEV)})
    a.update(kw)
    return types.SimpleNamespace(**a)


@pytest.mark.parametrize("rot", ["rotate_left", "rotate_right", None])
def test_waifu2x_process_image_composition(rot):
    from nunif_b200.nunif.rgb_noise import rgb_noise_like
    from nunif_b200.waifu2x.ui_utils import process_image
    args = _args(**({rot: True} if rot else {}))
    rgb = orn.golden_rgb((3, 45, 70), 12)
    alpha = torch.rand(1, 45, 70, generator=torch.Generator().manual_seed(2))
    got, galpha = process_image(_StubCtx(), rgb, alpha, args, seed=31)
    k = {"rotate_left": 1, "rotate_right": 3, None: 0}[rot]
    x = torch.rot90(rgb.to(DEV), k, (-2, -1))
    y, _ = _StubCtx().convert(x, None, "scale", 0, output_device=DEV)
    want = orn.apply_rgb_noise(y, rgb_noise_like(y, seed=31), strength=0.3 * 0.5)
    check_float(got, want, f"waifu2x_image/{rot}")
    assert torch.equal(galpha, torch.rot90(alpha.to(DEV), k, (-2, -1)))
    args.grain = False
    assert torch.equal(process_image(_StubCtx(), rgb, alpha, args)[0], y)


def test_waifu2x_video_composition():
    from nunif_b200.waifu2x.ui_utils import make_video_pipeline
    args = _args(rotate_right=True)
    frames = _frames(9, [(48, 80)] * 9, 8, 6)
    pipe = make_video_pipeline(_StubCtx(), args, batch_size=4, seed=17)
    got = []
    for f in frames:
        got += pipe(f)
    got += pipe.finish()
    conv = lambda x: _StubCtx().convert(torch.rot90(x, 3, (-2, -1)), None, "scale", 0, output_device=DEV)[0]   # noqa: E731
    want, _ = _reference_video(frames, 8, conv, args.grain_strength, args.grain_speed, 17)
    assert len(got) == 9
    for t, (u, y) in enumerate(zip(got, want)):
        assert tuple(u.shape) == (80, 48, 3)
        check_quantised(u, y, 8, f"waifu2x_video/frame{t}")
