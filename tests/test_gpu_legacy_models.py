"""GPU: waifu2x.upconv_7 / waifu2x.vgg_7 on the engine - forward and tiled_render parity against the reference's goldens and
the oracle on the same GPU (fp32 and fp16 autocast), the tensor-core vs SIMT output heads, CUDA-graph replay, the tile-size
floor, and the upconv_7/<style> checkpoint directory through the hub."""
import os

import pytest
import torch

from nunif_b200 import synth
from oracle import legacy as ol, seam_blending as osb
from tests.util import load_golden, t, stats, log_metric
from tests.test_gpu_models import check, amp, _fp32_ref
from tests.test_legacy_models import inputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

MODELS = [("upconv_7", synth.upconv7_state_dict, ol.upconv7_forward, ol.UPCONV_7),
          ("vgg_7", synth.vgg7_state_dict, ol.vgg7_forward, ol.VGG_7)]
IDS = [m[0] for m in MODELS]


def _model(name, sdf, seed=0):
    from nunif_b200.nunif.models import create_model
    return create_model("waifu2x." + name, sdf(seed), DEV)


@pytest.mark.parametrize("name,sdf,fn,spec", MODELS, ids=IDS)
def test_forward_matches_goldens(name, sdf, fn, spec):
    g = load_golden(name)
    inp = inputs(g)
    m = _model(name, sdf)
    assert (m.i2i_scale, m.i2i_offset, m.i2i_blend_size) == (spec["scale"], spec["offset"], None)
    for xk, zk in (("x", "z"), ("x_odd", "z_odd")):      # tile 104 and the odd tile 61
        x = inp[xk].to(DEV)
        z = m(x).float()
        assert z.shape == t(g[zk]).shape
        check(f"{name}_forward_{x.shape[-1]}", z, t(g[zk]), amp(fn, sdf(0), x))


@pytest.mark.parametrize("name,sdf,fn,spec", MODELS, ids=IDS)
def test_forward_at_production_shape(name, sdf, fn, spec):
    """tile 256, batch 4: the launch shapes of a 4K render, against the fp32 oracle (TF32 off) and the autocast oracle."""
    m = _model(name, sdf)
    x = torch.stack([synth.synth_image(500 + i, 3, 256, 256, smooth=(i % 2 == 0)) for i in range(4)]).to(DEV)
    z = m(x).float()
    check(f"{name}_forward_256x4", z, _fp32_ref(fn, sdf(0), x), amp(fn, sdf(0), x))


@pytest.mark.parametrize("name,sdf,fn,spec", MODELS, ids=IDS)
def test_smallest_tile_and_below(name, sdf, fn, spec):
    """Every tile size with input_tile_step = T - 14 > 0 is accepted (T = 15 is the smallest); below that the engine raises."""
    m = _model(name, sdf)
    x = torch.stack([synth.synth_image(600, 3, 15, 15), synth.synth_image(601, 3, 15, 15, smooth=False)]).to(DEV)
    z = m(x).float()
    want = _fp32_ref(fn, sdf(0), x)
    assert z.shape == want.shape == (2, 3, 15 * spec["scale"] - 2 * spec["offset"], 15 * spec["scale"] - 2 * spec["offset"])
    assert stats(z, want)["max"] < 1e-2, stats(z, want)
    from nunif_b200.nunif.render import tiled_render
    with torch.no_grad(), pytest.raises(RuntimeError, match="tile_size too small"):
        tiled_render(synth.synth_image(602, 3, 40, 50).to(DEV), m, tile_size=14, batch_size=2)
    with pytest.raises(RuntimeError):
        m(x[:, :, :14, :14].contiguous())              # an empty output tile


@pytest.mark.parametrize("name,sdf,fn,spec", MODELS, ids=IDS)
def test_tiled_render(name, sdf, fn, spec):
    from nunif_b200.nunif.render import tiled_render
    g = load_golden(name)
    img = inputs(g)["img"]
    m = _model(name, sdf)
    T, B = int(g["tile_size"]), int(g["batch_size"])
    with torch.no_grad():
        y = tiled_render(img.to(DEV), m, tile_size=T, batch_size=B)
        others = [tiled_render(img.to(DEV), m, tile_size=T, batch_size=b) for b in (1, 5)]
    assert y.shape == t(g["render"]).shape and y.is_contiguous()
    sdc = {k: v.to(DEV) for k, v in sdf(0).items()}

    def amp_model(b):
        with torch.autocast("cuda", dtype=torch.float16):
            return fn(sdc, b.to(DEV)).float().cpu()
    y_amp = osb.tiled_render(img, amp_model, spec["scale"], spec["offset"], 0, T, B)
    check(name + "_render", y, t(g["render"]), y_amp)
    for o in others:                                    # the batch size must not change the result
        assert torch.equal(o, y)


@pytest.mark.parametrize("name,sdf,fn,spec", MODELS, ids=IDS)
def test_tensor_core_and_simt_heads_agree(name, sdf, fn, spec):
    """nb200_tune_set(7, 1) runs the stem and the output head on their SIMT kernels (fp32 weights at fp16 precision, fp32
    accumulation in a different order); the result must agree with the mma.sync path up to that reordering, and pass the
    same parity criterion."""
    from nunif_b200 import _lib
    g = load_golden(name)
    inp = inputs(g)
    m = _model(name, sdf)
    for xk, zk in (("x", "z"), ("x_odd", "z_odd")):
        x = inp[xk].to(DEV)
        a = m(x).float()
        _lib.lib().nb200_tune_set(7, 1)
        try:
            b = m(x).float()
        finally:
            _lib.lib().nb200_tune_set(7, 0)
        s = stats(a, b)
        log_metric(f"{name}_tc_vs_simt_{x.shape[-1]}", **s)
        assert s["max"] < 1e-2 and s["mean"] < 2e-4, s
        check(f"{name}_simt_forward_{x.shape[-1]}", b, t(g[zk]), amp(fn, sdf(0), x))


@pytest.mark.parametrize("name,sdf,fn,spec", MODELS, ids=IDS)
def test_cuda_graph_replay_is_bit_identical(name, sdf, fn, spec):
    from nunif_b200 import _lib
    from nunif_b200.nunif.render import tiled_render
    m = _model(name, sdf)
    imgs = [synth.synth_image(70 + i, 3, 150, 200).to(DEV) for i in range(3)]
    with torch.no_grad():
        want = [tiled_render(im, m, tile_size=61, batch_size=5) for im in imgs]
        _lib.lib().nb200_tune_set(9, 1)
        try:
            for rep in range(3):
                for im, w in zip(imgs, want):
                    assert torch.equal(tiled_render(im, m, tile_size=61, batch_size=5), w), rep
            host = tiled_render(imgs[0].cpu().pin_memory(), m, tile_size=61, batch_size=5)
            torch.cuda.synchronize()
            assert torch.equal(host, want[0].cpu())
        finally:
            _lib.lib().nb200_tune_set(9, 0)


# ---- the upconv_7/<style> checkpoint directory -----------------------------------------------------------------------------
def _write(dirpath, filename, name, sd):
    os.makedirs(dirpath, exist_ok=True)
    # the dict nunif.models.save_model writes (nunif/models/utils.py:12-39)
    torch.save({"nunif_model": 1, "name": name, "kwargs": {}, "state_dict": sd, "updated_at": "0"}, os.path.join(dirpath, filename))


def _release_layout(d, skip=()):
    """scale2x.pth and noise{n}_scale2x.pth are upconv_7, noise{n}.pth are vgg_7 (waifu2x/docs/training.md:59-69)."""
    files = {"scale2x.pth": ("waifu2x.upconv_7", synth.upconv7_state_dict(0))}
    for n in range(4):
        files[f"noise{n}_scale2x.pth"] = ("waifu2x.upconv_7", synth.upconv7_state_dict(1 + n))
        files[f"noise{n}.pth"] = ("waifu2x.vgg_7", synth.vgg7_state_dict(n))
    for f, (name, sd) in files.items():
        if f not in skip:
            _write(d, f, name, sd)


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    root = tmp_path_factory.mktemp("pretrained_models")
    _release_layout(os.path.join(root, "upconv_7", "art"))
    _release_layout(os.path.join(root, "upconv_7", "photo"), skip=("noise2.pth",))
    return str(root)


def test_hub_upconv_7_directory(model_dir):
    from nunif_b200.waifu2x import waifu2x
    from nunif_b200.nunif.models import create_model
    from nunif_b200.nunif.render import tiled_render
    m = waifu2x("upconv_7/art", model_dir=model_dir, tile_size=64, batch_size=4)        # method=None: every slot
    ctx = m.ctx
    assert ctx.scale_model.name == "waifu2x.upconv_7" and ctx.scale4x_model is None
    assert all(s.name == "waifu2x.upconv_7" for s in ctx.noise_scale_models)
    assert all(s.name == "waifu2x.vgg_7" for s in ctx.noise_models)
    x = synth.synth_image(8, 3, 90, 130)

    def direct(name, sd, img, reduce=lambda y: y):
        with torch.no_grad():
            return reduce(tiled_render(img.to(DEV), create_model(name, sd, DEV), tile_size=64, batch_size=4)).cpu()
    rgb, alpha = m.infer(x, output_type="tensor", method="noise", noise_level=3)
    assert alpha is None and torch.equal(rgb, direct("waifu2x.vgg_7", synth.vgg7_state_dict(3), x))
    rgb, _ = m.infer(x, output_type="tensor", method="scale")
    assert torch.equal(rgb, direct("waifu2x.upconv_7", synth.upconv7_state_dict(0), x))
    rgb, _ = m.infer(x, output_type="tensor", method="noise_scale", noise_level=3)
    assert rgb.shape == (3, 180, 260) and torch.equal(rgb, direct("waifu2x.upconv_7", synth.upconv7_state_dict(4), x))
    with pytest.raises(ValueError):
        m.set_mode("scale4x")

    # RGBA through noise_scale: the alpha plane takes the second pass through the scale model (waifu2x/utils.py:282-287)
    a = torch.ones(1, 90, 130)
    a[:, 20:60, 30:90] = 0.25
    a[:, 70:, :40] = 0.0
    rgb, alpha = m.infer(x, output_type="tensor", alpha=a, method="noise_scale", noise_level=3)
    want_alpha = direct("waifu2x.upconv_7", synth.upconv7_state_dict(0), a.expand(3, 90, 130), lambda y: y.mean(0, keepdim=True))
    assert rgb.shape == (3, 180, 260) and alpha.shape == (1, 180, 260)
    assert torch.equal(alpha, want_alpha)


def test_hub_upconv_7_missing_noise_level(model_dir):
    from nunif_b200.waifu2x import waifu2x
    with pytest.raises(FileNotFoundError):
        waifu2x("upconv_7/photo", model_dir=model_dir, tile_size=64, batch_size=4)
    p = waifu2x("upconv_7/photo", method="noise", noise_level=1, model_dir=model_dir, tile_size=64, batch_size=4)
    assert p.infer(synth.synth_image(9, 3, 40, 50), output_type="tensor")[0].shape == (3, 40, 50)
