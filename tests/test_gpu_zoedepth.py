"""GPU parity of the ZoeD_N metric depth network (SURVEY.md 8a rows B1, B4, B5; BASELINE configs[4]'s depth stage) against
the oracle's restatement (oracle/zoedepth.py; third-party network, cross-checked against transformers on the CPU).

Criterion as for Depth-Anything: the engine computes in the reference's CUDA numerics (fp16 autocast), so its error
against the fp32 oracle is compared with the error of the oracle itself run under CUDA fp16 autocast."""
import numpy as np
import pytest
import torch

from tests.util import log_metric, stats, true_fp32
from nunif_b200 import synth
from oracle import zoedepth as oz

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _refs(sd, x, cfg):
    sdc = {k: v.to(DEV) for k, v in sd.items()}
    with torch.no_grad():
        with true_fp32():
            ref32 = oz.zoedepth_forward(sdc, x.to(DEV).float(), cfg)
        with torch.autocast("cuda", dtype=torch.float16):
            refamp = oz.zoedepth_forward(sdc, x.to(DEV), cfg).float()
    return ref32.cpu(), refamp.cpu()


def _check(tag, got, ref32, refamp):
    scale = float(ref32.abs().max())
    e_ref, e_our, e_amp = stats(refamp, ref32), stats(got, ref32), stats(got, refamp)
    log_metric(tag, ours_max=e_our["max"], ours_mean=e_our["mean"], ours_p999=e_our["p999"], refamp_max=e_ref["max"],
               refamp_mean=e_ref["mean"], refamp_p999=e_ref["p999"], ours_vs_amp_max=e_amp["max"], scale=scale)
    assert torch.isfinite(got).all()
    # mean and 99.9th percentile: no worse than the reference's own fp16 evaluation on maps of >= 10^5 pixels (p99.9: 1.1 x); on the
    # small test maps (6k .. 20k pixels, where p99.9 is the ~10th largest sample) 1.25 x / 1.5 x.  The maximum gets 4 x: the
    # log-binomial head divides its logits (k log p + (63 - k) log(1 - p)) by a temperature down to 0.0212, i.e. a 1-ulp fp16 change
    # of one pre-activation moves a logit by up to ~3000 ulp - the maximum is a heavy-tailed statistic of any two correct fp16
    # evaluations (measured: refamp 1.6e-2 .. 1.7e-2 on a 0.2 .. 3.8 m range at mean 4e-4; 3.4 m on the full-size network).  The
    # worst case seen is 3.4 x (mini 2x96x64: 0.052 vs 0.0155, three adjacent pixels of one low-temperature row, T = 0.3, while every
    # intermediate stage incl. the bin centres is at or below the autocast error)
    big = got.numel() >= 100_000
    assert e_our["mean"] <= max(5e-4 * scale, (1.0 if big else 1.25) * e_ref["mean"]), (tag, e_our, e_ref)
    assert e_our["p999"] <= max(1e-3 * scale, (1.1 if big else 1.5) * e_ref["p999"]), (tag, e_our, e_ref)
    assert e_our["max"] <= max(1e-3 * scale, 4.0 * e_ref["max"]), (tag, e_our, e_ref)


@pytest.mark.parametrize("B,H,W", [(1, 64, 96), (2, 96, 64), (1, 128, 160)])
def test_zoedepth_forward_mini(B, H, W):
    """Reduced widths (synth.ZOED_MINI), same code path: non-square grids resample the relative-position table."""
    from nunif_b200.iw3 import ZoeDepthNet
    sd = synth.zoedepth_state_dict(1, synth.ZOED_MINI)
    x = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(H + W))
    net = ZoeDepthNet(sd, DEV)
    got = net(x.to(DEV)).cpu()
    ref32, refamp = _refs(sd, x, oz.ZOED_MINI)
    assert got.shape == ref32.shape == (B, 1, H, W)
    assert float(ref32.std()) > 0.05
    _check(f"zoedepth_mini_{B}x{H}x{W}", got, ref32, refamp)


def test_zoedepth_mini_batch_invariant_and_grid_change():
    from nunif_b200.iw3 import ZoeDepthNet
    sd = synth.zoedepth_state_dict(2, synth.ZOED_MINI)
    net = ZoeDepthNet(sd, DEV)
    x = torch.randn(3, 3, 64, 96, generator=torch.Generator().manual_seed(3)).to(DEV)
    y3 = net(x)
    y1 = net(x[1:2])
    assert torch.equal(y3[1:2], y1)
    z = net(torch.randn(1, 3, 96, 96, generator=torch.Generator().manual_seed(4)).to(DEV))   # bias cache rebuilt for a new grid
    assert torch.isfinite(z).all()
    assert torch.equal(net(x[1:2]), y1)                                                       # ... and rebuilt back


def test_zoedepth_rejects_bad_input_and_keys():
    from nunif_b200.iw3 import ZoeDepthNet
    sd = synth.zoedepth_state_dict(1, synth.ZOED_MINI)
    net = ZoeDepthNet(sd, DEV)
    with pytest.raises(RuntimeError, match="multiples of 32"):
        net(torch.zeros(1, 3, 48, 64, device=DEV))
    bad = dict(sd)
    bad.pop("conv2.weight")
    with pytest.raises(RuntimeError, match="missing key"):
        ZoeDepthNet(bad, DEV)
    bad = dict(sd)
    bad["extra.weight"] = torch.zeros(3)
    with pytest.raises(RuntimeError, match="unexpected key"):
        ZoeDepthNet(bad, DEV)


def test_zoedepth_full_size_384x512():
    """The released configuration (BEiT-L/16, 24 blocks, 1024 wide) at the network input of a landscape frame."""
    from nunif_b200.iw3 import ZoeDepthNet
    sd = synth.zoedepth_state_dict(0)
    x = torch.randn(1, 3, 384, 512, generator=torch.Generator().manual_seed(11)).clamp_(-1, 1)
    net = ZoeDepthNet(sd, DEV)
    got = net(x.to(DEV)).cpu()
    ref32, refamp = _refs(sd, x, oz.ZOED_N)
    assert got.shape == (1, 1, 384, 512)
    _check("zoedepth_full_384x512", got, ref32, refamp)


def test_zoedepth_model_infer_pipeline_1080p():
    """ZoeDepthModel.infer on a 1080p frame: batch_preprocess (384x704 incl. reflection pad) -> network -> crop -> negate
    (+ flip TTA, + dilate_edge), against the same composition built from the oracle pieces; then the reference's
    process_image call sequence (get_ema_buffer_size -> infer -> minmax_normalize_chw, iw3/utils.py:505-520)."""
    from nunif_b200.iw3 import ZoeDepthModel
    from nunif_b200.iw3.zoedepth_preprocess import batch_preprocess
    sd = synth.zoedepth_state_dict(2, synth.ZOED_MINI)
    model = ZoeDepthModel("ZoeD_N").load_state_dict(sd, gpu=0)
    assert model.is_metric() and model.get_name() == "ZoeDepth" and model.loaded()
    x = torch.stack([synth.synth_image(90 + i, 3, 1080, 1920, smooth=False) for i in range(2)])
    with torch.inference_mode():
        d = model.infer(x.to(DEV), tta=False, edge_dilation=0)
        xp, pad_h, pad_w = batch_preprocess(x.to(DEV))
        assert xp.shape[-2:] == (384, 704)
        assert d.shape == (2, 1, 384 - 2 * pad_h, 704 - 2 * pad_w) and d.is_cuda and d.dtype == torch.float32
        ref32, refamp = _refs(sd, xp.cpu(), oz.ZOED_MINI)
        crop = (slice(None), slice(None), slice(pad_h, 384 - pad_h), slice(pad_w, 704 - pad_w))
        _check("zoedepth_1080p_infer", -d.cpu(), ref32[crop], refamp[crop])
        # flip TTA: average of the frame and its mirrored evaluation
        dt = model.infer(x[0].to(DEV), tta=True, edge_dilation=0)
        assert dt.shape == (1, 384 - 2 * pad_h, 704 - 2 * pad_w)
        xf = torch.cat([xp[:1], torch.flip(xp[:1], dims=[3])], dim=0)
        r32, ramp = _refs(sd, xf.cpu(), oz.ZOED_MINI)
        want32 = (r32[:1][crop] + torch.flip(r32[1:][crop], dims=[3])) * 0.5
        wantamp = (ramp[:1][crop] + torch.flip(ramp[1:][crop], dims=[3])) * 0.5
        _check("zoedepth_1080p_tta", -dt.cpu().unsqueeze(0), want32, wantamp)
        # dilation runs in negative space (zoedepth_model.py:125-127)
        from nunif_b200.iw3 import dilate_edge
        dd = model.infer(x.to(DEV), tta=False, edge_dilation=2)
        assert torch.allclose(dd, dilate_edge(d.clone(), 2), atol=1e-5)
        # process_image sequence
        assert model.get_ema_buffer_size() >= 1
        dn = model.minmax_normalize_chw(model.infer(x[0].to(DEV), tta=False, edge_dilation=2))
        assert dn.shape == d.shape[1:] and float(dn.min()) >= 0.0 and float(dn.max()) <= 1.0


def test_zoedepth_infer_matches_reference_batch_infer_golden():
    """ZoeDepthModel.infer against the REAL iw3/zoedepth_model.batch_infer run on the CPU in fp32 around the oracle network
    (tests/golden/zoedepth_infer.npz, oracle/gen_golden.py:gen_zoedepth_infer): landscape batch and a portrait single image (square
    reflection pad), flip TTA on / off, edge dilation 0 / 2.  Bounds: the fp16 error level of the reduced network measured by
    the tests above (mean 1e-4, p99.9 2e-3 of the range) with a safety factor; the exact criterion is in _check."""
    from tests.util import load_golden, t
    from nunif_b200.iw3 import ZoeDepthModel
    g = load_golden("zoedepth_infer")
    sd = synth.zoedepth_state_dict(5, synth.ZOED_MINI)
    model = ZoeDepthModel("ZoeD_N").load_state_dict(sd, gpu=0)
    model.model.prep_h_height, model.model.prep_v_height = 96, 128       # the sizes the golden was generated with
    land, port = t(g["land"]).to(DEV), t(g["port"]).to(DEV)
    with torch.inference_mode():
        for flip in (0, 1):
            for dil in (0, 2):
                for name, x in (("land", land), ("port", port)):
                    want = t(g[f"{name}_f{flip}_d{dil}"])
                    got = model.infer(x, tta=bool(flip), edge_dilation=dil).cpu()
                    assert got.shape == want.shape, (name, flip, dil, got.shape, want.shape)
                    scale = float(want.abs().max())
                    e = stats(got, want)
                    log_metric(f"zoedepth_infer_golden_{name}_f{flip}_d{dil}", max=e["max"], mean=e["mean"], p999=e["p999"], scale=scale)
                    assert torch.isfinite(got).all()
                    assert e["mean"] <= 1e-3 * scale and e["p999"] <= 1e-2 * scale and e["max"] <= 0.1 * scale, (name, flip, dil, e, scale)
