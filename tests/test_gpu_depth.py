"""GPU parity of the Depth-Anything-V2 ViT-S network (SURVEY.md 8a rows B1, B3, B5) against the oracle's restatement
(oracle/depth_anything.py; third-party network, cross-checked against transformers on the CPU).

Criterion as for the waifu2x models: the engine computes in the reference's CUDA numerics (fp16 autocast), so its
error against the fp32 oracle is compared with the error of the oracle itself run under CUDA fp16 autocast."""
import pytest
import torch

from tests.util import log_metric, stats, true_fp32
from nunif_b200 import synth
from oracle import depth_anything as oda

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _refs(sd, x):
    sdc = {k: v.to(DEV) for k, v in sd.items()}
    with torch.no_grad():
        with true_fp32():
            ref32 = oda.depth_anything_forward(sdc, x.to(DEV).float())
        with torch.autocast("cuda", dtype=torch.float16):
            refamp = oda.depth_anything_forward(sdc, x.to(DEV)).float()
    return ref32.cpu(), refamp.cpu()


def _check(tag, got, ref32, refamp):
    scale = float(ref32.abs().max())
    e_ref, e_our, e_amp = stats(refamp, ref32), stats(got, ref32), stats(got, refamp)
    log_metric(tag, ours_max=e_our["max"], ours_mean=e_our["mean"], refamp_max=e_ref["max"], refamp_mean=e_ref["mean"],
               ours_vs_amp_max=e_amp["max"], scale=scale)
    assert e_our["max"] <= max(1e-3 * scale, 1.5 * e_ref["max"]), (tag, e_our, e_ref)
    assert e_our["mean"] <= max(5e-4 * scale, 1.25 * e_ref["mean"]), (tag, e_our, e_ref)


@pytest.mark.parametrize("B,H,W", [(1, 14 * 6, 14 * 6), (2, 14 * 9, 14 * 13), (1, 14 * 5, 14 * 11)])
def test_depth_anything_forward_small(B, H, W):
    from nunif_b200.iw3 import DepthAnythingNet
    sd = synth.depth_anything_v2_state_dict(1)
    x = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(H + W))
    net = DepthAnythingNet(sd, DEV)
    got = net(x.to(DEV)).cpu()
    ref32, refamp = _refs(sd, x)
    assert got.shape == ref32.shape
    _check(f"depth_anything_{B}x{H}x{W}", got, ref32, refamp)


def test_depth_anything_1080p_infer_pipeline():
    """DepthAnythingModel.infer on 1080p frames: preprocess (392x686) -> network -> dilate_edge, against the same
    composition built from the oracle pieces; flip-TTA path included."""
    from nunif_b200.iw3 import DepthAnythingModel, batch_preprocess, dilate_edge
    sd = synth.depth_anything_v2_state_dict(2)
    model = DepthAnythingModel().load_state_dict(sd, gpu=0)
    x = torch.stack([synth.synth_image(70 + i, 3, 1080, 1920, smooth=False) for i in range(2)])
    with torch.inference_mode():
        d = model.infer(x.to(DEV), edge_dilation=0)
        assert d.shape == (2, 1, 392, 686) and d.is_cuda and d.dtype == torch.float32
        xp = batch_preprocess(x.to(DEV))
        ref32, refamp = _refs(sd, xp.cpu())
        _check("depth_anything_1080p", d[:, 0].cpu(), ref32, refamp)
        d1 = model.infer(x[0].to(DEV), edge_dilation=2)
        assert d1.shape == (1, 392, 686)
        assert torch.equal(d1, dilate_edge(d[:1], 2)[0])
        dt = model.infer(x.to(DEV), tta=True)
        flipped = model.infer(torch.flip(x, dims=[3]).to(DEV))
        # the network output is fp16-quantised (reference numerics) and the GEMM tiling depends on the batch size:
        # allow two fp16 ulps at the top of the range
        assert stats(dt, (d + torch.flip(flipped, dims=[3])) * 0.5)["max"] <= 2 ** -9 * float(d.abs().max())


def test_pos_table_interpolation_matches_oracle():
    """The bicubic position-table resample is host C++ in the engine; check it end to end through a network whose
    only non-zero signal is the position table."""
    from nunif_b200.iw3 import DepthAnythingNet
    sd = synth.depth_anything_v2_state_dict(4)
    x = torch.zeros(1, 3, 14 * 7, 14 * 10)
    got = DepthAnythingNet(sd, DEV)(x.to(DEV)).cpu()
    ref32, refamp = _refs(sd, x)
    _check("depth_anything_pos_only", got, ref32, refamp)


@pytest.mark.parametrize("encoder,H,W", [("vitb", 14 * 6, 14 * 9), ("vitl", 14 * 5, 14 * 7)])
def test_depth_anything_base_and_large_encoders(encoder, H, W):
    """Any_V2_B / Any_V2_L share the code path; only the table in depth_model.cu changes (dim, heads, depth, head widths)."""
    from nunif_b200.iw3 import DepthAnythingNet
    sd = synth.depth_anything_v2_state_dict(5, encoder=encoder, pos_grid=8)
    x = torch.randn(1, 3, H, W, generator=torch.Generator().manual_seed(H * W))
    got = DepthAnythingNet(sd, DEV, encoder=encoder)(x.to(DEV)).cpu()
    sdc = {k: v.to(DEV) for k, v in sd.items()}
    with torch.no_grad():
        ref32 = oda.depth_anything_forward(sdc, x.to(DEV).float(), encoder).cpu()
        with torch.autocast("cuda", dtype=torch.float16):
            refamp = oda.depth_anything_forward(sdc, x.to(DEV), encoder).float().cpu()
    _check(f"depth_anything_{encoder}", got, ref32, refamp)
