"""GPU: iw3.depth_aa (csrc/depth_aa.cu + wgmma GEMMs) against the reference-generated golden (tests/golden/depth_aa.npz,
oracle/gen_golden.py gen_depth_aa ran the REAL model) and against the oracle at other shapes.  The reference runs this filter in
fp32 (outside autocast, iw3/depth_anything_model.py:153-154); the engine's GEMMs are fp16 with fp32 accumulation."""
import numpy as np
import pytest
import torch

from tests.util import load_golden, log_metric
from nunif_b200 import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _model():
    from nunif_b200.iw3.depth_aa import DepthAA
    return DepthAA(synth.depth_aa_state_dict(0), DEV)


def _check(tag, got, want, scale=1.0):
    d = (got.float().cpu() - want).abs()
    mx, mean = d.max().item(), d.mean().item()
    log_metric("depth_aa", tag=tag, max=mx, mean=mean, range=float(want.max() - want.min()))
    # north-star tolerance 1e-3 of the value range (depth maps are normalised to [0, 1] for forward; `scale` for infer)
    assert mx <= 2e-3 * scale and mean <= 2e-4 * scale, (tag, mx, mean)


def test_depth_aa_golden():
    g = load_golden("depth_aa")
    m = _model()
    x, y = torch.from_numpy(g["x"]), torch.from_numpy(g["y"])
    _check("forward_golden", m(x.to(DEV)), y)
    xi, yi = torch.from_numpy(g["xi"]), torch.from_numpy(g["yi"])
    _check("infer_golden", m.infer(xi.to(DEV)), yi, scale=float(xi.max() - xi.min()))


@pytest.mark.parametrize("B,H,W", [(1, 16, 16), (2, 37, 53), (1, 392, 686), (4, 112, 96)])
def test_depth_aa_oracle(B, H, W):
    from oracle import depth_aa as oaa
    sd = synth.depth_aa_state_dict(0)
    m = _model()
    g = torch.Generator().manual_seed(B * 1000 + H + W)
    x = torch.rand(B, 1, H, W, generator=g)
    x = torch.nn.functional.avg_pool2d(x, 5, 1, 2)          # smooth-ish depth with edges
    x = (x - x.min()) / (x.max() - x.min())
    with torch.inference_mode():
        want = oaa.depth_aa_forward(sd, x)
        want_nc = oaa.depth_aa_forward(sd, x, clamp=False)
        xi = x * 7.5 + 1.25
        want_i = oaa.depth_aa_infer(sd, xi)
    _check(f"forward_{B}x{H}x{W}", m(x.to(DEV)), want)
    _check(f"forward_noclamp_{B}x{H}x{W}", m(x.to(DEV), clamp=False), want_nc)
    _check(f"infer_{B}x{H}x{W}", m.infer(xi.to(DEV)), want_i, scale=7.5)


def test_depth_anything_infer_with_depth_aa():
    """DepthAnythingModel.infer(depth_aa=True) = batch_infer with the filter between the network and dilate_edge (:153-156)."""
    from nunif_b200.iw3.depth_anything_model import DepthAnythingModel
    dm = DepthAnythingModel("Any_V2_S").load_state_dict(synth.depth_anything_v2_state_dict(0), gpu=0)
    x = synth.synth_image(5, 3, 126, 168).to(DEV)
    with pytest.raises(RuntimeError):
        dm.infer(x, depth_aa=True)
    dm.load_depth_aa(synth.depth_aa_state_dict(0))
    with torch.inference_mode():
        a = dm.infer(x, depth_aa=False, edge_dilation=0)
        b = dm.infer(x, depth_aa=True, edge_dilation=0)
        want = dm.depth_aa.infer(a.unsqueeze(0)).squeeze(0)
    assert a.shape == b.shape
    assert float((b - want).abs().max()) == 0.0
    assert float((b - a).abs().max()) > 0.0
