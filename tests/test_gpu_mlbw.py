"""GPU: sbs.mlbw (csrc/mlbw.cu + wgmma GEMMs) in delta_output mode and apply_divergence_nn_delta_weight against the
reference-generated golden (tests/golden/mlbw.npz: the REAL model, fp32 on the CPU) and against the oracle for the 4-layer and
`small` variants.  The engine runs the reference's CUDA numerics (fp16 autocast): bounds as for sbs.row_flow_v3."""
import pytest
import torch

from tests.util import load_golden, log_metric
from nunif_b200 import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def t(a, dev=None):
    x = torch.from_numpy(a)
    return x.to(dev) if dev else x


def stats(got, want):
    d = (got.float().cpu() - want.float()).abs()
    return {"max": d.max().item(), "mean": d.mean().item()}


def test_mlbw_delta_golden():
    from nunif_b200.iw3 import MLBW
    g = load_golden("mlbw")
    m = MLBW(synth.mlbw_state_dict(0), DEV)
    assert m.num_layers == 2
    delta, lw = m(t(g["x"], DEV))
    sd, sw = stats(delta, t(g["delta"])), stats(lw, t(g["layer_weight"]))
    rng = float(t(g["delta"]).abs().max())
    log_metric("mlbw_delta", delta_max=sd["max"], delta_mean=sd["mean"], delta_range=rng, lw_max=sw["max"], lw_mean=sw["mean"])
    # fp16 network vs the fp32 reference: relative to the +-range of the flow (pixels) / the [0, 1] weights
    assert sd["max"] < 2e-2 * max(rng, 1.0) and sd["mean"] < 2e-3 * max(rng, 1.0), sd
    assert sw["max"] < 2e-2 and sw["mean"] < 2e-3, sw
    assert float((lw.sum(1) - 1).abs().max()) < 1e-5


def test_mlbw_apply_divergence_golden():
    from nunif_b200.iw3 import MLBW, apply_divergence_nn_LR
    g = load_golden("mlbw")
    m = MLBW(synth.mlbw_state_dict(0), DEV)
    d = t(g["d"], DEV)
    c = torch.stack([synth.synth_image(4 + i, 3, 140, 260) for i in range(2)]).to(DEV)
    l, r = apply_divergence_nn_LR(m, c, d, 2.0, 0.5, steps=1)
    sl, sr = stats(l, t(g["left"])), stats(r, t(g["right"]))
    log_metric("mlbw_lr", left_max=sl["max"], right_max=sr["max"], left_mean=sl["mean"], right_mean=sr["mean"])
    assert sl["mean"] < 1e-3 and sr["mean"] < 1e-3 and sl["max"] < 3e-2 and sr["max"] < 3e-2, (sl, sr)


@pytest.mark.parametrize("L,small,B,h,w", [(4, False, 1, 70, 130), (2, True, 2, 33, 96), (2, False, 1, 392, 686)])
def test_mlbw_variants_oracle(L, small, B, h, w):
    """num_layers = 4 (C = 128, 4 heads) and the `small` layout (two blocks, shifted along x only) against the oracle, which
    tests/test_oracle_golden.py::test_mlbw_variants_oracle_matches_reference pins to the real model at the first two shapes."""
    from oracle import mlbw as om
    from oracle.row_flow import make_input
    from nunif_b200.iw3 import MLBW
    sd = synth.mlbw_state_dict(1, num_layers=L)
    if small:
        sd = {k: v for k, v in sd.items() if not (k.startswith("lv2.2.") or k.startswith("lv2.3."))}
    d = synth.synth_depth(7, B, h, w)
    x = make_input(d, 2.5, 0.4)
    with torch.inference_mode():
        wd, ww = om.mlbw_delta(sd, x, num_layers=L, small=small)
    m = MLBW(sd, DEV)
    assert m.num_layers == L
    delta, lw = m(x.to(DEV))
    sd_, sw = stats(delta, wd), stats(lw, ww)
    rng = float(wd.abs().max())
    log_metric(f"mlbw_L{L}_small{int(small)}_{h}x{w}", delta_max=sd_["max"], delta_mean=sd_["mean"], delta_range=rng, lw_max=sw["max"], lw_mean=sw["mean"])
    assert sd_["max"] < 2e-2 * max(rng, 1.0) and sd_["mean"] < 2e-3 * max(rng, 1.0), sd_
    assert sw["max"] < 2e-2 and sw["mean"] < 2e-3, sw
