"""CPU checks of iw3's auto-convergence (--convergence-mode sod_v1): the oracle (oracle/sod.py) against the real reference's
fp32 output (tests/golden/sod_v1.npz), the checkpoint loader, and the dispatcher's refusal of foreign convergence models."""
import types
import pytest
import torch
import torch.nn.functional as F

from tests.util import load_golden, t
from nunif_b200 import synth
from oracle import sod as osod
from oracle.gen_golden_sod import NET_CASES, POS, EMA_RESET, frames


def _d192(i):
    """SODV1.infer's depth_192 of NET_CASES[i]: the reference's own F.interpolate of the regenerated depth."""
    d = frames(*NET_CASES[i])[1]
    return F.interpolate(d, (192, 192), mode="bilinear", antialias=False, align_corners=False)


def test_state_dict_matches_the_network():
    sd = synth.sod_v1_state_dict(0)
    assert len(synth.sod_rebnconvs()) == 112
    assert len(sd) == 112 * 7 + 14
    assert all(float((sd[n + ".bn_s1.running_var"] - 1).abs().min()) > 0 for n, *_ in synth.sod_rebnconvs())


@pytest.mark.parametrize("i", range(len(NET_CASES)))
def test_oracle_network_golden(i):
    g = load_golden("sod_v1")
    rgb, d = frames(*NET_CASES[i])
    with torch.no_grad():
        sal, d192 = osod.sod_infer(synth.sod_v1_state_dict(0), rgb, d)
    assert float((sal - t(g[f"net{i}_sal"])).abs().max()) < 1e-5
    assert torch.equal(d192, _d192(i))
    assert torch.equal(d192[..., :16, :16], t(g[f"net{i}_d192c"]))
    frac = float((t(g[f"net{i}_sal"]) > 0.5).float().mean())
    assert 0.05 < frac < 0.95, frac


@pytest.mark.parametrize("i", range(len(NET_CASES)))
def test_oracle_position_golden(i):
    g = load_golden("sod_v1")
    sal, d192 = t(g[f"net{i}_sal"]), _d192(i)
    for k, pos in enumerate(POS):
        assert torch.equal(osod.depth_position(sal, d192, pos).flatten(), t(g[f"net{i}_zpos"][k]))


def test_oracle_position_edge_cases():
    g = load_golden("sod_v1")
    sal, d192 = t(g["net0_sal"]), _d192(0)
    bg = osod.depth_position(torch.zeros_like(sal), d192, 0.3)
    assert torch.equal(bg, t(g["bg_zpos"])) and bool((bg == 0.5).all())
    flat = osod.depth_position(sal, torch.full_like(d192, 0.37), 0.3)
    assert torch.equal(flat, t(g["flat_zpos"])) and bool((flat == torch.tensor(0.37)).all())


def test_oracle_ema_golden():
    g = load_golden("sod_v1")
    raw = t(g["ema_raw"])
    ema = osod.EMA(0.9)
    assert torch.equal(ema(raw, EMA_RESET), t(g["ema_a"]))
    assert torch.equal(ema(raw.flip(0)), t(g["ema_b"]))
    # the reset after frame 1 restarts the average at frame 2
    assert float(t(g["ema_a"])[2]) == float(raw[2])


def test_loader_never_downloads(tmp_path, monkeypatch):
    from nunif_b200.iw3 import convergence_estimator as ce
    monkeypatch.setattr(ce, "HUB_MODEL_DIR", str(tmp_path))
    with pytest.raises(FileNotFoundError):
        ce.load_sod_state_dict()
    (tmp_path / "checkpoints").mkdir()
    path = tmp_path / "checkpoints" / ce.SOD_CHECKPOINT
    sd = synth.sod_v1_state_dict(0)
    torch.save({"name": "sbs.row_flow_v3", "state_dict": sd}, path)
    with pytest.raises(ValueError):
        ce.load_sod_state_dict()
    for name in ("iw3.sod_v1", "iw3.dsod_v1"):
        torch.save({"name": name, "state_dict": sd}, path)
        got = ce.load_sod_state_dict()
        assert set(got) == set(sd)


def test_foreign_convergence_model_raises():
    from nunif_b200.iw3 import apply_divergence
    args = types.SimpleNamespace(method="backward", mapper="none", convergence=0.5, divergence=2.0, synthetic_view="both",
                                 state={"convergence_model": lambda im, depth, reset_pts=None: None})
    with pytest.raises(NotImplementedError, match="ConvergenceEstimator"):
        apply_divergence(torch.zeros(1, 1, 8, 8), torch.zeros(1, 3, 8, 8), args, None)


def test_tensor_convergence_feature_terms():
    c = torch.tensor([0.2, 0.5, 0.9]).reshape(3, 1, 1, 1)
    d = torch.rand(3, 1, 4, 5)
    shift = osod.backward_index_shift(d, 2.0, c)
    for i in range(3):
        # fp32(shift_size) * c[i]: the tensor path's rounding, not the double product of the scalar path
        want = d[i] * 0.02 - (torch.tensor(0.02, dtype=torch.float32) * c[i])
        assert torch.equal(shift[i], want)
    f = osod.convergence_feature(2.0, c, 640)
    assert torch.equal(f.flatten(), (torch.tensor(-(2.0 * 0.5 * 0.01 * 640), dtype=torch.float32) * c.flatten()) / 32.0)
