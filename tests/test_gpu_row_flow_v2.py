"""GPU parity of `--method row_flow_v2` (the fused sbs.row_flow_v2 kernel, csrc/rowflow_v2.cu) and `--method row_flow_v3_sym`
(one delta, both eyes in one warp launch) against the real reference's fp32 output (tests/golden/row_flow_v2.npz) and the
oracle run under CUDA autocast."""
import types
import pytest
import torch

from tests.util import load_golden, t, log_metric, stats, true_fp32
from nunif_b200 import synth
from oracle import row_flow as orf, row_flow_v2 as orf2
from oracle.gen_golden_row_flow_v2 import LR_CASES, SYM_CASES, VIEWS, lr_inputs, sym_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _sd(sd):
    return {k: v.to(DEV) for k, v in sd.items()}


def _amp_v2(sdc):
    def f(x):
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            return orf2.row_flow_v2_delta(sdc, x.to(DEV))       # fp16, as _forward_delta_only returns it
    return f


def _amp_v3(sdc):
    def f(x):
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            return orf.row_flow_delta(sdc, x.to(DEV)).float()  # row_flow_v3.py:103 casts to fp32
    return f


def _check_delta(got, x, sd, tag):
    """The engine's delta against the fp32 oracle, within the autocast oracle's own error (x 1.5 on the max, 1.25 on the mean)."""
    sdc = _sd(sd)
    with torch.no_grad(), true_fp32():
        ref32 = orf2.row_flow_v2_delta(sdc, x.to(DEV)).float()
    refamp = _amp_v2(sdc)(x).float()
    scale = float(ref32.abs().max())
    e_ref, e_our = stats(refamp, ref32), stats(got, ref32)
    log_metric("row_flow_v2_delta_" + tag, ours_max=e_our["max"], ours_mean=e_our["mean"], refamp_max=e_ref["max"],
               refamp_mean=e_ref["mean"], scale=scale)
    assert e_our["max"] <= max(1e-3 * scale, 1.5 * e_ref["max"]), (tag, e_our, e_ref)
    assert e_our["mean"] <= max(1e-3 * scale, 1.25 * e_ref["mean"]), (tag, e_our, e_ref)


def test_row_flow_v2_delta_golden():
    from nunif_b200.iw3 import RowFlowV2
    g = load_golden("row_flow_v2")
    sd = synth.row_flow_v2_state_dict(0)
    m = RowFlowV2(sd, DEV)
    sdc = _sd(sd)
    for i in range(4):
        x, ref32 = t(g[f"net{i}_x"], DEV), t(g[f"net{i}_delta"], DEV)
        got = m(x)
        assert got.shape == (x.shape[0], 2, x.shape[2], x.shape[3]) and float(got[:, 1].abs().max()) == 0.0
        got = got[:, :1]
        assert torch.equal(got, got.half().float())    # fp16 values
        refamp = _amp_v2(sdc)(x).float()
        scale = float(ref32.abs().max())
        e_ref, e_our = stats(refamp, ref32), stats(got, ref32)
        log_metric(f"row_flow_v2_delta_golden{i}", ours_max=e_our["max"], ours_mean=e_our["mean"], refamp_max=e_ref["max"],
                   refamp_mean=e_ref["mean"], scale=scale)
        assert e_our["max"] <= max(1e-3 * scale, 1.5 * e_ref["max"]), (i, e_our, e_ref)
        assert e_our["mean"] <= max(1e-3 * scale, 1.25 * e_ref["mean"]), (i, e_our, e_ref)


@pytest.mark.parametrize("B,h,w", [(1, 16, 109), (2, 16, 110), (1, 16, 111), (1, 15, 219), (3, 17, 220), (1, 31, 221),
                                   (2, 32, 64), (1, 33, 5), (4, 1, 130), (4, 1, 5), (1, 3, 1)])
def test_row_flow_v2_delta_tile_edges(B, h, w):
    """Widths one below, at and one above multiples of the 110-column tile, heights around the 16-row strip, h = 1, w = 5."""
    from nunif_b200.iw3 import RowFlowV2
    from nunif_b200.iw3.row_flow import make_input
    sd = synth.row_flow_v2_state_dict(1)
    m = RowFlowV2(sd, DEV)
    d = synth.synth_depth(40 + h + w, B, h, w).to(DEV)
    x = make_input(d, 2.5, 0.4)
    _check_delta(m.delta_x(x), x, sd, f"{B}x{h}x{w}")


@pytest.mark.parametrize("i", range(len(LR_CASES)))
def test_row_flow_v2_lr_golden(i):
    from nunif_b200.iw3 import RowFlowV2, apply_divergence_nn_LR
    g = load_golden("row_flow_v2")
    m = RowFlowV2(synth.row_flow_v2_state_dict(0), DEV)
    d, c = (v.to(DEV) for v in lr_inputs())
    div, conv, view, steps, psb = LR_CASES[i]
    l, r = apply_divergence_nn_LR(m, c, d, div, conv, steps=steps, synthetic_view=VIEWS[view], preserve_screen_border=bool(psb))
    for tag, eye in (("left", l), ("right", r)):
        if f"v2lr{i}_{tag}" in g:
            s = stats(eye, t(g[f"v2lr{i}_{tag}"]))
            log_metric(f"row_flow_v2_lr{i}_{tag}", max=s["max"], mean=s["mean"])
            assert s["mean"] < 1e-3 * steps and s["max"] < 3e-2 * steps, (tag, s)
        else:
            assert torch.equal(eye, c)


@pytest.mark.parametrize("i", range(len(SYM_CASES)))
def test_row_flow_v3_sym_golden(i):
    from nunif_b200.iw3 import RowFlowV3, apply_divergence_nn_LR
    g = load_golden("row_flow_v2")
    m = RowFlowV3(synth.row_flow_v3_state_dict(2), DEV, symmetric=True)
    div, conv, view, h, w, H, W = SYM_CASES[i]
    d, c = (v.to(DEV) for v in sym_inputs(i, h, w, H, W))
    l, r = apply_divergence_nn_LR(m, c, d, div, conv, steps=3, synthetic_view=VIEWS[view], preserve_screen_border=True)
    for tag, eye in (("left", l), ("right", r)):
        if f"sym{i}_{tag}" in g:
            s = stats(eye, t(g[f"sym{i}_{tag}"]))
            log_metric(f"row_flow_v3_sym{i}_{tag}", max=s["max"], mean=s["mean"])
            assert s["mean"] < 1e-3 and s["max"] < 3e-2, (tag, s)
        else:   # the un-warped eye of a single view is c, bit for bit
            assert torch.equal(eye, c)


def test_sym_warp_equals_two_delta_warps():
    """nb200_backward_warp_delta_sym against nb200_backward_warp_delta with +delta and -delta, bit for bit."""
    from nunif_b200 import _lib
    from nunif_b200.iw3.row_flow import _warp_delta
    for (H, W, h, w) in ((72, 130, 40, 65), (40, 66, 40, 66), (61, 37, 61, 37)):
        c = synth.synth_image(5, 3, H, W).unsqueeze(0).expand(2, -1, -1, -1).contiguous().to(DEV)
        delta = (torch.randn(2, 1, h, w, generator=torch.Generator().manual_seed(h)) * 3).to(DEV)
        scale = 1.0 / (w // 2 - 1)
        left, right = torch.empty_like(c), torch.empty_like(c)
        _lib.check(_lib.lib().nb200_backward_warp_delta_sym(_lib.ptr(c), _lib.ptr(delta), 2, H, W, h, w, scale, 1, 1, _lib.ptr(left),
                                                            _lib.ptr(right), _lib.stream_ptr(c.device)))
        assert torch.equal(left, _warp_delta(c, delta, scale)) and torch.equal(right, _warp_delta(c, -delta, scale)), (H, W)


def test_f16_warp_rounds_like_aten():
    """nb200_backward_warp_delta_f16 against the reference's backward_warp on an fp16 delta with a 0-dim fp32 CUDA delta_scale."""
    from nunif_b200.iw3.row_flow import _warp_delta
    H, W, h, w = 90, 160, 45, 80
    c = synth.synth_image(6, 3, H, W).unsqueeze(0).to(DEV)
    delta = (torch.randn(1, 1, h, w, generator=torch.Generator().manual_seed(1)) * 3).half().to(DEV)
    scale = 1.0 / (w // 2 - 1)
    got = _warp_delta(c, delta.float(), scale, f16=True)
    with true_fp32():
        want = orf2.backward_warp(c, delta, torch.tensor(scale, dtype=torch.float32, device=DEV))
    s = stats(got, want)
    assert s["max"] < 1e-4, s


def _frames(seed):
    c = torch.stack([synth.synth_image(seed + i, 3, 1080, 1920) for i in range(4)]).to(DEV)
    d = synth.synth_depth(seed + 10, 4, 392, 686).to(DEV)
    return c, d


def test_row_flow_v2_1080p_matches_oracle_amp():
    from nunif_b200.iw3 import RowFlowV2, apply_divergence_nn_LR
    sd = synth.row_flow_v2_state_dict(1)
    m = RowFlowV2(sd, DEV)
    c, d = _frames(50)
    l, r = apply_divergence_nn_LR(m, c, d, 2.0, 0.5)
    with torch.no_grad(), true_fp32():
        lo, ro = orf2.apply_divergence_nn_delta_LR(_amp_v2(_sd(sd)), c, d, 2.0, 0.5)
    sl, sr = stats(l, lo), stats(r, ro)
    log_metric("row_flow_v2_1080p", left_max=sl["max"], right_max=sr["max"], left_mean=sl["mean"], right_mean=sr["mean"])
    assert sl["mean"] < 1e-3 and sr["mean"] < 1e-3, (sl, sr)


def test_row_flow_v3_sym_1080p_matches_oracle_amp():
    from nunif_b200.iw3 import RowFlowV3, apply_divergence_nn_LR
    sd = synth.row_flow_v3_state_dict(3)
    m = RowFlowV3(sd, DEV, symmetric=True)
    c, d = _frames(60)
    l, r = apply_divergence_nn_LR(m, c, d, 2.0, 0.5)
    with torch.no_grad(), true_fp32():
        lo, ro = orf2.apply_divergence_nn_symmetric(_amp_v3(_sd(sd)), c, d, 2.0, 0.5)
    sl, sr = stats(l, lo), stats(r, ro)
    log_metric("row_flow_v3_sym_1080p", left_max=sl["max"], right_max=sr["max"], left_mean=sl["mean"], right_mean=sr["mean"])
    assert sl["mean"] < 1e-3 and sr["mean"] < 1e-3, (sl, sr)


@pytest.mark.parametrize("method", ["row_flow_v2", "row_flow_v3_sym", "row_flow_sym"])
def test_apply_divergence_with_loaded_model(method, tmp_path):
    from nunif_b200.iw3 import apply_divergence, load_row_flow_model, RowFlowV2
    name, sd = (("sbs.row_flow_v2", synth.row_flow_v2_state_dict(0)) if method == "row_flow_v2"
                else ("sbs.row_flow_v3", synth.row_flow_v3_state_dict(2)))
    p = tmp_path / "ckpt.pth"
    torch.save({"name": name, "state_dict": sd}, str(p))
    m = load_row_flow_model(method, DEV, path=str(p))
    assert isinstance(m, RowFlowV2) == (method == "row_flow_v2") and m.symmetric == (method != "row_flow_v2")
    args = types.SimpleNamespace(method=method, mapper="none", convergence=0.5, divergence=2.0, synthetic_view="both")
    d, c = (v.to(DEV) for v in sym_inputs(0, *SYM_CASES[0][3:]))
    left, right = apply_divergence(d[0], c[0], args, m)
    assert left.shape == right.shape == c[0].shape
    assert not torch.equal(left, right)
