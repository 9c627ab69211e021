"""GPU parity of the iw3 path (path B) against the oracle and the committed reference goldens.
All calls go through the C ABI (nunif_b200._lib)."""
import pytest
import torch

from tests.util import load_golden, t, log_metric, stats
from nunif_b200 import synth
from oracle import iw3 as oiw

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-3  # north_star: within 1e-3 max-abs of the reference output


def test_backward_warp_golden():
    from nunif_b200.iw3 import apply_divergence_grid_sample
    g = load_golden("backward_warp")
    c, d_lo, d_hi = t(g["c"], DEV), t(g["d_lo"], DEV), t(g["d_hi"], DEV)
    for sv in ("both", "left", "right"):
        l, r = apply_divergence_grid_sample(c, d_lo, 2.0, 0.5, sv)
        sl, sr = stats(l, t(g[f"bw_{sv}_l"])), stats(r, t(g[f"bw_{sv}_r"]))
        log_metric("backward_warp_" + sv, **sl)
        assert sl["max"] < TOL and sr["max"] < TOL, (sv, sl, sr)
    l, r = apply_divergence_grid_sample(c, d_hi, 5.0, 0.3, "both")
    assert stats(l, t(g["bw_hi_l"]))["max"] < TOL and stats(r, t(g["bw_hi_r"]))["max"] < TOL


def test_backward_warp_sbs_and_anaglyph_epilogues():
    from nunif_b200.iw3 import apply_divergence_grid_sample
    g = load_golden("backward_warp")
    c, d = t(g["c"], DEV), t(g["d_lo"], DEV)
    l, r = apply_divergence_grid_sample(c, d, 2.0, 0.5, "both")
    sbs = apply_divergence_grid_sample(c, d, 2.0, 0.5, "both", compose=1)
    assert torch.equal(sbs, torch.cat([l, r], dim=3))
    ana = apply_divergence_grid_sample(c, d, 2.0, 0.5, "both", compose=2)
    want = torch.stack([oiw.dubois(l[i].cpu(), r[i].cpu(), True) for i in range(l.shape[0])])
    assert stats(ana, want)["max"] < 2e-5


def test_backward_warp_1080p_properties():
    """Full-size, size-independent checks: zero divergence is the identity; constant depth is a pure shift."""
    from nunif_b200.iw3 import apply_divergence_grid_sample
    c = synth.synth_image(3, 3, 1080, 1920).unsqueeze(0).to(DEV)
    d = synth.synth_depth(4, 1, 392, 686).to(DEV)
    l, r = apply_divergence_grid_sample(c, d, 0.0, 0.5, "both")
    assert stats(l, c)["max"] < 1e-4 and stats(r, c)["max"] < 1e-4
    l, r = apply_divergence_grid_sample(c, torch.full_like(d, 0.5), 2.0, 0.5, "both")
    assert stats(l, c)["max"] < 1e-4
    # oracle at full size
    lo, ro = oiw.apply_divergence_grid_sample(c.cpu(), d.cpu(), 2.0, 0.5, "both")
    l, r = apply_divergence_grid_sample(c, d, 2.0, 0.5, "both")
    s = stats(l, lo)
    log_metric("backward_warp_1080p", **s)
    assert s["max"] < TOL and stats(r, ro)["max"] < TOL


def test_forward_warp_golden_exact_fullres_depth():
    """With a full-resolution depth there is no resize in the path: results must be bit-exact."""
    from nunif_b200.iw3 import apply_divergence_forward_warp
    g = load_golden("forward_warp")
    c, d_hi = t(g["c"], DEV), t(g["d_hi"], DEV)
    for tag, div, conv, wb in [("hi", 4.0, 0.5, False), ("hi_wb", 10.0, 0.3, True)]:
        for method in ("forward_fill", "forward"):
            l, r, lm, rm = apply_divergence_forward_warp(c, d_hi, div, conv, method=method, return_mask=True, width_base=wb)
            for got, key in ((l, "l"), (r, "r"), (lm, "lm"), (rm, "rm")):
                s = stats(got, t(g[f"fw_{tag}_{method}_{key}"]))
                log_metric(f"forward_warp_{tag}_{method}_{key}", **s)
                assert s["max"] == 0.0, (tag, method, key, s)
    for sv in ("left", "right"):
        l, r = apply_divergence_forward_warp(c, d_hi, 2.0, 0.5, method="forward_fill", synthetic_view=sv, width_base=False)
        assert stats(l, t(g[f"fw_{sv}_l"]))["max"] == 0.0 and stats(r, t(g[f"fw_{sv}_r"]))["max"] == 0.0


def test_forward_warp_iteration_cap():
    """Holes wider than 100 px: the reference's 100-iteration cap leaves negative cells (forward_warp.py:18,45)."""
    from nunif_b200.iw3 import apply_divergence_forward_warp
    g = load_golden("forward_warp")
    l, r = apply_divergence_forward_warp(t(g["cl"], DEV), t(g["dl"], DEV), 60.0, 0.0, method="forward_fill", width_base=True)
    assert (t(g["fw_long_l"]) < 0).any() or (t(g["fw_long_r"]) < 0).any()
    assert stats(l, t(g["fw_long_l"]))["max"] == 0.0 and stats(r, t(g["fw_long_r"]))["max"] == 0.0


def test_depth_resize_matches_aten():
    import ctypes
    from nunif_b200 import _lib
    g = load_golden("forward_warp")
    d = t(g["d_lo"], DEV)
    B, _, h, w = d.shape
    out = torch.empty((B, 1, 72, 128), device=DEV)
    _lib.check(_lib.lib().nb200_depth_resize_aa(_lib.ptr(d), B, h, w, 72, 128, _lib.ptr(out), _lib.stream_ptr()))
    want = oiw.upsample_depth(d.cpu(), (72, 128))
    s = stats(out, want)
    log_metric("depth_resize_aa", **s)
    assert s["max"] < 2e-6


def test_forward_warp_lowres_depth():
    """Low-res depth goes through the fused AA resize; ulp-level depth differences can move a splat across a
    pixel boundary, so parity is: >= 99.9% of pixels within 1e-3 (DESIGN.md 'forward warp parity')."""
    from nunif_b200.iw3 import apply_divergence_forward_warp
    g = load_golden("forward_warp")
    c, d_lo = t(g["c"], DEV), t(g["d_lo"], DEV)
    l, r = apply_divergence_forward_warp(c, d_lo, 4.0, 0.5, method="forward_fill", width_base=False)
    sl, sr = stats(l, t(g["fw_lo_forward_fill_l"])), stats(r, t(g["fw_lo_forward_fill_r"]))
    log_metric("forward_warp_lowres", **sl)
    assert sl["frac_gt_1e3"] < 1e-3 and sr["frac_gt_1e3"] < 1e-3, (sl, sr)


def test_forward_warp_1080p_vs_oracle():
    from nunif_b200.iw3 import apply_divergence_forward_warp
    c = synth.synth_image(5, 3, 1080, 1920).unsqueeze(0).to(DEV)
    d = synth.synth_depth(6, 1, 1080, 1920).to(DEV)
    l, r = apply_divergence_forward_warp(c, d, 2.0, 0.5, method="forward_fill", width_base=False)
    lo, ro = oiw.forward_warp(c.cpu(), d.cpu(), 2.0, 0.5, fill=True, width_base=False)
    sl, sr = stats(l, lo), stats(r, ro)
    log_metric("forward_warp_1080p", **sl)
    assert sl["max"] == 0.0 and sr["max"] == 0.0
    sbs = apply_divergence_forward_warp(c, d, 2.0, 0.5, method="forward_fill", width_base=False, compose=1)
    assert torch.equal(sbs, torch.cat([l, r], dim=3).clamp(0, 1))


def test_dilate_edge_minmax_mapper():
    from nunif_b200.iw3 import dilate_edge, minmax_normalize
    g = load_golden("dilation")
    x = t(g["x"], DEV)
    for key in g:
        if key.startswith("dil_"):
            n = [int(v) for v in key.split("_")[1:]]
            n = n[0] if len(n) == 1 else n
            s = stats(dilate_edge(x, n), t(g[key]))
            log_metric(key, **s)
            assert s["max"] < 1e-4, (key, s)
    mm = minmax_normalize(x[:1])
    assert stats(mm[0], t(g["minmax0"]))["max"] < 1e-6
    assert stats(minmax_normalize(x[:1], mapper="div_6")[0], t(g["div_6"]))["max"] < 1e-5
    assert stats(minmax_normalize(x[:1], mapper="div_1")[0], t(g["div_1"]))["max"] < 1e-5
    with pytest.raises(ValueError):
        dilate_edge(x, "3")
    # constant frame: scale == 0 branch (depth_scaler.py:13-15)
    z = torch.full((1, 1, 8, 8), 0.25, device=DEV)
    assert torch.equal(minmax_normalize(z), z)


def test_anaglyph_golden():
    from nunif_b200.iw3 import apply_anaglyph_redcyan
    g = load_golden("anaglyph")
    l, r = t(g["l"], DEV), t(g["r"], DEV)
    assert stats(apply_anaglyph_redcyan(l, r, "dubois"), t(g["dubois"]))["max"] < 2e-5
    assert stats(apply_anaglyph_redcyan(l, r, "dubois2"), t(g["dubois2"]))["max"] < 2e-5
    with pytest.raises(ValueError):
        apply_anaglyph_redcyan(l, r, "nope")
