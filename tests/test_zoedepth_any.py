"""CPU checks of ZoeD_Any_N / ZoeD_Any_K and the Depth-Anything V1 models: the oracle's restatement pinned against
transformers (the V1 encoder hooks, the "normed" bins head), the real iw3 batch_infer golden with prep_mod = 14, and the host
contracts of ZoeDepthAnythingModel, the V1 types and create_depth_model."""
import os
import numpy as np
import pytest
import torch

from nunif_b200 import synth
from tests.util import load_golden, t
from tests.test_oracle_golden import _da_to_hf, _zoe_to_hf


def test_depth_anything_v1_oracle_matches_transformers():
    """Any_S/B/L (and the ZoeD_Any core) hook the LAST FOUR blocks; transformers with out_features = the last four stages."""
    pytest.importorskip("transformers")
    from transformers import DepthAnythingConfig, DepthAnythingForDepthEstimation, Dinov2Config
    from oracle import depth_anything as oda
    from oracle import zoedepth_any as oza
    grid = 6
    sd = synth.depth_anything_v2_state_dict(3, pos_grid=grid)
    cfg = DepthAnythingConfig(
        backbone_config=Dinov2Config(hidden_size=384, num_hidden_layers=12, num_attention_heads=6, mlp_ratio=4, image_size=14 * grid,
                                     patch_size=14, out_features=["stage9", "stage10", "stage11", "stage12"],
                                     reshape_hidden_states=False, apply_layernorm=True, layer_norm_eps=1e-6),
        reassemble_hidden_size=384, neck_hidden_sizes=[48, 96, 192, 384], fusion_hidden_size=64, head_hidden_size=32,
        patch_size=14, reassemble_factors=[4, 2, 1, 0.5])
    hf = DepthAnythingForDepthEstimation(cfg).eval()
    missing, unexpected = hf.load_state_dict(_da_to_hf(sd), strict=False)
    assert not unexpected and all("position_ids" in m or "rel" in m for m in missing), (missing, unexpected)
    # the training grid: transformers resamples the position table by size, DINOv2 by scale factor + 0.1 (pinned elsewhere)
    x = torch.randn(2, 3, 14 * grid, 14 * grid, generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        want = hf(pixel_values=x).predicted_depth
        got = oda.depth_anything_forward(sd, x, oza.V1["vits"])
        v2 = oda.depth_anything_forward(sd, x, "vits")
    assert got.shape == want.shape == (2, 14 * grid, 14 * grid)
    assert float(want.std()) > 0.1
    assert float((got - want).abs().max()) < 2e-4 * float(want.abs().max())
    assert float((v2 - want).abs().max()) > 1e-2 * float(want.abs().max())     # the hook rule matters


def golden_inputs(g):
    """The frames of tests/golden/zoedepth_any_infer.npz, regenerated from their seeds (the file keeps a checksum and a
    corner of each, so that a change of synth.synth_image shows here)."""
    land = torch.stack([synth.synth_image(int(s), 3, *g["land_hw"].tolist(), smooth=False) for s in g["land_seeds"]])
    port = synth.synth_image(int(g["port_seed"]), 3, *g["port_hw"].tolist(), smooth=False)
    for x, name in ((land, "land"), (port, "port")):
        assert float(x.double().sum()) == pytest.approx(float(g[f"{name}_sum"]), rel=1e-9, abs=1e-6), name
        assert torch.equal(x[..., :8, :8], t(g[f"{name}_corner"])), name
    return land, port


def _beit_normed_sd(seed):
    """ZoeD_N's reduced BEiT core with ZoeD_Any_K's normed bins head (the same key names, attractors 2 x na wide)."""
    sd = synth.zoedepth_state_dict(seed, synth.ZOED_MINI)
    k = synth.zoedepth_any_state_dict(seed, synth.ZOED_ANY_MINI, normed=True)
    heads = ("conv2.", "seed_bin_regressor.", "seed_projector.", "projectors.", "attractors.", "conditional_log_binomial.")
    for name in list(sd):
        if name.startswith(heads):
            sd[name] = k[name]
    return sd


def test_normed_bins_head_matches_transformers():
    """The "normed" head (ZoeD_Any_K: SeedBinRegressor, AttractorLayer with the unnormalised first-of-pair attractor, sorted and
    clipped centres, max_depth 80) against transformers.ZoeDepthForDepthEstimation(bin_centers_type="normed")."""
    pytest.importorskip("transformers")
    from transformers import ZoeDepthConfig, ZoeDepthForDepthEstimation, BeitConfig
    from oracle import zoedepth as oz
    from oracle import zoedepth_any as oza
    cfg = oz.ZOED_MINI
    sd = _beit_normed_sd(3)
    assert sd["attractors.0._net.2.weight"].shape[0] == 32
    hf_cfg = ZoeDepthConfig(
        backbone_config=BeitConfig(image_size=16 * cfg["old_grid"], patch_size=16, hidden_size=cfg["dim"], num_hidden_layers=cfg["depth"],
                                   num_attention_heads=cfg["heads"], intermediate_size=4 * cfg["dim"], use_relative_position_bias=True,
                                   use_absolute_position_embeddings=False, use_mask_token=False, layer_scale_init_value=0.1,
                                   reshape_hidden_states=False, layer_norm_eps=1e-6,
                                   out_features=[f"stage{h + 1}" for h in cfg["hooks"]]),
        neck_hidden_sizes=list(cfg["oc"]), fusion_hidden_size=cfg["feat"], bottleneck_features=cfg["feat"], readout_type="project",
        reassemble_factors=[4, 2, 1, 0.5], num_relative_features=32, bin_embedding_dim=128, num_attractors=[16, 8, 4, 1],
        bin_centers_type="normed", bin_configurations=[{"n_bins": 64, "min_depth": 0.001, "max_depth": 80.0}])
    hf = ZoeDepthForDepthEstimation(hf_cfg).eval()
    missing, unexpected = hf.load_state_dict(_zoe_to_hf(sd, cfg), strict=False)
    assert not unexpected and all("relative_position_index" in m or "k_idx" in m or "k_minus_1" in m for m in missing), (missing, unexpected)
    x = torch.randn(2, 3, 64, 96, generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        want = hf(pixel_values=x).predicted_depth
        got = oza.zoedepth_normed_forward(sd, x, cfg)[:, 0]
    assert got.shape == want.shape == (2, 64, 96)
    assert float(want.std()) > 0.5 and float(want.max()) <= 80.0
    assert float((got - want).abs().max()) < 2e-4 * float(want.abs().max())


def test_dpt_head_taps_is_the_depth_anything_head():
    """oracle/zoedepth_any.dpt_head_taps restates oracle/depth_anything.dpt_head to expose the bins head's inputs; the two agree
    exactly, and the taps have the shapes the engine's taps 4..9 use."""
    from oracle import depth_anything as oda
    from oracle import zoedepth_any as oza
    sd = oza._core(synth.zoedepth_any_state_dict(2, synth.ZOED_ANY_MINI, False))
    x = torch.randn(2, 3, 98, 126, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        feats = oda.vit_intermediate(sd, x, oza.ZOED_ANY_MINI)
        got, taps = oza.dpt_head_taps(sd, feats, 7, 9, oza.ZOED_ANY_MINI)
        want = oda.dpt_head(sd, feats, 7, 9, oza.ZOED_ANY_MINI)
    assert torch.equal(got, want)
    assert [tuple(p.shape[-2:]) for p in taps["paths"]] == [(7, 9), (14, 18), (28, 36), (56, 72)]
    assert tuple(taps["l4_rn"].shape) == (2, 128, 4, 5) and tuple(taps["out_conv"].shape) == (2, 32, 98, 126)


def test_normed_bins_move_and_are_sorted():
    """Seeded ZoeD_Any_K weights: every attractor level moves the bins, the last level's centres reach the clip at max_depth and
    crowd into ties.  The sort never reorders them in exact arithmetic: b + inv_attractor(a - b) is non-decreasing in b (the
    slope 1 - (1 - 300 d^2) / (1 + 300 d^2)^2 is >= 0), a mean of such maps and the align_corners interpolation keep the order, and
    the seed centres are sorted.  So the sort only puts rounding-level inversions in order; this is checked, not assumed."""
    from oracle import zoedepth_any as oza
    import torch.nn.functional as F
    sd = synth.zoedepth_any_state_dict(1, synth.ZOED_ANY_MINI, normed=True)
    x = torch.randn(2, 3, 98, 126, generator=torch.Generator().manual_seed(0))
    with torch.no_grad():
        r = oza.zoedepth_any_forward(sd, x, oza.ZOED_ANY_MINI, normed=True, return_all=True)
    bins = r["bins"]
    for i in range(1, 4):
        prev = F.interpolate(bins[i - 1], bins[i].shape[-2:], mode="bilinear", align_corners=True)
        assert float((bins[i] - prev).abs().mean()) > 1e-3, i                         # the attractors move the bins
    c = r["centers"]
    assert float(c.min()) >= 1e-3 and float(c.max()) <= 80.0
    assert float((c == 80.0).float().mean()) > 1e-4                                  # the clip is reached
    scaled = (80.0 - 1e-3) * bins[3] + 1e-3
    gaps = scaled.diff(dim=1)
    assert float((gaps == 0).float().sum()) > 0                                      # crowded bins tie
    assert torch.equal(torch.sort(scaled, dim=1)[0].clip(1e-3, 80.0), c)
    assert float(gaps.min()) >= -1e-5                                                # order kept up to rounding
    assert float(r["metric_depth"].std()) > 1.0


def test_zoedepth_any_batch_infer_oracle_matches_reference_golden():
    """oracle/zoedepth_any.batch_infer against the REAL iw3/zoedepth_model.batch_infer with prep_mod = 14 (golden around a
    stand-in network, oracle/gen_golden_zoedepth_any.py): N and K, landscape batch and portrait image, flip TTA, dilation."""
    from oracle import zoedepth_any as oza
    g = load_golden("zoedepth_any_infer")
    land, port = golden_inputs(g)
    for normed, tag in ((False, "n"), (True, "k")):
        sd = synth.zoedepth_any_state_dict(5, synth.ZOED_ANY_MINI, normed=normed)
        with torch.no_grad():
            for flip in (0, 1):
                for dil in (0, 2):
                    kw = dict(flip_aug=bool(flip), edge_dilation=dil, h_height=56, v_height=70, cfg=oza.ZOED_ANY_MINI, normed=normed)
                    got = oza.batch_infer(sd, land, **kw)
                    want = t(g[f"{tag}_land_f{flip}_d{dil}"])
                    assert got.shape == want.shape and float((got - want).abs().max()) < 2e-4 * float(want.abs().max()), (tag, flip, dil)
                    got = oza.batch_infer(sd, port.unsqueeze(0), **kw)[0]
                    want = t(g[f"{tag}_port_f{flip}_d{dil}"])
                    assert got.shape == want.shape and float((got - want).abs().max()) < 2e-4 * float(want.abs().max()), (tag, flip, dil)


def test_zoedepth_any_size_rule_matches_reference_golden():
    """batch_preprocess with ensure_multiple_of = 14: network size and pads for 720p, 1080p, 4K, portrait, square, a frame smaller
    than 392 and resolution = 518, in the oracle and in the engine's host rule."""
    from oracle import frames as ofr
    from nunif_b200 import _lib
    import ctypes
    g = load_golden("zoedepth_any_infer")
    for H, W, hh, vh, oh, ow, ph, pw in g["sizes"].tolist():
        nh, nw, p_h, p_w, fh, fw = ofr.zoe_preprocess_size(H, W, hh, vh, 14)
        assert (fh + 2 * p_h, fw + 2 * p_w, p_h, p_w) == (oh, ow, ph, pw), (H, W, hh)
        o = [ctypes.c_int() for _ in range(6)]
        _lib.check(_lib.lib().nb200_zoe_preprocess_size(H, W, hh, vh, 14, *[ctypes.byref(v) for v in o]))
        nh, nw, p_h, p_w, fh, fw = (v.value for v in o)
        assert (fh + 2 * p_h, fw + 2 * p_w, p_h, p_w) == (oh, ow, ph, pw), (H, W, hh)
    assert [1080, 1920, 392, 518, 392, 700, 22, 31] in g["sizes"].tolist()


def test_zoedepth_any_model_host_contract():
    from nunif_b200.iw3 import ZoeDepthAnythingModel, ZoeDepthModel
    from nunif_b200.iw3 import zoedepth_any_model as zam
    for mt, f in (("ZoeD_Any_N", "depth_anything_metric_depth_indoor.pt"), ("ZoeD_Any_K", "depth_anything_metric_depth_outdoor.pt")):
        assert ZoeDepthAnythingModel.supported(mt) and not ZoeDepthModel.supported(mt)
        assert ZoeDepthAnythingModel.get_model_path(mt).endswith(os.path.join("checkpoints", f))
        m = ZoeDepthAnythingModel(mt)
        assert m.is_metric() and not m.loaded() and m.get_name() == "ZoeDepth"
        assert not ZoeDepthAnythingModel.multi_gpu_supported(mt)
        with pytest.raises(FileNotFoundError):
            m.load_model(mt, device=torch.device("cuda", 0))                   # never downloads
    for bad in ("ZoeD_N", "ZoeD_K", "Any_L"):
        with pytest.raises(ValueError):
            ZoeDepthAnythingModel(bad)
    with pytest.raises(ValueError, match="ZoeDepthAnythingModel"):
        ZoeDepthModel("ZoeD_Any_N")
    with pytest.raises(RuntimeError):
        zam.ZoeDepthAnythingNet({"a": torch.zeros(1)}, "cpu")                  # no CPU path
    with pytest.raises(ValueError):
        zam.ZoeDepthAnythingNet({}, "cuda:0", "ZoeD_N")


def test_depth_anything_v1_host_contract():
    from nunif_b200.iw3 import DepthAnythingModel
    for mt, f in (("Any_S", "depth_anything_vits14.pth"), ("Any_B", "depth_anything_vitb14.pth"), ("Any_L", "depth_anything_vitl14.pth")):
        assert DepthAnythingModel.supported(mt)
        assert DepthAnythingModel.get_model_path(mt).endswith(os.path.join("checkpoints", f))
        m = DepthAnythingModel(mt)
        assert not m.is_metric() and m.get_name() == "DepthAnything"
        with pytest.raises(ValueError, match="depth_aa"):
            m.load_depth_aa({})                                                # V2 only (AA_SUPPORTED_MODELS)


def test_create_depth_model_routes_and_refuses():
    from nunif_b200.iw3 import create_depth_model, ZoeDepthModel, ZoeDepthAnythingModel, DepthAnythingModel
    from nunif_b200.iw3.depth_model_factory import NOT_BUILT
    assert type(create_depth_model("ZoeD_N")) is ZoeDepthModel
    for mt in ("ZoeD_Any_N", "ZoeD_Any_K"):
        m = create_depth_model(mt)
        assert type(m) is ZoeDepthAnythingModel and m.model_type == mt
    for mt in ("Any_S", "Any_B", "Any_L", "Any_V2_S", "Any_V2_B", "Any_V2_L"):
        m = create_depth_model(mt)
        assert type(m) is DepthAnythingModel and m.model_type == mt
    for mt in ("ZoeD_K", "ZoeD_NK", "Any_V2_N_L", "Any_V2_K_S", "Any_V2_N", "Distill_Any_B", "DepthPro", "VDA_L", "VDA_Stream_Metric_S",
               "Any_V3_Mono"):
        assert mt in NOT_BUILT
        with pytest.raises(NotImplementedError, match=mt):
            create_depth_model(mt)
    with pytest.raises(ValueError, match="not supported"):
        create_depth_model("NoSuchModel")
