"""ORACLE (test infrastructure only - never imported by nunif_b200/): CPU/torch restatement of ZoeD_Any_N / ZoeD_Any_K, the
Depth-Anything metric depth networks the reference loads through torch.hub (iw3/zoedepth_model.py:154-170,
"nagadomi/Depth-Anything_iw3:main", DepthAnythingMetricDepth, model_type "indoor" / "outdoor") - THIRD-PARTY code
(LiheYoung/Depth-Anything metric_depth: ZoeDepth over DepthAnythingCore) that is not in the reference tree and cannot be
fetched here - and of the Depth-Anything V1 relative models Any_S/B/L.

PARITY UNPINNED against the reference's own copy: this file restates the published composition
  * the Depth-Anything V1 encoder: DINOv2 ViT/14, get_intermediate_layers(x, 4, return_class_token=True) = the LAST FOUR
    blocks through the final norm, class token ignored.  It runs oracle/depth_anything.vit_intermediate unchanged: the V1
    and ZoeD_Any configurations are entries of its ENCODERS table (registered below) whose hook indices are the last four
    blocks,
  * the Depth-Anything DPT head, with the points DepthAnythingCore hooks for the bins head: out_conv (the ReLU inside
    output_conv2), l4_rn, r4 .. r1, and the relative depth (dpt_head_taps; its depth output is checked equal to
    oracle/depth_anything.dpt_head in tests/test_zoedepth_any.py),
  * the ZoeDepth v1 bins head: "softplus" for indoor = oracle/zoedepth.metric_head (ZoeD_N's head, called as is), "normed"
    with max_depth 80 for outdoor (metric_head_normed, written line by line from the module code with the helpers of
    oracle/zoedepth.py),
with the checkpoint key names `core.core.pretrained.*`, `core.core.depth_head.*`, `conv2`, `seed_bin_regressor`, ...
(checkpoint saved as {"model": state_dict}).  Every part that has an independent implementation is pinned against
transformers 5.5 (tests/test_zoedepth_any.py): the V1 encoder + head against DepthAnythingForDepthEstimation with the last
four stages, the normed bins head against ZoeDepthForDepthEstimation with bin_centers_type="normed" (over ZoeD_N's BEiT
core, zoedepth_normed_forward).  The composition itself (which hooks feed which head input) is not pinned by either.

Functional style (state_dict in, tensors out) so the same code runs in fp32 on the CPU or under CUDA autocast in the GPU tests.
"""
import torch
import torch.nn.functional as F

from . import depth_anything as oda
from . import zoedepth as oz

PATCH = 14
PRE = "core.core."
MIN_DEPTH = 1e-3
MAX_DEPTH = {False: 10.0, True: 80.0}      # indoor ("softplus", unused by that head) / outdoor ("normed")


def _last4(dim, depth, heads, feat, oc):
    return (dim, depth, heads, tuple(range(depth - 4, depth)), feat, tuple(oc))


# ENCODERS entries (dim, depth, heads, hooked blocks, head features, head out_channels) with the V1 hook rule
V1 = {e: "v1_" + e for e in ("vits", "vitb", "vitl")}
ZOED_ANY = "zoed_any_vitl"
ZOED_ANY_MINI = "zoed_any_mini"            # reduced configuration for fast tests (same code path): head dim 64, 4 blocks
_CONFIGS = {**{V1[e]: _last4(c[0], c[1], c[2], c[4], c[5]) for e, c in oda.ENCODERS.items() if e in V1},
            ZOED_ANY: _last4(1024, 24, 16, 256, (256, 512, 1024, 1024)),
            ZOED_ANY_MINI: _last4(256, 4, 4, 128, (64, 128, 256, 256))}
for _k, _v in _CONFIGS.items():
    assert oda.ENCODERS.setdefault(_k, _v) == _v


def _core(sd):
    """ZoeD_Any's `core.core.pretrained.*` / `core.core.depth_head.*` under the Depth-Anything key names."""
    return {k[len(PRE):]: v for k, v in sd.items() if k.startswith(PRE)}


def dpt_head_taps(sd, feats, ph, pw, encoder):
    """oracle/depth_anything.dpt_head (Depth-Anything DPTHead.forward) -> (relative depth B,1,H,W after the model-level ReLU,
    taps): taps = the DepthAnythingCore hooks, "l4_rn", "paths" (refinenet4 .. refinenet1 outputs), "out_conv"."""
    dim = oda.ENCODERS[encoder][0]
    layers = []
    for i, (x, _cls) in enumerate(feats):
        B = x.shape[0]
        x = x.permute(0, 2, 1).reshape(B, dim, ph, pw)
        x = F.conv2d(x, sd[f"depth_head.projects.{i}.weight"], sd[f"depth_head.projects.{i}.bias"])
        if i == 0:
            x = F.conv_transpose2d(x, sd["depth_head.resize_layers.0.weight"], sd["depth_head.resize_layers.0.bias"], stride=4)
        elif i == 1:
            x = F.conv_transpose2d(x, sd["depth_head.resize_layers.1.weight"], sd["depth_head.resize_layers.1.bias"], stride=2)
        elif i == 3:
            x = F.conv2d(x, sd["depth_head.resize_layers.3.weight"], sd["depth_head.resize_layers.3.bias"], stride=2, padding=1)
        layers.append(F.conv2d(x, sd[f"depth_head.scratch.layer{i + 1}_rn.weight"], None, padding=1))
    l1, l2, l3, l4 = layers
    s = "depth_head.scratch."
    p4 = oda._fusion(sd, s + "refinenet4.", l4, None, size=l3.shape[2:])
    p3 = oda._fusion(sd, s + "refinenet3.", p4, l3, size=l2.shape[2:])
    p2 = oda._fusion(sd, s + "refinenet2.", p3, l2, size=l1.shape[2:])
    p1 = oda._fusion(sd, s + "refinenet1.", p2, l1)
    out = F.conv2d(p1, sd[s + "output_conv1.weight"], sd[s + "output_conv1.bias"], padding=1)
    out = F.interpolate(out, (ph * PATCH, pw * PATCH), mode="bilinear", align_corners=True)
    act = F.relu(F.conv2d(out, sd[s + "output_conv2.0.weight"], sd[s + "output_conv2.0.bias"], padding=1))
    out = F.relu(F.conv2d(act, sd[s + "output_conv2.2.weight"], sd[s + "output_conv2.2.bias"]))
    return F.relu(out), {"l4_rn": l4, "paths": [p4, p3, p2, p1], "out_conv": act}


def _seed_normed(sd, x, min_depth, max_depth):
    """SeedBinRegressor.forward (localbins_layers.py / transformers ZoeDepthSeedBinRegressor, "normed"), line by line and
    without added casts: under autocast B is fp16, sum / cumsum run in fp32."""
    B = oz._mlp2(sd, "seed_bin_regressor.", x, F.relu)
    eps = 1e-3
    B = B + eps
    B_widths_normed = B / B.sum(dim=1, keepdim=True)
    B_widths = (max_depth - min_depth) * B_widths_normed
    B_widths = F.pad(B_widths, (0, 0, 0, 0, 1, 0), mode="constant", value=min_depth)
    B_edges = torch.cumsum(B_widths, dim=1)
    B_centers = 0.5 * (B_edges[:, :-1, ...] + B_edges[:, 1:, ...])
    return B_widths_normed, B_centers


def _attractor_normed(sd, i, x, b_prev, prev_b_embedding, min_depth, max_depth):
    """AttractorLayer.forward (attractor.py / transformers ZoeDepthAttractorLayer; attractor_type "inv", kind "mean",
    memory_efficient False).  The 2 n_attractors outputs are viewed as (na, 2) and element 0 is kept WITHOUT the
    normalisation (upstream bug, kept: the weights were trained with it).  -> (b_new_centers, sorted clipped B_centers)."""
    prev_b_embedding = F.interpolate(prev_b_embedding, x.shape[-2:], mode="bilinear", align_corners=True)
    x = x + prev_b_embedding
    A = oz._mlp2(sd, f"attractors.{i}.", x, F.relu)
    eps = 1e-3
    A = A + eps
    n, c, h, w = A.shape
    A = A.view(n, oz.N_ATTRACTORS[i], 2, h, w)
    A_normed = A[:, :, 0, ...]
    b_prev = F.interpolate(b_prev, (h, w), mode="bilinear", align_corners=True)
    b_centers = b_prev
    delta_c = torch.mean(oz.inv_attractor(A_normed.unsqueeze(2) - b_centers.unsqueeze(1)), dim=1)
    b_new_centers = b_centers + delta_c
    B_centers = (max_depth - min_depth) * b_new_centers + min_depth
    B_centers, _ = torch.sort(B_centers, dim=1)
    B_centers = torch.clip(B_centers, min_depth, max_depth)
    return b_new_centers, B_centers


def metric_head_normed(sd, act, bottleneck, blocks, rel, internals=None, min_depth=MIN_DEPTH, max_depth=80.0):
    """zoedepth_v1.py ZoeDepth.forward after the core with bin_centers_type "normed" (ZoeD_Any_K).  internals["bins"]: the
    b_new of each level ([0, 1] units), internals["centers"]: the last level's sorted, clipped centres (the only ones the
    output uses)."""
    x = F.conv2d(bottleneck, sd["conv2.weight"], sd["conv2.bias"])
    _, seed_b_centers = _seed_normed(sd, x, min_depth, max_depth)
    b_prev = (seed_b_centers - min_depth) / (max_depth - min_depth)
    prev_b_embedding = oz._mlp2(sd, "seed_projector.", x)
    for i, feat in enumerate(blocks):
        b_embedding = oz._mlp2(sd, f"projectors.{i}.", feat)
        b, b_centers = _attractor_normed(sd, i, b_embedding, b_prev, prev_b_embedding, min_depth, max_depth)
        b_prev = b.clone()
        prev_b_embedding = b_embedding.clone()
        if internals is not None:
            internals.setdefault("bins", []).append(b)
    if internals is not None:
        internals["centers"] = b_centers
    last = torch.cat([act, F.interpolate(rel.unsqueeze(1), size=act.shape[2:], mode="bilinear", align_corners=True).to(act.dtype)], dim=1)
    b_embedding = F.interpolate(b_embedding, last.shape[-2:], mode="bilinear", align_corners=True)
    # ConditionalLogBinomial (bottleneck_factor 2, p_eps 1e-4, act softmax), as in oracle/zoedepth.metric_head
    y = F.gelu(F.conv2d(torch.cat([last, b_embedding], dim=1), sd["conditional_log_binomial.mlp.0.weight"],
                        sd["conditional_log_binomial.mlp.0.bias"]))
    pt = F.softplus(F.conv2d(y, sd["conditional_log_binomial.mlp.2.weight"], sd["conditional_log_binomial.mlp.2.bias"])).float()
    p = pt[:, :2] + 1e-4
    p = (p[:, 0] / (p[:, 0] + p[:, 1])).unsqueeze(1)
    tmp = pt[:, 2:] + 1e-4
    tmp = (tmp[:, 0] / (tmp[:, 0] + tmp[:, 1])).unsqueeze(1)
    tmp = (oz.MAX_TEMP - oz.MIN_TEMP) * tmp + oz.MIN_TEMP
    k = torch.arange(0, oz.N_BINS, device=p.device, dtype=torch.float32).view(1, -1, 1, 1)
    km1 = torch.tensor([oz.N_BINS - 1], device=p.device, dtype=torch.float32).view(1, -1, 1, 1)
    yk = oz.log_binom(km1, k) + k * torch.log(torch.clamp(p, 1e-4, 1)) + (km1 - k) * torch.log(torch.clamp(1 - p, 1e-4, 1))
    prob = torch.softmax(yk / tmp, dim=1)
    centers = F.interpolate(b_centers, prob.shape[-2:], mode="bilinear", align_corners=True)
    return torch.sum(prob * centers, dim=1, keepdim=True)


def zoedepth_normed_forward(sd, x, cfg=oz.ZOED_MINI):
    """ZoeD_N's BEiT core (oracle/zoedepth.py) under the normed bins head: the configuration the transformers cross-check
    of metric_head_normed uses (ZoeDepthForDepthEstimation builds its cores from BEiT, not from DINOv2)."""
    ph, pw = x.shape[-2] // oz.PATCH, x.shape[-1] // oz.PATCH
    feats = oz.beit_features(sd, x, cfg)
    blocks, bottleneck = oz.dpt_neck(sd, feats, ph, pw, cfg)
    rel, act = oz.relative_head(sd, blocks[-1])
    return metric_head_normed(sd, act, bottleneck, blocks, rel)


def zoedepth_any_forward(sd, x, cfg=ZOED_ANY, normed=False, return_all=False):
    """x: B,3,H,W normalised ((x - 0.5) / 0.5), H, W % 14 == 0 -> metric depth B,1,H,W (= model(x)['metric_depth']).
    normed: ZoeD_Any_K's bins head.  cfg: ZOED_ANY or ZOED_ANY_MINI."""
    ph, pw = x.shape[-2] // PATCH, x.shape[-1] // PATCH
    core = _core(sd)
    feats = oda.vit_intermediate(core, x, cfg)
    rel, taps = dpt_head_taps(core, feats, ph, pw, cfg)
    rel = rel.squeeze(1)              # DepthAnything.forward: interpolate to (h, w) = identity, ReLU (applied), squeeze
    internals = {} if return_all else None
    if normed:
        out = metric_head_normed(sd, taps["out_conv"], taps["l4_rn"], taps["paths"], rel, internals, MIN_DEPTH, MAX_DEPTH[True])
    else:
        out = oz.metric_head(sd, taps["out_conv"], taps["l4_rn"], taps["paths"], rel, internals)
    if return_all:
        return {"feats": feats, "blocks": taps["paths"], "bottleneck": taps["l4_rn"], "act": taps["out_conv"], "rel": rel,
                "metric_depth": out, **internals}
    return out


def batch_infer(sd, im, flip_aug=True, edge_dilation=0, h_height=392, v_height=518, cfg=ZOED_ANY, normed=False):
    """iw3/zoedepth_model.py:89-148 with prep_mod = 14 (:190-199) around zoedepth_any_forward (the preprocessing and
    dilation oracles are oracle/frames.py and oracle/iw3.py).  im: B,3,H,W in [0, 1] -> B,1,h,w (negated metric depth)."""
    import numpy as np
    from . import frames as ofr
    from . import iw3 as oiw3
    y, pad_h, pad_w = ofr.zoe_batch_preprocess(im.numpy() if torch.is_tensor(im) else im, h_height, v_height, 14)
    x = torch.from_numpy(np.ascontiguousarray(y)).float()
    if flip_aug:
        x = torch.cat([x, torch.flip(x, dims=[3])], dim=0)
    out = torch.nan_to_num(zoedepth_any_forward(sd, x, cfg, normed))
    out = out[:, :, pad_h:out.shape[2] - pad_h, pad_w:out.shape[3] - pad_w]
    out = oiw3.dilate_edge(-out, edge_dilation) if edge_dilation else -out
    if flip_aug:
        n = out.shape[0] // 2
        out = (out[:n] + torch.flip(out[n:], dims=[3])) * 0.5
    return out
