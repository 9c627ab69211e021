"""Fused per-frame stereo pipelines (what iw3/utils.py:292-391 apply_divergence +
:430-487 postprocess_image do for the SBS / anaglyph outputs of the BASELINE configs)."""
from .backward_warp import apply_divergence_grid_sample
from .forward_warp import apply_divergence_forward_warp
from .depth_scaler import minmax_normalize
from .dilation import dilate_edge, edge_dilation_is_enabled
from ._common import COMPOSE_SBS, COMPOSE_ANAGLYPH


def stereo_sbs(c, depth, divergence=2.0, convergence=0.5, method="forward_fill", mapper="none",
               edge_dilation=0, synthetic_view="both", anaglyph=None, side_model=None):
    """c: B,3,H,W frames; depth: B,1,h,w raw model output (larger = nearer).
    dilate_edge -> per-frame min/max -> mapper -> warp -> SBS (B,3,H,2W) or anaglyph (B,3,H,W)."""
    if edge_dilation_is_enabled(edge_dilation):
        depth = dilate_edge(depth, edge_dilation)
    depth = minmax_normalize(depth, mapper=mapper)
    if method in {"forward", "forward_fill"}:
        if anaglyph is not None:
            from .anaglyph import apply_anaglyph_redcyan
            l, r = apply_divergence_forward_warp(c, depth, divergence, convergence, method=method,
                                                 synthetic_view=synthetic_view, width_base=False)
            return apply_anaglyph_redcyan(l, r, anaglyph)
        return apply_divergence_forward_warp(c, depth, divergence, convergence, method=method,
                                             synthetic_view=synthetic_view, width_base=False, compose=COMPOSE_SBS)
    if method in {"grid_sample", "backward"}:
        compose = COMPOSE_SBS if anaglyph is None else COMPOSE_ANAGLYPH
        if anaglyph not in (None, "dubois"):
            raise NotImplementedError("fused anaglyph epilogue supports dubois only")
        return apply_divergence_grid_sample(c, depth, divergence, convergence, synthetic_view, compose=compose)
    if method in {"row_flow_v3", "row_flow"}:
        # the learned warp (iw3/utils.py:331-340 apply_divergence_nn_LR with args.side_model)
        if side_model is None:
            raise ValueError("method row_flow_v3 needs side_model (a nunif_b200.iw3.RowFlowV3)")
        import torch
        from .row_flow import apply_divergence_nn_LR
        l, r = apply_divergence_nn_LR(side_model, c, depth, divergence, convergence, steps=1, synthetic_view=synthetic_view)
        if anaglyph is not None:
            from .anaglyph import apply_anaglyph_redcyan
            return apply_anaglyph_redcyan(l, r, anaglyph)
        return torch.cat([l, r], dim=3)
    raise ValueError(f"method {method} is not on the H100 hot path")
