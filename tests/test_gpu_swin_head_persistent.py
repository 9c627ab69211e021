"""The persistent fused Swin-block head (csrc/swin_attention_mma.cu swin_attn_fused_kernel).  Each CTA runs tiles blockIdx.x +
k gridDim.x of 3 windows, gathers its next tile at tile + gridDim.x under the current one, and carries its weight ring, its two
A tiles, its two q|k|v chunk buffers and their barriers' parities from one tile to the next; the attention warps gather and
signal each tile at their first and second item of the previous one.  A tile's arithmetic does not depend on which CTA runs
it, so every grid size (nb200_tune_set(11, cap)) must give the same bits.  The default grid is min(tiles, SMs), so without the
cap only the schedule the device's SM count gives is ever run; with it, one CTA runs hundreds of tiles and wraps every
barrier parity many times.

The block tail (swin_block.cu) is launched as a programmatic dependent of the head.  A tail CTA can only become resident
beside a running head CTA when the head has fewer CTAs than SMs, so the head -> tail pair is run at both, with both grids
capped, and at network level (where the two launches are adjacent on the stream, eagerly and inside a CUDA graph) against
the default grids.
"""
import contextlib

import pytest
import torch

from nunif_b200 import _lib, synth
from tests.replay import DEV, swin_attn_check, window_attention64
from tests.util import log_metric

HEAD_CAP, TAIL_CAP, GRAPHS = 11, 10, 9   # nb200_tune_set keys
CS = {96: 16, 192: 48}                   # to_image's channels in the last block's tail
ONE_AXIS_MSG = "both equal to the 6-token window or both larger"


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@contextlib.contextmanager
def _knobs(settings):
    """nb200_tune_set(key, value) for each item of `settings` for the block; every key is back at 0 afterwards."""
    lib = _lib.lib()
    try:
        for k, v in settings.items():
            _lib.check(lib.nb200_tune_set(k, v))
        yield
        torch.cuda.synchronize()
    finally:
        for k in settings:
            lib.nb200_tune_set(k, 0)


def _head_inputs(B, H, W, C, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    rn = lambda *shape: torch.randn(*shape, generator=g, device=DEV)
    x = rn(B, H, W, C).half()
    return x, {"wqkv": (rn(3 * C, C) / C ** 0.5).half(), "bqkv": 0.1 * rn(3 * C), "table": 0.5 * rn(121, 6)}


def _head(x, w, att, shift):
    B, H, W, C = x.shape
    _lib.check(_lib.lib().nb200_swin_attn_fused_f16(_lib.ptr(x), _lib.ptr(w["wqkv"]), _lib.ptr(w["bqkv"]), _lib.ptr(w["table"]),
                                                    _lib.ptr(att), B, H, W, C, shift, _lib.stream_ptr()))


def _nan_like(x):
    return torch.full_like(x, float("nan"))


# ------------------------------------------------------------------------------------------------------------ grid sizes
def _grid_shapes():
    """(B, H, W): 1 window (one partial tile); 4 windows (the last tile holds 1); 20 windows over 5 images (tiles straddle
    images); SMs + 1 tiles, the last one partial; the two tile-256 production stages (534 and 2134 tiles); a non-square map
    whose tiles straddle images."""
    S = _sms()
    n = 3 * S + 1 if (3 * S + 1) % 2 == 0 else 3 * S + 2   # windows: ceil(n / 3) = S + 1 tiles
    return [(1, 6, 6), (1, 12, 12), (5, 12, 12), (1, 12, 3 * n), (16, 60, 60), (16, 120, 120), (7, 24, 42)]


@pytest.mark.gpu
@pytest.mark.parametrize("shift", [0, 3])
@pytest.mark.parametrize("C", [96, 192])
@pytest.mark.parametrize("si", range(7))
def test_head_grid_size_bit_identical(si, C, shift):
    B, H, W = _grid_shapes()[si]
    S = _sms()
    caps = (1, 2, 3, 11, S - 1, 0)   # 0: the default grid, min(tiles, SMs)
    x, w = _head_inputs(B, H, W, C, 1000 * si + C + shift)
    x0 = x.clone()
    outs = {}
    for cap in caps:
        att = _nan_like(x)
        with _knobs({HEAD_CAP: cap}):
            _head(x, w, att, shift)
        outs[cap] = att
    tiles = -(-B * (H // 6) * (W // 6) // 3)
    assert torch.equal(x.view(torch.int16), x0.view(torch.int16)), "x changed"
    assert not bool(torch.isnan(outs[0]).any()), f"NaN (or an unwritten element) at the default grid, {tiles} tiles"
    for cap in caps[:-1]:
        d = outs[cap].view(torch.int16) != outs[0].view(torch.int16)
        assert not bool(d.any()), (f"grid cap {cap} differs from the default grid in {int(d.sum())} elements "
                                   f"(B, H, W = {B, H, W}, C = {C}, shift = {shift}, {tiles} tiles, {S} SMs)")


# ------------------------------------------------------------------------------------------------------------ one CTA vs float64
@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,C,shift", [(16, 60, 60, 96, 3), (5, 12, 12, 192, 3), (2, 60, 60, 192, 0)])
def test_head_one_cta_against_float64(B, H, W, C, shift):
    """Every tile through one CTA, against the float64 reference and per-element bound of the kernel replay."""
    with _knobs({HEAD_CAP: 1}):
        worst, over, bad = swin_attn_check(dict(B=B, H=H, W=W, C=C, shift=shift), 7919 * B + H + C + shift)
    tiles = -(-B * (H // 6) * (W // 6) // 3)
    log_metric("swin_head_one_cta", B=B, H=H, W=W, C=C, shift=shift, tiles=tiles, err_over_bound=f"{worst:.3g}", over=over)
    print(f"\none CTA, {tiles} tiles, B, H, W, C, shift = {B, H, W, C, shift}: worst err/bound {worst:.3g}, {over} elements over")
    assert not bad and over == 0, (bad, worst, over)


# ------------------------------------------------------------------------------------------------------------ head -> tail
def _tail_weights(C, cs, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    rn = lambda *shape: torch.randn(*shape, generator=g, device=DEV)
    w = {"wp": (rn(C, C) / C ** 0.5).half(), "bp": 0.1 * rn(C), "w1": (rn(2 * C, C) / C ** 0.5).half(), "b1": 0.1 * rn(2 * C),
         "w2": (rn(C, 2 * C) / (2 * C) ** 0.5).half(), "b2": 0.1 * rn(C)}
    if cs:
        w["wy"], w["by"] = (rn(cs, C) / C ** 0.5).half(), rn(cs)
    return w


def _tail(x, att, w, y=None):
    """the block tail on the head's output: x updated in place, or with y, to_image's Linear into y and x unchanged."""
    lib = _lib.lib()
    T, C = x.numel() // x.shape[-1], x.shape[-1]
    p = {k: _lib.ptr(v) for k, v in w.items()}
    if y is not None:
        _lib.check(lib.nb200_swin_mlp_fused_y_f16(_lib.ptr(x), _lib.ptr(att), T, C, p["wp"], p["bp"], p["w1"], p["b1"], p["w2"],
                                                  p["b2"], _lib.ptr(y), y.shape[-1], p["wy"], p["by"], _lib.stream_ptr()))
    else:
        _lib.check(lib.nb200_swin_mlp_fused_f16(_lib.ptr(x), _lib.ptr(att), T, C, p["wp"], p["bp"], p["w1"], p["b1"], p["w2"],
                                                p["b2"], _lib.stream_ptr()))


def _pair_shapes():
    """(B, H, W): 11 head tiles (fewer than SMs: tail CTAs can be resident beside head CTAs), and more head and tail tiles
    than SMs."""
    S = _sms()
    return [(2, 24, 24), (-(-(S + 1) * 3 // 100) + 1, 60, 60)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["proj", "y"])
@pytest.mark.parametrize("C", [96, 192])
@pytest.mark.parametrize("pi", range(2))
def test_head_then_tail_without_sync(pi, C, mode):
    """Head and tail back to back on one stream (the tail a programmatic dependent of the head), under (head cap, tail cap),
    bit-identical to the two calls separated by a device synchronisation at the default grids.  The head's entry point frees
    its bias fragments (stream-ordered) between the two launches; the network test runs them adjacent, as the model does."""
    B, H, W = _pair_shapes()[pi]
    x0, wh = _head_inputs(B, H, W, C, 31 * pi + C)
    wt = _tail_weights(C, CS[C] if mode == "y" else 0, 37 * pi + C)

    def run(sync):
        x, att = x0.clone(), _nan_like(x0)
        y = torch.full((B, H, W, CS[C]), float("nan"), dtype=torch.float16, device=DEV) if mode == "y" else None
        _head(x, wh, att, 3)
        if sync:
            torch.cuda.synchronize()
        _tail(x, att, wt, y)
        torch.cuda.synchronize()
        if y is not None:
            assert torch.equal(x.view(torch.int16), x0.view(torch.int16)), "x changed although y was requested"
        return att, (x if y is None else y)

    att0, want = run(True)
    assert not bool(torch.isnan(want).any())
    for hc, tc in ((1, 0), (2, 0), (0, 1), (3, 7), (0, 0)):
        with _knobs({HEAD_CAP: hc, TAIL_CAP: tc}):
            att, got = run(False)
        assert torch.equal(att.view(torch.int16), att0.view(torch.int16)), f"head output, caps (head {hc}, tail {tc}), {B, H, W}"
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), f"tail output, caps (head {hc}, tail {tc}), {B, H, W}"


# ------------------------------------------------------------------------------------------------------------ networks
@pytest.mark.gpu
@pytest.mark.parametrize("scale", [1, 2, 4])
def test_network_grid_caps_bit_identical(scale):
    """SwinUNet forwards at tile 64 batch 3 and tile 112 batch 1 (every head and tail grid below the SM count, so tail CTAs
    start beside head CTAs) with the head and tail grids capped, eagerly and through CUDA-graph replay (nb200_tune_set(9, 1):
    captured at the second call on the same buffers, replayed at the third), bit-identical to the default-grid eager output."""
    from nunif_b200.nunif.models import create_model
    lib = _lib.lib()
    m = create_model(f"waifu2x.swin_unet_{scale}x", synth.swin_unet_state_dict(0, scale), DEV)
    for T, B in ((64, 3), (112, 1)):
        assert m.find_valid_tile_size(T) == T
        x = torch.rand(B, 3, T, T, generator=torch.Generator().manual_seed(T + scale)).to(DEV)
        xh = torch.zeros((B, T, T, 8), device=DEV, dtype=torch.float16)
        xh[..., :3] = x.permute(0, 2, 3, 1)
        S = T * m.i2i_scale - 2 * m.i2i_offset
        z = torch.empty((B, 3, S, S), device=DEV, dtype=torch.float16)

        def forward():
            z.fill_(float("nan"))
            _lib.check(lib.nb200_model_forward(m._h, _lib.ptr(xh), B, T, 1, _lib.ptr(z), _lib.stream_ptr()))
            torch.cuda.synchronize()
            return z.view(torch.int16).clone()

        want = forward()
        assert not bool(torch.isnan(z).any())
        for hc in (1, 5):
            for tc in (0, 3):
                with _knobs({HEAD_CAP: hc, TAIL_CAP: tc}):
                    assert torch.equal(forward(), want), f"eager, caps (head {hc}, tail {tc}), tile {T} batch {B}"
                with _knobs({HEAD_CAP: hc, TAIL_CAP: tc, GRAPHS: 1}):
                    for call in range(3):
                        assert torch.equal(forward(), want), f"graphs, call {call}, caps (head {hc}, tail {tc}), tile {T} batch {B}"


# ------------------------------------------------------------------------------------------------------------ per-axis shift
@pytest.mark.parametrize("H,W", [(12, 6), (6, 12), (12, 18), (6, 6)])
def test_reference_shifts_each_axis_as_torchvision(H, W):
    """window_attention64 against torchvision's own shifted_window_attention (float64, identity proj), which zeroes the shift
    of each axis the window covers on its own."""
    tv = pytest.importorskip("torchvision.models.swin_transformer")
    C = 96
    g = torch.Generator().manual_seed(H * 100 + W)
    x = torch.randn(2, H, W, C, generator=g, dtype=torch.float64)
    wqkv = torch.randn(3 * C, C, generator=g, dtype=torch.float64) / C ** 0.5
    bqkv = 0.1 * torch.randn(3 * C, generator=g, dtype=torch.float64)
    table = 0.5 * torch.randn(121, 6, generator=g, dtype=torch.float64)
    rpb = table[synth.relative_position_index(6)].view(36, 36, -1).permute(2, 0, 1).contiguous().unsqueeze(0)
    want = tv.shifted_window_attention(x, wqkv, torch.eye(C, dtype=torch.float64), rpb, [6, 6], 6, [3, 3], qkv_bias=bqkv,
                                       proj_bias=torch.zeros(C, dtype=torch.float64), training=False)
    got = window_attention64(x @ wqkv.t() + bqkv, table, C, 3)[0]
    assert (got - want).abs().max().item() < 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize("C", [96, 192])
@pytest.mark.parametrize("H,W", [(12, 6), (6, 12)])
def test_shift_on_one_axis_is_refused(H, W, C):
    """torchvision shifts only the axis longer than the window; the kernels take one shift for both axes, so a shifted call
    with exactly one side of 6 is refused (fused head and unfused window attention).  Unshifted, the same map is computed."""
    B = 2
    x, w = _head_inputs(B, H, W, C, H + W + C)
    att = _nan_like(x)
    with pytest.raises(RuntimeError, match=ONE_AXIS_MSG):
        _head(x, w, att, 3)
    qkv = torch.randn(3, B, H, W, C, generator=torch.Generator(device=DEV).manual_seed(C), device=DEV).half()
    with pytest.raises(RuntimeError, match=ONE_AXIS_MSG):
        _lib.check(_lib.lib().nb200_window_attention_f16(_lib.ptr(qkv), _lib.ptr(w["table"]), _lib.ptr(att), B, H, W, C, 6, 3,
                                                         _lib.stream_ptr()))
    torch.cuda.synchronize()
    assert bool(torch.isnan(att).all()), "a refused call wrote its output"
    worst, over, bad = swin_attn_check(dict(B=B, H=H, W=W, C=C, shift=0), H + W + C)
    assert not bad and over == 0, (bad, worst, over)
