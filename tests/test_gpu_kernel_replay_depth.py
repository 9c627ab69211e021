"""Replay every launch of the depth networks' own kernels against float64 references: the patch im2col, token assembly, ZoeD_N's
hook cast and readout concat (csrc/depth_kernels.cu, zoe_kernels.cu), the DPT reassemble-0 depth-to-space, reassemble-3 stride-2
im2col, the fusion blocks' relu / add and output_conv2's last 1x1 conv; and, on the CPU, the two host resamples of the position
tables (csrc/depth_model.cu interp_pos_table, zoe_model.cu zoe_resample_table).  The GEMMs, attention, add + LayerNorm, DPT
upsample and bins head of these networks are replayed by the other modules.

The discipline of tests/test_gpu_kernel_replay.py, with the helpers of tests/replay.py: a module fixture turns on bit 5 of the
launch recorder and records the depth networks of MODELS (Depth-Anything V2 S / B / L and V1 S on a 1080p batch, ZoeD_N on a 4K
batch, ZoeD_Any_N on a 1080p landscape and a portrait frame: odd token-grid widths and heights), and each unique configuration,
plus a synthetic list for the edges production does not reach (one-token grids and rows, odd and even grids for the stride-2
pad, batches whose rows straddle images, every embedding width, counts that are not a multiple of the block size), is replayed
through the kernel's test entry point on fresh seeded data.  Outputs sit between guard blocks whose NaN sentinel must survive,
and inputs must keep their bits.  The references are written from the network's semantics (F.unfold, torch.cat, F.pad and
reshapes of the documented layouts), never from the kernels' index arithmetic.  All but the last 1x1 conv are data movement or
one rounding, so they must match bit for bit.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from tests.util import log_metric
from tests.replay import (DEV, MODELS, Tally, bits, body, configurations, guarded, guarded32, record_networks, replay, rounded)
from nunif_b200 import _lib
from nunif_b200._lib import ptr

U = 2.0 ** -24                 # fp32 unit roundoff
REC_DEPTH = 32                 # nb200_record_launches bit of the kinds replayed here
TINY = 1e-300                  # bound floor: an exact element has err / bound 0

DEPTH_KINDS = ("dapatch", "zpatch", "datok", "ztok", "zcast", "zreadout", "d2s4", "im2s2", "reluadd", "headfin")
DEPTH_MODELS = [(n, fn) for n, fn in MODELS if n.startswith(("depth_anything", "zoed"))]
# the launches of one forward, from vit_encoder / dpt_fuse / dpt_output (csrc/depth_model.cu): one patch embedding and token
# assembly, ZoeD_N's four hooks through zoe_add_cast and its four ProjectReadout concats, one reassemble 0 and 3, relu_add once
# in refinenet4 (no second input) and twice in each of the other three, and one head_final.  ZoeD_Any_N runs two frames.
_DA = {"dapatch": 1, "datok": 1, "d2s4": 1, "im2s2": 1, "reluadd": 7, "headfin": 1}
EXPECTED = {
    "depth_anything_v2_s": _DA,
    "depth_anything_v2_b": _DA,
    "depth_anything_v2_l": _DA,
    "depth_anything_v1_s": _DA,
    "zoed_n": {"zpatch": 1, "ztok": 1, "zcast": 4, "zreadout": 4, "d2s4": 1, "im2s2": 1, "reluadd": 7, "headfin": 1},
    "zoed_any_n": {k: 2 * n for k, n in _DA.items()},
}


@pytest.fixture(scope="module")
def production():
    """name -> every record (kind, config) of one forward of each depth network of MODELS (configurations() deduplicates)."""
    return record_networks(REC_DEPTH, DEPTH_MODELS, unique=False)


@pytest.mark.gpu
def test_every_network_records_its_launches(production):
    assert [n for n, _ in DEPTH_MODELS] == list(EXPECTED)
    for name, _ in DEPTH_MODELS:
        counts = {k: sum(1 for kk, _ in production[name] if kk == k) for k in DEPTH_KINDS}
        log_metric("replay_depth_launches", model=name, **counts)
        assert {k: n for k, n in counts.items() if n} == EXPECTED[name], name
    # the recorded grids include an odd token-grid width (Depth-Anything's 28 x 49) and an odd height (ZoeD_Any's portrait frame)
    s2 = [r for recs in production.values() for k, r in recs if k == "im2s2"]
    assert any(r["w"] % 2 for r in s2) and any(r["h"] % 2 for r in s2)
    assert {(r["c"] < r["cpad"]) for recs in production.values() for k, r in recs if k == "d2s4"} == {False, True}
    assert {r["has_sum"] for recs in production.values() for k, r in recs if k == "reluadd"} == {0, 1}


# ------------------------------------------------------------------------------------------------------------ helpers
def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g, device=DEV) * scale


def _sync():
    torch.cuda.synchronize()


def filled(t):
    """A guarded buffer holding t (fp16 or fp32) -> (buffer, the view the kernel gets, element count)."""
    n = t.numel()
    buf = guarded(n) if t.dtype == torch.float16 else guarded32(n)
    v = body(buf, n).view(t.shape)
    v.copy_(t)
    return buf, v, n


def same_bits(tally, what, buf, buf0):
    """An input buffer (with its guards) still holds the bits it was given."""
    view = torch.int16 if buf.dtype == torch.float16 else torch.int32
    tally.exact(what, buf.view(view), buf0.view(view))


def exact32(tally, what, got, want):
    tally.exact(what, got.contiguous().view(torch.int32), want.float().contiguous().view(torch.int32))


# token grids (ph, pw) of the synthetic configurations: one token, one row, one column, odd and even sides
GRIDS = [(1, 1), (1, 5), (6, 1), (2, 3), (3, 4), (5, 7)]


# ------------------------------------------------------------------------------------------------------------ patch im2col
def patch_check(r, seed, patch):
    """Bit-exact: A = F.unfold(x, p, stride=p).transpose(1, 2).half() (Conv2d weight order c, ky, kx), and for the 14-px
    patch the columns 588..kpad-1 exactly zero."""
    B, H, W = r["B"], r["H"], r["W"]
    K = 3 * patch * patch
    kpad = r.get("kpad", K)
    ph, pw = H // patch, W // patch
    g = _gen(seed)
    xb, x, _ = filled(_randn(g, B, 3, H, W, scale=3.0))
    x0 = xb.clone()
    no = B * ph * pw * kpad
    out = guarded(no)
    if patch == 14:
        _lib.check(_lib.lib().nb200_da_patch_im2col_f16(ptr(x), B, H, W, kpad, ptr(body(out, no)), _lib.stream_ptr()))
    else:
        _lib.check(_lib.lib().nb200_zoe_patch_im2col_f16(ptr(x), B, H, W, ptr(body(out, no)), _lib.stream_ptr()))
    _sync()
    tally = Tally()
    tally.guards("A", out, no)
    same_bits(tally, "x", xb, x0)
    want = torch.zeros(B * ph * pw, kpad, dtype=torch.float16, device=DEV)
    want[:, :K] = F.unfold(x, patch, stride=patch).transpose(1, 2).reshape(-1, K).half()
    tally.exact("A", bits(body(out, no).view(B * ph * pw, kpad)), bits(want))
    return tally.result()


@pytest.mark.gpu
def test_patch_im2col_replay(production):
    synth = [dict(B=B, H=14 * ph, W=14 * pw, kpad=kpad) for (ph, pw), B, kpad in
             zip(GRIDS, (1, 2, 1, 3, 1, 2), (640, 640, 588, 640, 600, 640))]
    replay("dapatch", configurations(production, "dapatch", synth), lambda r, s: patch_check(r, s, 14))


@pytest.mark.gpu
def test_zoe_patch_im2col_replay(production):
    synth = [dict(B=B, H=16 * ph, W=16 * pw) for (ph, pw), B in zip(GRIDS, (1, 2, 1, 3, 1, 2))]
    replay("zpatch", configurations(production, "zpatch", synth), lambda r, s: patch_check(r, s, 16))


# ------------------------------------------------------------------------------------------------------------ tokens
def tokens_check(r, seed, with_pos):
    """Bit-exact: X32 = cat([cls, T.float()]) + pos in float64, rounded once to fp32 (fp32 + fp32 rounded through float64 is
    the fp32 sum: 53 >= 2 * 24 + 2); without pos (BEiT) X32 = cat([cls, T.float()])."""
    B, P, dim = r["B"], r["P"], r["dim"]
    g = _gen(seed)
    tb, T, _ = filled(_randn(g, B * P, dim, scale=2.0).half())
    cb, cls, _ = filled(_randn(g, dim))
    pb, pos, _ = filled(_randn(g, P + 1, dim, scale=0.3)) if with_pos else (None, None, 0)
    ins = [(n, b, b.clone()) for n, b in (("T", tb), ("cls", cb), ("pos", pb)) if b is not None]
    no = B * (P + 1) * dim
    out = guarded32(no)
    _lib.check(_lib.lib().nb200_vit_assemble_tokens_f32(ptr(T), ptr(cls), ptr(pos) if with_pos else None, ptr(body(out, no)),
                                                        B, P, dim, _lib.stream_ptr()))
    _sync()
    tally = Tally()
    tally.guards("X32", out, no)
    for n, b, b0 in ins:
        same_bits(tally, n, b, b0)
    want = torch.cat([cls.double().expand(B, 1, dim), T.double().view(B, P, dim)], 1)
    if with_pos:
        want = want + pos.double()
    exact32(tally, "X32", body(out, no).view(B, P + 1, dim), want)
    return tally.result()


def _token_synthetic():
    """Every embedding width in use (ViT-S / B / L and the reduced 256 of the synth configurations) on one-token, one-row and
    one-column grids, with batches whose rows straddle images; B (P + 1) dim is not a multiple of the 256-thread block for
    the odd B (P + 1) at dim 384."""
    return [dict(B=B, P=ph * pw, dim=dim) for dim in (256, 384, 768, 1024) for (ph, pw), B in zip(GRIDS[:4], (1, 2, 3, 1))]


@pytest.mark.gpu
def test_assemble_tokens_replay(production):
    replay("datok", configurations(production, "datok", _token_synthetic()), lambda r, s: tokens_check(r, s, True))


@pytest.mark.gpu
def test_zoe_assemble_tokens_replay(production):
    replay("ztok", configurations(production, "ztok", _token_synthetic()), lambda r, s: tokens_check(r, s, False))


# ------------------------------------------------------------------------------------------------------------ ZoeD_N hooks
def zcast_check(r, seed):
    """With delta: X32 bit-exact fp32(x + d) (float64 sum rounded once), the hook bit-exact fp16 of that (overflowing elements
    become inf like torch's cast); without delta X32 keeps its bits and the hook is fp16(x)."""
    n, has_delta = r["n"], r["has_delta"]
    g = _gen(seed)
    x = _randn(g, n, scale=4.0)
    x[::97] *= 3e4                       # some beyond fp16's range, and fp16 subnormals below
    x[1::89] *= 1e-6
    xb, X, _ = filled(x)
    x0 = X.clone()
    db, d, _ = filled(_randn(g, n, scale=2.0).half()) if has_delta else (None, None, 0)
    d0 = db.clone() if has_delta else None
    out = guarded(n)
    _lib.check(_lib.lib().nb200_zoe_add_cast_f16(ptr(X), ptr(d) if has_delta else None, ptr(body(out, n)), n, _lib.stream_ptr()))
    _sync()
    tally = Tally()
    tally.guards("hook", out, n)
    tally.guards("X32", xb, n)
    want = (x0.double() + d.double()).float() if has_delta else x0
    exact32(tally, "X32", X, want)
    if has_delta:
        same_bits(tally, "delta", db, d0)
    tally.exact("hook", bits(body(out, n)), bits(want.half()))
    return tally.result()


@pytest.mark.gpu
def test_zoe_add_cast_replay(production):
    synth = [dict(n=n, has_delta=hd) for n in (4, 12, 1028, 4 * 257 * 3) for hd in (1, 0)]
    replay("zcast", configurations(production, "zcast", synth), zcast_check)


def zreadout_check(r, seed):
    """Bit-exact: A = cat(tokens, cls.expand) of each image, in that order: A[b P + n] = [F[b][1 + n], F[b][0]]."""
    B, P, dim = r["B"], r["P"], r["dim"]
    g = _gen(seed)
    fb, Fh, _ = filled(_randn(g, B, P + 1, dim).half())
    f0 = fb.clone()
    no = B * P * 2 * dim
    out = guarded(no)
    _lib.check(_lib.lib().nb200_zoe_readout_concat_f16(ptr(Fh), B, P, dim, ptr(body(out, no)), _lib.stream_ptr()))
    _sync()
    tally = Tally()
    tally.guards("A", out, no)
    same_bits(tally, "F", fb, f0)
    want = torch.cat([Fh[:, 1:], Fh[:, :1].expand(B, P, dim)], -1).reshape(B * P, 2 * dim)
    tally.exact("A", bits(body(out, no).view(B * P, 2 * dim)), bits(want))
    return tally.result()


@pytest.mark.gpu
def test_zoe_readout_concat_replay(production):
    synth = [dict(B=B, P=ph * pw, dim=dim) for dim in (64, 256, 1024) for (ph, pw), B in zip(GRIDS[:4], (1, 2, 3, 1))]
    replay("zreadout", configurations(production, "zreadout", synth), zreadout_check)


# ------------------------------------------------------------------------------------------------------------ DPT reassemble
def d2s4_check(r, seed):
    """Bit-exact: generate the NHWC image Y [B][4h][4w][c], build the GEMM output T [B h w][16 c] in the documented column order
    n = (dy * 4 + dx) * c + co, and the kernel must return F.pad(Y, (0, cpad - c)): channels c..cpad-1 exactly zero."""
    B, h, w, c, cpad = r["B"], r["h"], r["w"], r["c"], r["cpad"]
    g = _gen(seed)
    Y = _randn(g, B, 4 * h, 4 * w, c).half()
    T = Y.view(B, h, 4, w, 4, c).permute(0, 1, 3, 2, 4, 5).reshape(B * h * w, 16 * c)
    tb, Td, _ = filled(T)
    t0 = tb.clone()
    no = B * 16 * h * w * cpad
    out = guarded(no)
    _lib.check(_lib.lib().nb200_dpt_depth_to_space4_f16(ptr(Td), B, h, w, c, cpad, ptr(body(out, no)), _lib.stream_ptr()))
    _sync()
    tally = Tally()
    tally.guards("out", out, no)
    same_bits(tally, "T", tb, t0)
    tally.exact("out", bits(body(out, no).view(B, 4 * h, 4 * w, cpad)), bits(F.pad(Y, (0, cpad - c))))
    return tally.result()


@pytest.mark.gpu
def test_depth_to_space4_replay(production):
    # c0pad > c (ViT-S: 48 -> 64, a width that is not a multiple of 32: 40 -> 64) and c0pad == c, on the synthetic grids
    synth = [dict(B=B, h=ph, w=pw, c=c, cpad=cp) for (ph, pw), B in zip(GRIDS, (1, 2, 1, 3, 1, 2))
             for c, cp in ((48, 64), (40, 64), (96, 96), (256, 256))]
    replay("d2s4", configurations(production, "d2s4", synth), d2s4_check)


def im2s2_check(r, seed):
    """Bit-exact: F.unfold(x_nchw, 3, padding=1, stride=2) (columns c, ky, kx) reordered to k = (ky * 3 + kx) * C + c, fp16
    zeros at the pad."""
    B, h, w, C = r["B"], r["h"], r["w"], r["C"]
    g = _gen(seed)
    xb, x, _ = filled(_randn(g, B, h, w, C).half())
    x0 = xb.clone()
    ho, wo = (h + 1) // 2, (w + 1) // 2
    no = B * ho * wo * 9 * C
    out = guarded(no)
    _lib.check(_lib.lib().nb200_dpt_im2col_s2_f16(ptr(x), B, h, w, C, ptr(body(out, no)), _lib.stream_ptr()))
    _sync()
    tally = Tally()
    tally.guards("A", out, no)
    same_bits(tally, "x", xb, x0)
    cols = F.unfold(x.permute(0, 3, 1, 2).float(), 3, padding=1, stride=2)
    assert cols.shape[-1] == ho * wo
    want = cols.view(B, C, 9, ho * wo).permute(0, 3, 2, 1).reshape(B * ho * wo, 9 * C).half()
    tally.exact("A", bits(body(out, no).view(B * ho * wo, 9 * C)), bits(want))
    return tally.result()


@pytest.mark.gpu
def test_im2col_s2_replay(production):
    # odd and even sides (the (h + 1) / 2 output and the bottom / right pad), one-row and one-column grids, every reassemble-3
    # width in use (384, 768, 1024 and the synth 256) and narrow ones
    synth = [dict(B=B, h=ph, w=pw, C=C) for (ph, pw), B in zip(GRIDS, (1, 2, 1, 3, 1, 2)) for C in (8, 256, 384)]
    synth += [dict(B=2, h=7, w=9, C=768), dict(B=1, h=4, w=6, C=1024)]
    replay("im2s2", configurations(production, "im2s2", synth), im2s2_check)


# ------------------------------------------------------------------------------------------------------------ DPT fusion and output
def reluadd_check(r, seed):
    """y bit-exact relu(x) (a zero input may give either signed zero); s bit-exact fp16(x0 + x) computed in float64: the kernel
    rounds the sum of two fp16 values to fp32 and then to fp16, which equals one correct rounding (24 >= 2 * 11 + 2)."""
    n, has_sum = r["n"], r["has_sum"]
    g = _gen(seed)
    x = _randn(g, n, scale=3.0).half()
    x[::101] = 0.0
    x[1::103] = -0.0
    xb, xd, _ = filled(x)
    x0b, x0d, _ = filled(_randn(g, n, scale=3.0).half())
    ins = [("x", xb, xb.clone()), ("x0", x0b, x0b.clone())]
    y = guarded(n)
    s = guarded(n)
    _lib.check(_lib.lib().nb200_dpt_relu_add_f16(ptr(xd), ptr(x0d) if has_sum else None, ptr(body(y, n)),
                                                 ptr(body(s, n)) if has_sum else None, n, _lib.stream_ptr()))
    _sync()
    tally = Tally()
    tally.guards("y", y, n)
    for what, b, b0 in ins:
        same_bits(tally, what, b, b0)
    tally.exact("y", bits(body(y, n) + 0.0), bits(torch.where(xd > 0, xd, torch.zeros_like(xd))))
    if has_sum:
        tally.guards("s", s, n)
        tally.exact("s", bits(body(s, n)), bits((x0d.double() + xd.double()).half()))
    else:                                # no sum: the buffer the kernel was not given keeps its sentinel
        tally.guards("s", s, 0)
    return tally.result()


@pytest.mark.gpu
def test_relu_add_replay(production):
    synth = [dict(n=n, has_sum=hs) for n in (8, 24, 8 * 257, 64 * 3 * 5 * 7) for hs in (1, 0)]
    replay("reluadd", configurations(production, "reluadd", synth), reluadd_check)


def headfin_check(r, seed):
    """depth = relu(fp16(x . w + b)) against float64: the fp32 fma chain of C terms and the fp32 bias add are within
    E = (C + 1) U sum|x w| + U |b| of x . w + b; rounded() carries that through the fp16 rounding point (ReLU is 1-Lipschitz),
    so an output may differ only where an fp16 boundary lies within E.  Every output must be an fp16 value and >= 0."""
    npix, C = r["npix"], r["C"]
    g = _gen(seed)
    xb, x, _ = filled(_randn(g, npix, C).half())
    x0 = xb.clone()
    wb, w, _ = filled(_randn(g, C, scale=C ** -0.5))
    w0 = wb.clone()
    bias = float(torch.randn(1, generator=torch.Generator().manual_seed(seed)).float() * 0.5)
    out = guarded32(npix)
    _lib.check(_lib.lib().nb200_dpt_head_final_f32(ptr(x), npix, C, ptr(w), bias, ptr(body(out, npix)), _lib.stream_ptr()))
    _sync()
    tally = Tally()
    got = body(out, npix)
    tally.guards("depth", out, npix)
    same_bits(tally, "x", xb, x0)
    same_bits(tally, "w", wb, w0)
    tally.no_nan("depth", got)
    xd, wd = x.double(), w.double()
    v = xd @ wd + bias
    ref, e = rounded(v, (C + 1) * U * (xd.abs() @ wd.abs()) + U * abs(bias))
    tally.add(got, ref.clamp(min=0), e.clamp(min=TINY))
    exact32(tally, "depth as fp16 values", got, got.half().float())
    if bool((got < 0).any()):
        tally.bad.append("negative depth")
    return tally.result()


@pytest.mark.gpu
def test_head_final_replay(production):
    synth = [dict(npix=n, C=32) for n in (1, 255, 257, 1000, 3 * 98 * 126)]
    replay("headfin", configurations(production, "headfin", synth), headfin_check)


# ------------------------------------------------------------------------------------------------------------ host resamples (CPU)
def pos_table(table, g, ph, pw):
    """nb200_vit_pos_table_f32: table [1 + g*g][dim] fp32 (CPU) -> [1 + ph*pw][dim]."""
    dim = table.shape[-1]
    out = torch.empty(1 + ph * pw, dim)
    _lib.check(_lib.lib().nb200_vit_pos_table_f32(ptr(table), g, dim, ph, pw, ptr(out)))
    return out


def _axis_ec(n_out, s):
    """The fp32 source coordinate's error on one axis: s * (o + 0.5) - 0.5 with s rounded to fp32 (U), the product (U) and the
    subtraction (U |result| <= U s (o + 0.5) + U / 2), and t = c - floor(c) when c < 0 (U / 2): 3 U s (o + 0.5) + U."""
    return 3 * U * s * (torch.arange(n_out, dtype=torch.float64) + 0.5) + U


# bicubic (Keys, A = -0.75): over t in [0, 1) the four weights have sum |w| <= 1.375 and sum |w'| <= 3.0
CUBIC_SUM_W, CUBIC_SUM_DW = 1.375, 3.0
# one cubic weight evaluated in fp32 (Horner, |t| <= 2): at most 9 U for an inner tap (1.25 t - 2.25, * t, * t, + 1, and the
# 1 - t argument) and 43 U for an outer one (intermediates up to 6 in magnitude, earlier errors scaled by t <= 2)
CUBIC_DW = (43 + 9 + 9 + 43) * U
# weights and accumulation of the separable sum, per unit of M = max |table|: each row sum h (four products and adds: 4 U
# sum |x w|, plus the weights' errors) is within (4 * 1.375 U + CUBIC_DW) M; the column sum scales that by 1.375 and adds
# its own 4 U sum |h w| and the weights' errors on |h| <= 1.375 M
CUBIC_ACC = 1.375 * (4 * 1.375 * U + CUBIC_DW) + 4 * 1.375 ** 2 * U + CUBIC_DW * 1.375


def pos_table_reference(table, g, ph, pw):
    """float64 dinov2 interpolate_pos_encoding: the class row, then F.interpolate(bicubic, scale_factor=((ph + 0.1) / g,
    (pw + 0.1) / g), align_corners=False) of the g x g grid, or the table itself when ph == pw == g; and the bound on the host
    code's fp32 arithmetic, per element:
      slope: the sample's derivative along an axis is sum_j w'_j x_j times the other axis's weights, <= 3.0 * 1.375 M, times
        that axis's source-coordinate error (_axis_ec)
      weights and accumulation: CUBIC_ACC M
    with M the largest |entry| of that channel (the taps a coordinate within its error can use lie in the table)."""
    dim = table.shape[-1]
    t64 = table.double()
    if ph == g and pw == g:
        return t64, torch.zeros_like(t64)
    grid = t64[1:].reshape(1, g, g, dim).permute(0, 3, 1, 2)
    sy, sx = (ph + 0.1) / g, (pw + 0.1) / g
    res = F.interpolate(grid, scale_factor=(sy, sx), mode="bicubic", align_corners=False)
    assert res.shape[-2:] == (ph, pw)
    ref = torch.cat([t64[:1], res.permute(0, 2, 3, 1).reshape(ph * pw, dim)])
    M = t64[1:].abs().amax(0)
    ec = _axis_ec(ph, 1 / sy).view(ph, 1) + _axis_ec(pw, 1 / sx).view(1, pw)
    bound = (CUBIC_SUM_DW * CUBIC_SUM_W * ec.reshape(-1, 1) + CUBIC_ACC) * M
    return ref, torch.cat([torch.zeros(1, dim, dtype=torch.float64), bound])


# (g, ph, pw, dim): Depth-Anything's 1080p grid (28 x 49) and ZoeD_Any's landscape (28 x 50) and portrait (37 rows: one axis
# at the training size still interpolates) on the released 37 grid; the training grid itself (a copy); grids smaller than g on
# both axes and on one; 1 x 1, 1 x N and N x 1; ph * pw == g * g with ph != pw (still interpolated); the synth 6 and 8 grids
POS_CASES = [(37, 28, 49, 384), (37, 28, 50, 64), (37, 37, 21, 64), (37, 37, 37, 64), (37, 10, 12, 64), (37, 40, 5, 64),
             (37, 1, 1, 64), (37, 1, 30, 64), (37, 30, 1, 64), (8, 4, 16, 64), (8, 8, 8, 32), (6, 7, 10, 384), (6, 2, 3, 256)]


def test_vit_pos_table_matches_float64():
    """Host only, no device needed: nb200_vit_pos_table_f32 (the table every Depth-Anything and ZoeD_Any forward uploads)
    against float64 interpolate_pos_encoding within pos_table_reference's bound; ph == pw == g is a bit-exact copy and the
    class row always is.  The largest difference from torch's fp32 CPU F.interpolate is logged, not gated."""
    worst, fails = 0.0, []
    for g, ph, pw, dim in POS_CASES:
        table = torch.randn(1 + g * g, dim, generator=torch.Generator().manual_seed(g * 1000 + ph * 37 + pw)) * 0.2
        got = pos_table(table, g, ph, pw)
        ref, bound = pos_table_reference(table, g, ph, pw)
        if not torch.equal(got[0], table[0]):
            fails.append(f"{g} {ph}x{pw}: class row changed")
        if ph == g and pw == g:
            if not torch.equal(got, table):
                fails.append(f"{g} {ph}x{pw}: not a copy")
            ratio, fp32 = 0.0, 0.0
        else:
            ratio = float(((got.double() - ref).abs()[1:] / bound[1:]).max())
            grid = table[1:].reshape(1, g, g, dim).permute(0, 3, 1, 2)
            t32 = F.interpolate(grid, scale_factor=((ph + 0.1) / g, (pw + 0.1) / g), mode="bicubic", align_corners=False)
            fp32 = float((got[1:] - t32.permute(0, 2, 3, 1).reshape(ph * pw, dim)).abs().max())
        log_metric("replay_pos_table", g=g, ph=ph, pw=pw, dim=dim, err_over_bound=f"{ratio:.3g}", max_diff_torch_fp32=fp32)
        worst = max(worst, ratio)
        if ratio > 1:
            fails.append(f"{g} {ph}x{pw}: err/bound {ratio:.3g}")
    print(f"\npos table: {len(POS_CASES)} grids, worst err/bound {worst:.3g}")
    assert not fails, fails


def beit_table_reference(table, g, heads, ph, pw):
    """float64 MiDaS _get_rel_pos_bias: F.interpolate(bilinear, size=(2 ph - 1, 2 pw - 1), align_corners=False) of the
    (2g - 1)^2 sub-table, the 3 class rows copied; and the bound on the host code's fp32 arithmetic, per element:
      slope: a bilinear sample moves by at most 2 M per unit of source coordinate on either axis (M the largest |entry| of
        that head), times that axis's coordinate error (_axis_ec; the clamp at 0 is exact on both sides)
      weights and accumulation: 8 U M (1 - l rounded, the four products and three adds of hy (hx a + lx b) + ly (hx c + lx d))."""
    S, nh, nw = 2 * g - 1, 2 * ph - 1, 2 * pw - 1
    t64 = table.double()
    sub = t64[:S * S].reshape(1, S, S, heads).permute(0, 3, 1, 2)
    res = F.interpolate(sub, size=(nh, nw), mode="bilinear", align_corners=False).permute(0, 2, 3, 1).reshape(nh * nw, heads)
    ref = torch.cat([res, t64[S * S:]])
    M = t64[:S * S].abs().amax(0)
    ec = _axis_ec(nh, S / nh).view(nh, 1) + _axis_ec(nw, S / nw).view(1, nw)
    bound = (2 * ec.reshape(-1, 1) + 8 * U) * M
    return ref, torch.cat([bound, torch.zeros(3, heads, dtype=torch.float64)])


# (g, ph, pw, heads): ZoeD_N's 4K grid (24 x 44) on the released 24 grid, the training grid (a copy), 1 x 1, 1 x N, N x 1, a
# portrait grid, grids smaller than g, and the synth 6 grid
BEIT_CASES = [(24, 24, 44, 16), (24, 24, 24, 16), (24, 1, 1, 16), (24, 1, 30, 4), (24, 30, 1, 4), (24, 44, 24, 16),
              (24, 12, 20, 4), (24, 5, 5, 4), (6, 4, 6, 4), (6, 6, 9, 4), (6, 12, 2, 4)]


def test_beit_rel_table_matches_float64():
    """Host only, no device needed: nb200_zoe_rel_pos_table (the table every ZoeD_N forward expands) against float64
    _get_rel_pos_bias within beit_table_reference's bound; the class rows are copied bit for bit and the training grid is a
    bit-exact copy.  The largest difference from torch's fp32 CPU F.interpolate is logged, not gated."""
    worst, fails = 0.0, []
    for g, ph, pw, heads in BEIT_CASES:
        S, nh, nw = 2 * g - 1, 2 * ph - 1, 2 * pw - 1
        table = torch.randn(S * S + 3, heads, generator=torch.Generator().manual_seed(g * 1000 + ph * 41 + pw))
        out = torch.empty(nh * nw + 3, heads)
        _lib.check(_lib.lib().nb200_zoe_rel_pos_table(ptr(table), g, heads, ph, pw, ptr(out)))
        ref, bound = beit_table_reference(table, g, heads, ph, pw)
        if not torch.equal(out[-3:], table[-3:]):
            fails.append(f"{g} {ph}x{pw}: class rows changed")
        if (ph, pw) == (g, g) and not torch.equal(out, table):
            fails.append(f"{g} {ph}x{pw}: not a copy")
        ratio = float(((out.double() - ref).abs()[:-3] / bound[:-3]).max())
        sub = table[:S * S].reshape(1, S, S, heads).permute(0, 3, 1, 2)
        t32 = F.interpolate(sub, size=(nh, nw), mode="bilinear", align_corners=False).permute(0, 2, 3, 1).reshape(nh * nw, heads)
        fp32 = float((out[:-3] - t32).abs().max())
        log_metric("replay_beit_table", g=g, ph=ph, pw=pw, heads=heads, err_over_bound=f"{ratio:.3g}", max_diff_torch_fp32=fp32)
        worst = max(worst, ratio)
        if ratio > 1:
            fails.append(f"{g} {ph}x{pw}: err/bound {ratio:.3g}")
    print(f"\nBEiT table: {len(BEIT_CASES)} grids, worst err/bound {worst:.3g}")
    assert not fails, fails
