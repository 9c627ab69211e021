"""GPU: replay every launch that the engine's networks make of the fp32 / fp16 kernels between their GEMMs, at the production
shapes, against float64 references: the WindowMHA2d core and replication pad of the WABlock (row_flow_v3, mlbw, depth_aa), the
ViT residual add + LayerNorm and the DPT head's bilinear upsample (Depth-Anything, ZoeDepth), and the ZoeDepth bins head
(softplus / normed seed, attractors with the bitonic sort, the ConditionalLogBinomial concat and mixture, the BEiT relative
position bias expansion).

The discipline of tests/test_gpu_kernel_replay.py, with the helpers of tests/replay.py: a module fixture turns on bit 1 of the
launch recorder (the kinds between the GEMMs; bit 0 keeps the GEMM replay's kinds) and records one forward of each network of
AUX_MODELS, and each unique configuration (plus a synthetic list that reaches the edges production
does not) is replayed through the kernel's test entry point on fresh seeded data.  Inputs outside the view a launch reads are
NaN, every buffer sits between guard blocks that hold a sentinel bit pattern (a NaN) and must survive bit for bit, and every
output element is checked against a float64 reference written from the reference network's semantics (oracle/wa_block.py,
oracle/depth_anything.py, oracle/zoedepth*.py, ATen's align_corners=True index arithmetic), within a per-element bound derived
from the kernel's arithmetic (stated in each check's docstring; U = 2^-24 is the fp32 unit roundoff).
"""
import math

import pytest
import torch

from tests.util import log_metric
from tests.replay import (DEV, MODELS, SENTINEL32, Tally, bits, body, configurations, guarded, guarded32, record_networks, replay,
                          round16_bound, rounded, zoe_any)
from nunif_b200 import _lib
from nunif_b200._lib import ptr

pytestmark = pytest.mark.gpu
U = 2.0 ** -24                 # fp32 unit roundoff
CHUNK = 1 << 24                # elements of the largest float64 temporary of one reference chunk
LOG2E = 1.4426950408889634
REC_AUX = 2                    # nb200_record_launches bit of the kinds replayed here (bit 0: the GEMM / attention / Swin kinds)

AUX_KINDS = ("wmha", "reppad", "ln", "upbl", "zadd_up", "zsoftplus", "zseed", "zattr", "zclb_concat", "zclb_final", "zrelbias")
# window_mha's instantiations: (window, heads, head dim)
WMHA_INST = {(3, 2, 32), (4, 2, 32), (4, 4, 32), (8, 2, 16)}
LN_DIMS = {256, 384, 768, 1024}


# ------------------------------------------------------------------------------------------------------------ networks
_NETS = dict(MODELS)
AUX_MODELS = [(n, _NETS[n]) for n in ("depth_anything_v2_s", "depth_anything_v2_b", "depth_anything_v2_l", "depth_anything_v1_s",
                                      "zoed_n", "zoed_any_n")] + [("zoed_any_k", zoe_any(True, "ZoeD_Any_K", 9))] + \
             [(n, _NETS[n]) for n in ("row_flow_v3", "mlbw_l2", "mlbw_l4", "depth_aa")]


@pytest.fixture(scope="module")
def production():
    """name -> unique records (kind, config) of the kinds of AUX_KINDS in one forward of each network of AUX_MODELS."""
    return record_networks(REC_AUX, AUX_MODELS)


def test_every_network_records_its_launches(production):
    lines = []
    for name, _ in AUX_MODELS:
        counts = {k: sum(1 for kk, _ in production[name] if kk == k) for k in AUX_KINDS}
        lines.append(f"{name:20s} unique: " + " ".join(f"{k} {n}" for k, n in counts.items() if n))
        log_metric("replay_aux_configs", model=name, **counts)
    print("\n" + "\n".join(lines))
    kinds = {k for recs in production.values() for k, _ in recs}
    assert kinds == set(AUX_KINDS), f"never recorded: {set(AUX_KINDS) - kinds}"
    for name in ("row_flow_v3", "mlbw_l2", "mlbw_l4", "depth_aa"):
        assert {"wmha", "reppad"} <= {k for k, _ in production[name]}, name
    for name in ("depth_anything_v2_s", "depth_anything_v2_l", "zoed_n", "zoed_any_n", "zoed_any_k"):
        assert {"ln", "upbl"} <= {k for k, _ in production[name]}, name
    assert "zrelbias" in {k for k, _ in production["zoed_n"]}
    assert any(k == "zattr" and r["normed"] == 0 for k, r in production["zoed_any_n"])
    assert any(k == "zattr" and r["normed"] == 1 and r["has_sorted"] == 1 for k, r in production["zoed_any_k"])
    assert any(k == "zseed" for k, _ in production["zoed_any_k"])


# ------------------------------------------------------------------------------------------------------------ helpers
# ATen upsample_bilinear2d(align_corners=True): the source coordinate of output index i is the fp32 product
# ((in - 1) / (out - 1) in fp32) * i, its integer part the first tap and its fraction the weight of the second
def ac_index(n_in, n_out):
    """-> (i0, i1, w0, w1) per output index; the weights in float64."""
    if n_out > 1:
        scale = torch.tensor(float(n_in - 1), dtype=torch.float32, device=DEV) / torch.tensor(float(n_out - 1), dtype=torch.float32, device=DEV)
    else:
        scale = torch.zeros((), dtype=torch.float32, device=DEV)
    f = scale * torch.arange(n_out, dtype=torch.float32, device=DEV)
    i0 = f.long().clamp(max=n_in - 1)
    i1 = (i0 + 1).clamp(max=n_in - 1)
    w1 = f.double() - i0.double()
    return i0, i1, 1.0 - w1, w1


def bilinear64(x, H, W):
    """x [h][w][C] -> (float64 bilinear(align_corners=True) [H][W][C], sum of |the four corners|).  A fp32 blend of the corners with
    weights in [0, 1] (two products and a sum per level, the weight 1 - w1) is within 8 U sum |corners| of it: 2^-21 sum |corners|."""
    h, w, C = x.shape
    yi0, yi1, wy0, wy1 = ac_index(h, H)
    xi0, xi1, wx0, wx1 = ac_index(w, W)
    x = x.double()
    a, b = x[yi0][:, xi0], x[yi0][:, xi1]
    c, d = x[yi1][:, xi0], x[yi1][:, xi1]
    wy0, wy1, wx0, wx1 = wy0.view(H, 1, 1), wy1.view(H, 1, 1), wx0.view(1, W, 1), wx1.view(1, W, 1)
    return wy0 * (wx0 * a + wx1 * b) + wy1 * (wx0 * c + wx1 * d), a.abs() + b.abs() + c.abs() + d.abs()


# ------------------------------------------------------------------------------------------------------------ window_mha
def _synthetic_wmha():
    """Every instantiation unshifted, the even windows also shifted in each direction; 15 windows per image (plus padding) so
    that CTAs of 7, 4 or 2 windows straddle two images; and a grid of one window."""
    out = []
    for ws, heads, hd in sorted(WMHA_INST):
        pads = [(0, 0)] + ([(0, ws // 2), (ws // 2, 0), (ws // 2, ws // 2)] if ws % 2 == 0 else [])
        for py, px in pads:
            for B, H, W in ((3, 5 * ws, 3 * ws), (1, ws, ws)):
                out.append(dict(B=B, H=H, W=W, C=heads * hd, ws=ws, heads=heads, pad_y=py, pad_x=px))
    return out


def wmha_inputs(r, mode, seed):
    """-> (qkv fp16 [B][H][W][3C], qkv_bias fp32 [3C], bias fp32 [N][N]).  mode "random": scores of standard deviation ~2;
    "bias": the bias makes the last key of every window take the softmax and masks key 0 with a -1e4 entry; "pad": every query
    points at the k bias, so in windows that hold padded tokens those keys take the softmax (and their v is the v bias)."""
    B, H, W, C, ws, heads = (r[f] for f in ("B", "H", "W", "C", "ws", "heads"))
    d, N = C // heads, ws * ws
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B, H, W, 3, heads, d, generator=g, device=DEV)
    qkv_bias = torch.randn(3, heads, d, generator=g, device=DEV)
    bias = torch.randn(N, N, generator=g, device=DEV)
    if mode == "random":
        x[..., :2, :, :] *= 1.5
    elif mode == "bias":
        bias[:, N - 1] += 12.0
        bias[:, 0] = -1e4
    else:
        kb = qkv_bias[1]
        lam = 10.0 / (d ** -0.5 * (kb * kb).sum(-1))
        x[..., :2, :, :] *= 0.3
        x[..., 0, :, :] += lam[:, None] * kb
    return x.reshape(B, H, W, 3 * C).half(), qkv_bias.reshape(3 * C).float(), bias.float()


def wmha_reference(qkv16, qkv_bias, bias, r):
    """float64 WindowMHA2d core (oracle/wa_block.py window_mha2d between the Linears): the token grid zero padded by pad_y / pad_x
    BEFORE the qkv projection, so a padded token's k | v is the (fp16) projection bias; softmax(q k^T / sqrt(d) + bias) v per
    window and head.  -> iterator of (first padded row, reference, bound E on |kernel's fp32 value - reference|) per chunk of
    window rows of the padded grid.

    E: each score is an fp32 dot product of d fma (error (d + 2) U scale sum|q k| with the scale and bias roundings) plus 2 U |s|;
    __expf(s - max) is within 2^-23 (2 + 1.173 |s - max|) relative (CUDA's documented maximum) after the U |s - max| rounding of
    its argument.  A relative error r_j on key j's weight moves the output by sum_j p_j r_j (v_j - o) (first order, 1.1 margin);
    the row sum, the reciprocal, p_j and the PV fma chain add (2N + 4) U sum_j p_j |v_j|."""
    B, H, W, C, ws, heads, py, px = (r[f] for f in ("B", "H", "W", "C", "ws", "heads", "pad_y", "pad_x"))
    d, N, scale = C // heads, ws * ws, (C // heads) ** -0.5
    Hp, Wp = H + 2 * py, W + 2 * px
    pad = torch.cat([torch.zeros(C, dtype=torch.float64, device=DEV), qkv_bias[C:].half().double()])
    xp = pad.expand(B, Hp, Wp, 3 * C).clone()
    xp[:, py:py + H, px:px + W] = qkv16.double()
    nh, nw = Hp // ws, Wp // ws
    bias = bias.double()
    rows = max(1, CHUNK // (B * nw * heads * N * N))
    for r0 in range(0, nh, rows):
        r1 = min(nh, r0 + rows)
        t = xp[:, r0 * ws:r1 * ws].reshape(B, r1 - r0, ws, nw, ws, 3, heads, d).permute(5, 0, 1, 3, 6, 2, 4, 7).reshape(3, -1, heads, N, d)
        q, k, v = t[0], t[1], t[2]
        s = q @ k.transpose(-1, -2) * scale + bias
        p = torch.softmax(s, -1)
        o = p @ v
        xm = (s - s.amax(-1, keepdim=True)).abs()
        rr = U * ((d + 2) * scale * (q.abs() @ k.abs().transpose(-1, -2)) + 2 * bias.abs() + 2 * s.abs()) + 2.0 ** -23 * (2 + 1.173 * xm) + U * xm
        pr = p * rr
        pv = p @ v.abs()
        E = 1.1 * (pr @ v.abs() + pr.sum(-1, keepdim=True) * o.abs()) + (2 * N + 4) * U * pv
        del s, p, xm, rr, pr, pv, t, q, k

        def back(a):
            return a.reshape(B, r1 - r0, nw, heads, ws, ws, d).permute(0, 1, 4, 2, 5, 3, 6).reshape(B, (r1 - r0) * ws, Wp, C)
        yield r0 * ws, back(o), back(E)


def wmha_check(r, seed):
    B, H, W, C, ws, heads, py, px = (r[f] for f in ("B", "H", "W", "C", "ws", "heads", "pad_y", "pad_x"))
    M, tally = B * H * W, Tally()
    for mode in ("random", "bias") + (("pad",) if py or px else ()):
        qkv16, qkv_bias, bias = wmha_inputs(r, mode, seed)
        qb = guarded(M * 3 * C)
        body(qb, M * 3 * C).copy_(qkv16.flatten())
        q0 = qb.clone()
        out = guarded(M * C)
        _lib.check(_lib.lib().nb200_window_mha_f16(ptr(body(qb, M * 3 * C)), ptr(qkv_bias), ptr(bias), ptr(body(out, M * C)), B, H, W, C,
                                                   ws, heads, py, px, _lib.stream_ptr()))
        torch.cuda.synchronize()
        got = body(out, M * C).view(B, H, W, C)
        tally.no_nan(f"{mode} output", got)
        tally.guards(f"{mode} output", out, M * C)
        tally.exact(f"{mode} qkv", bits(qb), bits(q0))
        for Y0, ref, E in wmha_reference(qkv16, qkv_bias, bias, r):
            y0, y1 = max(Y0, py), min(Y0 + ref.shape[1], py + H)
            if y0 < y1:
                sl = (slice(None), slice(y0 - Y0, y1 - Y0), slice(px, px + W))
                tally.add(got[:, y0 - py:y1 - py], ref[sl], round16_bound(ref[sl], E[sl]))
    return tally.result()


def test_window_mha_replay(production):
    have = {(r["ws"], r["heads"], r["C"] // r["heads"]) for recs in production.values() for k, r in recs if k == "wmha"}
    print(f"\nwindow_mha instantiations recorded: {sorted(have)}")
    cases = configurations(production, "wmha", _synthetic_wmha())
    assert {(r["ws"], r["heads"], r["C"] // r["heads"]) for _, r in cases} == WMHA_INST
    for ws, heads, hd in WMHA_INST:
        pads = {(r["pad_y"], r["pad_x"]) for _, r in cases if (r["ws"], r["heads"], r["C"] // r["heads"]) == (ws, heads, hd)}
        assert pads >= ({(0, 0)} | ({(0, ws // 2), (ws // 2, 0), (ws // 2, ws // 2)} if ws % 2 == 0 else set())), (ws, heads, pads)
    replay("wmha", cases, wmha_check)


def test_window_mha_refuses_bad_padding():
    """Padding other than 0 or ws / 2, or a padded grid that does not tile into whole windows (odd ws with padding: the last
    row / column of windows would be dropped), is refused before any launch.  Real buffers, so nothing is read out of them
    even if a check were missing."""
    lib = _lib.lib()
    qkv = torch.zeros(4 * 3 * 4 * 3 * 64, dtype=torch.float16, device=DEV)
    out = torch.zeros(4 * 3 * 4 * 64, dtype=torch.float16, device=DEV)
    qb, bias = torch.zeros(3 * 64, device=DEV), torch.zeros(64 * 64, device=DEV)
    for ws, H, W, py, px, msg in ((3, 3, 3, 1, 0, b"padded token grid"), (3, 3, 3, 0, 1, b"padded token grid"),
                                  (4, 4, 4, 1, 0, b"padding must be"), (4, 4, 4, 2, 4, b"padding must be")):
        assert lib.nb200_window_mha_f16(ptr(qkv), ptr(qb), ptr(bias), ptr(out), 1, H, W, 64, ws, 2, py, px, _lib.stream_ptr()) != 0
        assert msg in lib.nb200_last_error(), lib.nb200_last_error()
    assert lib.nb200_window_mha_f16(ptr(qkv), None, ptr(bias), ptr(out), 1, 4, 4, 64, 4, 2, 2, 0, _lib.stream_ptr()) != 0
    assert b"qkv bias" in lib.nb200_last_error()
    torch.cuda.synchronize()
    assert not bool(out.any())


# ------------------------------------------------------------------------------------------------------------ replication pad
SYNTH_REPPAD = [dict(B=2, H=1, W=1, C=8), dict(B=3, H=7, W=5, C=24), dict(B=1, H=2, W=33, C=64)]


def reppad_check(r, seed):
    """Bit-exact against ReplicationPad2d(1) built from clamped indices."""
    B, H, W, C = (r[f] for f in ("B", "H", "W", "C"))
    g = torch.Generator(device=DEV).manual_seed(seed)
    n, no = B * H * W * C, B * (H + 2) * (W + 2) * C
    xb, out = guarded(n), guarded(no)
    body(xb, n).copy_(torch.randn(n, generator=g, device=DEV).half())
    x0 = xb.clone()
    _lib.check(_lib.lib().nb200_reppad1_f16(ptr(body(xb, n)), B, H, W, C, ptr(body(out, no)), _lib.stream_ptr()))
    torch.cuda.synchronize()
    tally = Tally()
    x = body(x0, n).view(B, H, W, C)
    iy = torch.arange(-1, H + 1, device=DEV).clamp(0, H - 1)
    ix = torch.arange(-1, W + 1, device=DEV).clamp(0, W - 1)
    tally.exact("output", bits(body(out, no)).view(B, H + 2, W + 2, C), bits(x[:, iy][:, :, ix].contiguous()))
    tally.guards("output", out, no)
    tally.exact("input", bits(xb), bits(x0))
    return tally.result()


def test_reppad_replay(production):
    replay("reppad", configurations(production, "reppad", SYNTH_REPPAD), reppad_check)


# ------------------------------------------------------------------------------------------------------------ add + LayerNorm
SYNTH_LN = [dict(rows=rows, dim=dim, has_delta=hd, has_out=ho) for dim in sorted(LN_DIMS) for rows, hd, ho in ((8 * 5 + 3, 1, 1), (1, 1, 1), (13, 0, 1))] + \
           [dict(rows=21, dim=384, has_delta=1, has_out=0)]


def ln_inputs(r, seed):
    """Rows cycle through: constant (variance 0), near-constant (variance 1e-6, where eps matters), a 1e3 common offset, one
    massive outlier channel, and plain N(0, 1) rows.  The first two get a zero delta so that they stay (near-)constant."""
    rows, dim = r["rows"], r["dim"]
    g = torch.Generator(device=DEV).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    x = rn(rows, dim)
    kind = torch.arange(rows, device=DEV) % 6
    c = 3 * rn(rows, 1)
    x = torch.where(kind[:, None] == 0, c.expand(rows, dim), x)
    x = torch.where(kind[:, None] == 1, c + 1e-3 * x, x)
    x = torch.where(kind[:, None] == 2, x + 1e3, x)
    out_col = (torch.arange(rows, device=DEV) * 37) % dim
    x[(kind == 3).nonzero().flatten(), out_col[kind == 3]] = 3e4
    delta = None
    if r["has_delta"]:
        delta = torch.where((kind[:, None] <= 1), 0.0, rn(rows, dim)).half()
    return x, delta, 1 + 0.2 * rn(dim), 0.1 * rn(dim)


def ln_check(r, seed):
    """The residual write-back x32 + fp32(delta) is bit-exact against torch's fp32 add (x32 is not written without a delta);
    the fp16 output is within round16_bound of the float64 LayerNorm (eps 1e-6) of the updated stream, with E per element:
    the warp's sums are trees of depth D = dim / 128 + 7, so the mean is within e_m = D U mean|x| + U |mean|; the variance's
    relative error is (D + 5) U plus e_m^2 / var (Sum(x - mean) = 0 cancels the first-order term), rsqrtf adds 2 ulp and eps one
    rounding, so rstd is within e_r = ((D + 5) U var + e_m^2) / (2 (var + eps)) + U / 2 + 2^-22 relative; the affine tail
    (x - m) rstd w + b rounds three times.  E = 1.1 (|w| rstd (e_m + |x - mean| (e_r + 3 U)) + 2 U (|y| + |b|))."""
    rows, dim, has_delta, has_out = (r[f] for f in ("rows", "dim", "has_delta", "has_out"))
    x, delta, w, b = ln_inputs(r, seed)
    n = rows * dim
    xb = guarded32(n)
    body(xb, n).copy_(x.flatten())
    db = None
    if has_delta:
        db = guarded(n)
        body(db, n).copy_(delta.flatten())
        d0 = db.clone()
    out = guarded(n) if has_out else None
    _lib.check(_lib.lib().nb200_add_layernorm_f32(ptr(body(xb, n)), ptr(body(db, n)) if has_delta else None, ptr(w), ptr(b),
                                                  ptr(body(out, n)) if has_out else None, rows, dim, _lib.stream_ptr()))
    torch.cuda.synchronize()
    tally = Tally()
    xn = x + delta.float() if has_delta else x
    tally.exact("residual stream", body(xb, n).view(torch.int32), xn.flatten().view(torch.int32))
    tally.guards("residual stream", xb, n)
    if has_delta:
        tally.exact("delta", bits(db), bits(d0))
    if has_out:
        got = body(out, n).view(rows, dim)
        tally.no_nan("output", got)
        tally.guards("output", out, n)
        X = xn.double()
        mean = X.mean(-1, keepdim=True)
        dev = X - mean
        var = (dev * dev).mean(-1, keepdim=True)
        rstd = 1.0 / torch.sqrt(var + 1e-6)
        y = dev * rstd * w.double() + b.double()
        D = dim // 128 + 7
        e_m = D * U * X.abs().mean(-1, keepdim=True) + U * mean.abs()
        e_r = ((D + 5) * U * var + e_m ** 2) / (2 * (var + 1e-6)) + U / 2 + 2.0 ** -22
        E = 1.1 * (w.double().abs() * rstd * (e_m + dev.abs() * (e_r + 3 * U)) + 2 * U * (y.abs() + b.double().abs()))
        tally.add(got, y, round16_bound(y, E))
    return tally.result()


def test_add_layernorm_replay(production):
    cases = configurations(production, "ln", SYNTH_LN)
    assert {r["dim"] for _, r in cases} == LN_DIMS
    assert {(r["has_delta"], r["has_out"]) for _, r in cases} >= {(1, 1), (0, 1), (1, 0)}
    replay("ln", cases, ln_check)


# ------------------------------------------------------------------------------------------------------------ bilinear upsample
SYNTH_UPBL = [dict(B=2, h=9, w=13, C=8, H=9, W=13), dict(B=1, h=7, w=5, C=16, H=19, W=23), dict(B=2, h=1, w=3, C=8, H=4, W=1),
              dict(B=1, h=11, w=11, C=32, H=3, W=29)]


def _upsample_case(r, seed, fn, with_e):
    B, h, w, C, H, W = (r[f] for f in ("B", "h", "w", "C", "H", "W"))
    g = torch.Generator(device=DEV).manual_seed(seed)
    ni, no = B * h * w * C, B * H * W * C
    xb, out = guarded(ni), guarded(no)
    body(xb, ni).copy_((torch.randn(ni, generator=g, device=DEV) * 4).half())
    eb = None
    if with_e:
        eb = guarded(no)
        body(eb, no).copy_((torch.randn(no, generator=g, device=DEV) * 4).half())
    snap = [t.clone() for t in (xb, eb) if t is not None]
    fn(xb, eb, out, ni, no)
    torch.cuda.synchronize()
    tally = Tally()
    got = body(out, no).view(B, H, W, C)
    tally.no_nan("output", got)
    tally.guards("output", out, no)
    for t, t0 in zip([t for t in (xb, eb) if t is not None], snap):
        tally.exact("input", bits(t), bits(t0))
    x = body(xb, ni).view(B, h, w, C)
    for i in range(B):
        up, s = bilinear64(x[i], H, W)
        E = 2.0 ** -21 * s
        if with_e:
            # the interpolated embedding is rounded to fp16 first (an fp16 tensor in the reference), then fp16 + fp16
            up_r, eu = rounded(up, E)
            ref = body(eb, no).view(B, H, W, C)[i].double() + up_r
            tally.add(got[i], ref, round16_bound(ref, eu))
        else:
            tally.add(got[i], up, round16_bound(up, E))
    return tally.result()


def upbl_check(r, seed):
    """One fp16 rounding of the bilinear (align_corners=True) resize: round16_bound with E = 2^-21 sum |corners| (bilinear64)."""
    def run(xb, eb, out, ni, no):
        _lib.check(_lib.lib().nb200_upsample_bilinear_f16(ptr(body(xb, ni)), r["B"], r["h"], r["w"], r["C"], ptr(body(out, no)), r["H"],
                                                          r["W"], _lib.stream_ptr()))
    return _upsample_case(r, seed, run, False)


def zadd_up_check(r, seed):
    """y = fp16(e + fp16(bilinear(prev))): the inner rounding carries E = 2^-21 sum |corners| forward through rounded(), the
    outer one is round16_bound of that."""
    def run(xb, eb, out, ni, no):
        _lib.check(_lib.lib().nb200_zoe_add_upsampled_f16(ptr(body(eb, no)), ptr(body(xb, ni)), r["B"], r["h"], r["w"], r["C"], r["H"],
                                                          r["W"], ptr(body(out, no)), _lib.stream_ptr()))
    return _upsample_case(r, seed, run, True)


def test_upsample_bilinear_replay(production):
    replay("upbl", configurations(production, "upbl", SYNTH_UPBL), upbl_check)


def test_zoe_add_upsampled_replay(production):
    replay("zadd_up", configurations(production, "zadd_up", SYNTH_UPBL), zadd_up_check)


# ------------------------------------------------------------------------------------------------------------ clb concat
SYNTH_CLB_CONCAT = [dict(B=2, h=9, w=13, H=9, W=13), dict(B=1, h=5, w=7, H=19, W=23), dict(B=3, h=1, w=2, H=2, W=5)]


def clb_concat_check(r, seed):
    """A[pix] = [bilinear(emb) 128 | act 32 | fp16(rel) | 31 zeros]: the copy groups (act, rel at this size: the reference's
    interpolate of rel to act's size is the identity, then .to(fp16)) and the zeros bit-exact, the interpolated groups one fp16
    rounding as in upbl_check."""
    B, h, w, H, W = (r[f] for f in ("B", "h", "w", "H", "W"))
    g = torch.Generator(device=DEV).manual_seed(seed)
    npix, ne = B * H * W, B * h * w * 128
    act, eb, relb, out = guarded(npix * 32), guarded(ne), guarded32(npix), guarded(npix * 192)
    body(act, npix * 32).copy_((torch.randn(npix * 32, generator=g, device=DEV) * 2).half())
    body(eb, ne).copy_((torch.randn(ne, generator=g, device=DEV) * 4).half())
    body(relb, npix).copy_(torch.rand(npix, generator=g, device=DEV) * 10)
    snap = [t.clone() for t in (act, eb, relb)]
    _lib.check(_lib.lib().nb200_zoe_clb_concat_f16(ptr(body(act, npix * 32)), ptr(body(relb, npix)), ptr(body(eb, ne)), B, h, w, H, W,
                                                   ptr(body(out, npix * 192)), _lib.stream_ptr()))
    torch.cuda.synchronize()
    tally = Tally()
    got = body(out, npix * 192).view(B, H, W, 192)
    tally.no_nan("output", got)
    tally.guards("output", out, npix * 192)
    for t, t0 in zip((act, eb, relb), snap):
        tally.exact("input", t.view(torch.int16), t0.view(torch.int16))
    want = torch.zeros(B, H, W, 64, dtype=torch.float16, device=DEV)
    want[..., :32] = body(act, npix * 32).view(B, H, W, 32)
    want[..., 32] = body(relb, npix).view(B, H, W).half()
    tally.exact("act | rel | zeros", bits(got[..., 128:].contiguous()), bits(want))
    emb = body(eb, ne).view(B, h, w, 128)
    for i in range(B):
        up, s = bilinear64(emb[i], H, W)
        tally.add(got[i, ..., :128], up, round16_bound(up, 2.0 ** -21 * s))
    return tally.result()


def test_zoe_clb_concat_replay(production):
    replay("zclb_concat", configurations(production, "zclb_concat", SYNTH_CLB_CONCAT), clb_concat_check)


# ------------------------------------------------------------------------------------------------------------ softplus
def softplus64(x):
    """F.softplus (beta 1, threshold 20) in float64."""
    return torch.where(x > 20, x, torch.log1p(torch.exp(x)))


def softplus_check(r, seed):
    """fp32 softplus of fp16 inputs: expf and log1pf are within 2 ulp each and softplus's condition number in its input is
    below 1, so the bound is 2^-21 |ref| (plus 2^-126 where exp underflows)."""
    n = r["n"]
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = (torch.randn(n, generator=g, device=DEV) * 8).half()
    special = torch.tensor([20.0, 20.015625, 19.984375, -20.0, 0.0, -0.0, 65504.0, -65504.0, -100.0, 2.0 ** -24, -17.0, 88.0],
                           device=DEV).half()
    x[:min(n, special.numel())] = special[:n]
    xb, out = guarded(n), guarded32(n)
    body(xb, n).copy_(x)
    _lib.check(_lib.lib().nb200_zoe_softplus_f32(ptr(body(xb, n)), ptr(body(out, n)), n, _lib.stream_ptr()))
    torch.cuda.synchronize()
    tally = Tally()
    got = body(out, n)
    tally.no_nan("output", got)
    tally.guards("output", out, n)
    ref = softplus64(x.double())
    tally.add(got, ref, 2.0 ** -21 * ref.abs() + 2.0 ** -126)
    return tally.result()


def test_zoe_softplus_replay(production):
    replay("zsoftplus", configurations(production, "zsoftplus", [dict(n=1), dict(n=12), dict(n=64 * 1001 + 3)]), softplus_check)


# ------------------------------------------------------------------------------------------------------------ normed seed
def seed_check(r, seed):
    """SeedBinRegressor (normed; oracle/zoedepth_any.py _seed_normed): w = fp16 tensor + 1e-3 (ATen: fp32 add, fp16 result), edges
    min + cumsum((max - min) w / sum w), centres the edge midpoints, out = (centres - min) / (max - min), in float64 from the fp16
    w.  The kernel's fp32 sum (6 levels), widths (2 roundings), scan (6 levels) and the edges in depth units (a few roundings of
    values up to min + span) put it within E = 2^-19 (1 + min / span) of the reference on the [0, 1] scale."""
    npix, lo, hi = r["npix"], float(r["min"]), float(r["max"])
    lo32, hi32 = torch.tensor(lo, dtype=torch.float32).item(), torch.tensor(hi, dtype=torch.float32).item()
    g = torch.Generator(device=DEV).manual_seed(seed)
    s = torch.relu(torch.randn(npix, 64, generator=g, device=DEV) * 2)
    kind = torch.arange(npix, device=DEV) % 5
    s[kind == 1] = 0.0
    s[kind == 2, 17] = 6e4
    s[kind == 3] = torch.exp(torch.randn(int((kind == 3).sum()), 64, generator=g, device=DEV) * 3).clamp(max=6e4)
    s = s.half()
    n = npix * 64
    sb, out = guarded(n), guarded32(n)
    body(sb, n).copy_(s.flatten())
    _lib.check(_lib.lib().nb200_zoe_seed_normed_f32(ptr(body(sb, n)), npix, lo32, hi32, ptr(body(out, n)), _lib.stream_ptr()))
    torch.cuda.synchronize()
    tally = Tally()
    got = body(out, n).view(npix, 64)
    tally.no_nan("output", got)
    tally.guards("output", out, n)
    w = (s.float() + 1e-3).half().double()
    cw = torch.cumsum(w, -1)
    ref = (cw - 0.5 * w) / cw[:, -1:]
    span = hi32 - lo32
    tally.add(got, ref, torch.full_like(ref, 2.0 ** -19 * (1 + abs(lo32) / span)))
    return tally.result()


def test_zoe_seed_normed_replay(production):
    cases = configurations(production, "zseed", [dict(npix=1, min=0.001, max=80), dict(npix=8 * 37 + 5, min=0.5, max=10.0)])
    replay("zseed", cases, seed_check)


# ------------------------------------------------------------------------------------------------------------ attractors
def inv_attractor(dx):
    """attractor.py inv_attractor with its default alpha = 300, gamma = 2 (what the upstream layers call)."""
    return dx / (1 + 300.0 * dx * dx)


SYNTH_ZATTR = [
    # normed: identity resize (the sort sees prev's patterns unchanged), the production attractor count, sorted centres
    dict(B=2, h=9, w=13, H=9, W=13, lda=32, na=16, normed=1, min=0.001, max=80, has_sorted=1),
    dict(B=1, h=5, w=7, H=19, W=23, lda=2, na=1, normed=1, min=0.5, max=10.0, has_sorted=1),
    dict(B=1, h=3, w=3, H=10, W=6, lda=8, na=4, normed=1, min=0.001, max=80, has_sorted=0),
    dict(B=2, h=9, w=13, H=9, W=13, lda=16, na=16, normed=0, min=0, max=0, has_sorted=0),
    dict(B=1, h=1, w=4, H=4, W=11, lda=8, na=1, normed=0, min=0, max=0, has_sorted=0),
]


def attractor_check(r, seed):
    """AttractorLayer (normed: a_j = fp16(apre[2j] + 1e-3)) / AttractorLayerUnnormed (a_j = softplus(apre[j]), fp32, within
    2^-21 a_j): c = bilinear(prev) (within e_c = 2^-21 sum |corners|), out = c + mean_j inv_attractor(a_j - c), in float64.
    |d inv / d dx| <= 1, so E = 2.25 e_c + mean_j(e_a_j + 2 U |dx_j| + 6 U |inv_j|) + na U mean_j |inv_j| + 2 U |out| (the
    na-term fp32 sum, the divide, the final add).  Sorted (normed): clip(sort(span out + min), min, max) of the kernel's own
    unsorted output, computed in fp32 by torch, within 1 fp32 ulp (the kernel may fuse span out + min into one FMA).

    prev's pixels cycle through random values in [-0.3, 1.3] (beyond [0, 1] so that the clip acts), ascending and descending
    bins, and bins drawn from 5 levels (ties); with an identity resize the sort sees them unchanged."""
    B, h, w, H, W, lda, na, normed = (r[f] for f in ("B", "h", "w", "H", "W", "lda", "na", "normed"))
    g = torch.Generator(device=DEV).manual_seed(seed)
    npix, nprev = B * H * W, B * h * w * 64
    ab, pb, out = guarded(npix * lda), guarded32(nprev), guarded32(npix * 64)
    sb = guarded32(npix * 64) if r["has_sorted"] else None
    apre = body(ab, npix * lda).view(npix, lda)       # columns the kernel does not read stay NaN
    cols = slice(0, 2 * na, 2) if normed else slice(0, na)
    if normed:
        apre[:, cols] = (torch.rand(npix, na, generator=g, device=DEV) * 1.2).half()
        u = torch.rand(B * h * w, 64, generator=g, device=DEV)
        kind = torch.arange(B * h * w, device=DEV) % 4
        prev = -0.3 + 1.6 * u
        prev = torch.where(kind[:, None] == 1, prev.sort(-1).values, prev)
        prev = torch.where(kind[:, None] == 2, prev.sort(-1, descending=True).values, prev)
        prev = torch.where(kind[:, None] == 3, -0.3 + 0.4 * (u * 5).floor(), prev)
    else:
        apre[:, cols] = (torch.randn(npix, na, generator=g, device=DEV) + 0.5).half()
        prev = 0.2 + 2.8 * torch.rand(B * h * w, 64, generator=g, device=DEV)
    body(pb, nprev).copy_(prev.flatten())
    snap = [ab.clone(), pb.clone()]
    lo, hi = (torch.tensor(float(v), dtype=torch.float32).item() for v in (r["min"], r["max"]))
    _lib.check(_lib.lib().nb200_zoe_attractor_f32(ptr(body(ab, npix * lda)), lda, na, ptr(body(pb, nprev)), B, h, w, H, W, normed, lo, hi,
                                                  ptr(body(out, npix * 64)), ptr(body(sb, npix * 64)) if sb is not None else None,
                                                  _lib.stream_ptr()))
    torch.cuda.synchronize()
    tally = Tally()
    got = body(out, npix * 64).view(B, H, W, 64)
    tally.no_nan("output", got)
    tally.guards("output", out, npix * 64)
    tally.exact("apre", bits(ab), bits(snap[0]))
    tally.exact("prev", pb.view(torch.int32), snap[1].view(torch.int32))
    a_all = apre[:, cols].reshape(B, H, W, na)
    for i in range(B):
        c, s = bilinear64(body(pb, nprev).view(B, h, w, 64)[i], H, W)
        if normed:
            a = (a_all[i].float() + 1e-3).half().double()
            ea = torch.zeros_like(a)
        else:
            a = softplus64(a_all[i].double())
            ea = 2.0 ** -21 * a
        delta = torch.zeros_like(c)
        err = torch.zeros_like(c)
        sinv = torch.zeros_like(c)
        for j in range(na):
            dx = a[..., j:j + 1] - c
            v = inv_attractor(dx)
            delta += v
            sinv += v.abs()
            err += ea[..., j:j + 1] + 2 * U * dx.abs() + 6 * U * v.abs()
        ref = c + delta / na
        E = 2.25 * 2.0 ** -21 * s + err / na + U * sinv + 2 * U * ref.abs()
        tally.add(got[i], ref, E)
    if sb is not None:
        gs = body(sb, npix * 64).view(B, H, W, 64)
        tally.no_nan("sorted", gs)
        tally.guards("sorted", sb, npix * 64)
        span = torch.tensor(hi, dtype=torch.float32, device=DEV) - torch.tensor(lo, dtype=torch.float32, device=DEV)
        want = (span * got + lo).sort(-1).values.clamp(lo, hi).double()
        tally.add(gs, want, 2.0 ** -23 * want.abs() + 2.0 ** -149)
    return tally.result()


def test_zoe_attractor_replay(production):
    cases = configurations(production, "zattr", SYNTH_ZATTR)
    na_max = max(r["na"] for _, r in cases)
    for normed in (0, 1):
        assert {r["na"] for _, r in cases if r["normed"] == normed} >= {1, na_max}, normed
    assert any(r["has_sorted"] and r["h"] == r["H"] and r["w"] == r["W"] for _, r in cases)
    replay("zattr", cases, attractor_check)


# ------------------------------------------------------------------------------------------------------------ log-binomial mixture
def _synthetic_clb_final():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    # npix = 3 (64 sms) + 39: the persistent warps of the capped grid (8 warps x 8 blocks per SM) loop 4 times, the last partly
    return [dict(B=1, h=2, w=37, H=3, W=64 * sms + 13, ldg=80), dict(B=2, h=9, w=13, H=9, W=13, ldg=104),
            dict(B=1, h=5, w=7, H=19, W=23, ldg=96)]


def clb_final_check(r, seed):
    """ConditionalLogBinomial after its GELU (oracle/zoedepth.py metric_head): t_o = softplus(g w2_o + b2_o), p = (t0 + 1e-4) /
    (t0 + t1 + 2e-4), temperature = 49.9788 (t2 + 1e-4) / (t2 + t3 + 2e-4) + 0.0212, logits (log_binom(63, k) + k log clamp(p) +
    (63 - k) log clamp(1 - p)) / temperature, softmax over 64 bins, depth = sum prob_k bilinear(bins)_k, in float64.  The 4-output
    conv is kept in fp32 (the kernel's documented choice; the autocast reference rounds it to fp16).

    Bound, first order with the kernel's fp32 steps: the conv sums (depth 8) are within e_acc = 9 U (sum|g w2| + |b2|), so
    e_t = e_acc sigmoid(acc + e_acc) + 2^-20 t; p and the
    temperature fraction carry e_t / t of each term plus 2 U; log clamp(x) moves by e_x / max(x - e_x, 1e-4) plus one logf ulp;
    log_binom's three fp32 n log n terms (a logf ulp and a product
    rounding each, two subtractions) are within 5 U of their magnitudes (+ 2e-6 for the 1e-7 epsilons fp32 cannot hold); the
    logit error e_y = (e_lb + k e_lp + (63 - k) e_lq + 4 U |terms|) / temp + |y| (e_temp / temp + U) is amplified by up to
    1 / 0.0212; expf adds 2 ulp after its argument's rounding.  A relative error r_k on bin k's weight moves the depth by
    sum_k p_k r_k |c_k - depth| (1.1 margin), the centres add e_c = 2^-21 sum |corners| and the two 64-term warp sums and the
    divide 8 U sum p_k |c_k| + U |depth|.

    The first four hidden channels steer t: w2 = [I_4 | 0.05 N(0, 1)], so rows cycle through p near 0 / 1 (clamped at 1e-4 and
    1 - 1e-4), the temperature at its minimum (0.0212) and maximum (50), and random values."""
    B, h, w, H, W, ldg = (r[f] for f in ("B", "h", "w", "H", "W", "ldg"))
    g = torch.Generator(device=DEV).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    npix, nb = B * H * W, B * h * w * 64
    gb, bb, out = guarded(npix * ldg), guarded32(nb), guarded32(npix)
    G = body(gb, npix * ldg).view(npix, ldg)
    ctrl = 4 * rn(npix, 4)
    kind = torch.arange(npix, device=DEV) % 6
    big, small = 12.0, -18.0
    for kd, vals in ((1, (big, small, None, None)), (2, (small, big, None, None)), (3, (None, None, small, big)),
                     (4, (None, None, big, small)), (5, (big, small, small, big))):
        for o, v in enumerate(vals):
            if v is not None:
                ctrl[kind == kd, o] = v
    G[:, :4] = ctrl.half()
    G[:, 4:80] = rn(npix, 76).half()
    w2 = torch.cat([torch.eye(4, device=DEV), 0.05 * rn(4, 76)], 1).contiguous()
    b2 = 0.1 * rn(4)
    bins = (0.5 + 9.5 * torch.rand(B * h * w, 64, generator=g, device=DEV)).sort(-1).values
    body(bb, nb).copy_(bins.flatten())
    snap = [gb.clone(), bb.clone()]
    _lib.check(_lib.lib().nb200_zoe_clb_final_f32(ptr(body(gb, npix * ldg)), ldg, ptr(w2), ptr(b2), ptr(body(bb, nb)), B, h, w, H, W,
                                                  ptr(body(out, npix)), _lib.stream_ptr()))
    torch.cuda.synchronize()
    tally = Tally()
    got = body(out, npix).view(B, H, W)
    tally.no_nan("depth", got)
    tally.guards("depth", out, npix)
    tally.exact("hidden", bits(gb), bits(snap[0]))
    tally.exact("bins", bb.view(torch.int32), snap[1].view(torch.int32))
    from oracle.zoedepth import MAX_TEMP, MIN_TEMP
    k = torch.arange(64, dtype=torch.float64, device=DEV)
    n63, eps = 63.0 + 1e-7, 1e-7
    kk = k + eps
    lb_terms = [n63 * math.log(n63) * torch.ones_like(k), kk * torch.log(kk), (n63 - kk) * torch.log(n63 - kk + eps)]
    lb = lb_terms[0] - lb_terms[1] - lb_terms[2]
    e_lb = 5 * U * sum(t.abs() for t in lb_terms) + 2e-6
    Gd = G[:, :80].double().reshape(B, H, W, 80)
    w2d, b2d = w2.double(), b2.double()
    for i in range(B):
        acc = Gd[i] @ w2d.t() + b2d
        e_acc = 9 * U * (Gd[i].abs() @ w2d.abs().t() + b2d.abs())
        t = softplus64(acc) + 1e-4
        e_t = e_acc * torch.sigmoid(acc + e_acc) + 2.0 ** -20 * t
        rel = e_t / t

        def frac(a, b):
            f = t[..., a] / (t[..., a] + t[..., b])
            return f, f * (rel[..., a] + (e_t[..., a] + e_t[..., b]) / (t[..., a] + t[..., b]) + 2 * U)
        p, e_p = frac(0, 1)
        tn, e_tn = frac(2, 3)
        temp = (MAX_TEMP - MIN_TEMP) * tn + MIN_TEMP
        e_temp = (MAX_TEMP - MIN_TEMP) * e_tn + 2 * U * temp
        q, e_q = 1 - p, e_p + U * (1 - p)
        lp, lq = torch.log(p.clamp(1e-4, 1)), torch.log(q.clamp(1e-4, 1))
        e_lp = e_p / (p - e_p).clamp_min(1e-4) + 2.0 ** -23 * (1 + lp.abs())
        e_lq = e_q / (q - e_q).clamp_min(1e-4) + 2.0 ** -23 * (1 + lq.abs())
        Y = lb + k * lp[..., None] + (63 - k) * lq[..., None]
        T = temp[..., None]
        y = Y / T
        e_Y = e_lb + k * e_lp[..., None] + (63 - k) * e_lq[..., None] + 4 * U * (lb.abs() + k * lp.abs()[..., None] + (63 - k) * lq.abs()[..., None])
        e_y = e_Y / T + y.abs() * (e_temp[..., None] / T + U)
        xm = (y - y.amax(-1, keepdim=True)).abs()
        prob = torch.softmax(y, -1)
        c, s = bilinear64(body(bb, nb).view(B, h, w, 64)[i], H, W)
        d = (prob * c).sum(-1)
        rk = e_y + U * xm + 2.0 ** -22
        E = 1.1 * (prob * rk * (c - d[..., None]).abs()).sum(-1) + (prob * 2.0 ** -21 * s).sum(-1) + 8 * U * (prob * c.abs()).sum(-1) + U * d.abs()
        tally.add(got[i], d, E)
    return tally.result()


def test_zoe_clb_final_replay(production):
    cases = configurations(production, "zclb_final", _synthetic_clb_final())
    assert any(r["ldg"] > 80 for _, r in cases) and any(r["ldg"] == 80 for _, r in cases)
    replay("zclb_final", cases, clb_final_check)


# ------------------------------------------------------------------------------------------------------------ BEiT bias expansion
SYNTH_ZRELBIAS = [dict(ph=1, pw=1, heads=2, ldb=3), dict(ph=3, pw=5, heads=4, ldb=20), dict(ph=2, pw=7, heads=3, ldb=15)]


def relbias_check(r, seed):
    """Bit-exact: bias[h][q][k] = fp32(table[index(q, k)][h] * log2 e) with the index table of MiDaS beit.py
    gen_relative_position_index (oracle/zoedepth.py relative_position_index, not the kernel's formula); columns N..ldb-1 keep
    their sentinel."""
    from oracle.zoedepth import relative_position_index
    ph, pw, heads, ldb = (r[f] for f in ("ph", "pw", "heads", "ldb"))
    N, rows = ph * pw + 1, (2 * ph - 1) * (2 * pw - 1) + 3
    g = torch.Generator(device=DEV).manual_seed(seed)
    table = torch.randn(rows, heads, generator=g, device=DEV)
    n = heads * N * ldb
    out = guarded32(n)
    _lib.check(_lib.lib().nb200_zoe_expand_rel_bias_f32(ptr(table), ph, pw, heads, ptr(body(out, n)), ldb, _lib.stream_ptr()))
    torch.cuda.synchronize()
    tally = Tally()
    got = body(out, n).view(heads, N, ldb)
    idx = relative_position_index(ph, pw).to(DEV)
    want = (table[idx.view(-1)].view(N, N, heads).permute(2, 0, 1) * torch.tensor(LOG2E, dtype=torch.float32, device=DEV)).contiguous()
    tally.exact("bias", got[..., :N].contiguous().view(torch.int32), want.view(torch.int32))
    tally.exact("columns N..ldb", got[..., N:].contiguous().view(torch.int32),
                torch.full((heads, N, ldb - N), SENTINEL32, dtype=torch.int32, device=DEV))
    tally.guards("bias", out, n)
    return tally.result()


def test_zoe_expand_rel_bias_replay(production):
    replay("zrelbias", configurations(production, "zrelbias", SYNTH_ZRELBIAS), relbias_check)
