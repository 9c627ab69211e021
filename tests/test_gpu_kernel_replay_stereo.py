"""GPU: replay every launch of the learned stereo networks' own kernels against float64 references: the input and output stages
of row_flow_v3 (csrc/rowflow_kernels.cu), mlbw (csrc/mlbw.cu) and depth_aa (csrc/depth_aa.cu), the fused row_flow_v2 delta
kernel (csrc/rowflow_v2.cu) and the hole mask of mask_mlbw_l2.  Their window-attention blocks and GEMMs are replayed by the
other three modules.

The discipline of tests/test_gpu_kernel_replay.py, with the helpers of tests/replay.py: a module fixture turns on bit 3 of the
launch recorder and records the networks of STEREO_MODELS, and each unique configuration (plus a synthetic list for the edges
production does not reach: every tap clamped, one-row images, widths around the pack and tile sizes, batches whose tokens and
strips straddle images) is replayed through the kernel's test entry point on fresh seeded data.  Outputs sit between guard
blocks whose NaN sentinel must survive, and input elements the reference never reads are NaN.  The references follow the
oracle's structure (oracle/row_flow.py, row_flow_v2.py, mlbw.py, depth_aa.py): real F.pad replicate pads, pixel (un)shuffles,
crops and F.conv2d in float64, never the kernels' clamp arithmetic.  Each element's bound comes from the kernel's arithmetic
(U = 2^-24 is the fp32 unit roundoff): an fp32 fma chain of n terms is within (n + 1) U sum|a w| of the exact sum, a chain of
L mma.sync k16 steps within 2^-20 L sum|a w|, and an fp16 rounding point carries a difference forward only where a rounding
boundary lies within the bound (rounded()).
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from tests.util import log_metric
from tests.replay import (DEV, STEREO_MODELS, Tally, bits, body, configurations, guarded, guarded32, record_networks, replay,
                          round16_bound, rounded)
from nunif_b200 import _lib, synth
from nunif_b200._lib import ptr

pytestmark = pytest.mark.gpu
U = 2.0 ** -24                 # fp32 unit roundoff
ACC = 2.0 ** -20               # per chained mma.sync k16 step: |fp32 accumulator - exact| <= ACC * L * sum |a w|
REC_STEREO = 8                 # nb200_record_launches bit of the kinds replayed here
FP16_MAX = 65520.0             # fp16 rounds a value at or beyond this magnitude to inf
TINY = 1e-300                  # bound floor: an exact element has err / bound 0

STEREO_KINDS = ("rfprep", "rflast", "rf2", "mlprep", "mlout", "holemask", "aaminmax", "aaprep", "aaout")
# the launches of one forward of each network (both frames of STEREO_FRAMES, or both eyes)
EXPECTED = {
    "row_flow_v3": {"rfprep": 2, "rflast": 2},
    "row_flow_v2": {"rf2": 2},
    "mlbw_l2": {"mlprep": 2, "mlout": 2},
    "mlbw_l4": {"mlprep": 2, "mlout": 2},
    "mask_mlbw_l2": {"mlprep": 2, "mlout": 2},
    "mlbw_l2_inpaint": {"mlprep": 2, "mlout": 2, "holemask": 2},
    "depth_aa": {"aaminmax": 1, "aaprep": 1, "aaout": 1},
}


@pytest.fixture(scope="module")
def production():
    """name -> every record (kind, config) of one forward of each network of STEREO_MODELS (configurations() deduplicates)."""
    return record_networks(REC_STEREO, STEREO_MODELS, unique=False)


def test_every_network_records_its_launches(production):
    for name, _ in STEREO_MODELS:
        counts = {k: sum(1 for kk, _ in production[name] if kk == k) for k in STEREO_KINDS}
        log_metric("replay_stereo_launches", model=name, **counts)
        assert {k: n for k, n in counts.items() if n} == EXPECTED[name], name
    assert {r["hole"] for k, r in production["mask_mlbw_l2"] if k == "mlout"} == {1}
    assert {r["hole"] for n in ("mlbw_l2", "mlbw_l4") for k, r in production[n] if k == "mlout"} == {0}
    assert {r["mirror"] for k, r in production["mlbw_l2_inpaint"] if k == "holemask"} == {0, 1}
    assert [(r["norm"], r["clamp"]) for k, r in production["depth_aa"] if k == "aaout"] == [(1, 0)]


# ------------------------------------------------------------------------------------------------------------ helpers
def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def host(t):
    """A host fp32 copy for the entry points' weight arguments (keep it alive across the call)."""
    return t.detach().float().cpu().contiguous()


def unshuffle18(x):
    """pixel_unshuffle (1, 8) of [B][C][Hp][8 Wt] as the oracle writes it -> tokens [B][Hp][Wt][8 C], channel c * 8 + s."""
    B, C, Hp, Wp = x.shape
    return x.reshape(B, C, Hp, 1, Wp // 8, 8).permute(0, 2, 4, 1, 3, 5).reshape(B, Hp, Wp // 8, C * 8)


def shuffle18(t):
    """pixel_shuffle (1, 8): tokens [B][Hp][Wt][8 C] -> [B][C][Hp][8 Wt] (the inverse of unshuffle18)."""
    B, Hp, Wt, C8 = t.shape
    return t.reshape(B, Hp, Wt, C8 // 8, 1, 8).permute(0, 3, 1, 4, 2, 5).reshape(B, C8 // 8, Hp, Wt * 8)


def conv64(x, w, b=None, pad=None):
    """float64 F.conv2d of x (optionally replicate padded first) -> (conv, sum |x w| + |b|)."""
    if pad is not None:
        x = F.pad(x, pad, mode="replicate")
    w = w.double()
    y = F.conv2d(x, w, None if b is None else b.double())
    a = F.conv2d(x.abs(), w.abs())
    return y, a if b is None else a + b.double().abs().view(1, -1, 1, 1)


def add16(tally, what, got, ref, E):
    """One fp16 rounding of a value within E of ref (round16_bound), where ref may lie beyond fp16's range: an element whose
    whole interval [ref - E, ref + E] is beyond FP16_MAX must be inf of ref's sign, one whose interval reaches it may be
    either; the others are tallied."""
    over = ref.abs() - E >= FP16_MAX
    maybe = (ref.abs() + E >= FP16_MAX) & ~over
    if bool(over.any()):
        tally.exact(f"{what} beyond fp16", got[over], torch.copysign(torch.full_like(ref[over], math.inf), ref[over]).to(got.dtype))
    rest = ~(over | maybe)
    if bool(rest.any()):
        tally.add(got[rest], ref[rest], round16_bound(ref[rest], E[rest]))


def rf_geom(B, h, w):
    """row_flow_v3's padding (row_flow_v3.py:59-60, always pads): -> (Hp, Wt)."""
    return h + 12 - h % 12, (w + 96 - w % 96) // 8


def ml_geom(B, H, W):
    """mlbw's _calc_pad (mlbw.py:72-88, always pads) -> dict of the recorded geometry fields."""
    pad_w, pad_h = 32 - W % 32, 4 - H % 4
    return dict(B=B, H=H, W=W, ph1=pad_h // 2, pw1=pad_w // 2, Hp=H + pad_h, Wt=(W + pad_w) // 8)


def aa_geom(B, H, W):
    """depth_aa's padding (depth_aa.py:61-62, always pads) -> dict of the recorded geometry fields."""
    pad_w, pad_h = 16 - W % 16, 16 - H % 16
    return dict(B=B, H=H, W=W, ph1=pad_h // 2, pw1=pad_w // 2, Hh=(H + pad_h) // 2, Wh=(W + pad_w) // 2)


# (B, h, w): every tap clamped (w < 8, w < 14, h = 1, 2, 3), heights around 4, 12 and 16, widths where w % 8, w % 32 and
# w % 96 are 0, 1 and 7 (w % 96 == 0 pads a whole extra block), and batches whose tokens straddle images
SHAPES = [(1, 1, 1), (2, 2, 7), (1, 3, 13), (3, 4, 96), (1, 12, 97), (2, 11, 103), (1, 13, 32), (2, 16, 33), (1, 17, 39),
          (2, 5, 64), (1, 15, 65), (1, 3, 191), (2, 12, 192)]


# ------------------------------------------------------------------------------------------------------------ row_flow_v3
def rfprep_check(r, seed):
    """Bit-exact: fp16(pixel_unshuffle (1, 8) of F.pad(x, (0, 8 Wt - w, 0, Hp - h), replicate)), channels 24..31 zero."""
    B, h, w, Hp, Wt = (r[f] for f in ("B", "h", "w", "Hp", "Wt"))
    g = _gen(seed)
    n, no = B * 3 * h * w, B * Hp * Wt * 32
    xb, out = guarded32(n), guarded(no)
    x = body(xb, n).view(B, 3, h, w)
    x.copy_(torch.randn(B, 3, h, w, generator=g, device=DEV) * 2)
    x0 = xb.clone()
    _lib.check(_lib.lib().nb200_row_flow_prep_f16(ptr(x), B, h, w, Hp, Wt, ptr(body(out, no)), _lib.stream_ptr()))
    torch.cuda.synchronize()
    tally = Tally()
    tally.guards("tokens", out, no)
    tally.exact("x", xb.view(torch.int32), x0.view(torch.int32))
    want = torch.zeros(B, Hp, Wt, 32, dtype=torch.float16, device=DEV)
    want[..., :24] = unshuffle18(F.pad(x, (0, 8 * Wt - w, 0, Hp - h), mode="replicate")).half()
    tally.exact("tokens", bits(body(out, no).view(B, Hp, Wt, 32)), bits(want))
    return tally.result()


def _rf_synthetic():
    return [dict(B=B, h=h, w=w, Hp=rf_geom(B, h, w)[0], Wt=rf_geom(B, h, w)[1]) for B, h, w in SHAPES]


def test_row_flow_prep_replay(production):
    replay("rfprep", configurations(production, "rfprep", _rf_synthetic()), rfprep_check)


def rflast_check(r, seed):
    """conv3x3(ReplicationPad2d(1)(pixel_shuffle(x)[:, :, :h, :w])) (oracle/row_flow.py:30-33) in float64: one fp16 rounding after
    an fp32 fma chain of 72 terms from the bias, round16_bound with E = 73 U (sum|a w| + |b|).  The token rows >= h and the
    pixels of columns >= w are NaN: cropping after the pad would read them."""
    B, Hp, Wt, h, w = (r[f] for f in ("B", "Hp", "Wt", "h", "w"))
    g = _gen(seed)
    n, no = B * Hp * Wt * 64, B * h * w
    S = torch.randn(B, 8, Hp, 8 * Wt, generator=g, device=DEV) * 2
    S[:, :, h:] = math.nan
    S[..., w:] = math.nan
    xb, out = guarded(n), guarded32(no)
    body(xb, n).copy_(unshuffle18(S).half().flatten())
    x0 = xb.clone()
    wt = torch.randn(1, 8, 3, 3, generator=g, device=DEV) * (1.5 / 72 ** 0.5)
    bias = torch.randn(1, generator=g, device=DEV) * 0.1
    wh, bh = host(wt), host(bias)
    _lib.check(_lib.lib().nb200_row_flow_last_conv_f32(ptr(body(xb, n)), B, Hp, Wt, h, w, ptr(wh), ptr(bh), ptr(body(out, no)),
                                                       _lib.stream_ptr()))
    torch.cuda.synchronize()
    tally = Tally()
    got = body(out, no).view(B, 1, h, w)
    tally.no_nan("delta", got)
    tally.guards("delta", out, no)
    tally.exact("tokens", bits(xb), bits(x0))
    Sd = shuffle18(body(x0, n).view(B, Hp, Wt, 64).double())[:, :, :h, :w]
    y, a = conv64(Sd, wt, bias, (1, 1, 1, 1))
    tally.add(got, y, round16_bound(y, 73 * U * a))
    return tally.result()


def test_row_flow_last_conv_replay(production):
    replay("rflast", configurations(production, "rflast", _rf_synthetic()), rflast_check)


# ------------------------------------------------------------------------------------------------------------ row_flow_v2
def rf2_reference(sd, x, single=False, band=64):
    """RowFlowV2._forward_delta_only (oracle/row_flow_v2.py) in float64 with the kernel's rounding points, for x [1][3][h][w]:
    x and the weights fp16 (autocast), every conv -> fp16, + fp16 bias -> fp16 (an fp32 add), ReLU; non_overlap +
    overlap_residual an fp32 add rounded to fp16.  The 28-pixel pre-pad, the inner pads and the crop are the oracle's.
    Everything before the 3x3 conv is row-local, so output rows [y0, y1) need only padded rows y0 + 27 .. y1 + 28 of x: the
    reference runs in bands of `band` rows, the 3x3 conv on a band's own halo rows (the oracle's row pad of that conv lies
    outside the crop).

    Each conv's accumulator is within acc * sum|a w| of the float64 sum (10 U for the 9-term feature fma chain, 17 U for the
    16-term head, 2^-20 L for an mma chain of L k16 steps), plus the differences carried in through |w|.  `single`: every
    output channel of every conv has one nonzero weight (rf2_single_state_dict), so each sum is one exact fp16 x fp16 product
    whatever the order of the zeros: acc = 0, and E = 0 everywhere.  A rounding point whose input is exactly the
    reference's gives exactly the reference's fp16 value, and the fp32 bias add of two equal fp16 pairs is equal too; only
    where a difference is carried do the adds contribute 2 U |v|.  -> iterator of (y0, the fp32 sum before the final fp16
    rounding, bound E on the kernel's difference from it: 0 where the kernel's final value must be that sum's fp16 rounding)."""
    w16 = {k: v.to(DEV).half().double() for k, v in sd.items()}
    _, _, h, w = x.shape
    xp = F.pad(x.half().double(), (28,) * 4, mode="replicate")

    def fp32_add(a, b, e):
        v = (a.float() + b.float()).double()
        return v, torch.where(e > 0, e + 2 * U * v.abs(), torch.zeros_like(e))

    def layer(a, ea, key, pad, acc, relu=True):
        y, s = conv64(a, w16[key + ".weight"], None, pad)
        e = acc * s + F.conv2d(F.pad(ea, pad, mode="replicate") if pad else ea, w16[key + ".weight"].abs())
        c, e1 = rounded(y, e)
        o, e2 = rounded(*fp32_add(c, w16[key + ".bias"].view(1, -1, 1, 1).expand_as(c), e1))
        return (o.clamp_min(0), e2) if relu else (o, e2)

    a1 = 0.0 if single else 1.0
    for y0 in range(0, h, band):
        y1 = min(h, y0 + band)
        xb = xp[:, :, y0 + 27:y1 + 29]
        f, ef = layer(xb, torch.zeros_like(xb), "feature.0", (1, 1, 0, 0), a1 * 10 * U)
        nv, env = layer(f, ef, "non_overlap", None, a1 * 17 * U, relu=False)
        r1, e1 = layer(f, ef, "overlap_residual.0", (4, 4, 0, 0), a1 * 9 * ACC)
        r2, e2 = layer(r1, e1, "overlap_residual.2", (4, 4, 0, 0), a1 * 9 * ACC)
        r3, e3 = layer(r2, e2, "overlap_residual.4", (4, 4, 0, 0), a1 * 18 * ACC)
        r4, e4 = layer(r3, e3, "overlap_residual.6", (1, 1, 0, 0), a1 * 18 * ACC, relu=False)
        out, E = fp32_add(nv[:, :, 1:-1], r4, env[:, :, 1:-1] + e4)
        yield y0, out[..., 28:28 + w], E[..., 28:28 + w]


def rf2_single_state_dict(seed):
    """row_flow_v2 weights that make every rounding point of the kernel observable: each output channel of every conv reads one
    input (channel, tap) picked at random, with a weight of two or three significant bits (+-0.75, 1, 1.25, 1.5, positive three
    times in four), so its fp32 product keeps bits below fp16's precision and the conv -> fp16 -> + bias -> fp16 double rounding
    differs from a single rounding in a good share of the elements.  The 3x3 conv's tap is in the row above or the row below
    (never the middle one), so a row read out of order changes the output.  Biases N(0, 0.3)."""
    g = torch.Generator().manual_seed(seed)
    sd = synth.row_flow_v2_state_dict(seed)
    vals = torch.tensor([0.75, 1.0, 1.25, 1.5])

    def pick(n):
        sign = torch.where(torch.rand(n, generator=g) < 0.75, 1.0, -1.0)
        return vals[torch.randint(0, 4, (n,), generator=g)] * sign
    for key in ("feature.0", "non_overlap", "overlap_residual.0", "overlap_residual.2", "overlap_residual.4", "overlap_residual.6"):
        co, ci, kh, kw = sd[key + ".weight"].shape
        wt = torch.zeros(co, ci * kh * kw)
        if key == "overlap_residual.6":
            ky = 2 * int(torch.randint(0, 2, (1,), generator=g))
            wt[0, int(torch.randint(0, ci, (1,), generator=g)) * 9 + ky * 3 + int(torch.randint(0, 3, (1,), generator=g))] = pick(1)[0]
        else:
            wt[torch.arange(co), torch.randint(0, ci * kh * kw, (co,), generator=g)] = pick(co)
        sd[key + ".weight"] = wt.view(co, ci, kh, kw)
        sd[key + ".bias"] = torch.randn(co, generator=g) * 0.3
    return sd


def _rf2_synthetic():
    """Widths around the 110-column tile and heights around the 16-row strip, every tap clamped, batches of strips."""
    return [dict(B=B, h=h, w=w) for B, h, w in ((1, 1, 1), (2, 3, 5), (1, 2, 13), (3, 4, 14), (2, 15, 109), (1, 16, 110),
                                                (1, 17, 111), (2, 31, 219), (1, 33, 220), (1, 16, 221), (2, 33, 111))]


def rf2_check(r, seed, single):
    """The whole delta network through nb200_row_flow_v2_delta and a model packed from the weights, so that the packer's
    B-fragment order is checked too, against rf2_reference: where E = 0 the kernel's delta must be the reference's fp16 value
    bit for bit, elsewhere within round16_bound.  x's guards are NaN (the clamp-to-edge must never reach them); depth in
    [0, 1], the two feature planes N(0, 0.5) so that every tap matters.

    single = 0: synth.row_flow_v2_state_dict(seed).  Carried through five layers of He-scaled weights, the bound grows to a
    few times the output's own size (median E about 3 |ref|), so these weights catch only gross faults.  single = 1:
    rf2_single_state_dict(seed), where every conv is exact: E is 0 on every element and delta must be bit-exact, so a
    missing, extra or misplaced rounding point, a wrong tap, row or channel moves it off its fp16 value."""
    from nunif_b200.iw3 import RowFlowV2
    B, h, w = r["B"], r["h"], r["w"]
    g = _gen(seed)
    sd = rf2_single_state_dict(seed) if single else synth.row_flow_v2_state_dict(seed)
    net = RowFlowV2(sd, DEV)
    n, no = B * 3 * h * w, B * h * w
    xb, out = guarded32(n), guarded32(no)
    x = body(xb, n).view(B, 3, h, w)
    x[:, :1].copy_(torch.rand(B, 1, h, w, generator=g, device=DEV))
    x[:, 1:].copy_(torch.randn(B, 2, h, w, generator=g, device=DEV) * 0.5)
    x0 = xb.clone()
    _lib.check(_lib.lib().nb200_row_flow_v2_delta(net._h, ptr(x), B, h, w, ptr(body(out, no)), _lib.stream_ptr()))
    torch.cuda.synchronize()
    tally = Tally()
    got = body(out, no).view(B, 1, h, w)
    tally.no_nan("delta", got)
    tally.guards("delta", out, no)
    tally.exact("x", xb.view(torch.int32), x0.view(torch.int32))
    n_exact = 0
    for b in range(B):
        for y0, ref, E in rf2_reference(sd, x[b:b + 1], bool(single)):
            gb = got[b:b + 1, :, y0:y0 + ref.shape[2]]
            ex = E == 0
            n_exact += int(ex.sum())
            tally.exact("delta where E = 0", gb[ex].view(torch.int32), ref[ex].float().half().float().view(torch.int32))
            if bool((~ex).any()):
                tally.add(gb[~ex], ref[~ex], round16_bound(ref[~ex], E[~ex]))
    log_metric("replay_rf2_exact", cfg=f"B={B},h={h},w={w}", single=single, exact=n_exact, of=no)
    if single and n_exact != no:
        tally.bad.append(f"only {n_exact} of {no} elements with E = 0")
    return tally.result()


def test_row_flow_v2_replay(production):
    cases = configurations(production, "rf2", _rf2_synthetic())
    replay("rf2", cases, rf2_check, variant=("single", (0, 1)))


# ------------------------------------------------------------------------------------------------------------ mlbw
def mlprep_check(r, seed):
    """lv1_in (oracle/mlbw.py:24-27): F.pad(x, (pw1, pw2, ph1, ph2)) and F.pad((4, 4, 0, 0)), both replicate, conv (1, 9)
    3 -> C1, LeakyReLU(0.2), pixel_unshuffle (1, 8).  The kernel convolves the fp32 input with the fp32 weights (the exact
    operation, which the autocast reference approximates with fp16 operands): an fp32 fma chain of 27 terms from the bias, 0.2f
    (within U / 4 of 0.2) and its product, then one fp16 rounding: round16_bound with E = 28 U (sum|a w| + |b|) + 2 U |y|."""
    B, H, W, ph1, pw1, Hp, Wt, C1 = (r[f] for f in ("B", "H", "W", "ph1", "pw1", "Hp", "Wt", "C1"))
    g = _gen(seed)
    n, no = B * 3 * H * W, B * Hp * Wt * 8 * C1
    xb, out = guarded32(n), guarded(no)
    x = body(xb, n).view(B, 3, H, W)
    x.copy_(torch.randn(B, 3, H, W, generator=g, device=DEV))
    x0 = xb.clone()
    wt = torch.randn(C1, 3, 1, 9, generator=g, device=DEV) / 27 ** 0.5
    bias = torch.randn(C1, generator=g, device=DEV) * 0.05
    wh, bh = host(wt), host(bias)
    _lib.check(_lib.lib().nb200_mlbw_prep_f16(ptr(x), B, H, W, ph1, pw1, Hp, Wt, C1, ptr(wh), ptr(bh), ptr(body(out, no)),
                                              _lib.stream_ptr()))
    torch.cuda.synchronize()
    tally = Tally()
    got = body(out, no).view(B, Hp, Wt, 8 * C1)
    tally.no_nan("tokens", got)
    tally.guards("tokens", out, no)
    tally.exact("x", xb.view(torch.int32), x0.view(torch.int32))
    xp = F.pad(x.double(), (pw1, 8 * Wt - W - pw1, ph1, Hp - H - ph1), mode="replicate")
    a, s = conv64(xp, wt, bias, (4, 4, 0, 0))
    y = F.leaky_relu(a, 0.2)
    tally.add(got, unshuffle18(y), round16_bound(unshuffle18(y), unshuffle18(28 * U * s + 2 * U * y.abs())))
    return tally.result()


def _ml_synthetic(C1s=(8, 16)):
    return [dict(ml_geom(B, h, w), C1=C1) for B, h, w in SHAPES for C1 in C1s]


def test_mlbw_prep_replay(production):
    cases = configurations(production, "mlprep", _ml_synthetic())
    assert {r["C1"] for _, r in cases} == {8, 16}
    replay("mlprep", cases, mlprep_check)


def mlout_check(r, seed):
    """lv1_out and the heads (oracle/mlbw.py:31-35): v = fp16(t + t0) (the fp16 tensor sum, computed here as the kernel and
    ATen do: an fp32 add rounded once), y = conv (1, 9)(F.pad(pixel_shuffle(v), (4, 4, 0, 0), replicate)) cropped to the image,
    in float64.  Each output is an fp32 fma chain of 9 C1 terms from the bias, E = (9 C1 + 1) U (sum|v w| + |b|): delta and the
    hole logit are one fp16 rounding (round16_bound); the L logits are rounded (rounded()) and go through the kernel's softmax,
    whose relative error per layer is the wmha row's first-order __expf bound, 2^-23 (2 + 1.173 |x|) + U |x| for x = logit -
    max, plus the logit's rounding difference, and (L + 2) U for the sum, reciprocal and product.  The token rows outside
    [ph1, ph1 + H) of both inputs are NaN."""
    B, H, W, ph1, pw1, Hp, Wt, C1, L, hole = (r[f] for f in ("B", "H", "W", "ph1", "pw1", "Hp", "Wt", "C1", "L", "hole"))
    g = _gen(seed)
    NO = 2 * L + hole
    n, no = B * Hp * Wt * 8 * C1, B * H * W
    tb, t0b = guarded(n), guarded(n)
    for buf in (tb, t0b):
        t = torch.randn(B, Hp, Wt, 8 * C1, generator=g, device=DEV)
        t[:, :ph1] = math.nan
        t[:, ph1 + H:] = math.nan
        body(buf, n).copy_(t.half().flatten())
    snap = [tb.clone(), t0b.clone()]
    wt = torch.randn(NO, C1, 1, 9, generator=g, device=DEV) * (1.5 / (9 * C1) ** 0.5)
    bias = torch.randn(NO, generator=g, device=DEV) * 0.1
    wh, bh = host(wt), host(bias)
    db, lb = guarded32(L * no), guarded32(L * no)
    hb = guarded32(no) if hole else None
    _lib.check(_lib.lib().nb200_mlbw_out_f32(ptr(body(tb, n)), ptr(body(t0b, n)), B, H, W, ph1, pw1, Hp, Wt, C1, L, ptr(wh), ptr(bh),
                                             ptr(body(db, L * no)), ptr(body(lb, L * no)), ptr(body(hb, no)) if hole else None,
                                             _lib.stream_ptr()))
    torch.cuda.synchronize()
    tally = Tally()
    for what, buf, m in (("delta", db, L * no), ("layer weight", lb, L * no)) + ((("hole", hb, no),) if hole else ()):
        tally.no_nan(what, body(buf, m))
        tally.guards(what, buf, m)
    tally.exact("t", bits(tb), bits(snap[0]))
    tally.exact("t0", bits(t0b), bits(snap[1]))
    tok = lambda buf: body(buf, n).view(B, Hp, Wt, 8 * C1)
    v = (tok(tb).float() + tok(t0b).float()).half().double()
    y, s = conv64(shuffle18(v), wt, bias, (4, 4, 0, 0))
    y, E = (t[..., ph1:ph1 + H, pw1:pw1 + W] for t in (y, (9 * C1 + 1) * U * s))
    tally.add(body(db, L * no).view(B, L, H, W), y[:, :L], round16_bound(y[:, :L], E[:, :L]))
    if hole:
        tally.add(body(hb, no).view(B, 1, H, W), y[:, 2 * L:], round16_bound(y[:, 2 * L:], E[:, 2 * L:]))
    lg, elg = rounded(y[:, L:2 * L], E[:, L:2 * L])
    p = torch.softmax(lg, 1)
    xm = (lg - lg.amax(1, keepdim=True)).abs()
    rr = 2.0 ** -23 * (2 + 1.173 * xm) + U * xm + elg
    Ep = 1.1 * p * (rr + (p * rr).sum(1, keepdim=True)) + (L + 2) * U * p + 2.0 ** -126
    tally.add(body(lb, L * no).view(B, L, H, W), p, Ep)
    return tally.result()


def _mlout_synthetic():
    return [dict(ml_geom(B, h, w), C1=4 * L, L=L, hole=hole) for B, h, w in SHAPES for L, hole in ((2, 0), (4, 0), (2, 1))]


def test_mlbw_out_replay(production):
    cases = configurations(production, "mlout", _mlout_synthetic())
    assert {(r["L"], r["hole"]) for _, r in cases} == {(2, 0), (4, 0), (2, 1)}
    replay("mlout", cases, mlout_check)


# ------------------------------------------------------------------------------------------------------------ hole mask
def ac_lambda(n_in, n_out):
    """ATen's upsample_bilinear2d(align_corners=True) source indices and weights along one axis, in fp32 as ATen computes them:
    scale = fp32(n_in - 1) / fp32(n_out - 1) (0 for one output), src = scale * i, i0 = min(floor(src), n_in - 1),
    i1 = i0 + (i0 < n_in - 1), l1 = src - i0, l0 = 1 - l1 -> (i0, i1, l0, l1), the weights as float64."""
    one = lambda v: torch.tensor(float(v), dtype=torch.float32, device=DEV)
    scale = one(n_in - 1) / one(n_out - 1) if n_out > 1 else one(0)
    src = scale * torch.arange(n_out, dtype=torch.float32, device=DEV)
    i0 = src.floor().long().clamp(max=n_in - 1)
    i1 = torch.where(i0 < n_in - 1, i0 + 1, i0)
    l1 = (src - i0.float()).clamp(0, 1)
    return i0, i1, (1 - l1).double(), l1.double()


def closing(x):
    """iw3/dilation.py closing with n_iter = 1: a 3x3 max (dilation), then a 3x3 min (erosion), max_pool2d's -inf padding."""
    return -F.max_pool2d(-F.max_pool2d(x, 3, 1, 1), 3, 1, 1)


def holemask_check(r, seed):
    """postprocess_hole_mask up to the threshold (iw3/backward_warp.py:382-388), with forward_left's flips for mirror = 1: the
    closing of the (flipped) logits, the align_corners=True bilinear resize with ATen's fp32 indices and weights (ac_lambda)
    against float64 interpolation, flipped back.  The kernel blends in fp32 (two products and a sum per axis), within
    E = 5 U sum|l v| of that.  Threshold NaN (the resized closed logits): within E, and bit-exact against the fp32 closing when
    both axes copy.  A real threshold: the mask must equal z > logit(threshold) wherever the reference z is farther than
    E + 2^-19 (1 + |logit|) (expf and the fp32 sigmoid) from the logit; the ambiguous elements are counted and capped."""
    B, h, w, H, W, mirror, thr = (r[f] for f in ("B", "h", "w", "H", "W", "mirror", "threshold"))
    g = _gen(seed)
    n, no = B * h * w, B * H * W
    lb, out = guarded32(n), guarded32(no)
    logits = body(lb, n).view(B, 1, h, w)
    logits.copy_(torch.randn(B, 1, h, w, generator=g, device=DEV) * 3 - 1.7)
    l0 = lb.clone()
    _lib.check(_lib.lib().nb200_hole_mask(ptr(logits), B, h, w, H, W, ctypes.c_float(thr), mirror, ptr(body(out, no)), _lib.stream_ptr()))
    torch.cuda.synchronize()
    tally = Tally()
    got = body(out, no).view(B, 1, H, W)
    tally.no_nan("mask", got)
    tally.guards("mask", out, no)
    tally.exact("logits", lb.view(torch.int32), l0.view(torch.int32))
    src = torch.flip(logits, (3,)) if mirror else logits
    cl = closing(src).double()
    yi0, yi1, ly0, ly1 = ac_lambda(h, H)
    xi0, xi1, lx0, lx1 = ac_lambda(w, W)
    ly0, ly1, lx0, lx1 = ly0.view(H, 1), ly1.view(H, 1), lx0.view(1, W), lx1.view(1, W)
    a00, a01 = cl[:, :, yi0][..., xi0], cl[:, :, yi0][..., xi1]
    a10, a11 = cl[:, :, yi1][..., xi0], cl[:, :, yi1][..., xi1]
    z = ly0 * (lx0 * a00 + lx1 * a01) + ly1 * (lx0 * a10 + lx1 * a11)
    E = 5 * U * (ly0 * (lx0 * a00.abs() + lx1 * a01.abs()) + ly1 * (lx0 * a10.abs() + lx1 * a11.abs()))
    if mirror:
        z, E = torch.flip(z, (3,)), torch.flip(E, (3,))
    if math.isnan(thr):
        tally.add(got, z, E + TINY)
        if h == H and w == W:
            tally.exact("closing", got.view(torch.int32), closing(logits).view(torch.int32))
        return tally.result()
    tally.exact("mask values", ((got == 0) | (got == 1)).all().view(1), torch.ones(1, dtype=torch.bool, device=DEV))
    t32 = float(torch.tensor(thr, dtype=torch.float32))
    lt = math.log(t32 / (1 - t32))
    clear = (z - lt).abs() > E + 2.0 ** -19 * (1 + abs(lt))
    tally.exact("mask", got[clear], (z[clear] > lt).float())
    amb = int((~clear).sum())
    log_metric("replay_holemask_ambiguous", cfg=str(r), ambiguous=amb)
    if amb > max(8, no // 1000):
        tally.bad.append(f"{amb} elements within the sigmoid's ambiguity band")
    return tally.result()


def _holemask_synthetic():
    """The copy axes (h = H, w = W), a one-row / one-column output (scale 0), non-integer ratios up and down, each axis alone,
    mirror 0 and 1, threshold NaN and the production 0.15."""
    shapes = [(2, 7, 9, 7, 9), (1, 5, 6, 1, 13), (1, 4, 5, 9, 1), (1, 1, 1, 3, 4), (1, 7, 9, 23, 31), (2, 23, 31, 7, 9),
              (1, 6, 11, 6, 29), (1, 13, 8, 5, 8)]
    t15 = float(torch.tensor(0.15, dtype=torch.float32))
    return [dict(B=B, h=h, w=w, H=H, W=W, mirror=m, threshold=t) for B, h, w, H, W in shapes for m in (0, 1) for t in (math.nan, t15)]


def test_hole_mask_replay(production):
    replay("holemask", configurations(production, "holemask", _holemask_synthetic()), holemask_check)


# ------------------------------------------------------------------------------------------------------------ depth_aa
def aaminmax_check(r, seed):
    """Bit-exact against x.amin() / x.amax(); negative depth, the extremes at the first and the last element."""
    n = r["n"]
    g = _gen(seed)
    xb, mm = guarded32(n), guarded32(2)
    x = body(xb, n)
    x.copy_(torch.randn(n, generator=g, device=DEV) * 2 - 0.5)
    if n > 1:
        x[0], x[-1] = float(x.max()) + 1, float(x.min()) - 1
    _lib.check(_lib.lib().nb200_depth_aa_minmax_f32(ptr(x), n, ptr(body(mm, 2)), _lib.stream_ptr()))
    torch.cuda.synchronize()
    tally = Tally()
    tally.guards("min / max", mm, 2)
    tally.exact("min / max", body(mm, 2).view(torch.int32), torch.stack([x.amin(), x.amax()]).view(torch.int32))
    return tally.result()


def test_depth_aa_minmax_replay(production):
    cases = configurations(production, "aaminmax", [dict(n=n) for n in (1, 5, 1023, 1024, 1025, 3 * 1024 + 7, 33 * 1024 + 1)])
    replay("aaminmax", cases, aaminmax_check)


# data modes of the normalised kinds: a random depth map (negative values included), a constant map (mx = mn: the 0 / 0 -> 0
# branch of nan_to_num) and a random map under min = max = its first value (the +-x / 0 -> +-FLT_MAX branch)
AA_MODES = ("random", "constant", "x/0")


def aa_inputs(r, mode, g):
    """-> x [B][1][H][W] fp32 and the min / max pair the kernel gets (None without normalisation)."""
    B, H, W = r["B"], r["H"], r["W"]
    x = torch.rand(B, 1, H, W, generator=g, device=DEV) * 3 - 1
    if not r["norm"]:
        return torch.rand(B, 1, H, W, generator=g, device=DEV) * 1.4 - 0.2, None   # both sides of the clamp
    if mode == "constant":
        x = torch.full_like(x, 0.37)
    mm = torch.stack([x.amin(), x.amax()]) if mode != "x/0" else x.flatten()[:1].repeat(2)
    return x, mm


def normalised(x, mm):
    """DepthAA.infer's nan_to_num((x - min) / (max - min)) in torch's fp32, as the reference computes it."""
    return x if mm is None else torch.nan_to_num((x - mm[0]) / (mm[1] - mm[0]))


def aaprep_check(r, seed):
    """proj_in of pixel_unshuffle(2) of F.pad(normalised x, (pw1, pw2, ph1, ph2), replicate) (oracle/depth_aa.py:21-23) in
    float64 from torch's fp32 normalised values (the kernel divides with IEEE rounding too; a one-ulp difference there would
    lie within the bound, so this is not a bit-exact check of the division): a 4-term fma chain from the bias, one fp16 rounding,
    E = 5 U (sum|a w| + |b|); beyond fp16's range the tokens must be inf (add16).  Normalised cases run every AA_MODES."""
    B, H, W, ph1, pw1, Hh, Wh, norm = (r[f] for f in ("B", "H", "W", "ph1", "pw1", "Hh", "Wh", "norm"))
    tally = Tally()
    g = _gen(seed)
    for mode in AA_MODES if norm else AA_MODES[:1]:
        x, mm = aa_inputs(r, mode, g)
        # the x / 0 mode's FLT_MAX inputs: weights small enough that no fp32 partial sum overflows
        wt = torch.randn(32, 4, 1, 1, generator=g, device=DEV) * (0.05 if mode == "x/0" else 0.5)
        bias = torch.randn(32, generator=g, device=DEV) * 0.05
        wh, bh = host(wt), host(bias)
        n, no = B * H * W, B * Hh * Wh * 32
        xb, out = guarded32(n), guarded(no)
        body(xb, n).copy_(x.flatten())
        x0 = xb.clone()
        _lib.check(_lib.lib().nb200_depth_aa_prep_f16(ptr(body(xb, n)), ptr(mm), B, H, W, ph1, pw1, Hh, Wh, ptr(wh), ptr(bh),
                                                      ptr(body(out, no)), _lib.stream_ptr()))
        torch.cuda.synchronize()
        got = body(out, no).view(B, Hh, Wh, 32)
        tally.no_nan(f"{mode} tokens", got)
        tally.guards(f"{mode} tokens", out, no)
        tally.exact(f"{mode} x", xb.view(torch.int32), x0.view(torch.int32))
        y = F.pad(normalised(x, mm).double(), (pw1, 2 * Wh - W - pw1, ph1, 2 * Hh - H - ph1), mode="replicate")
        a, s = conv64(F.pixel_unshuffle(y, 2), wt, bias)
        add16(tally, mode, got, a.permute(0, 2, 3, 1), 5 * U * s.permute(0, 2, 3, 1))
    return tally.result()


def _aa_synthetic(kind):
    shapes = [(1, 1, 1), (2, 3, 5), (1, 16, 16), (3, 17, 31), (2, 8, 33), (1, 15, 1)]
    flags = ((0, 0), (0, 1), (1, 0)) if kind == "aaout" else ((0, None), (1, None))
    out = []
    for B, H, W in shapes:
        for norm, clamp in flags:
            d = dict(aa_geom(B, H, W), norm=norm)
            if clamp is not None:
                d["clamp"] = clamp
            out.append(d)
    return out


def test_depth_aa_prep_replay(production):
    cases = configurations(production, "aaprep", _aa_synthetic("aaprep"))
    replay("aaprep", cases, aaprep_check)


def aaout_check(r, seed):
    """proj_out, pixel_shuffle(2), crop and residual (oracle/depth_aa.py:26-30, :38): acc = the float64 1x1 conv of the fp16
    tokens, within E_acc = 33 U (sum|t w| + |b|) (a 32-term fma chain from the bias).  Without normalisation out = fp32(x + acc)
    (+ U |out|), clamped to [0, 1] with clamp; with it out = ((norm + acc) scale) + min in three fp32 roundings, the conv error
    scaled by |scale|: E = |scale| (E_acc + U |norm + acc|) + U |(norm + acc) scale| + U |out|.  scale = 0 (AA_MODES' constant
    and x / 0 maps) must give min exactly.  The tokens whose 2x2 pixels all lie outside the crop window are NaN."""
    B, H, W, ph1, pw1, Hh, Wh, norm, clamp = (r[f] for f in ("B", "H", "W", "ph1", "pw1", "Hh", "Wh", "norm", "clamp"))
    tally = Tally()
    g = _gen(seed)
    nt, n = B * Hh * Wh * 32, B * H * W
    ty, tx = torch.arange(Hh, device=DEV), torch.arange(Wh, device=DEV)
    inside = (((2 * ty + 1 >= ph1) & (2 * ty < ph1 + H)).view(Hh, 1) & ((2 * tx + 1 >= pw1) & (2 * tx < pw1 + W)).view(1, Wh))
    for mode in AA_MODES if norm else AA_MODES[:1]:
        x, mm = aa_inputs(r, mode, g)
        tok = torch.randn(B, Hh, Wh, 32, generator=g, device=DEV)
        tok[:, ~inside] = math.nan
        wt = torch.randn(4, 32, 1, 1, generator=g, device=DEV) * 0.05
        bias = torch.randn(4, generator=g, device=DEV) * 0.01
        wh, bh = host(wt), host(bias)
        tb, xb, out = guarded(nt), guarded32(n), guarded32(n)
        body(tb, nt).copy_(tok.half().flatten())
        body(xb, n).copy_(x.flatten())
        snap = [tb.clone(), xb.clone()]
        _lib.check(_lib.lib().nb200_depth_aa_out_f32(ptr(body(tb, nt)), ptr(body(xb, n)), ptr(mm), B, H, W, ph1, pw1, Hh, Wh, ptr(wh),
                                                     ptr(bh), clamp, ptr(body(out, n)), _lib.stream_ptr()))
        torch.cuda.synchronize()
        got = body(out, n).view(B, 1, H, W)
        tally.no_nan(f"{mode} out", got)
        tally.guards(f"{mode} out", out, n)
        tally.exact(f"{mode} tokens", bits(tb), bits(snap[0]))
        tally.exact(f"{mode} x", xb.view(torch.int32), snap[1].view(torch.int32))
        a, s = conv64(body(tb, nt).view(B, Hh, Wh, 32).permute(0, 3, 1, 2).double(), wt, bias)
        acc, s = (F.pixel_shuffle(t, 2)[..., ph1:ph1 + H, pw1:pw1 + W] for t in (a, s))
        e_acc = 33 * U * s
        if mm is None:
            ref = x.double() + acc
            E = e_acc + U * ref.abs()
            if clamp:
                ref = ref.clamp(0, 1)
        else:
            scale = float(mm[1] - mm[0])
            v = normalised(x, mm).double() + acc
            ref = v * scale + float(mm[0])
            E = abs(scale) * (e_acc + U * v.abs()) + U * (v * scale).abs() + U * ref.abs()
            if scale == 0:
                tally.exact(f"{mode} out = min", got.view(torch.int32), torch.full_like(got, float(mm[0])).view(torch.int32))
                continue
        tally.add(got, ref, E + TINY)
    return tally.result()


def test_depth_aa_out_replay(production):
    cases = configurations(production, "aaout", _aa_synthetic("aaout"))
    assert {(r["norm"], r["clamp"]) for _, r in cases} == {(0, 0), (0, 1), (1, 0)}
    replay("aaout", cases, aaout_check)
