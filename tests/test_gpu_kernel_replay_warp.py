"""GPU: replay every launch of the backward stereo warps (csrc/warp_backward.cu) and of the antialiased depth resize
(nb200_depth_resize_aa) against float64 references.  Most iw3 output pixels come out of this warp: the grid_sample /
backward method with its SBS and dubois epilogues (nb200_backward_warp, and _conv for a per-frame convergence), and the
learned methods' warps (nb200_backward_warp_delta, _f16 for row_flow_v2, _sym for row_flow_v3_sym).

The discipline of tests/test_gpu_kernel_replay.py, with the helpers of tests/replay.py: a module fixture turns on bit 4 of
the launch recorder and records the production flows of WARP_FLOWS, and each unique configuration, plus a synthetic list
for the edges production does not reach, is replayed through the C entry point on fresh seeded data.  A depth-driven
configuration runs on both kernels (the row-staged one and the gather-from-global one that wide rows take) and with every
compose mode; every kind also runs with the colour input and the outputs one float off 16-byte alignment, so that both
kernels take their scalar paths.  Outputs sit between guard blocks whose NaN sentinel must survive, the inputs must keep
their bits, and the recorder confirms the kernel each call took.

The references restate oracle/iw3.py's structure in float64 on the device, never the kernels' arithmetic: make_grid from
torch.linspace, grid + delta * delta_scale, F.interpolate(bilinear, align_corners=True) to the frame, F.grid_sample
(bilinear, border, align_corners=True) and clamp, SBS a cat, dubois oracle.iw3.dubois's formula.  They take the fp32
scalars the upstream code rounds itself (shift, shift_conv, delta_scale, and fp32(shift) * conv[b] for a convergence
tensor).  Each element's bound comes from the kernels' arithmetic, U = 2^-24 being the fp32 unit roundoff (eye_reference,
dubois_reference and aa_axis name each term).
"""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.util import log_metric
from tests.replay import (DEV, GUARD, SENTINEL32, U, WARP_FLOWS, Tally, aa_resize_reference, configurations, guarded32,
                          record_networks, recorded, replay, rounded)
from nunif_b200 import _lib
from nunif_b200._lib import ptr

pytestmark = pytest.mark.gpu
REC_WARP = 16                  # nb200_record_launches bit of the kinds replayed here
TINY = 1e-300                  # bound floor: an exact element has err / bound 0
SECOND_ORDER = 1 + 2.0 ** -20  # the first-order bounds below leave out products of two roundings
# |fp32 linspace(-1, 1, n)[j] - exact|: the step 2 / (n - 1) rounded (U step, j times: at most 2U), the product j * step
# (U |j step| <= 2U) and the sum with -1 or 1 (U), whichever end the evaluation starts from
E_LIN = 5 * U
POWF = 2.0 ** -21              # CUDA powf: 4 ulp (CUDA C++ Programming Guide, single-precision functions), 4 * 2^-23 relative
SMEM_ROW = 200 * 1024          # the row-staged kernel's shared-memory limit (warp_backward.cu)

WARP_KINDS = ("bwarp", "bwdelta", "aaresize")
# the launches of each flow of WARP_FLOWS
EXPECTED = {
    "stereo_sbs_1080p": {"bwarp": 1},
    "stereo_sbs_4k_dubois": {"bwarp": 1},
    "grid_sample_views": {"bwarp": 9},
    "grid_sample_conv_tensor": {"bwarp": 1},
    "row_flow_v3": {"bwdelta": 2},                          # one warp per eye
    "row_flow_v3_steps2": {"bwdelta": 6},                   # per eye: the depth re-warp, then one warp per step
    "row_flow_v2": {"bwdelta": 2},
    "row_flow_v3_sym": {"bwdelta": 2},                      # both eyes in one launch, per view
    "mlbw_l2": {"bwdelta": 4, "aaresize": 2},               # per eye: the layer-weight resize and one warp per layer
    "mlbw_l4": {"bwdelta": 8, "aaresize": 2},
    "mask_mlbw_l2": {"bwdelta": 4, "aaresize": 2},
    "row_flow_v3_stereo_width": {"bwdelta": 2, "aaresize": 1},   # --stereo-width: the depth resized to 1080 x 1920 once
}


@pytest.fixture(scope="module")
def production():
    """name -> every record (kind, config) of each flow of WARP_FLOWS (configurations() deduplicates)."""
    return record_networks(REC_WARP, WARP_FLOWS, unique=False)


def test_every_flow_records_its_launches(production):
    for name, _ in WARP_FLOWS:
        counts = {k: sum(1 for kk, _ in production[name] if kk == k) for k in WARP_KINDS}
        log_metric("replay_warp_launches", model=name, **counts)
        assert {k: n for k, n in counts.items() if n} == EXPECTED[name], name
    recs = lambda name, kind: [r for k, r in production[name] if k == kind]
    assert [(r["compose"], r["B"], r["H"], r["W"], r["h"], r["w"]) for r in recs("stereo_sbs_1080p", "bwarp")] == [(1, 4, 1080, 1920, 392, 686)]
    assert [(r["compose"], r["B"], r["H"], r["W"], r["h"], r["w"]) for r in recs("stereo_sbs_4k_dubois", "bwarp")] == [(2, 2, 2160, 3840, 384, 704)]
    assert sorted({(r["H"], r["W"], r["view"]) for r in recs("grid_sample_views", "bwarp")}) == sorted(
        {(H, W, v) for H, W in ((1080, 1920), (1920, 1080), (240, 320)) for v in (0, 1, 2)})
    assert [(r["B"], r["conv"]) for r in recs("grid_sample_conv_tensor", "bwarp")] == [(4, 1)]
    assert {r["path"] for n, _ in WARP_FLOWS for r in recs(n, "bwarp")} == {0}
    assert {r["mode"] for r in recs("row_flow_v2", "bwdelta")} == {1}
    assert [(r["warp_left"], r["warp_right"]) for r in recs("row_flow_v3_sym", "bwdelta")] == [(1, 1), (1, 0)]
    assert {r["mode"] for n in ("row_flow_v3", "mlbw_l2", "mlbw_l4", "mask_mlbw_l2") for r in recs(n, "bwdelta")} == {0}
    assert [(r["h"], r["w"], r["H"], r["W"]) for r in recs("row_flow_v3_stereo_width", "aaresize")] == [(392, 686, 1080, 1920)]
    assert {(r["H"], r["W"]) for r in recs("row_flow_v3_stereo_width", "bwdelta")} == {(2160, 3840)}


# ------------------------------------------------------------------------------------------------------------ helpers
def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def f32(v):
    """v rounded to fp32 (a recorded value prints 9 significant digits: this recovers the value the kernel got)."""
    return float(torch.tensor(float(v), dtype=torch.float32))


def buf32(n, off):
    """A guarded fp32 buffer whose body of n elements starts `off` elements after the front guard (off = 1: 4-byte aligned
    only, so no kernel may use its 16-byte vector path) -> (buffer, body)."""
    b = guarded32(n + off)
    return b, b[GUARD + off:GUARD + off + n]


def guards(tally, what, b, n, off):
    """Everything outside the body of buf32(n, off) still holds the sentinel."""
    bits = b.view(torch.int32)
    if not (bool((bits[:GUARD + off] == SENTINEL32).all()) and bool((bits[GUARD + off + n:] == SENTINEL32).all())):
        tally.bad.append(f"{what}: guard changed")


def one_launch(tally, kind, call, want, path=None):
    """Run call() under the recorder: one launch of `kind` whose fields include `want` (fp32 values compared as fp32), on
    the kernel path expected."""
    recs = recorded(REC_WARP, call)
    if len(recs) != 1 or recs[0][0] != kind:
        tally.bad.append(f"recorded {recs}, expected one {kind}")
        return
    got = recs[0][1]
    for f, v in want.items():
        if (f32(got[f]) != f32(v)) if isinstance(v, float) else got[f] != v:
            tally.bad.append(f"{kind} recorded {f}={got[f]}, expected {v}")
    if path is not None and got["path"] != path:
        tally.bad.append(f"{kind} took path {got['path']}, expected {path}")


def lin64(n):
    return torch.linspace(-1, 1, n, dtype=torch.float64, device=DEV)


def ac_pos(n_in, n_out):
    """The exact align_corners=True source position of every output index and its tap floor(pos) -> (pos, i0)."""
    s = (n_in - 1) / (n_out - 1) if n_out > 1 else 0.0
    pos = torch.arange(n_out, dtype=torch.float64, device=DEV) * s
    return pos, pos.floor().long().clamp(max=n_in - 1)


def near(m):
    """Max over the 5 x 5 neighbourhood of each depth pixel: the taps a position within a fraction of a pixel of the
    exact one can reach."""
    return F.max_pool2d(m, 5, 1, 2)


# ------------------------------------------------------------------------------------------------------------ warp reference
def eye_reference(c64, d, shift, sc, ds, sign, f16=False):
    """One warped eye of oracle/iw3.py's backward_warp in float64: index_shift = d * shift - sc (sc one value per frame),
    grid x = linspace(-1, 1, w) + sign * index_shift * delta_scale, F.interpolate to the frame (bilinear, align_corners),
    F.grid_sample (bilinear, border, align_corners) at row y, clamp.  f16: the product delta * delta_scale is an fp16
    rounding point (rounded()).  -> (reference [B][3][H][W], bound).

    The bound follows the kernels' arithmetic.  Per depth pixel (grid table t = lx +- fp32(is * ds)):
      E_is   = U |d shift| + U |is|               fp32(d * shift), then - shift_conv, each rounded
      E_prod = |ds| E_is + U |is ds|              the product's rounding (then rounded() in f16 mode)
      E_t    = E_LIN + E_prod + U (|lx| + |prod|) linspace's own error, and the sum's rounding
    Per output pixel, from the 5 x 5 depth neighbourhood of its taps:
      E_grid = E_t + 6 U |t|                      the align-corners blend: two fp32 products and a sum per axis, and
                                                  lx0 = 1 - lx1 / ly0 = 1 - ly1 rounded (mix2_rn)
               + slope_x 2U pos_x + slope_y 2U pos_y   the fp32 scales (h-1)/(H-1), (w-1)/(W-1) (U each) and the products
                                                  sy * y, sx * x (U each) move the source position; the grid is piecewise
                                                  linear in it with the slopes |t[j+1] - t[j]| (|t[i+1] - t[i]|)
      E_ix   = (W-1)/2 E_grid + 2U |ix|           unnormalise: (g + 1) and * (W - 1) rounded; the clamp is 1-Lipschitz
      E_out  = L E_ix + 3U max|c| + E_y           the sample is piecewise linear in ix with slopes |c[k+1] - c[k]|: L the
                                                  largest over the segments within E_ix of ix; the blend's two products,
                                                  its sum and wa = (fx + 1) - ix rounded; E_y = the float64 grid's
                                                  distance from row y times the largest row difference
    The final clamp is 1-Lipschitz."""
    B, _, H, W = c64.shape
    h, w = d.shape[-2:]
    d = d.double()
    sc = sc.double().view(-1, 1, 1, 1)
    lin = lin64(w).view(1, 1, 1, w)
    is_ = d * shift - sc
    e_is = U * ((d * shift).abs() + is_.abs())
    prod = sign * is_ * ds
    e_prod = abs(ds) * e_is + U * prod.abs()
    if f16:
        prod, e_prod = rounded(prod, e_prod)      # round to nearest even is odd-symmetric: the sign commutes with it
    t = lin + prod
    e_t = E_LIN + e_prod + U * (lin.abs() + prod.abs())
    g = F.interpolate(t, size=(H, W), mode="bilinear", align_corners=True)
    posy, i0 = ac_pos(h, H)
    posx, j0 = ac_pos(w, W)
    at = lambda m: near(m)[:, :, i0][:, :, :, j0]
    dx = F.pad((t[..., 1:] - t[..., :-1]).abs(), (0, 1))
    dy = F.pad((t[:, :, 1:] - t[:, :, :-1]).abs(), (0, 0, 0, 1))
    e_grid = (at(e_t) + 6 * U * at(t.abs()) + at(dx) * (2 * U * posx.view(1, 1, 1, W)) + at(dy) * (2 * U * posy.view(1, 1, H, 1)))
    del dx, dy
    ixu = (g + 1) * 0.5 * (W - 1)
    e_ix = (W - 1) / 2 * e_grid + 2 * U * ixu.abs()
    ix = ixu.clamp(0, W - 1)
    gy = lin64(H).view(1, H, 1, 1).expand(B, H, W, 1)
    out = F.grid_sample(c64, torch.cat([g.permute(0, 2, 3, 1), gy], 3), mode="bilinear", padding_mode="border",
                        align_corners=True).clamp(0, 1)
    cmax = float(c64.abs().max())
    e_y = ((lin64(H) + 1) * 0.5 * (H - 1) - torch.arange(H, device=DEV)).abs().view(1, 1, H, 1) * 2 * cmax
    if W > 1:
        seg = (c64[..., 1:] - c64[..., :-1]).abs()
        klo = (ix - e_ix).floor().clamp(0, W - 2).long().expand(B, 3, H, W)
        khi = (ix + e_ix).floor().clamp(0, W - 2).long().expand(B, 3, H, W)
        L = torch.maximum(seg.gather(3, klo), seg.gather(3, khi))
        L = torch.where(khi - klo > 1, seg.amax(3, keepdim=True), L)
        del seg
    else:
        L = torch.zeros_like(c64)
    bound = SECOND_ORDER * (L * e_ix + 3 * U * cmax + e_y)
    return out, bound


LM = ((0.437, 0.449, 0.164), (-0.062, -0.062, -0.024), (-0.048, -0.050, -0.017))
RM = ((-0.011, -0.032, -0.007), (0.377, 0.761, 0.009), (-0.026, -0.093, 1.234))
T1, T2 = 0.04045, 0.0031308    # the sRGB transfer's breakpoints (iw3/anaglyph.py)
# the transfer's gap at each breakpoint (the two branches differ by this much there), and how far the kernel's fp32
# breakpoints lie from them: an input within that distance plus its error may take the other branch
J1 = abs(T1 / 12.92 - ((T1 + 0.055) / 1.055) ** 2.4)
J2 = abs(T2 * 12.92 - (1.055 * T2 ** (1 / 2.4) - 0.055))
D1, D2 = abs(f32(T1) - T1), abs(f32(T2) - T2)


def to_linear(x):
    return torch.where(x <= T1, x / 12.92, ((x + 0.055) / 1.055) ** 2.4)


def to_srgb(x):
    return torch.where(x <= T2, x * 12.92, 1.055 * x ** (1 / 2.4) - 0.055)


def dubois_reference(l, r, el, er):
    """oracle.iw3.dubois (clip_before=True) in float64 on eyes l, r within el, er -> (reference, bound).  Per term:
      to_linear: its largest slope on [.., max input] (2.4 / 1.055 ((x + 0.055) / 1.055)^1.4 at the largest x) times the
        input's error; powf's 4 ulp plus 2.4 times the argument's four roundings (x + 0.055f, / 1.055f, both constants) and
        one, relative; the gap J1 where the input is within its error (and the fp32 breakpoint's offset) of T1
      the 3-term dot products: |m| times those, plus 5U sum |m L| (the fp32 constants, two products and two sums)
      the sum a + b after the clamps: U |a + b|
      to_srgb on the clamped sum: its largest slope on [0, 1] (12.92, the linear branch; the power branch's is 12.70 at
        T2) times that; 1.055 P (powf's 4 ulp, fp32(1 / 2.4)'s exponent error times |ln x| <= 5.8, 1.055f and the
        product: 7U) with P <= 1, and 2U for - 0.055f and its rounding; the gap J2 near T2.
    The clamps are 1-Lipschitz."""
    xmax = max(float(l.max()), float(r.max()), 1.0)
    k1 = 2.4 / 1.055 * ((xmax + 0.055) / 1.055) ** 1.4

    def linear(x, e):
        y = to_linear(x)
        return y, k1 * e + (POWF + 10 * U) * y.abs() + torch.where((x - T1).abs() <= e + D1, J1, 0.0)
    L, EL = linear(l, el)
    R, ER = linear(r, er)
    out, bound = [], []
    for k in range(3):
        a = sum(LM[k][m] * L[:, m] for m in range(3))
        ea = sum(abs(LM[k][m]) * (EL[:, m] + 5 * U * L[:, m].abs()) for m in range(3))
        b = sum(RM[k][m] * R[:, m] for m in range(3))
        eb = sum(abs(RM[k][m]) * (ER[:, m] + 5 * U * R[:, m].abs()) for m in range(3))
        s = (a.clamp(0, 1) + b.clamp(0, 1))
        es = ea + eb + U * s.abs()
        s = s.clamp(0, 1)
        out.append(to_srgb(s).clamp(0, 1))
        bound.append(12.92 * es + 1.055 * (POWF + 7 * U) + 2 * U + torch.where((s - T2).abs() <= es + D2, J2, 0.0))
    return torch.stack(out, 1), SECOND_ORDER * torch.stack(bound, 1)


# ------------------------------------------------------------------------------------------------------------ bwarp
_cache = {}


def cached(seed, make):
    """The inputs and references of one configuration, shared by its variants (replay() runs them one after another)."""
    if seed not in _cache:
        _cache.clear()
        _cache[seed] = make()
    return _cache[seed]


def bwarp_data(r, seed):
    """Seeded inputs (colour in [-0.1, 1.1] and depth in [-0.25, 1.25]: both sides of every clamp, and depth beyond [0, 1]
    as nb200_backward_warp accepts; per-frame convergence in [-0.5, 1]) and the float64 eyes with their bounds (an eye the
    view does not warp is c itself, bound 0)."""
    B, H, W, h, w, view = (r[f] for f in ("B", "H", "W", "h", "w", "view"))
    g = _gen(seed)
    c = torch.rand(B, 3, H, W, generator=g, device=DEV) * 1.2 - 0.1
    depth = torch.rand(B, 1, h, w, generator=g, device=DEV) * 1.5 - 0.25
    conv = torch.rand(B, generator=g, device=DEV) * 1.5 - 0.5
    shift, ds = f32(r["shift"]), f32(r["delta_scale"])
    # the convergence tensor's product is the fp32 tensor op fp32(shift) * conv[b]
    sc = (torch.tensor(shift, dtype=torch.float32, device=DEV) * conv) if r["conv"] else torch.full((B,), f32(r["shift_conv"]), device=DEV)
    c64 = c.double()
    zero = torch.zeros_like(c64)
    left = eye_reference(c64, depth, shift, sc, ds, -1) if view != 2 else (c64, zero)
    right = eye_reference(c64, depth, shift, sc, ds, 1) if view != 1 else (c64, zero)
    return dict(c=c, depth=depth, conv=conv, left=left, right=right)


def bwarp_check(r, seed, variant):
    """nb200_backward_warp (or _conv) on the kernel, alignment and compose mode of `variant` = 100 gather + 10 offset +
    compose: gather forces the gather-from-global kernel (tuning knob 3), offset puts c and the outputs one float off
    16-byte alignment.  Compose 0 checks both eyes, 1 the SBS frame (cat), 2 the dubois anaglyph (dubois_reference)."""
    B, H, W, h, w, view = (r[f] for f in ("B", "H", "W", "h", "w", "view"))
    gather, off, compose = variant // 100, variant // 10 % 10, variant % 10
    data = cached(seed, lambda: bwarp_data(r, seed))
    if compose == 2 and "dubois" not in data:
        (lr, le), (rr, re) = data["left"], data["right"]
        data["dubois"] = dubois_reference(lr, rr, le, re)
    tally = Tally()
    n = B * 3 * H * W
    cb, c = buf32(n, off)
    c.copy_(data["c"].flatten())
    db, d = buf32(B * h * w, 0)
    d.copy_(data["depth"].flatten())
    vb, v = buf32(B, 0)
    v.copy_(data["conv"])
    snap = [cb.clone(), db.clone(), vb.clone()]
    no = 2 * n if compose == 1 else n
    lb, left = buf32(no, off)
    rb, right = buf32(n, off) if compose == 0 else (None, None)
    shift = f32(r["shift"])
    divergence = shift / 0.01 / (1 if view == 0 else 2)
    shift_d = divergence * (1 if view == 0 else 2) * 0.01     # the host's double shift_size, as backward_warp() computes it
    convergence = f32(r["shift_conv"]) / shift_d if shift_d else 0.0
    lib = _lib.lib()
    smem = 16 * (w + 1) + 12 * ((W + 4) & ~3)
    path = 1 if gather or smem > SMEM_ROW else 0
    want = dict(B=B, H=H, W=W, h=h, w=w, view=view, compose=compose, conv=r["conv"], shift=shift,
                shift_conv=0.0 if r["conv"] else f32(r["shift_conv"]), delta_scale=f32(r["delta_scale"]))

    def call():
        rp = ptr(right) if right is not None else None
        if r["conv"]:
            _lib.check(lib.nb200_backward_warp_conv(ptr(c), ptr(d), B, H, W, h, w, divergence, ptr(v), view, compose, ptr(left), rp,
                                                    _lib.stream_ptr()))
        else:
            _lib.check(lib.nb200_backward_warp(ptr(c), ptr(d), B, H, W, h, w, divergence, convergence, view, compose, ptr(left), rp,
                                               _lib.stream_ptr()))
    lib.nb200_tune_set(3, gather)
    try:
        one_launch(tally, "bwarp", call, want, path)
    finally:
        lib.nb200_tune_set(3, 0)
    for what, b, s in (("c", cb, snap[0]), ("depth", db, snap[1]), ("convergence", vb, snap[2])):
        tally.exact(what, b.view(torch.int32), s.view(torch.int32))
    guards(tally, "left", lb, no, off)
    tally.no_nan("left", left)
    (lr, le), (rr, re) = data["left"], data["right"]
    if compose == 0:
        guards(tally, "right", rb, n, off)
        tally.no_nan("right", right)
        tally.add(left.view(B, 3, H, W), lr, le + TINY)
        tally.add(right.view(B, 3, H, W), rr, re + TINY)
    elif compose == 1:
        tally.add(left.view(B, 3, H, 2 * W), torch.cat([lr, rr], 3), torch.cat([le, re], 3) + TINY)
    else:
        ref, bound = data["dubois"]
        tally.add(left.view(B, 3, H, W), ref, bound + TINY)
    return tally.result()


def _bwarp(B, H, W, h, w, view=0, conv=0, shift=0.02, convergence=0.5):
    """A synthetic configuration: the fp32 scalars the host computes for divergence = 100 shift (twice for one view)."""
    s = f32(shift * (1 if view == 0 else 2))
    return dict(B=B, H=H, W=W, h=h, w=w, view=view, compose=0, conv=conv, shift=s, shift_conv=0.0 if conv else f32(s * convergence),
                delta_scale=f32(max(h, w) / w))


def _bwarp_synthetic():
    out = [_bwarp(1, 7, 9, 5, 1)]                                                     # one depth column: linspace(-1, 1, 1) = [-1]
    out += [_bwarp(1, H, W, h, w) for H in (1, 2) for W in (1, 2) for h in (1, 2) for w in (1, 2)]
    out += [_bwarp(1, 5, 13, 3, 7), _bwarp(2, 6, 14, 4, 5), _bwarp(1, 4, 15, 4, 6)]  # W % 4 = 1, 2, 3
    out += [_bwarp(1, 8, 64, 8, 64), _bwarp(1, 6, 33, 6, 33)]                         # full-resolution depth
    out += [_bwarp(1, 9, 11, 23, 31)]                                                 # depth larger than the frame
    out += [_bwarp(1, 3, 7312, 3, 7312), _bwarp(1, 3, 7313, 3, 7313)]                 # either side of the 200 KB row
    out += [_bwarp(1, 16, 40, 9, 21, shift=1.0)]                                      # clamps at both borders
    out += [_bwarp(1, 12, 50, 7, 19, convergence=-0.5)]                               # negative convergence
    out += [_bwarp(3, 12, 50, 7, 19, conv=1), _bwarp(2, 5, 30, 9, 17, view=1, conv=1)]   # per-frame convergence
    out += [_bwarp(2, 10, 24, 6, 13, view=1), _bwarp(2, 10, 24, 6, 13, view=2)]
    # the three shapes the row-staged / gather agreement test covered (divergence 3, convergence 0.4)
    out += [_bwarp(2, H, W, h, w, shift=0.03, convergence=0.4) for H, W, h, w in ((270, 480, 98, 170), (37, 101, 37, 101), (64, 258, 20, 33))]
    return out


BWARP_VARIANTS = tuple(100 * g + 10 * o + k for g in (0, 1) for o in (0, 1) for k in (0, 1, 2))


def test_backward_warp_replay(production):
    cases = configurations(production, "bwarp", _bwarp_synthetic())
    replay("bwarp", cases, bwarp_check, variant=("gather_offset_compose", BWARP_VARIANTS))
    _cache.clear()


# ------------------------------------------------------------------------------------------------------------ bwdelta
MODES = ("nb200_backward_warp_delta", "nb200_backward_warp_delta_f16", "nb200_backward_warp_delta_sym")


def bwdelta_data(r, seed):
    """Seeded colour in [-0.1, 1.1] and a delta whose grid offset delta * delta_scale spans +-0.15 (fp16 values in mode
    1), and the float64 references: mode 0 / 1 the "+" warp of the one output; mode 2 left = grid + delta * delta_scale,
    right = grid - delta * delta_scale, an eye not warped being c itself (bound 0)."""
    B, H, W, h, w, mode = (r[f] for f in ("B", "H", "W", "h", "w", "mode"))
    g = _gen(seed)
    ds = f32(r["delta_scale"])
    c = torch.rand(B, 3, H, W, generator=g, device=DEV) * 1.2 - 0.1
    delta = (torch.rand(B, 1, h, w, generator=g, device=DEV) * 2 - 1) * (0.15 / ds)
    if mode == 1:
        delta = delta.half().float()
    c64 = c.double()
    zero = torch.zeros(B, device=DEV)
    if mode < 2:
        return dict(c=c, delta=delta, outs=[eye_reference(c64, delta, 1.0, zero, ds, 1, f16=mode == 1)])
    left = eye_reference(c64, delta, -1.0, zero, ds, -1) if r["warp_left"] else (c64, torch.zeros_like(c64))
    right = eye_reference(c64, delta, -1.0, zero, ds, 1) if r["warp_right"] else (c64, torch.zeros_like(c64))
    return dict(c=c, delta=delta, outs=[left, right])


def bwdelta_check(r, seed, off):
    B, H, W, h, w, mode = (r[f] for f in ("B", "H", "W", "h", "w", "mode"))
    data = cached(seed, lambda: bwdelta_data(r, seed))
    tally = Tally()
    n = B * 3 * H * W
    cb, c = buf32(n, off)
    c.copy_(data["c"].flatten())
    db, d = buf32(B * h * w, 0)
    d.copy_(data["delta"].flatten())
    snap = [cb.clone(), db.clone()]
    outs = [buf32(n, off) for _ in data["outs"]]
    fn = getattr(_lib.lib(), MODES[mode])
    ds = f32(r["delta_scale"])
    want = {f: r[f] for f in ("B", "H", "W", "h", "w", "mode", "warp_left", "warp_right")}
    want["delta_scale"] = ds
    if mode < 2:
        call = lambda: _lib.check(fn(ptr(c), ptr(d), B, H, W, h, w, ds, ptr(outs[0][1]), _lib.stream_ptr()))
    else:
        call = lambda: _lib.check(fn(ptr(c), ptr(d), B, H, W, h, w, ds, r["warp_left"], r["warp_right"], ptr(outs[0][1]),
                                     ptr(outs[1][1]), _lib.stream_ptr()))
    one_launch(tally, "bwdelta", call, want)
    tally.exact("c", cb.view(torch.int32), snap[0].view(torch.int32))
    tally.exact("delta", db.view(torch.int32), snap[1].view(torch.int32))
    for k, ((b, got), (ref, bound)) in enumerate(zip(outs, data["outs"])):
        guards(tally, f"out {k}", b, n, off)
        tally.no_nan(f"out {k}", got)
        tally.add(got.view(B, 3, H, W), ref, bound + TINY)
    return tally.result()


def _bwdelta(B, H, W, h, w, mode=0, wl=None, wr=1):
    """A synthetic configuration with the drivers' delta_scale 1 / (w // 2 - 1) (0.5 where that is not positive), fp16 in
    mode 1; wl defaults to 0 for the one-output modes and 1 for mode 2."""
    ds = 1.0 / (w // 2 - 1) if w // 2 > 1 else 0.5
    ds = float(torch.tensor(ds).half()) if mode == 1 else f32(ds)
    return dict(B=B, H=H, W=W, h=h, w=w, mode=mode, warp_left=(1 if mode == 2 else 0) if wl is None else wl,
                warp_right=wr if mode == 2 else 1, delta_scale=ds)


def _bwdelta_synthetic():
    out = [_bwdelta(1, 7, 9, 5, 1, m) for m in (0, 1, 2)]                                # one delta column
    out += [_bwdelta(1, H, W, h, w) for H in (1, 2) for W in (1, 2) for h in (1, 2) for w in (1, 2)]
    out += [_bwdelta(1, 5, 13, 3, 7, m) for m in (0, 1, 2)] + [_bwdelta(2, 6, 14, 4, 5), _bwdelta(1, 4, 15, 4, 6, 1)]
    out += [_bwdelta(1, 8, 64, 8, 64, m) for m in (0, 1, 2)]                             # full-resolution delta
    out += [_bwdelta(1, 9, 11, 23, 31, m) for m in (0, 1, 2)]                            # delta larger than the frame
    out += [_bwdelta(1, 2, 7312, 2, 7312, m) for m in (0, 1, 2)]                         # the widest row the kernel takes
    out += [_bwdelta(2, 10, 24, 6, 13, 2, 1, 0), _bwdelta(2, 10, 24, 6, 13, 2, 0, 1), _bwdelta(3, 12, 50, 7, 19, 1)]
    return out


def test_backward_warp_delta_replay(production):
    cases = configurations(production, "bwdelta", _bwdelta_synthetic())
    assert {r["mode"] for _, r in cases} == {0, 1, 2}
    replay("bwdelta", cases, bwdelta_check, variant=("offset", (0, 1)))
    _cache.clear()


# ------------------------------------------------------------------------------------------------------------ aaresize
def aaresize_check(r, seed, off):
    """F.interpolate(depth, (H, W), bilinear, align_corners=True, antialias=True) in float64, on depth in [-0.25, 1.25],
    within aa_resize_reference's bound."""
    B, h, w, H, W = (r[f] for f in ("B", "h", "w", "H", "W"))
    g = _gen(seed)
    tally = Tally()
    n, no = B * h * w, B * H * W
    xb, x = buf32(n, off)
    x.copy_(torch.rand(n, generator=g, device=DEV) * 1.5 - 0.25)
    x0 = xb.clone()
    ob, out = buf32(no, off)
    one_launch(tally, "aaresize", lambda: _lib.check(_lib.lib().nb200_depth_resize_aa(ptr(x), B, h, w, H, W, ptr(out), _lib.stream_ptr())),
               dict(B=B, h=h, w=w, H=H, W=W))
    tally.exact("depth", xb.view(torch.int32), x0.view(torch.int32))
    guards(tally, "out", ob, no, off)
    tally.no_nan("out", out)
    ref, bound = aa_resize_reference(x.view(B, 1, h, w).double(), H, W)
    tally.add(out.view(B, 1, H, W), ref, SECOND_ORDER * bound + TINY)
    return tally.result()


def _aaresize_synthetic():
    out = [dict(B=1, h=h, w=w, H=H, W=W) for h in (1, 2) for w in (1, 2) for H in (1, 2) for W in (1, 2)]
    out += [dict(B=B, h=h, w=w, H=H, W=W) for B, h, w, H, W in (
        (2, 7, 9, 23, 31),       # upsampling, odd ratios
        (1, 23, 31, 7, 9),       # downsampling
        (1, 6, 40, 17, 11),      # one axis up, the other down
        (1, 64, 200, 5, 13),     # downsampling by a large factor (wide tap windows)
        (1, 8, 9, 8, 9),         # the same size
        (8, 5, 7, 11, 13),       # B * L layer-weight planes
        (1, 3, 1, 1, 9))]        # one column up to nine, three rows down to one
    return out


def test_depth_resize_aa_replay(production):
    cases = configurations(production, "aaresize", _aaresize_synthetic())
    replay("aaresize", cases, aaresize_check, variant=("offset", (0, 1)))
