"""GPU: replay every launch that the engine's networks make of the hand-written convolutions outside the wgmma GEMM, at the
production shapes, against float64 references: the first 3x3 conv of every waifu2x model (stem_conv_mma_kernel), the CUNet /
UpCUNet tails (tail_conv_mma_kernel), the UpConv7 / VGG7 output heads (head_conv_mma_kernel), the SE block, SwinUNet's
to_image (pixel shuffle and the bicubic-antialias 2x / 1x views) and every REBNCONV of iw3.sod_v1 (sod_conv_kernel).

The discipline of tests/test_gpu_kernel_replay.py and tests/test_gpu_kernel_replay_aux.py, with the helpers of tests/replay.py:
a module fixture turns on bit 2 of the launch recorder and records one forward of each waifu2x network of MODELS (tile 256, batch 16),
of swin_unet_4x.to_1x() and of SODV1.infer at B = 4 and B = 1; small forwards at other tiles and batches, and a synthetic list,
add the edges production does not reach.  Each unique configuration is replayed through the kernel's test entry point on fresh
seeded data, once on the production path and, for the stem / tail / head, once on their SIMT kernels (nb200_tune_set(7, 1));
the recorder confirms which kernel ran.  Weights are passed in the PyTorch layout and packed by the networks' own packers, so
the fp16 fragment order is under test as well.

Inputs outside the view a launch reads are NaN: a SOD input's channels outside its slice, the pad channels of to_image's
input, z1's channels 3..7 and the pixels outside its 20-pixel crop.  The one exception is the stem's NHWC8 input: its
mma.sync multiplies channel 3 by a zero weight, so channel 3 must hold 0 (what the tile unfold writes), while channels 4..7
are never read and hold NaN.  Every output buffer sits between guard blocks holding a sentinel bit pattern (a NaN) that must
survive bit for bit, as must the output channels a launch does not own (a SOD output slice, the stem's channels past
cout_pad).  Each output element is checked against a float64 reference written from the reference networks' semantics
(Conv2d / ConvTranspose2d with the fp16-rounded weights the packers make, the SE block of nunif/modules/attention.py, ATen's
upsample_bicubic2d_aa, the REBNCONV under autocast) within a bound derived from the kernel's arithmetic, stated in each check's
docstring (U = 2^-24 is the fp32 unit roundoff).
"""
import time

import pytest
import torch
import torch.nn.functional as F

from tests.util import log_metric
from tests.replay import (DEV, MODELS, SENTINEL, Tally, _gen, bits, body, configurations, guarded, guarded32, guards_ok,
                          record_networks, recorded, replay, round16_bound, rounded, swin_sd, waifu2x)
from nunif_b200 import _lib, synth
from nunif_b200._lib import ptr

pytestmark = pytest.mark.gpu
U = 2.0 ** -24                 # fp32 unit roundoff
REC_CONV = 4                   # nb200_record_launches bit of the kinds replayed here
ACC = 2.0 ** -20               # per chained mma.sync k-step: |fp32 accumulator - exact| <= ACC * L * sum |a w|

CONV_KINDS = ("stem", "tail", "head", "se", "toimg", "sodconv")
WAIFU2X = ("swin_unet_4x", "swin_unet_4x.to_2x", "swin_unet_2x", "swin_unet_1x", "upcunet", "cunet", "upconv_7", "vgg_7")
SOD_CONVS = 112                # REBNCONVs per SODV1 forward (csrc/sod_kernels.h sod_layer_list)
T0 = None                      # start of the module's recording fixture


# ------------------------------------------------------------------------------------------------------------ networks
def _sod(B):
    def run():
        from nunif_b200.iw3 import SODV1
        rgb = torch.rand(B, 3, 1080, 1920, generator=_gen(12)).to(DEV)
        depth = torch.rand(B, 1, 392, 686, generator=_gen(13)).to(DEV)
        SODV1(synth.sod_v1_state_dict(0), DEV).infer(rgb, depth)
    return run


_NETS = dict(MODELS)
CONV_MODELS = [(n, _NETS[n]) for n in WAIFU2X] + [
    ("swin_unet_4x.to_1x", waifu2x("waifu2x.swin_unet_4x", swin_sd(4), view="to_1x", seed=11)),   # down 4: no network of MODELS
    ("sod_v1_b4", _sod(4)),    # iw3 --convergence-mode sod_v1 on the iw3_1080p batch: 4 frames, 392 x 686 depth
    ("sod_v1_b1", _sod(1)),
]
# other tiles and batches: Swin / CUNet / UpCUNet at tile 64, the legacy models at tiles 15 (head output of 1 or 2 rows), 61
# and 104, batches 1 and 3
EDGE_MODELS = [
    ("swin_unet_4x T64 n3", waifu2x("waifu2x.swin_unet_4x", swin_sd(4), 64, 3, seed=11)),
    ("swin_unet_4x.to_2x T64 n1", waifu2x("waifu2x.swin_unet_4x", swin_sd(4), 64, 1, "to_2x", 11)),
    ("swin_unet_4x.to_1x T64 n3", waifu2x("waifu2x.swin_unet_4x", swin_sd(4), 64, 3, "to_1x", 11)),
    ("swin_unet_2x T64 n1", waifu2x("waifu2x.swin_unet_2x", swin_sd(2), 64, 1, seed=11)),
    ("swin_unet_1x T64 n3", waifu2x("waifu2x.swin_unet_1x", swin_sd(1), 64, 3, seed=11)),
    ("cunet T64 n3", waifu2x("waifu2x.cunet", synth.cunet_state_dict, 64, 3, seed=11)),
    ("cunet T64 n1", waifu2x("waifu2x.cunet", synth.cunet_state_dict, 64, 1, seed=11)),
    ("upcunet T64 n1", waifu2x("waifu2x.upcunet", synth.upcunet_state_dict, 64, 1, seed=11)),
    ("upcunet T64 n3", waifu2x("waifu2x.upcunet", synth.upcunet_state_dict, 64, 3, seed=11)),
] + [(f"{m} T{T} n{n}", waifu2x(f"waifu2x.{m}", sd, T, n, seed=11))
     for m, sd in (("upconv_7", synth.upconv7_state_dict), ("vgg_7", synth.vgg7_state_dict)) for T, n in ((15, 3), (61, 1), (104, 3))]


@pytest.fixture(scope="module")
def production():
    """name -> [(kind, config)] of every recorded launch (not deduplicated: the coverage test counts them), for the networks
    of CONV_MODELS and EDGE_MODELS."""
    global T0
    T0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    return record_networks(REC_CONV, CONV_MODELS + EDGE_MODELS, unique=False)


def test_every_network_records_its_launches(production):
    lines = []
    for name in production:
        counts = {k: sum(1 for kk, _ in production[name] if kk == k) for k in CONV_KINDS}
        lines.append(f"{name:28s} launches: " + " ".join(f"{k} {n}" for k, n in counts.items() if n))
        log_metric("replay_conv_launches", model=name, **counts)
    print("\n" + "\n".join(lines))
    for name in WAIFU2X + ("swin_unet_4x.to_1x",):
        assert any(k == "stem" for k, _ in production[name]), name
    for name in ("sod_v1_b4", "sod_v1_b1"):
        assert sum(1 for k, _ in production[name] if k == "sodconv") == SOD_CONVS, name
    # production runs every recorded kernel on its mma.sync path
    assert all(r["path"] == 0 for recs in production.values() for k, r in recs if "path" in r)


# ------------------------------------------------------------------------------------------------------------ helpers
def host(t):
    return t.detach().float().cpu().contiguous()


def nchw64(x):
    return x.double().permute(0, 3, 1, 2)


def conv64(x, w, b=None, transposed=False, dil=1, pad=0):
    """x NHWC (fp16 values), w float64 in the PyTorch layout -> NHWC float64 (conv + b, conv(|x|, |w|) + |b|)."""
    def f(a, ww):
        if transposed:
            return F.conv_transpose2d(a, ww, stride=2, padding=3)
        return F.conv2d(a, ww, dilation=dil, padding=pad)
    xd = nchw64(x)
    y, s = f(xd, w), f(xd.abs(), w.abs())
    if b is not None:
        y, s = y + b.view(1, -1, 1, 1), s + b.abs().view(1, -1, 1, 1)
    return y.permute(0, 2, 3, 1), s.permute(0, 2, 3, 1)


def h64(w):
    """Weights as the packers store them: rounded to fp16, in float64 on the device."""
    return w.half().double().to(DEV)


def leaky64(v):
    return torch.where(v > 0, v, 0.1 * v)


def path_check(tally, kind, fn, path):
    """Launch fn() under the recorder: exactly one launch of `kind`, on the kernel path expected."""
    got = [r["path"] for k, r in recorded(REC_CONV, fn) if k == kind]
    if got != [path]:
        tally.bad.append(f"{kind}: recorded paths {got}, expected [{path}]")


def on_path(check):
    """check(r, seed, path) with the stem / tail / head kernel knob set for the call (nb200_tune_set(7, path): 0 mma.sync,
    1 SIMT)."""
    def run(r, seed, path):
        lib = _lib.lib()
        _lib.check(lib.nb200_tune_set(7, path))
        try:
            return check(r, seed, path)
        finally:
            lib.nb200_tune_set(7, 0)
    return run


# ------------------------------------------------------------------------------------------------------------ stem
SYNTH_STEM = [dict(n=2, Hi=67, Wi=67, cout_pad=64, ldo=72, path=0),     # partial row pair, a 1-column last block, ldo > cout_pad
              dict(n=1, Hi=9, Wi=130, cout_pad=32, ldo=40, path=0)]


def stem_check(r, seed, path):
    """out = fp16(LeakyReLU(conv3x3(x[..., :3]) + b)) for channels < cout, exactly +0 for cout..cout_pad-1 (UpConv7's 16 of 32),
    sentinel for cout_pad..ldo-1.  K = 36 in L = 3 chained k16 steps (the SIMT kernel's 27 fp32 FMAs are within the same
    bound): the pre-activation is within E = ACC L sum|x w| + 2^-22 (|z| + |b|) (bias add, LeakyReLU product), then one fp16
    rounding.  Run with cout = cout_pad and, at cout_pad 32, with UpConv7's cout = 16."""
    n, Hi, Wi, cp, ldo = (r[f] for f in ("n", "Hi", "Wi", "cout_pad", "ldo"))
    Ho, Wo = Hi - 2, Wi - 2
    ni, no = n * Hi * Wi * 8, n * Ho * Wo * ldo
    tally = Tally()
    for cout in (cp, 16) if cp == 32 else (cp,):
        g = torch.Generator(device=DEV).manual_seed(seed + cout)
        xb, out = guarded(ni), guarded(no)
        x = body(xb, ni).view(n, Hi, Wi, 8)
        x[..., :3] = (torch.rand(n, Hi, Wi, 3, generator=g, device=DEV) * 1.4 - 0.2).half()
        x[..., 3] = 0.0
        x0 = xb.clone()
        w = torch.randn(cout, 3, 3, 3, generator=g, device=DEV) * 0.4
        b = torch.randn(cout, generator=g, device=DEV) * 0.3
        wh, bh = host(w), host(b)
        path_check(tally, "stem", lambda: _lib.check(_lib.lib().nb200_stem_conv_f16(
            ptr(body(xb, ni)), ptr(wh), ptr(bh), cout, cp, n, Hi, Wi, ptr(body(out, no)), ldo, _lib.stream_ptr())), path)
        tally.exact("input", bits(xb), bits(x0))
        tally.guards("output", out, no)
        got = body(out, no).view(n, Ho, Wo, ldo)
        tally.no_nan("output", got[..., :cp])
        tally.exact("padded channels", bits(got[..., cout:cp]), torch.zeros_like(bits(got[..., cout:cp])))
        tally.exact("channels past cout_pad", bits(got[..., cp:]), torch.full_like(bits(got[..., cp:]), SENTINEL))
        w64 = h64(w)
        for i in range(n):
            z, s = conv64(x[i:i + 1, ..., :3], w64, b.double())
            E = ACC * 3 * s + 2.0 ** -22 * (z.abs() + b.double().abs())
            y = leaky64(z)
            tally.add(got[i:i + 1, ..., :cout], y, round16_bound(y, E))
    return tally.result()


def test_stem_replay(production):
    cases = configurations(production, "stem", SYNTH_STEM)
    assert {r["cout_pad"] for _, r in cases} == {32, 64}
    replay("stem", cases, on_path(stem_check), variant=("path", (0, 1)))


# ------------------------------------------------------------------------------------------------------------ tail
def tail_check(r, seed, path):
    """mode 0: Conv2d(64, 3, 3) valid; mode 1: ConvTranspose2d(64, 3, 4, stride 2, padding 3).  The accumulator is within
    E = ACC L sum|x w| + 2^-22 (|z| + |b|) with L = 4 k16 steps per tap x 9 taps (mode 0) or the 4 taps of one output parity
    (mode 1).  epi 0: NHWC8 fp16(clamp(z, 0, 1) if clip else z) in channels 0..2, exactly +0 in 3..7.  epi 1: planar
    fp16(clamp(z + z1[20 + y][20 + x][c], 0, 1)) with one more fp32 rounding (U |z + z1|) before the clamp.  Inputs reach
    beyond [0, 1] so that every clamp acts."""
    mode, epi, n, Hi, Wi, z1H, z1W, clip = (r[f] for f in ("mode", "epi", "n", "Hi", "Wi", "z1H", "z1W", "clip"))
    Ho, Wo = (Hi - 2, Wi - 2) if mode == 0 else (2 * Hi - 4, 2 * Wi - 4)
    taps, L = (9, 36) if mode == 0 else (16, 16)
    g = torch.Generator(device=DEV).manual_seed(seed)
    ni = n * Hi * Wi * 64
    no = n * Ho * Wo * 8 if epi == 0 else n * 3 * Ho * Wo
    xb, out = guarded(ni), guarded(no)
    x = body(xb, ni).view(n, Hi, Wi, 64)
    x.copy_((torch.randn(n, Hi, Wi, 64, generator=g, device=DEV) * 0.5 + 0.1).half())
    wshape = (3, 64, 3, 3) if mode == 0 else (64, 3, 4, 4)
    w = torch.randn(*wshape, generator=g, device=DEV) * (1.2 / (0.5 * (64 * taps) ** 0.5))
    b = 0.5 + 0.2 * torch.randn(3, generator=g, device=DEV)
    z1b, z1 = None, None
    if epi == 1:
        z1b = guarded(n * z1H * z1W * 8)
        z1 = body(z1b, n * z1H * z1W * 8).view(n, z1H, z1W, 8)
        z1[:, 20:20 + Ho, 20:20 + Wo, :3] = (torch.rand(n, Ho, Wo, 3, generator=g, device=DEV) * 1.2 - 0.1).half()
    snap = [t.clone() for t in (xb, z1b) if t is not None]
    wh, bh = host(w), host(b)
    tally = Tally()
    path_check(tally, "tail", lambda: _lib.check(_lib.lib().nb200_tail_conv_f16(
        ptr(body(xb, ni)), ptr(wh), ptr(bh), mode, epi, n, Hi, Wi, ptr(body(out, no)),
        ptr(body(z1b, n * z1H * z1W * 8)) if epi else None, z1H, z1W, clip, _lib.stream_ptr())), path)
    for t, t0 in zip([t for t in (xb, z1b) if t is not None], snap):
        tally.exact("input", bits(t), bits(t0))
    tally.guards("output", out, no)
    got = body(out, no).view(n, Ho, Wo, 8) if epi == 0 else body(out, no).view(n, 3, Ho, Wo).permute(0, 2, 3, 1)
    tally.no_nan("output", got)
    if epi == 0:
        tally.exact("channels 3..7", bits(got[..., 3:].contiguous()), torch.zeros_like(bits(got[..., 3:].contiguous())))
    w64 = h64(w)
    for i in range(n):
        z, s = conv64(x[i:i + 1], w64, b.double(), transposed=mode == 1)
        E = ACC * L * s + 2.0 ** -22 * (z.abs() + b.double().abs())
        if epi == 1:
            z = z + z1[i:i + 1, 20:20 + Ho, 20:20 + Wo, :3].double()
            E = E + U * z.abs()
        y = z.clamp(0, 1) if clip or epi == 1 else z
        tally.add(got[i:i + 1, ..., :3], y, round16_bound(y, E))
    return tally.result()


def test_tail_replay(production):
    cases = configurations(production, "tail", [dict(mode=0, epi=0, n=2, Hi=9, Wi=131, z1H=0, z1W=0, clip=1, path=0),
                                        dict(mode=1, epi=0, n=1, Hi=5, Wi=67, z1H=0, z1W=0, clip=0, path=0)])
    assert {(r["mode"], r["epi"]) for _, r in cases} == {(0, 0), (0, 1), (1, 0)}
    assert {r["clip"] for _, r in cases if r["epi"] == 0} == {0, 1}
    replay("tail", cases, on_path(tail_check), variant=("path", (0, 1)))


# ------------------------------------------------------------------------------------------------------------ head
def head_check(r, seed, path):
    """mode 0: Conv2d(128, 3, 3) valid; mode 1: ConvTranspose2d(256, 3, 4, 2, 3); planar fp16(clamp(z, 0, 1)).  L = 4 k16
    steps per tap x taps per output (9, or 4 of one parity) x CIN / 64 chunks; E = ACC L sum|x w| + 2^-22 (|z| + |b|)."""
    mode, cin, n, Hi, Wi = (r[f] for f in ("mode", "cin", "n", "Hi", "Wi"))
    Ho, Wo = (Hi - 2, Wi - 2) if mode == 0 else (2 * Hi - 4, 2 * Wi - 4)
    L = (9 if mode == 0 else 4) * 4 * cin // 64
    g = torch.Generator(device=DEV).manual_seed(seed)
    ni, no = n * Hi * Wi * cin, n * 3 * Ho * Wo
    xb, out = guarded(ni), guarded(no)
    x = body(xb, ni).view(n, Hi, Wi, cin)
    x.copy_((torch.randn(n, Hi, Wi, cin, generator=g, device=DEV) * 0.5 + 0.1).half())
    x0 = xb.clone()
    taps = 9 if mode == 0 else 16
    w = torch.randn(*((3, cin, 3, 3) if mode == 0 else (cin, 3, 4, 4)), generator=g, device=DEV) * (1.2 / (0.5 * (cin * taps) ** 0.5))
    b = 0.5 + 0.2 * torch.randn(3, generator=g, device=DEV)
    wh, bh = host(w), host(b)
    tally = Tally()
    path_check(tally, "head", lambda: _lib.check(_lib.lib().nb200_head_conv_f16(
        ptr(body(xb, ni)), ptr(wh), ptr(bh), mode, cin, n, Hi, Wi, ptr(body(out, no)), _lib.stream_ptr())), path)
    tally.exact("input", bits(xb), bits(x0))
    tally.guards("output", out, no)
    got = body(out, no).view(n, 3, Ho, Wo).permute(0, 2, 3, 1)
    tally.no_nan("output", got)
    w64 = h64(w)
    for i in range(n):
        z, s = conv64(x[i:i + 1], w64, b.double(), transposed=mode == 1)
        E = ACC * L * s + 2.0 ** -22 * (z.abs() + b.double().abs())
        y = z.clamp(0, 1)
        tally.add(got[i:i + 1], y, round16_bound(y, E))
    return tally.result()


def test_head_replay(production):
    cases = configurations(production, "head")
    assert {(r["mode"], r["cin"]) for _, r in cases} == {(0, 128), (1, 256)}
    assert {r["Hi"] for _, r in cases} >= {3, 49, 92, 244}
    replay("head", cases, on_path(head_check), variant=("path", (0, 1)))


# ------------------------------------------------------------------------------------------------------------ SE
SYNTH_SE = [dict(n=n, H=H, W=W, C=C) for C in (64, 128) for n, H, W in ((3, 7, 9), (1, 32, 64), (3, 3, 683), (1, 122, 122))]


def se_check(r, seed):
    """x *= sigmoid(conv2(relu(conv1(mean_HW x)))) with the 1x1 convs' weights and biases rounded to fp16, in float64.

    First-order bound: a thread sums 2048 / ROWS pixels of its chunk (ROWS = 2048 / C pixel rows per block), the block ROWS
    partials, se_fc the nchunks chunk sums, then one divide: the mean is within e_m = (2048 / ROWS + ROWS + nchunks + 2) U
    mean|x|.  fc1 (C fp32 FMAs from its bias) adds sum|w1| e_m + (C + 1) U (|b1| + sum|w1 m|), ReLU keeps it; fc2 the same
    with R = C / 8; sigmoid's slope s (1 - s) carries that, and __expf's 2^-23 (2 + 1.173 |a|) relative error on e^-a moves
    the sigmoid by (1 - s) s times it (plus 2 U for the add and divide).  The scaled output is one fp32 product (U) and one fp16
    rounding; E = 1.1 |x| e_scale + U |x s|."""
    n, H, W, C = (r[f] for f in ("n", "H", "W", "C"))
    HW, R = H * W, C // 8
    rows = 2048 // C
    nchunks = -(-HW // 2048)
    g = torch.Generator(device=DEV).manual_seed(seed)
    ne = n * HW * C
    xb = guarded(ne)
    x = body(xb, ne).view(n, HW, C)
    x.copy_((torch.randn(n, HW, C, generator=g, device=DEV) + 0.3 * torch.randn(n, 1, C, generator=g, device=DEV)).half())
    x0 = x.clone()
    w1 = torch.randn(R, C, generator=g, device=DEV) * (2.0 / C ** 0.5)
    b1 = torch.randn(R, generator=g, device=DEV) * 0.3
    w2 = torch.randn(C, R, generator=g, device=DEV) * (3.0 / R ** 0.5)
    b2 = torch.randn(C, generator=g, device=DEV) * 0.5
    hs = [host(t) for t in (w1, b1, w2, b2)]
    _lib.check(_lib.lib().nb200_se_block_f16(ptr(body(xb, ne)), *(ptr(t) for t in hs), n, H, W, C, _lib.stream_ptr()))
    torch.cuda.synchronize()
    tally = Tally()
    tally.guards("x", xb, ne)
    got = body(xb, ne).view(n, HW, C)
    tally.no_nan("x", got)
    W1, B1, W2, B2 = (h64(t) for t in (w1, b1, w2, b2))
    X = x0.double()
    m = X.mean(1)                                                    # [n][C]
    e_m = (2048 // rows + rows + nchunks + 2) * U * X.abs().mean(1)
    a1 = m @ W1.t() + B1
    e1 = e_m @ W1.abs().t() + (C + 1) * U * (B1.abs() + m.abs() @ W1.abs().t())
    hid = a1.clamp_min(0)
    a2 = hid @ W2.t() + B2
    e2 = e1 @ W2.abs().t() + (R + 1) * U * (B2.abs() + hid @ W2.abs().t())
    sg = torch.sigmoid(a2)
    e_s = sg * (1 - sg) * (e2 + 2.0 ** -23 * (2 + 1.173 * a2.abs())) + 2 * U * sg
    ref = X * sg[:, None, :]
    E = 1.1 * X.abs() * e_s[:, None, :] + U * ref.abs()
    tally.add(got, ref, round16_bound(ref, E))
    return tally.result()


def test_se_replay(production):
    cases = configurations(production, "se", SYNTH_SE)
    assert {r["C"] for _, r in cases} == {64, 128}
    hw = {r["H"] * r["W"] for _, r in cases}
    assert 14884 in hw and 2048 in hw and 2049 in hw and min(hw) < 2048
    replay("se", cases, se_check)


# ------------------------------------------------------------------------------------------------------------ to_image
SYNTH_TOIMG = [dict(n=2, Hs=21, Ws=21, cs=48, r=4, down=2),     # S = 42: the last 32-wide output tile is partial
               dict(n=1, Hs=21, Ws=21, cs=48, r=4, down=4),     # S = 21: the last 16-wide output tile is partial
               dict(n=3, Hs=5, Ws=5, cs=48, r=4, down=1),
               dict(n=2, Hs=7, Ws=7, cs=16, r=2, down=1), dict(n=1, Hs=9, Ws=9, cs=16, r=1, down=1),
               dict(n=1, Hs=10, Ws=10, cs=16, r=2, down=2)]


def toimg_variant(r):
    if r["r"] == 4 and r["cs"] == 48:
        return {1: "r4", 2: "down2", 4: "down4"}[r["down"]]
    return "generic"


def aa_weights(n_in, scale):
    """ATen upsample_bicubic2d_aa (align_corners=False, A = -0.5) for an integer downscale: -> float64 [n_out][n_in] weights,
    each row renormalised over the taps that fall inside the input."""
    n_out = n_in // scale
    center = scale * (torch.arange(n_out, dtype=torch.float64) + 0.5)
    support = 2.0 * scale
    xmin = (center - support + 0.5).floor().clamp_min(0)
    xmax = (center + support + 0.5).floor().clamp(max=n_in)
    j = torch.arange(n_in, dtype=torch.float64)
    t = ((j[None, :] - center[:, None] + 0.5) / scale).abs()
    a = -0.5
    w = torch.where(t < 1, ((a + 2) * t - (a + 3)) * t * t + 1, torch.where(t < 2, (((t - 5) * t + 8) * t - 4) * a, torch.zeros_like(t)))
    w = torch.where((j[None, :] >= xmin[:, None]) & (j[None, :] < xmax[:, None]), w, torch.zeros_like(w))
    return (w / w.sum(1, keepdim=True)).to(DEV)


def toimg_check(r, seed):
    """down 1: bit-exact against clamp(pixel_shuffle(y), 0, 1) in fp16 (an fp16 value clamped in fp32 is fp16 again).
    down 2 / 4: fp32 against the float64 bicubic-antialias resize of that clamp (aa_weights, horizontal then vertical) and a
    clamp after it.  The tap arguments are exact (a power-of-two scale); the cubic's four or five fp32 roundings of terms below 8
    and the division by the sum t >= 1 put every fp32 tap weight within e_w = 2^-20 of the normalised float64 one.  With inputs
    in [0, 1], NT = 4 down taps and Sx, Sy the sums of |weights|: the horizontal pass is within
    NT (e_w + U Sx), the vertical one E = Sy NT (e_w + U Sx) + NT e_w Sx + NT U Sy Sx.  Channels 3 r^2 .. cs-1 of y are NaN."""
    n, Hs, Ws, cs, rr, down = (r[f] for f in ("n", "Hs", "Ws", "cs", "r", "down"))
    S_full = Hs * rr
    S = S_full // down
    g = torch.Generator(device=DEV).manual_seed(seed)
    ny, nz = n * Hs * Ws * cs, n * 3 * S * S
    yb = guarded(ny)
    y = body(yb, ny).view(n, Hs, Ws, cs)
    y[..., :3 * rr * rr] = (torch.randn(n, Hs, Ws, 3 * rr * rr, generator=g, device=DEV) * 0.6 + 0.5).half()
    y0 = yb.clone()
    if down == 1:
        out = guarded(nz)
        zp = body(out, nz)
    else:
        out = guarded32(nz)
        zp = body(out, nz)
    _lib.check(_lib.lib().nb200_to_image_f16(ptr(body(yb, ny)), n, Hs, Ws, cs, rr, down, ptr(zp), _lib.stream_ptr()))
    torch.cuda.synchronize()
    tally = Tally()
    tally.exact("input", bits(yb), bits(y0))
    tally.guards("output", out, nz)
    img = F.pixel_shuffle(y[..., :3 * rr * rr].permute(0, 3, 1, 2).float(), rr).clamp(0, 1)   # [n][3][S_full][S_full]
    if down == 1:
        tally.exact("image", bits(zp.view(n, 3, S, S)), bits(img.half()))
        return tally.result()
    got = zp.view(n, 3, S, S)
    tally.no_nan("image", got)
    Wt = aa_weights(S_full, down)
    Sa = Wt.abs().sum(1)
    NT = 4 * down
    e_w = 2.0 ** -20
    ref = (Wt @ img.double() @ Wt.t()).clamp(0, 1)
    Sy, Sx = Sa.view(S, 1), Sa.view(1, S)
    E = Sy * NT * (e_w + U * Sx) + NT * e_w * Sx + NT * U * Sy * Sx
    tally.add(got, ref, E.expand_as(ref))
    return tally.result()


def test_to_image_replay(production):
    cases = configurations(production, "toimg", SYNTH_TOIMG)
    assert {toimg_variant(r) for _, r in cases} == {"r4", "down2", "down4", "generic"}
    replay("toimg", cases, toimg_check)


# ------------------------------------------------------------------------------------------------------------ SOD REBNCONV
SOD_PAIRS = ((16, 64), (64, 64), (128, 64), (64, 16), (16, 16), (32, 16), (32, 64))   # (cin_pad, cout) of sod_layer_list


def _sod_cfg(B, H, cin, cout, dil, res):
    return dict(B=B, H=H, W=H, cin=cin, cout=cout, dil=dil, in_ld=cin + 16, in_off=8, out_ld=cout + 8, out_off=6, has_res=res,
                res_ld=cout + 8 if res else 0)


SYNTH_SOD = [_sod_cfg(B, H, cin, cout, 8, res) for H, B in ((6, 3), (12, 1)) for cin, cout in SOD_PAIRS for res in (0, 1)] + \
            [_sod_cfg(2, H, cin, cout, d, 1) for H in (6, 12) for cin, cout in ((64, 64), (16, 16)) for d in (2, 4)]


def sod_check(r, seed):
    """REBNCONV under autocast, with the kernel's rounding points (csrc/sod.cu): a = fp16(conv3x3_dil(x)) (cuDNN's fp16 output),
    fp16(a + bias), ReLU, then + res (fp32) and one fp16 rounding.  The accumulator is within ACC L sum|x w| with
    L = 9 cin / 16 k16 steps; each fp16 rounding point carries forward only the difference that a rounding boundary within the
    bound allows (rounded()); the bias add and the residual add are fp32 (U |v| each).  The input slice sits in a wider buffer
    whose other channels are NaN; the output slice's neighbours keep their sentinel."""
    B, H, W, cin, cout, dil, in_ld, in_off, out_ld, out_off, has_res, res_ld = (
        r[f] for f in ("B", "H", "W", "cin", "cout", "dil", "in_ld", "in_off", "out_ld", "out_off", "has_res", "res_ld"))
    g = torch.Generator(device=DEV).manual_seed(seed)
    npx = B * H * W
    xb, out = guarded(npx * in_ld), guarded(npx * out_ld)
    x = body(xb, npx * in_ld).view(B, H, W, in_ld)[..., in_off:in_off + cin]
    x.copy_((torch.rand(B, H, W, cin, generator=g, device=DEV) * 2.0).half())
    rb = None
    if has_res:
        rb = guarded(npx * res_ld)
        res = body(rb, npx * res_ld).view(B, H, W, res_ld)[..., :cout]
        res.copy_((torch.randn(B, H, W, cout, generator=g, device=DEV) * 0.25).half())
    wt = (torch.randn(cout, 9, cin, generator=g, device=DEV) * (2.0 / (9 * cin) ** 0.5)).half()
    bias = (torch.randn(cout, generator=g, device=DEV) * 0.5).half().float()
    snap = [t.clone() for t in (xb, rb) if t is not None]
    _lib.check(_lib.lib().nb200_sod_conv_f16(ptr(body(xb, npx * in_ld)), in_ld, in_off, cin, ptr(wt), ptr(bias), cout, dil,
                                             ptr(body(out, npx * out_ld)), out_ld, out_off,
                                             ptr(body(rb, npx * res_ld)) if has_res else None, res_ld, B, H, W, _lib.stream_ptr()))
    torch.cuda.synchronize()
    tally = Tally()
    for t, t0 in zip([t for t in (xb, rb) if t is not None], snap):
        tally.exact("input", bits(t), bits(t0))
    o = body(out, npx * out_ld).view(B, H, W, out_ld)
    written = torch.zeros(out_ld, dtype=torch.bool, device=DEV)
    written[out_off:out_off + cout] = True
    tally.exact("channels outside the output slice", bits(o[..., ~written].contiguous()),
                torch.full((B, H, W, out_ld - cout), SENTINEL, dtype=torch.int16, device=DEV))
    if not guards_ok(out, npx * out_ld):
        tally.bad.append("output: guard changed")
    got = o[..., out_off:out_off + cout]
    tally.no_nan("output", got)
    w64 = wt.double().view(cout, 3, 3, cin).permute(0, 3, 1, 2)
    L = 9 * cin // 16
    for i in range(B):
        a, s = conv64(x[i:i + 1], w64, dil=dil, pad=dil)
        h1, e1 = rounded(a, ACC * L * s)
        v2 = h1 + bias.double()
        h2, e3 = rounded(v2, e1 + U * v2.abs())
        v = h2.clamp_min(0)
        if has_res:
            v = v + res[i:i + 1].double()
            e3 = e3 + U * v.abs()
        tally.add(got[i:i + 1], v, round16_bound(v, e3))
    return tally.result()


def test_sod_conv_replay(production):
    cases = configurations(production, "sodconv", SYNTH_SOD)
    have = {(r["cout"], r["dil"]) for _, r in cases}
    assert have >= {(c, d) for c in (16, 64) for d in (1, 2, 4, 8)}, have
    assert {(r["cin"], r["cout"]) for _, r in cases} == set(SOD_PAIRS)
    replay("sodconv", cases, sod_check)


def test_wall_time_and_device(production):
    """Runs last: the module's wall time and peak device memory, with the card and its power limit they were measured on."""
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    wall, peak = time.time() - T0, torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"\nconv replay module: {wall:.1f} s, peak device memory {peak:.1f} GiB on {q.stdout.strip() or torch.cuda.get_device_name(0)}")
    log_metric("replay_conv_module", wall_s=f"{wall:.1f}", peak_gib=f"{peak:.2f}", device=q.stdout.strip())
