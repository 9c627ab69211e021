"""Float64 references of each stage of the light_inpaint_v1 forward, one function per stage (TEST INFRASTRUCTURE).

Every function takes the engine's own input of that stage (the debug taps of nb200_light_inpaint, DESIGN.md §5) in the
engine's layout (NHWC, fp16 activations) and evaluates the stage alone in float64, so an error can be pinned on one kernel.
The math follows oracle/light_inpaint.py and the lines of the reference it cites (iw3/models/light_inpaint_v1.py,
nunif/modules/attention.py).  With ``r16=True`` a stage rounds to fp16 exactly where the engine stores fp16 inside it (the
stem's normalised input, the token mixing's LN2(v)·g2), and the weights enter at the precision the engine packs them: GEMM
weights, Ws and the stem weights fp16-rounded, LN gains and biases fp32.  With ``r16=False`` nothing is rounded and `forward`
chains the stages into the whole network (tests/test_light_inpaint_stages.py pins that chain to oracle.light_inpaint).

Each stage returns ``(ref, abs_sum)``: abs_sum is Σ|a·w| per output element (bias and residual terms included), the scale of
the rounding error of an fp32 evaluation of the same sum.  For the elementwise stages it is the analogous scale (see each
docstring).  Tensors stay on the device they come on.
"""
import torch
import torch.nn.functional as F

# (state-dict prefix, window, shifted, channels) of the six GMLP blocks, in forward order (light_inpaint_v1.py:55-86)
BLOCKS = [("enc1", 16, True, 96)] + [(f"enc2.{i}", 8, i % 2 == 1, 192) for i in range(4)] + [("dec1", 16, False, 96)]
GELU_SLOPE = 1.13   # max |d/dx x·Phi(x)| = 1.1289 (at x = sqrt 2): an input error δ moves GELU's output by at most 1.13 δ


def padded(H, W):
    """light_inpaint_v1.py:134-139: replicate pad to the next multiple of 64 (64, not 0, when already a multiple)."""
    return H + 64 - H % 64, W + 64 - W % 64


def ulp16(r):
    """fp16 spacing at |r|, with the subnormal floor 2^-24."""
    _, e = torch.frexp(r.abs())
    return torch.where(r.abs() < 2.0 ** -14, torch.full_like(r, 2.0 ** -24), torch.ldexp(torch.ones_like(r), e - 11))


def _q(x, r16):
    return x.half().double() if r16 else x


def _w(sd, k, r16, dev):
    """A GEMM / Ws / stem weight: fp16-rounded when the engine packs it so."""
    return _q(sd[k].to(dev).double(), r16)


def _f(sd, k, dev):
    """An fp32 parameter (LN gain, bias, mask_bias)."""
    return sd[k].to(dev).double()


def _conv(x, w, b, stride=1):
    """NHWC conv (valid) and its Σ|a·w| + |b|."""
    xc = x.permute(0, 3, 1, 2)
    y = F.conv2d(xc, w, b, stride=stride)
    a = F.conv2d(xc.abs(), w.abs(), b.abs(), stride=stride)
    return y.permute(0, 2, 3, 1), a.permute(0, 2, 3, 1)


def _linear(x, w, b):
    return x @ w.t() + b, x.abs() @ w.abs().t() + b.abs()


def _rep_pad(x, p=1):
    """Replicate pad of NHWC by p on H and W."""
    return F.pad(x.permute(0, 3, 1, 2), (p, p, p, p), mode="replicate").permute(0, 2, 3, 1)


def _ln(x, g):
    """LayerNorm without bias, eps 1e-5, over the last dim; also the rstd."""
    mu = x.mean(-1, keepdim=True)
    r = torch.rsqrt(((x - mu) ** 2).mean(-1, keepdim=True) + 1e-5)
    return (x - mu) * r * g, r


# ---- stem and tail (light_inpaint_v1.py:113-118, 125-126, 132-154) --------------------------------------------------------------
def stem(sd, x, hole, blur, mirror, r16=True):
    """x [B][3][H][W] fp32 and the binary hole [B][1][H][W] in image coordinates, blur [B][H][W] (or [B][1][H][W]) in network
    coordinates (the engine's tap 100, so the > 0.99 token test sees the engine's values) -> X1 [B][H4][W4][96] and the mask
    token map [B][H4][W4].  Mirror, hole zeroing, (x - 0.5)/0.5 (fp32 then fp16 with r16, as the engine computes it: x·keep
    is exact for a binary hole), the replicate pad to Hp×Wp, pixel_unshuffle(4), the 1×1 48 -> 96 conv, LeakyReLU(0.2)."""
    dev = x.device
    B, _, H, W = x.shape
    if mirror:
        x, hole = x.flip(-1), hole.flip(-1)
    if r16:
        n = ((x.float() * (1 - hole.float()) - 0.5) / 0.5).half().double()
    else:
        n = (x.double() * (1 - hole.double()) - 0.5) / 0.5
    Hp, Wp = padded(H, W)
    n = F.pad(n, (0, Wp - W, 0, Hp - H), mode="replicate")
    m = F.pad(blur.reshape(B, 1, H, W).double(), (0, Wp - W, 0, Hp - H), mode="replicate")
    u = F.pixel_unshuffle(n, 4).permute(0, 2, 3, 1)
    y, a = _conv(u, _w(sd, "patch.0.weight", r16, dev), _f(sd, "patch.0.bias", dev))
    y = torch.where(y >= 0, y, 0.2 * y)
    tok = F.pixel_unshuffle(m, 4).amax(dim=1) > 0.99
    mb = _f(sd, "mask_bias", dev).reshape(96)
    t = tok[..., None]
    return torch.where(t, mb, y), torch.where(t, torch.zeros_like(a), a), tok


def tail(Y, x, hole, blur, mirror, shuffle_order="c_dy_dx"):
    """Y [B][H4][W4][48] (to_image's output) -> the output frame [B][3][H][W] in image coordinates: pixel_shuffle(4), crop,
    composite src·(1 - m) + net·m with the hole-zeroed frame and the blur, clamp, un-mirror.  No fp16 rounding: the engine
    runs it in fp32.  shuffle_order="dy_dx_c" reads the 48 channels in the wrong order (a test of the test)."""
    B, H4, W4, _ = Y.shape
    H, W = x.shape[2:]
    y = Y.double().permute(0, 3, 1, 2)
    if shuffle_order == "dy_dx_c":
        y = y.reshape(B, 4, 4, 3, H4, W4).permute(0, 3, 1, 2, 4, 5).reshape(B, 48, H4, W4)
    net = F.pixel_shuffle(y, 4)[:, :, :H, :W]
    if mirror:
        x, hole = x.flip(-1), hole.flip(-1)
    src = x.double() * (1 - hole.double())
    m = blur.reshape(B, 1, H, W).double()
    out = (src * (1 - m) + net * m).clamp(0, 1)
    return out.flip(-1) if mirror else out


# ---- GMLP block (light_inpaint_v1.py:37-49, attention.py:621-693) -----------------------------------------------------------------
def ln_pad(sd, p, x, pad):
    """Stage 1: LN1 of the block input x [B][H][W][C] with the shifted block's zero ring of width pad -> T [B][Hq][Wq][C].
    abs_sum = (|x| + mean|x|)·rstd·|g|: the scale of the fp32 errors of the mean, the centring and the variance."""
    x = x.double()
    g = _f(sd, p + ".norm1.weight", x.device)
    y, r = _ln(x, g)
    a = (x.abs() + x.abs().mean(-1, keepdim=True)) * r * g.abs()
    pz = (0, 0, pad, pad, pad, pad)
    return F.pad(y, pz), F.pad(a, pz)


def proj_in(sd, p, T, r16=True):
    """Stage 2: U = GELU(proj_in(T)) (erf form), [B][Hq][Wq][4C]; abs_sum is the pre-activation one times GELU's slope."""
    g = p + ".gmlp.gmlp.proj_in"
    y, a = _linear(T.double(), _w(sd, g + ".weight", r16, T.device), _f(sd, g + ".bias", T.device))
    return F.gelu(y), GELU_SLOPE * a


def _windows(t, ws, col_major):
    B, H, W, C = t.shape
    t = t.reshape(B, H // ws, ws, W // ws, ws, C)
    t = t.permute(0, 1, 3, 4, 2, 5) if col_major else t.permute(0, 1, 3, 2, 4, 5)
    return t.reshape(B, H // ws, W // ws, ws * ws, C)


def _unwindows(t, ws, col_major):
    B, nh, nw, _, C = t.shape
    t = t.reshape(B, nh, nw, ws, ws, C)
    t = t.permute(0, 1, 4, 2, 3, 5) if col_major else t.permute(0, 1, 3, 2, 4, 5)
    return t.reshape(B, nh * ws, nw * ws, C)


def token_mix(sd, p, U, ws, r16=True, ws_transposed=False, ln_over_u=False, ring=0, col_major=False):
    """Stage 3 (attention.py:643-660): v' = LN2(v)·g2 over all 2C channels of v (fp16 with r16), then per window of
    _to_windows order (tokens row-major, windows over the grid U covers, ring included) Ws·v' + bs, and the gate u·.
    U [B][Hq][Wq][4C] = u | v -> U with u replaced by u·(Ws·v' + bs); v passes unchanged (abs_sum 0 there).
    The third result, `flip`, is an absolute allowance for the one rounding the engine and this reference cannot share: the
    engine evaluates LN2(v)·g2 in fp32 before rounding it to fp16, so where the exact v'_m lies within that fp32 error
    (2^-16·(|v| + mean|v|)·rstd·|g2|, as for LN1) of an fp16 rounding midpoint, the engine may store the other neighbour, an
    input error of one ulp16(v'_m) that reaches the output as |u·Ws[n][m]|·ulp16(v'_m).  flip sums that over such m.
    The keyword arguments build wrong variants for the tests of the tests: Ws transposed, LN2 over u, windows over the grid
    without a ring of width `ring`, tokens column-major."""
    dev = U.device
    U = U.double()
    C2 = U.shape[-1] // 2
    u, v = U[..., :C2], U[..., C2:]
    g = p + ".gmlp.gmlp.proj_spatial"
    src, g2 = u if ln_over_u else v, _f(sd, p + ".norm2.weight", dev)
    vx, r = _ln(src, g2)
    vn = _q(vx, r16)
    fl = torch.zeros_like(vx)
    if r16:
        below = ulp16(vn * (1 - 2.0 ** -12))   # the fp16 spacing on the lower side of vn (half of ulp16(vn) at a power of 2)
        near = (vx - vn).abs() >= below / 2 - 2.0 ** -16 * (src.abs() + src.abs().mean(-1, keepdim=True)) * r * g2.abs()
        fl = torch.where(near, ulp16(vn), fl)
    N = ws * ws
    Ws = _w(sd, g + ".weight", r16, dev).reshape(N, N)
    if ws_transposed:
        Ws = Ws.t()
    bs = _f(sd, g + ".bias", dev)[:, None]
    H, W = U.shape[1] - 2 * ring, U.shape[2] - 2 * ring
    crop = (slice(None), slice(ring, ring + H), slice(ring, ring + W))
    wv = _windows(vn[crop], ws, col_major)
    mix = _unwindows(torch.einsum("nm,bijmc->bijnc", Ws, wv) + bs, ws, col_major)
    amix = _unwindows(torch.einsum("nm,bijmc->bijnc", Ws.abs(), wv.abs()) + bs.abs(), ws, col_major)
    fmix = _unwindows(torch.einsum("nm,bijmc->bijnc", Ws.abs(), _windows(fl[crop], ws, col_major)), ws, col_major)
    ref, a, flip = U.clone(), torch.zeros_like(U), torch.zeros_like(U)
    ref[crop + (slice(0, C2),)] = u[crop] * mix
    a[crop + (slice(0, C2),)] = u[crop].abs() * amix
    flip[crop + (slice(0, C2),)] = u[crop].abs() * fmix
    return ref, a, flip


def proj_out(sd, p, Umix, x, pad, r16=True, residual=2.0):
    """Stage 4: x + (proj_out(u·v') + x) on the cropped view: 2x + proj_out(Umix[ring-cropped, :2C]) -> [B][H][W][C].
    x is the block input (stage 0); `residual` = 1 is a wrong variant."""
    x = x.double()
    B, H, W, C = x.shape
    g = p + ".gmlp.gmlp.proj_out"
    uv = Umix.double()[:, pad:pad + H, pad:pad + W, :2 * C]
    y, a = _linear(uv, _w(sd, g + ".weight", r16, x.device), _f(sd, g + ".bias", x.device))
    return y + residual * x, a + residual * x.abs()


def w1(sd, p, x, r16=True):
    """Stage 5: glu_conv.w1, a 1×1 C -> C conv."""
    C = x.shape[-1]
    return _linear(x.double(), _w(sd, p + ".glu_conv.w1.weight", r16, x.device).reshape(C, C), _f(sd, p + ".glu_conv.w1.bias", x.device))


def pad_glu(h, cpad):
    """Stage 6: replicate pad 1 + GLU (a·sigmoid(b), halves of the C channels) into [B][H+2][W+2][cpad], channels >= C/2 zero.
    abs_sum = |a·sigmoid(b)|·(1 + |b|): the engine's __expf has a relative error of about 2^-21·(1 + |b|)."""
    h = _rep_pad(h.double())
    C = h.shape[-1]
    a, b = h[..., :C // 2], h[..., C // 2:]
    gl = a * torch.sigmoid(b)
    out = torch.zeros(*h.shape[:3], cpad, dtype=torch.float64, device=h.device)
    ab = torch.zeros_like(out)
    out[..., :C // 2] = gl
    ab[..., :C // 2] = gl.abs() * (1 + b.abs())
    return out, ab


def conv3_res(sd, p, P, x, r16=True):
    """Stage 7: x + glu_conv.w2 (valid 3×3, C/2 -> C) over P's first C/2 channels."""
    C = x.shape[-1]
    y, a = _conv(P.double()[..., :C // 2], _w(sd, p + ".glu_conv.w2.weight", r16, P.device), _f(sd, p + ".glu_conv.w2.bias", P.device))
    return y + x.double(), a + x.double().abs()


def block(sd, k, x, r16=True):
    """The eight stages of GMLP block k chained (stage 0 = x); the list of stage outputs 0..7."""
    p, ws, shift, C = BLOCKS[k]
    pad = ws // 2 if shift else 0
    s = [x]
    s.append(ln_pad(sd, p, x, pad)[0])
    s.append(proj_in(sd, p, s[1], r16)[0])
    s.append(token_mix(sd, p, s[2], ws, r16)[0])
    s.append(proj_out(sd, p, s[3], x, pad, r16)[0])
    s.append(w1(sd, p, s[4], r16)[0])
    s.append(pad_glu(s[5], (C // 2 + 31) // 32 * 32)[0])
    s.append(conv3_res(sd, p, s[6], s[4], r16)[0])
    return s


# ---- down, up, to_image (light_inpaint_v1.py:119-126) ---------------------------------------------------------------------------------
def down(sd, x, r16=True):
    """Tap 170: conv 2×2 stride 2, 96 -> 192."""
    return _conv(x.double(), _w(sd, "down.weight", r16, x.device), _f(sd, "down.bias", x.device), stride=2)


def up(sd, x2, x1, r16=True, swap_dy_dx=False):
    """Tap 171: pixel_shuffle(2) of the 1×1 192 -> 384 conv, plus the x1 skip.  swap_dy_dx is a wrong variant."""
    y, a = _conv(x2.double(), _w(sd, "up.weight", r16, x2.device), _f(sd, "up.bias", x2.device))

    def shuffle(t):
        t = t.permute(0, 3, 1, 2)
        if swap_dy_dx:
            B, _, h, w = t.shape
            t = t.reshape(B, 96, 2, 2, h, w).transpose(2, 3).reshape(B, 384, h, w)
        return F.pixel_shuffle(t, 2).permute(0, 2, 3, 1)

    return shuffle(y) + x1.double(), shuffle(a) + x1.double().abs()


def toimg_pad(x):
    """Tap 172: replicate pad 1 (exact)."""
    return _rep_pad(x.double())


def toimg(sd, P, r16=True):
    """Tap 173: valid 3×3 96 -> 48."""
    return _conv(P.double(), _w(sd, "to_image.1.weight", r16, P.device), _f(sd, "to_image.1.bias", P.device))


def forward(sd, x, hole, blur, mirror=0, r16=False):
    """The stages chained into LightInpaintV1.forward: x, hole [B][.][H][W] image coordinates, blur network coordinates."""
    x1 = stem(sd, x, hole, blur, mirror, r16)[0]
    x1 = block(sd, 0, x1, r16)[-1]
    x2 = down(sd, x1, r16)[0]
    for k in range(1, 5):
        x2 = block(sd, k, x2, r16)[-1]
    x5 = block(sd, 5, up(sd, x2, x1, r16)[0], r16)[-1]
    return tail(toimg(sd, toimg_pad(x5), r16)[0], x, hole, blur, mirror)
