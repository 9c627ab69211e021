"""GPU: the wgmma implicit-GEMM against torch fp32 on fp16-rounded operands."""
import pytest
import torch
import torch.nn.functional as F

from tests.util import log_metric
from nunif_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def run(A, kind, Wt, bias, act, out, out_mode=0, cout=0, res=None, res_crop=0, res_before_act=0, Cin=None):
    B, Hi, Wi, Ci = A.shape
    N = Wt.shape[0]
    rH = res.shape[1] if res is not None else 0
    rW = res.shape[2] if res is not None else 0
    _lib.check(_lib.lib().nb200_conv_gemm_f16(
        _lib.ptr(A), B, Hi, Wi, Ci, Cin or Ci, kind, _lib.ptr(Wt), N, _lib.ptr(bias), act, _lib.ptr(out), out.shape[-1],
        out_mode, cout, _lib.ptr(res), res.shape[-1] if res is not None else 0, rH, rW, res_crop, res_crop,
        res_before_act, _lib.stream_ptr()))
    torch.cuda.synchronize()


def act_ref(x, act):
    x = x.half().float()
    return {0: lambda v: v, 1: lambda v: F.leaky_relu(v, 0.1), 2: F.gelu, 3: F.relu}[act](x)


@pytest.mark.parametrize("M,K,N,act,use_res", [
    (1000, 96, 288, 0, False), (129, 192, 576, 0, False), (4096, 192, 192, 0, True), (777, 96, 192, 2, False),
    (2048, 384, 192, 0, True), (640, 192, 768, 0, False), (512, 192, 48, 0, False), (300, 96, 96, 0, True),
    (256, 64, 64, 1, False), (200, 32, 16, 3, False), (57600, 192, 384, 2, False),
    (200000, 192, 192, 0, True), (150001, 96, 288, 0, False), (99999, 384, 192, 0, True), (64, 192, 576, 0, False),
])
def test_linear_flat(M, K, N, act, use_res):
    g = torch.Generator(device="cpu").manual_seed(M + K + N)
    A = (torch.randn(M, K, generator=g)).half().to(DEV)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).half().to(DEV)
    b = torch.randn(N, generator=g).to(DEV)
    res = torch.randn(M, N, generator=g).half().to(DEV) if use_res else None
    out = torch.full((M, N), 7.0, dtype=torch.float16, device=DEV)
    run(A.view(1, 1, M, K), 0, W, b, act, out.view(1, 1, M, N), res=res.view(1, 1, M, N) if use_res else None)
    ref = act_ref(A.float() @ W.float().t() + b, act)
    if use_res:
        ref = ref.half().float() + res.float()
    err = (out.float() - ref).abs().max().item()
    log_metric("gemm_linear", M=M, K=K, N=N, act=act, res=use_res, err=err)
    assert err < 2e-2 * max(1.0, ref.abs().max().item()) / 4, err


@pytest.mark.parametrize("B,H,W,Cin,N,act", [(2, 37, 41, 64, 128, 1), (1, 20, 52, 32, 64, 1), (3, 18, 18, 128, 256, 1),
                                               (1, 30, 30, 256, 128, 0), (2, 26, 26, 64, 96, 1), (4, 130, 134, 64, 64, 1), (16, 50, 50, 128, 64, 1)])
def test_conv3(B, H, W, Cin, N, act):
    g = torch.Generator(device="cpu").manual_seed(H * W + Cin)
    A = torch.randn(B, H, W, Cin, generator=g).half().to(DEV)
    Wc = (torch.randn(N, Cin, 3, 3, generator=g) / (9 * Cin) ** 0.5).half().to(DEV)
    b = torch.randn(N, generator=g).to(DEV)
    Wt = Wc.permute(0, 2, 3, 1).reshape(N, 9 * Cin).contiguous()
    out = torch.full((B, H - 2, W - 2, N), 7.0, dtype=torch.float16, device=DEV)
    run(A, 2, Wt, b, act, out)
    ref = act_ref(F.conv2d(A.permute(0, 3, 1, 2).float(), Wc.float(), b), act).permute(0, 2, 3, 1)
    err = (out.float() - ref).abs().max().item()
    log_metric("gemm_conv3", H=H, W=W, Cin=Cin, N=N, err=err)
    assert err < 1e-2, err


@pytest.mark.parametrize("B,H,W,Cin,N,act,use_res", [(2, 28, 49, 64, 64, 3, False), (1, 14, 25, 384, 64, 0, False), (2, 56, 98, 96, 64, 0, True),
                                                       (3, 9, 7, 32, 32, 3, False), (1, 112, 196, 64, 32, 0, True), (2, 5, 3, 192, 64, 0, False)])
def test_conv3_same_padding(B, H, W, Cin, N, act, use_res):
    """kind 4: 3x3 conv with zero padding 1 - the halo is the tensor map's out-of-bounds zero fill (DPT head convs)."""
    g = torch.Generator(device="cpu").manual_seed(H * W + Cin + 1)
    A = torch.randn(B, H, W, Cin, generator=g).half().to(DEV)
    Wc = (torch.randn(N, Cin, 3, 3, generator=g) / (9 * Cin) ** 0.5).half().to(DEV)
    b = torch.randn(N, generator=g).to(DEV)
    res = torch.randn(B, H, W, N, generator=g).half().to(DEV) if use_res else None
    Wt = Wc.permute(0, 2, 3, 1).reshape(N, 9 * Cin).contiguous()
    out = torch.full((B, H, W, N), 7.0, dtype=torch.float16, device=DEV)
    run(A, 4, Wt, b, act, out, res=res)
    ref = act_ref(F.conv2d(A.permute(0, 3, 1, 2).float(), Wc.float(), b, padding=1), act).permute(0, 2, 3, 1)
    if use_res:
        ref = ref.half().float() + res.float()
    err = (out.float() - ref).abs().max().item()
    log_metric("gemm_conv3_same", H=H, W=W, Cin=Cin, N=N, err=err)
    assert err < 1e-2, err


@pytest.mark.parametrize("B,H,C,N", [(2, 24, 96, 192), (1, 36, 192, 192), (2, 20, 64, 64), (1, 12, 128, 128)])
def test_down2(B, H, C, N):
    g = torch.Generator(device="cpu").manual_seed(H + C)
    A = torch.randn(B, H, H, C, generator=g).half().to(DEV)
    Wc = (torch.randn(N, C, 2, 2, generator=g) / (4 * C) ** 0.5).half().to(DEV)
    b = torch.randn(N, generator=g).to(DEV)
    Wt = Wc.permute(0, 2, 3, 1).reshape(N, 4 * C).contiguous()
    out = torch.empty((B, H // 2, H // 2, N), dtype=torch.float16, device=DEV)
    run(A, 3, Wt, b, 0, out)
    ref = F.conv2d(A.permute(0, 3, 1, 2).float(), Wc.float(), b, stride=2).permute(0, 2, 3, 1)
    err = (out.float() - ref).abs().max().item()
    log_metric("gemm_down2", H=H, C=C, N=N, err=err)
    assert err < 1e-2, err


@pytest.mark.parametrize("B,H,Cin,cout,crop", [(2, 23, 64, 64, 4), (1, 15, 128, 128, 4), (1, 30, 192, 192, 0), (2, 12, 192, 96, 0)])
def test_convT2_pixshuf_with_cropped_skip(B, H, Cin, cout, crop):
    g = torch.Generator(device="cpu").manual_seed(H + Cin + cout)
    A = torch.randn(B, H, H, Cin, generator=g).half().to(DEV)
    Wc = (torch.randn(Cin, cout, 2, 2, generator=g) / Cin ** 0.5).half().to(DEV)   # ConvTranspose2d weight
    b = torch.randn(cout, generator=g).to(DEV)
    skip = torch.randn(B, 2 * H + 2 * crop, 2 * H + 2 * crop, cout, generator=g).half().to(DEV)
    Wt = Wc.permute(2, 3, 1, 0).reshape(4 * cout, Cin).contiguous()                  # n = (dy*2+dx)*cout + co
    bias4 = b.repeat(4)
    out = torch.empty((B, 2 * H, 2 * H, cout), dtype=torch.float16, device=DEV)
    run(A, 1, Wt, bias4, 1, out, out_mode=1, cout=cout, res=skip, res_crop=crop)
    y = F.leaky_relu(F.conv_transpose2d(A.permute(0, 3, 1, 2).float(), Wc.float(), b, stride=2).half().float(), 0.1)
    sk = skip.float().permute(0, 3, 1, 2)
    if crop:
        sk = sk[:, :, crop:-crop, crop:-crop]
    ref = (y.half().float() + sk).permute(0, 2, 3, 1)
    err = (out.float() - ref).abs().max().item()
    log_metric("gemm_convT2", H=H, Cin=Cin, cout=cout, err=err)
    assert err < 2e-2, err


@pytest.mark.parametrize("B,H,W,C,shift", [(2, 12, 12, 96, 0), (2, 12, 18, 96, 3), (1, 24, 24, 192, 0), (3, 18, 12, 192, 3),
                                             (1, 6, 6, 192, 3)])
def test_window_attention_core(B, H, W, C, shift):
    """qkv -> attention output (pre-projection) against a torch fp32 evaluation of torchvision's
    shifted_window_attention body (swin_transformer.py:166-221)."""
    heads, ws = 6, 6
    d = C // heads
    g = torch.Generator(device="cpu").manual_seed(C + H + shift)
    qkv = torch.randn(B, H, W, 3 * C, generator=g).half().to(DEV)
    table = (torch.randn(121, heads, generator=g) * 0.5).to(DEV)
    out = torch.full((B, H, W, C), 9.0, dtype=torch.float16, device=DEV)
    planes = qkv.view(B, H, W, 3, C).permute(3, 0, 1, 2, 4).contiguous()   # q | k | v as three dense [B,H,W,C] planes
    _lib.check(_lib.lib().nb200_window_attention_f16(_lib.ptr(planes), _lib.ptr(table), _lib.ptr(out), B, H, W, C, heads, shift,
                                                     _lib.stream_ptr()))
    torch.cuda.synchronize()
    from nunif_b200.synth import relative_position_index
    s = shift if ws < H else 0
    x = qkv.float()
    if s > 0:
        x = torch.roll(x, shifts=(-s, -s), dims=(1, 2))
    nh, nw = H // ws, W // ws
    xw = x.view(B, nh, ws, nw, ws, 3 * C).permute(0, 1, 3, 2, 4, 5).reshape(B * nh * nw, ws * ws, 3, heads, d).permute(2, 0, 3, 1, 4)
    q, k, v = xw[0] * d ** -0.5, xw[1], xw[2]
    attn = q @ k.transpose(-2, -1)
    idx = relative_position_index(ws).to(DEV)
    attn = attn + table[idx].view(ws * ws, ws * ws, -1).permute(2, 0, 1).unsqueeze(0)
    if s > 0:
        m = torch.zeros((H, W), device=DEV)
        cnt = 0
        for hs in ((0, -ws), (-ws, -s), (-s, None)):
            for ws_ in ((0, -ws), (-ws, -s), (-s, None)):
                m[hs[0]:hs[1], ws_[0]:ws_[1]] = cnt
                cnt += 1
        m = m.view(nh, ws, nw, ws).permute(0, 2, 1, 3).reshape(nh * nw, ws * ws)
        m = m.unsqueeze(1) - m.unsqueeze(2)
        m = m.masked_fill(m != 0, -100.0).masked_fill(m == 0, 0.0)
        attn = (attn.view(B, nh * nw, heads, ws * ws, ws * ws) + m.unsqueeze(1).unsqueeze(0)).view(-1, heads, ws * ws, ws * ws)
    o = (attn.softmax(-1) @ v).transpose(1, 2).reshape(-1, ws * ws, C)
    o = o.view(B, nh, nw, ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, C)
    if s > 0:
        o = torch.roll(o, shifts=(s, s), dims=(1, 2))
    err = (out.float() - o).abs().max().item()
    log_metric("window_attention", H=H, W=W, C=C, shift=shift, err=err)
    assert err < 1e-2, err
