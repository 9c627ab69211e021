"""GPU: the fused Swin-block kernels (csrc/swin_attention_mma.cu swin_attn_fused_kernel: wgmma qkv GEMM + window attention;
csrc/swin_block.cu swin_mlp_fused_kernel: proj + fc1 + GELU + fc2 on wgmma) against torch fp32 on fp16-rounded operands, and
the head against the unfused engine path (qkv GEMM -> window_attention_mma_kernel)."""
import pytest
import torch
import torch.nn.functional as F

from tests.util import log_metric
from nunif_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _mlp_ref(x, att, wp, bp, w1, b1, w2, b2):
    """fp32 math on the fp16 operands, rounding to fp16 where the engine stores (x1, hidden, output)."""
    x1 = x.float()
    if att is not None:
        x1 = (x1 + att.float() @ wp.float().t() + bp).half().float()
    h = F.gelu(x1 @ w1.float().t() + b1).half().float()
    return (x1 + h @ w2.float().t() + b2).half()


@pytest.mark.parametrize("T,C,proj", [
    (128, 192, False), (128, 192, True), (1000, 192, True), (128, 96, False), (128, 96, True), (777, 96, True),
    (148 * 128 * 3 + 55, 192, True), (148 * 128 * 2 + 1, 96, True), (57600, 192, True), (230400, 96, True),
])
def test_swin_mlp_fused(T, C, proj):
    g = torch.Generator(device="cpu").manual_seed(T + C + int(proj))
    x = torch.randn(T, C, generator=g).half().to(DEV)
    att = torch.randn(T, C, generator=g).half().to(DEV) if proj else None
    wp = (torch.randn(C, C, generator=g) / C ** 0.5).half().to(DEV)
    bp = (0.1 * torch.randn(C, generator=g)).to(DEV)
    w1 = (torch.randn(2 * C, C, generator=g) / C ** 0.5).half().to(DEV)
    b1 = (0.1 * torch.randn(2 * C, generator=g)).to(DEV)
    w2 = (torch.randn(C, 2 * C, generator=g) / (2 * C) ** 0.5).half().to(DEV)
    b2 = (0.1 * torch.randn(C, generator=g)).to(DEV)
    want = _mlp_ref(x, att, wp, bp, w1, b1, w2, b2)
    got = x.clone()
    _lib.check(_lib.lib().nb200_swin_mlp_fused_f16(
        _lib.ptr(got), _lib.ptr(att), T, C, _lib.ptr(wp), _lib.ptr(bp), _lib.ptr(w1), _lib.ptr(b1), _lib.ptr(w2), _lib.ptr(b2),
        _lib.stream_ptr()))
    torch.cuda.synchronize()
    d = (got.float() - want.float()).abs()
    err, mean = d.max().item(), d.mean().item()
    log_metric("swin_mlp_fused", T=T, C=C, proj=proj, err=err, mean=mean)
    # one fp16 ulp at |x| ~ 4-8 is 4e-3..8e-3: the two evaluations may round x1 / hidden / output differently
    assert err < 2e-2 and mean < 6e-4, (err, mean)


def _attn_ref(x, wqkv, bqkv, table, shift):
    """oracle.swin_unet.window_attention with an identity proj = everything up to the proj Linear, fp32 on fp16 operands."""
    from oracle import swin_unet as osw
    C = x.shape[-1]
    idx = torch.zeros(36 * 36, dtype=torch.long)
    for i in range(36):
        for j in range(36):
            idx[i * 36 + j] = (i // 6 - j // 6 + 5) * 11 + (i % 6 - j % 6 + 5)
    sd = {"a.qkv.weight": wqkv.float().cpu(), "a.qkv.bias": bqkv.float().cpu(),
          "a.relative_position_bias_table": table.float().cpu(), "a.relative_position_index": idx,
          "a.proj.weight": torch.eye(C), "a.proj.bias": torch.zeros(C)}
    return osw.window_attention(x.float().cpu(), "a", sd, 6, shift)


@pytest.mark.parametrize("B,H,W,C,shift", [
    (1, 12, 12, 192, 0), (1, 12, 12, 192, 3), (2, 18, 24, 192, 3), (1, 6, 6, 192, 3), (1, 12, 12, 96, 0), (2, 24, 18, 96, 3),
    (3, 48, 48, 192, 3), (2, 60, 60, 96, 3), (5, 30, 30, 192, 0), (16, 60, 60, 192, 3),
])
def test_swin_attn_fused(B, H, W, C, shift):
    g = torch.Generator(device="cpu").manual_seed(B * H + W + C + shift)
    x = torch.randn(B, H, W, C, generator=g).half().to(DEV)
    wqkv = (torch.randn(3 * C, C, generator=g) / C ** 0.5).half().to(DEV)
    bqkv = (0.1 * torch.randn(3 * C, generator=g)).to(DEV)
    table = (0.5 * torch.randn(121, 6, generator=g)).to(DEV)
    att = torch.full((B, H, W, C), 7.0, dtype=torch.float16, device=DEV)
    _lib.check(_lib.lib().nb200_swin_attn_fused_f16(_lib.ptr(x), _lib.ptr(wqkv), _lib.ptr(bqkv), _lib.ptr(table), _lib.ptr(att),
                                                    B, H, W, C, shift, _lib.stream_ptr()))
    torch.cuda.synchronize()
    want = _attn_ref(x, wqkv, bqkv, table, shift)
    d = (att.float().cpu() - want).abs()
    err, mean = d.max().item(), d.mean().item()
    # the unfused engine path: qkv GEMM (three planes) -> window_attention_mma_kernel; same rounding points
    T = B * H * W
    qkv = torch.empty(3, T, C, dtype=torch.float16, device=DEV)
    for i in range(3):
        _lib.check(_lib.lib().nb200_conv_gemm_f16(_lib.ptr(x), 1, 1, T, C, C, 0, _lib.ptr(wqkv[i * C:(i + 1) * C].contiguous()), C,
                                                  _lib.ptr(bqkv[i * C:(i + 1) * C].contiguous()), 0, _lib.ptr(qkv[i]), C, 0, 0,
                                                  None, 0, 0, 0, 0, 0, 0, _lib.stream_ptr()))
    ref2 = torch.empty_like(att)
    _lib.check(_lib.lib().nb200_window_attention_f16(_lib.ptr(qkv), _lib.ptr(table), _lib.ptr(ref2), B, H, W, C, 6, shift, _lib.stream_ptr()))
    torch.cuda.synchronize()
    d2 = (att.float() - ref2.float()).abs().max().item()
    log_metric("swin_attn_fused", B=B, H=H, W=W, C=C, shift=shift, err=err, mean=mean, vs_unfused=d2)
    assert err < 1.5e-2 and mean < 1e-3, (err, mean)
    assert d2 < 4e-3, d2
