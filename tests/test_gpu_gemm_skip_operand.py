"""GPU: the pixel-shuffle GEMM with a second A operand (a Linear of the full-resolution skip tensor folded into the GEMM, as
swin_unet 4x runs up1(x) + proj2(x3)) against torch fp32 on fp16-rounded operands."""
import pytest
import torch
import torch.nn.functional as F

from tests.util import log_metric
from nunif_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


# (2, 12, 192, 192, 96, 0): the swin_unet 4x up1 + proj2 channel counts; odd H and B * H not a multiple of the 8-row tile
# cover the edge tiles, whose rows past the image read the next image (or nothing) and are clipped at the store
@pytest.mark.parametrize("B,H,Cin,cout,Cin2,act", [(2, 12, 192, 192, 96, 0), (1, 23, 64, 64, 32, 1), (3, 20, 128, 64, 64, 0),
                                                   (2, 15, 192, 96, 96, 1)])
def test_convT2_pixshuf_with_linear_skip(B, H, Cin, cout, Cin2, act):
    g = torch.Generator(device="cpu").manual_seed(H + Cin + cout + Cin2)
    A = torch.randn(B, H, H, Cin, generator=g).half().to(DEV)
    Wc = (torch.randn(Cin, cout, 2, 2, generator=g) / Cin ** 0.5).half().to(DEV)   # ConvTranspose2d weight
    b = torch.randn(cout, generator=g).to(DEV)
    ld2 = Cin2 + 32                                                                  # the skip's channel stride > Cin2
    A2 = torch.randn(B, 2 * H, 2 * H, ld2, generator=g).half().to(DEV)
    Ws = (torch.randn(cout, Cin2, generator=g) / Cin2 ** 0.5).half().to(DEV)
    bs = torch.randn(cout, generator=g).to(DEV)
    Wt = torch.cat([Wc.permute(2, 3, 1, 0).reshape(4 * cout, Cin), Ws.repeat(4, 1)], 1).contiguous()   # n = (dy*2+dx)*cout + co
    bias4 = (b + bs).repeat(4).contiguous()
    out = torch.full((B, 2 * H, 2 * H, cout), 7.0, dtype=torch.float16, device=DEV)
    _lib.check(_lib.lib().nb200_conv_gemm_pixshuf_a2_f16(
        _lib.ptr(A), B, H, H, Cin, _lib.ptr(Wt), 4 * cout, _lib.ptr(bias4), act, _lib.ptr(out), cout, cout, _lib.ptr(A2), Cin2,
        ld2, _lib.stream_ptr()))
    torch.cuda.synchronize()
    y = F.conv_transpose2d(A.permute(0, 3, 1, 2).float(), Wc.float(), b, stride=2).permute(0, 2, 3, 1)
    ref = y + A2[..., :Cin2].float() @ Ws.float().t() + bs
    if act:
        ref = F.leaky_relu(ref, 0.1)
    err = (out.float() - ref).abs().max().item()
    log_metric("gemm_convT2_linear_skip", H=H, Cin=Cin, cout=cout, Cin2=Cin2, err=err)
    assert err < 2e-2, err
