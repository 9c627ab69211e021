"""GPU: the persistent fused Swin-block tail (csrc/swin_block.cu swin_mlp_fused_kernel).  Each CTA runs every gridDim-th
128-token tile, and the weight ring, the activation buffers and their barriers carry over from one tile to the next.  A
tile's arithmetic does not depend on which CTA runs it, so every grid size (nb200_tune_set(10, cap)) must give the same bits;
a grid of one CTA runs every tile through one CTA and wraps each barrier's parity many times."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from nunif_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CAPS = (1, 2, 7, 0)   # 0: the default grid, min(tiles, SMs)
CS = {96: 16, 192: 48}


def _mlp_ref(x, att, wp, bp, w1, b1, w2, b2):
    """fp32 math on the fp16 operands, rounding to fp16 where the engine stores (x1, hidden, output)."""
    x1 = x.float()
    if att is not None:
        x1 = (x1 + att.float() @ wp.float().t() + bp).half().float()
    h = F.gelu(x1 @ w1.float().t() + b1).half().float()
    return (x1 + h @ w2.float().t() + b2).half()


def _weights(C, seed, cs=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    w = {"wp": (torch.randn(C, C, generator=g) / C ** 0.5).half(), "bp": 0.1 * torch.randn(C, generator=g),
         "w1": (torch.randn(2 * C, C, generator=g) / C ** 0.5).half(), "b1": 0.1 * torch.randn(2 * C, generator=g),
         "w2": (torch.randn(C, 2 * C, generator=g) / (2 * C) ** 0.5).half(), "b2": 0.1 * torch.randn(C, generator=g)}
    if cs:
        w["wy"] = (torch.randn(cs, C, generator=g) / C ** 0.5).half()
        w["by"] = torch.randn(cs, generator=g)
    return {k: v.to(DEV) for k, v in w.items()}


def _run(x, att, w, cs=0, y=None, xp=None):
    """one tail call; x is updated in place (cs == 0) or y is written (cs > 0).  xp: x's address, if not x.data_ptr()."""
    lib = _lib.lib()
    T, C = x.shape
    xp = ctypes.c_void_p(x.data_ptr()) if xp is None else xp
    if cs:
        _lib.check(lib.nb200_swin_mlp_fused_y_f16(xp, _lib.ptr(att), T, C, _lib.ptr(w["wp"]), _lib.ptr(w["bp"]), _lib.ptr(w["w1"]),
                                                  _lib.ptr(w["b1"]), _lib.ptr(w["w2"]), _lib.ptr(w["b2"]), _lib.ptr(y), cs,
                                                  _lib.ptr(w["wy"]), _lib.ptr(w["by"]), _lib.stream_ptr()))
    else:
        _lib.check(lib.nb200_swin_mlp_fused_f16(xp, _lib.ptr(att), T, C, _lib.ptr(w["wp"]), _lib.ptr(w["bp"]), _lib.ptr(w["w1"]),
                                                _lib.ptr(w["b1"]), _lib.ptr(w["w2"]), _lib.ptr(w["b2"]), _lib.stream_ptr()))


def _with_cap(cap, fn):
    lib = _lib.lib()
    _lib.check(lib.nb200_tune_set(10, cap))
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        lib.nb200_tune_set(10, 0)


def _token_counts():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return [100, 128 * sms + 1, 148 * 128 * 3 + 55, 57600, 921600]


@pytest.mark.parametrize("mode", ["proj", "noproj", "y"])
@pytest.mark.parametrize("C", [96, 192])
@pytest.mark.parametrize("ti", range(5))
def test_tail_grid_size_bit_identical(ti, C, mode):
    T = _token_counts()[ti]
    cs = CS[C] if mode == "y" else 0
    w = _weights(C, 1000 * ti + C, cs)
    g = torch.Generator(device=DEV).manual_seed(7 * T + C)
    x0 = torch.randn(T, C, generator=g, device=DEV).half()
    att = torch.randn(T, C, generator=g, device=DEV).half() if mode != "noproj" else None
    outs = {}
    for cap in CAPS:
        x = x0.clone()
        y = torch.empty(T, cs, dtype=torch.float16, device=DEV) if cs else None
        _with_cap(cap, lambda: _run(x, att, w, cs, y))
        if cs:
            assert torch.equal(x, x0), "x changed although y was requested"
        outs[cap] = y if cs else x
    assert not bool(torch.isnan(outs[0]).any())
    for cap in CAPS[:-1]:
        assert torch.equal(outs[cap], outs[0]), f"grid cap {cap} differs from the default grid (T = {T}, C = {C}, {mode})"


@pytest.mark.parametrize("C", [96, 192])
def test_tail_one_cta_against_reference(C):
    """every tile through one CTA, against torch fp32 on the fp16 operands (the tolerance of test_gpu_fused)."""
    T = 128 * 37 + 5
    w = _weights(C, C + 1)
    g = torch.Generator(device=DEV).manual_seed(C + 2)
    x = torch.randn(T, C, generator=g, device=DEV).half()
    att = torch.randn(T, C, generator=g, device=DEV).half()
    want = _mlp_ref(x, att, w["wp"], w["bp"], w["w1"], w["b1"], w["w2"], w["b2"])
    got = x.clone()
    _with_cap(1, lambda: _run(got, att, w))
    d = (got.float() - want.float()).abs()
    err, mean = d.max().item(), d.mean().item()
    assert err < 2e-2 and mean < 6e-4, (err, mean)


@pytest.mark.parametrize("cap", [1, 0])
@pytest.mark.parametrize("C", [96, 192])
def test_tail_leaves_rows_outside_the_call(C, cap):
    """x is a slice of a larger buffer: the rows before it and past T (including those of the last, partial tile) keep their
    sentinel bits, and the rows inside equal the same call on a tensor of its own."""
    T, pad = 128 * 5 + 77, 300
    w = _weights(C, C + 3)
    g = torch.Generator(device=DEV).manual_seed(C + 4)
    x0 = torch.randn(T, C, generator=g, device=DEV).half()
    att = torch.randn(T, C, generator=g, device=DEV).half()
    big = torch.full((pad + T + pad, C), -1234.0, dtype=torch.float16, device=DEV)
    big[pad:pad + T] = x0
    ref = x0.clone()
    _with_cap(cap, lambda: _run(big[pad:pad + T], att, w))
    _with_cap(cap, lambda: _run(ref, att, w))
    assert bool((big[:pad] == -1234.0).all()) and bool((big[pad + T:] == -1234.0).all()), "rows outside the call changed"
    assert torch.equal(big[pad:pad + T], ref)
    assert not torch.equal(ref, x0)
