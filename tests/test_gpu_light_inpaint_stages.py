"""GPU: every stage of the light_inpaint_v1 forward (nb200_light_inpaint) against a float64 reference of that stage alone
(oracle/light_inpaint_stages.py), fed the engine's own input of the stage through the debug taps (DESIGN.md §5).

Criterion for an fp16 stage output `got` against its reference `ref`, elementwise:
    |got - ref| <= k·ulp16(ref) + 2^-16·Σ|a·w| + 2^-20 (+ flip for the token mixing)
k = 1 for stages with one rounding, 2 for the token mixing (LN2(v)·g2 is rounded to fp16 before the product with Ws) and the
GEMMs with a residual.  flip (ols.token_mix) allows for a v'_m that the engine's fp32 LN2 rounds to the other fp16 neighbour
than the exact value does: without it, outputs with cancellation exceeded the rest of the bound by up to 2.7x on an H100,
identically in the tensor-core and SIMT kernels (they share that LN2 code).  Σ|a·w| bounds the fp32 accumulation error (n·2^-24·Σ|a·w| for n terms, n <= 384 here, and far less
for the pairwise and tensor-core sums in practice), and 2^-20 covers the 5.3e-7 error of the engine's gelu_erf.  The
single-rounding stages must also round at most 1 % of the elements differently from fp16(ref).  The tests of the tests at the
end show that each wrong variant of a reference breaks its bound at least 10 times over."""
import pytest
import torch

from tests.util import log_metric
from nunif_b200 import synth, _lib
from oracle import light_inpaint as oli
from oracle import light_inpaint_stages as ols

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# name: (B, H, W, mirror, seed)
CASES = {
    "70x150": (2, 70, 150, 0, 0),           # W8 = 24: ragged 16-wide x-tiles of proj_out at C = 192; B > 1 with the shift ring
    "70x150_mirror": (2, 70, 150, 1, 0),
    "64x256": (1, 64, 256, 0, 1),           # multiples of 64: the pad is 64, not 0
    "1080p": (1, 1080, 1920, 0, 0),         # production: H4 x W4 = 272 x 496, 576 windows in each shifted block
}
SINGLE, DOUBLE = 1, 2


def tap_specs(B, H, W):
    """id -> (shape, dtype) of the debug taps (DESIGN.md §5)."""
    Hp, Wp = ols.padded(H, W)
    H4, W4 = Hp // 4, Wp // 4
    H8, W8 = H4 // 2, W4 // 2
    f16 = torch.float16
    s = {100: ((B, H, W), torch.float32), 101: ((B, H4, W4, 96), f16)}
    for k, (_, ws, shift, C) in enumerate(ols.BLOCKS):
        h, w = (H8, W8) if C == 192 else (H4, W4)
        p = ws // 2 if shift else 0
        hq, wq, cpad = h + 2 * p, w + 2 * p, (C // 2 + 31) // 32 * 32
        shapes = [(h, w, C), (hq, wq, C), (hq, wq, 4 * C), (hq, wq, 4 * C), (h, w, C), (h, w, C), (h + 2, w + 2, cpad), (h, w, C)]
        for st, sh in enumerate(shapes):
            s[110 + 10 * k + st] = ((B,) + sh, f16)
    s[170] = ((B, H8, W8, 192), f16)
    s[171] = ((B, H4, W4, 96), f16)
    s[172] = ((B, H4 + 2, W4 + 2, 96), f16)
    s[173] = ((B, H4, W4, 48), f16)
    return s


def forward(model, x, hole, mirror, tap_id=None, shape=None, dtype=None):
    """One nb200_light_inpaint call; with tap_id, the tap's buffer (filled with NaN beforehand) too."""
    lib = _lib.lib()
    buf = None
    if tap_id is not None:
        buf = torch.full(shape, float("nan"), dtype=dtype, device=DEV)
        _lib.check(lib.nb200_debug_tap(tap_id, _lib.ptr(buf), buf.numel() * buf.element_size()))
    try:
        out = model.infer(x, hole, mirror=bool(mirror))
    finally:
        lib.nb200_debug_tap(-1, None, 0)
    torch.cuda.synchronize()
    return out, buf


class Run:
    """The output of one case and every tap, each from its own forward."""

    def __init__(self, model, name):
        self.name = name
        self.B, self.H, self.W, self.mirror, seed = CASES[name]
        x, hole = oli.net_inputs(seed, self.B, self.H, self.W)
        self.x, self.hole = x.to(DEV), hole.to(DEV)
        self.out, _ = forward(model, self.x, self.hole, self.mirror)
        self.taps = {}
        for tid, (shape, dtype) in tap_specs(self.B, self.H, self.W).items():
            out, buf = forward(model, self.x, self.hole, self.mirror, tid, shape, dtype)
            assert torch.equal(out, self.out), f"arming tap {tid} changed the output"
            assert not buf.isnan().any(), f"tap {tid} copied short"
            self.taps[tid] = buf
        # stages 2 and 3 again with the SIMT token-mixing kernel (from enc1 on, its rounding changes every later input)
        self.simt = {}
        _lib.lib().nb200_tune_set(7, 1)
        try:
            for tid in [112 + 10 * k + s for k in range(len(ols.BLOCKS)) for s in (0, 1)]:
                shape, dtype = tap_specs(self.B, self.H, self.W)[tid]
                self.simt[tid] = forward(model, self.x, self.hole, self.mirror, tid, shape, dtype)[1]
                assert not self.simt[tid].isnan().any(), f"tap {tid} copied short"
        finally:
            _lib.lib().nb200_tune_set(7, 0)


@pytest.fixture(scope="module")
def sd():
    return {k: v.to(DEV) for k, v in synth.light_inpaint_v1_state_dict(0).items()}


@pytest.fixture(scope="module")
def runs(sd):
    from nunif_b200.iw3 import LightInpaintV1
    model = LightInpaintV1({k: v.cpu() for k, v in sd.items()}, DEV)
    cache = {}

    def get(name):
        if name not in cache:   # all cases stay: the 1080p taps take about 1.5 GB
            cache[name] = Run(model, name)
        return cache[name]

    yield get
    cache.clear()


ulp16 = ols.ulp16


def bound(ref, a, k, flip=0.0):
    return k * ulp16(ref) + 2.0 ** -16 * a + 2.0 ** -20 + flip


def measure(got, ref, a, k, flip=0.0):
    """(max of |got - ref| / bound, max error in ulps of ref, fraction of elements that are not fp16(ref))."""
    err = (got.double() - ref).abs()
    return (float((err / bound(ref, a, k, flip)).max()), float((err / ulp16(ref)).max()),
            float((got.double() != ref.half().double()).double().mean()))


def check(run, stage, got, ref_a, k):
    ref, a = ref_a[0], ref_a[1]
    assert got.shape == ref.shape, (stage, got.shape, ref.shape)
    ratio, ulps, frac = measure(got, ref, a, k, *ref_a[2:])
    log_metric(f"light_inpaint_stage_{run.name}_{stage}", max_ulp=f"{ulps:.3g}", max_over_bound=f"{ratio:.3g}",
               frac_not_rn=f"{frac:.3g}", k=k)
    assert ratio <= 1.0, (run.name, stage, ratio, ulps)
    if k == SINGLE:
        assert frac <= 0.01, (run.name, stage, frac)


def bits(t):
    return t.contiguous().view(torch.int16)


def blocks():
    for k, (p, ws, shift, C) in enumerate(ols.BLOCKS):
        yield k, 110 + 10 * k, p, ws, (ws // 2 if shift else 0), C


BLOCK_STAGES = ["ln_pad", "proj_in", "token_mix", "token_mix_simt", "proj_out", "w1", "pad_glu", "conv3_res"]


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("stage", BLOCK_STAGES)
def test_block_stage(runs, sd, case, stage):
    run = runs(case)
    T = run.taps
    with torch.no_grad():
        for k, b, p, ws, pad, C in blocks():
            name = f"{ols.BLOCKS[k][0]}_{stage}"
            if stage == "ln_pad":
                check(run, name, T[b + 1], ols.ln_pad(sd, p, T[b], pad), SINGLE)
            elif stage == "proj_in":
                check(run, name, T[b + 2], ols.proj_in(sd, p, T[b + 1]), SINGLE)
            elif stage == "token_mix":
                check(run, name, T[b + 3], ols.token_mix(sd, p, T[b + 2], ws), DOUBLE)
            elif stage == "token_mix_simt":
                check(run, name, run.simt[b + 3], ols.token_mix(sd, p, run.simt[b + 2], ws), DOUBLE)
            elif stage == "proj_out":
                check(run, name, T[b + 4], ols.proj_out(sd, p, T[b + 3], T[b], pad), DOUBLE)
            elif stage == "w1":
                check(run, name, T[b + 5], ols.w1(sd, p, T[b + 4]), SINGLE)
            elif stage == "pad_glu":
                check(run, name, T[b + 6], ols.pad_glu(T[b + 5], T[b + 6].shape[-1]), SINGLE)
            else:
                check(run, name, T[b + 7], ols.conv3_res(sd, p, T[b + 6], T[b + 4]), DOUBLE)


@pytest.mark.parametrize("case", list(CASES))
def test_outer_stages(runs, sd, case):
    """The stem, down, up + skip, to_image and the tail."""
    run = runs(case)
    T = run.taps
    with torch.no_grad():
        ref, a, tok = ols.stem(sd, run.x, run.hole, T[100], run.mirror)
        check(run, "stem", T[101], (ref, a), SINGLE)
        check(run, "down", T[170], ols.down(sd, T[117]), SINGLE)
        check(run, "up", T[171], ols.up(sd, T[157], T[117]), DOUBLE)
        check(run, "to_image", T[173], ols.toimg(sd, T[172]), SINGLE)
        d = float((run.out.double() - ols.tail(T[173], run.x, run.hole, T[100], run.mirror)).abs().max())
        log_metric(f"light_inpaint_stage_{run.name}_tail", max_abs=f"{d:.3g}")
        assert d <= 1e-6, d
        # the mask tokens are fp16(mask_bias), bit for bit, and the test sees some
        assert tok.any() and not tok.all()
        mb = sd["mask_bias"].reshape(96).half()
        assert torch.equal(bits(T[101][tok]), bits(mb.expand(int(tok.sum()), 96)))


@pytest.mark.parametrize("case", list(CASES))
def test_exact_invariants(runs, case):
    run = runs(case)
    T = run.taps
    # the taps chain: each block's input is the previous stage's output, bit for bit
    for b, src in ((110, 101), (120, 170), (130, 127), (140, 137), (150, 147), (160, 171)):
        assert torch.equal(bits(T[b]), bits(T[src])), (b, src)
    for k, b, p, ws, pad, C in blocks():
        t1 = bits(T[b + 1])
        if pad:   # the ring rows and columns of T are +0
            ring = torch.ones(t1.shape[1:3], dtype=torch.bool, device=DEV)
            ring[pad:-pad, pad:-pad] = False
            assert (t1[:, ring] == 0).all(), k
        # the token mixing leaves the v half of U alone
        assert torch.equal(bits(T[b + 3][..., 2 * C:]), bits(T[b + 2][..., 2 * C:])), k
        assert torch.equal(bits(run.simt[b + 3][..., 2 * C:]), bits(run.simt[b + 2][..., 2 * C:])), k
        # P: the ring replicates its source, channels >= C/2 are +0
        P = T[b + 6]
        assert torch.equal(bits(P), bits(ols.toimg_pad(P[:, 1:-1, 1:-1]).half())), k
        assert (bits(P[..., C // 2:]) == 0).all(), k
    assert torch.equal(bits(T[172]), bits(ols.toimg_pad(T[167]).half()))


def test_unrelated_tap_leaves_output_unchanged(runs, sd):
    """A ZoeDepth tap id armed during nb200_light_inpaint copies nothing and changes nothing."""
    run = runs("70x150")
    from nunif_b200.iw3 import LightInpaintV1
    model = LightInpaintV1({k: v.cpu() for k, v in sd.items()}, DEV)
    out, buf = forward(model, run.x, run.hole, run.mirror, 5, (1024,), torch.float32)
    assert torch.equal(out, run.out)
    assert buf.isnan().all()


# ---- tests of the tests: a subtly wrong reference fails its stage bound by 10x somewhere ----------------------------------------------------
VARIANTS = ["ws_transposed", "ln2_over_u", "shift_windows_unpadded", "window_tokens_column_major", "stem_without_mirror",
            "tail_without_mirror", "tail_shuffle_dy_dx_c", "up_dy_dx_swapped", "proj_out_1x_residual"]


@pytest.mark.parametrize("variant", VARIANTS)
def test_wrong_reference_fails(runs, sd, variant):
    run = runs("70x150_mirror")
    T = run.taps
    with torch.no_grad():
        if variant.startswith("tail"):
            ref = ols.tail(T[173], run.x, run.hole, T[100], 0 if variant == "tail_without_mirror" else run.mirror,
                           shuffle_order="dy_dx_c" if variant == "tail_shuffle_dy_dx_c" else "c_dy_dx")
            ratio = float((run.out.double() - ref).abs().max()) / 1e-6
        else:
            _, b, p, ws, pad, C = next(blocks())   # enc1: shifted, 16x16 windows
            flip = 0.0
            if variant == "stem_without_mirror":
                got, k, (ref, a, _) = T[101], SINGLE, ols.stem(sd, run.x, run.hole, T[100], 0)
            elif variant == "up_dy_dx_swapped":
                got, k, (ref, a) = T[171], DOUBLE, ols.up(sd, T[157], T[117], swap_dy_dx=True)
            elif variant == "proj_out_1x_residual":
                got, k, (ref, a) = T[b + 4], DOUBLE, ols.proj_out(sd, p, T[b + 3], T[b], pad, residual=1.0)
            else:
                kw = {"ws_transposed": dict(ws_transposed=True), "ln2_over_u": dict(ln_over_u=True),
                      "shift_windows_unpadded": dict(ring=pad), "window_tokens_column_major": dict(col_major=True)}[variant]
                got, k, (ref, a, flip) = T[b + 3], DOUBLE, ols.token_mix(sd, p, T[b + 2], ws, **kw)
            ratio = measure(got, ref, a, k, flip)[0]
    log_metric(f"light_inpaint_wrong_{variant}", max_over_bound=f"{ratio:.3g}")
    assert ratio >= 10, (variant, ratio)
