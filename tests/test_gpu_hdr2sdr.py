"""GPU: the fused hdr2sdr kernel (csrc/hdr2sdr.cu) against the oracle evaluated on CUDA - the reference's own op sequence
(nunif/utils/video.py:309-416) with device= the GPU - and against the reference's CPU output (tests/golden/hdr2sdr.npz); its
float output against hwc_to_chw_float of its uint16 output; FrameBatchPipeline(hdr2sdr=...) against tone-mapping first.

Against the reference's CPU output a sample may differ by 1 code more than the reference's own GPU run (the oracle on
CUDA) differs from it: at most 1 code for HLG, a few codes in PQ's darks (see test_uint16_matches_oracle_and_reference).

Where the kernel may differ from the CUDA oracle: only the 3x3 colour matrix.  torch.mm (cuBLAS) sums its three products
in an unspecified order; each of two evaluations lies within gamma_3 * S of the exact sum (S = sum_j |m_ij * s_j|,
gamma_3 ~ 3u, u = 2^-24), so they differ by at most 6u * S.  The clamps are 1-Lipschitz; the OETF's slope is 4.5 below
0.018 and 1.099 * 0.45 * v^-0.55 above, so the value the cast truncates moves by at most 65535 * slope * 6u * S, plus a
few ulps of the scaled value (2^-5 code) for the OETF's own roundings of a different input.  A pixel may therefore be
off by 1 code where the oracle's scaled value lies within that bound of an integer, and by up to the OETF's jump at 0.018
(OETF_JUMP codes) where the oracle's linear value lies within 6u * S of 0.018.  Everything else must be equal.

The oracle runs on CUDA with TF32 matmul off (PyTorch's default)."""
import numpy as np
import pytest
import torch

from oracle import hdr2sdr as ohs
from tests.util import load_golden, log_metric, true_fp32

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24
# 65535 * (1.099 * 0.018^0.45 - 0.099 - 4.5 * 0.018) rounded up: the codes the OETF jumps by at its switch
OETF_JUMP = int(np.ceil(65535 * abs(1.099 * 0.018 ** 0.45 - 0.099 - 4.5 * 0.018))) + 1


def oracle_cuda(x, trc, cs, **kw):
    """The oracle on the GPU, frame by frame: uint16 [B][H][W][3], and the allowance of each sample ([B][H][W][3] int:
    0 = must be equal, 1 = may differ by 1 code, OETF_JUMP = near the OETF switch)."""
    outs, allow = [], []
    mat = torch.tensor(ohs.MATRIX[cs], dtype=torch.float64, device=DEV)
    for f in x:
        taps = {}
        with true_fp32():
            outs.append(ohs.hdr2sdr(f, trc, cs, device=DEV, taps=taps, **kw))
        s = taps["sdr"].double()
        S = (mat.abs()[:, :, None, None] * s.abs()[None]).sum(1)               # [3][H][W]
        dlin = 6 * U * S
        lin, scaled = taps["linear"].double(), taps["scaled"].double()
        slope = torch.where(lin - dlin < 0.018, torch.full_like(lin, 4.5), 1.099 * 0.45 * (lin - dlin).clamp_min(0.018) ** -0.55)
        bound = 65535 * slope * dlin + 2.0 ** -5
        a = torch.where((scaled - scaled.round()).abs() <= bound, 1, 0)
        a = torch.where((lin - np.float32(0.018).item()).abs() <= dlin, OETF_JUMP, a)
        allow.append(a.permute(1, 2, 0))
    return torch.stack(outs), torch.stack(allow)


def check_against_oracle(got, x, trc, cs, tag, **kw):
    want, allow = oracle_cuda(x, trc, cs, **kw)
    d = (got.to(DEV).int() - want.int()).abs()
    assert bool((d <= allow).all()), f"{tag}: {int((d > allow).sum())} samples off beyond the matrix-order bound, max {int(d.max())}"
    log_metric("hdr2sdr_vs_cuda_oracle", case=tag, samples=d.numel(), differ=int((d > 0).sum()), max=int(d.max()),
               allowed_1=int((allow == 1).sum()), near_switch=int((allow == OETF_JUMP).sum()))
    assert int((d > 0).sum()) <= max(16, d.numel() // 1000), tag          # the reordered matrix sum rarely matters
    return want


@pytest.fixture(scope="module")
def golden():
    return load_golden("hdr2sdr")


@pytest.mark.parametrize("config", ohs.CONFIGS, ids=[c[0] for c in ohs.CONFIGS])
def test_uint16_matches_oracle_and_reference(config, golden):
    from nunif_b200.nunif.video import hdr2sdr
    cname, trc, cs, kw = config
    for name, x in ohs.golden_inputs().items():
        got = hdr2sdr(x, trc, cs, device=DEV, **kw)
        assert got.shape == x.shape and got.dtype == torch.uint16 and got.is_cuda
        want = check_against_oracle(got[None], x[None], trc, cs, f"{cname}/{name}", **kw)[0]
        ref = torch.from_numpy(ohs.reference_output(golden, config, name, x).astype(np.int32))
        d = (got.cpu().int() - ref).abs()
        d_gpu_ref = (want.cpu().int() - ref).abs()
        log_metric("hdr2sdr_vs_cpu_reference", case=f"{cname}/{name}", differ=int((d > 0).sum()), max=int(d.max()),
                   oracle_cuda_max=int(d_gpu_ref.max()))
        # the reference's own CPU and GPU runs differ where libdevice's powf / expf and the CPU's differ by an ulp; in PQ's
        # darks x^(1/m2) - c1 cancels and the quotient is raised to 1/m1 ~ 6.28, which grows that ulp into a few codes
        assert bool((d <= d_gpu_ref + 1).all()), (cname, name, int(d.max()))
        if trc == ohs.HLG:
            assert int(d.max()) <= 1, (cname, name, int(d.max()))


@pytest.mark.parametrize("B,H,W", [(1, 2160, 3840), (3, 2160, 3837)])
@pytest.mark.parametrize("trc,cs", [(ohs.PQ, "bt709"), (ohs.HLG, "bt601")])
def test_4k_batches_match_oracle(B, H, W, trc, cs):
    from nunif_b200.nunif.video import hdr2sdr
    g = torch.Generator().manual_seed(7 + B)
    x = torch.randint(0, 65536, (B, H, W, 3), generator=g, dtype=torch.int32).to(torch.uint16)
    got = hdr2sdr(x.to(DEV), trc, cs)
    check_against_oracle(got, x, trc, cs, f"4k/{B}x{H}x{W}/{trc}/{cs}")


def test_float_output_is_hwc_to_chw_of_uint16_output():
    from nunif_b200.nunif.video import hdr2sdr
    from nunif_b200.iw3 import hwc_to_chw_float
    g = torch.Generator().manual_seed(3)
    x = torch.randint(0, 65536, (2, 361, 643, 3), generator=g, dtype=torch.int32).to(torch.uint16).to(DEV)
    for trc, cs, kw in ((16, "bt709", {}), (18, "bt601", {}), (18, "bt709", dict(hlg_saturation_gain=1.0))):
        u = hdr2sdr(x, trc, cs, **kw)
        f = hdr2sdr(x, trc, cs, output="float", **kw)
        assert f.shape == (2, 3, 361, 643) and f.dtype == torch.float32
        assert torch.equal(f, hwc_to_chw_float(u))
        assert torch.equal(hdr2sdr(x[1], trc, cs, output="float", **kw), f[1])


def test_unaligned_and_partial_blocks():
    """A frame whose data pointer is not 16-byte aligned (the per-element staging path) and a pixel count that leaves a
    partial last block give the same pixels as an aligned copy."""
    from nunif_b200.nunif.video import hdr2sdr
    g = torch.Generator().manual_seed(4)
    H, W = 37, 53
    flat = torch.randint(0, 65536, (H * W * 3 + 1,), generator=g, dtype=torch.int32).to(torch.uint16).to(DEV)
    x = flat[1:].view(1, H, W, 3)
    assert x.data_ptr() % 16 != 0
    for trc, cs in ((16, "bt601"), (18, "bt709")):
        want = hdr2sdr(x.clone(), trc, cs)
        assert torch.equal(hdr2sdr(x, trc, cs), want)
        assert torch.equal(hdr2sdr(x, trc, cs, output="float"), hdr2sdr(x.clone(), trc, cs, output="float"))
        check_against_oracle(want, x.cpu(), trc, cs, f"unaligned/{trc}/{cs}")


@pytest.mark.parametrize("batch,depth,n", [(3, 3, 8), (4, 2, 9), (1, 2, 3)])
def test_pipeline_hdr2sdr_equals_tone_mapping_first(batch, depth, n):
    from nunif_b200.nunif.video import FrameBatchPipeline, hdr2sdr
    g = torch.Generator().manual_seed(9)
    frames = [torch.randint(0, 65536, (72, 130, 3), generator=g, dtype=torch.int32).to(torch.uint16) for _ in range(n)]
    for trc, cs in ((16, "bt709"), (18, "bt601")):
        seen = []

        def cb(x):
            seen.append(x.shape[0])
            return x
        pipe = FrameBatchPipeline(cb, batch, DEV, depth=depth, use_16bit=True, hdr2sdr=(trc, cs))
        out = []
        for f in frames:
            out += pipe(f)
        out += pipe(None)
        plain = FrameBatchPipeline(lambda x: x, batch, DEV, depth=depth, use_16bit=True)
        want = []
        for f in frames:
            want += plain(hdr2sdr(f, trc, cs, device=DEV).cpu())
        want += plain(None)
        assert len(out) == len(want) == n and seen[-1] == (n % batch or batch)
        for o, w in zip(out, want):
            assert torch.equal(o, w)
