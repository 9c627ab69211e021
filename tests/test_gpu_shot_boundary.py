"""GPU parity of TransNetV2 and detect_boundary (iw3 --scene-detect, csrc/transnet.cu + the wgmma GEMM): logits within a
small multiple of the PyTorch GPU path's own error, the exact histogram taps, batch invariance, the segment sets of the real
reference (tests/golden/transnetv2.npz), no host synchronisation before the end, and the scene flags driving the EMA
normaliser's flushes."""
import contextlib
import numpy as np
import pytest
import torch

from tests.util import load_golden, log_metric, stats
from nunif_b200 import synth
from oracle import transnetv2 as otn
from oracle.gen_golden_transnetv2 import LENGTHS, U16_SEED, U16_LEN, pts_of

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CASES = [(f"len{n}", n, n, False) for n in LENGTHS] + [("u16", U16_SEED, U16_LEN, True)]


@pytest.fixture(scope="module")
def sd():
    return synth.transnetv2_state_dict(0)


@pytest.fixture(scope="module")
def model(sd):
    from nunif_b200.nunif.transnetv2 import TransNetV2
    return TransNetV2(sd, DEV)


@pytest.fixture(scope="module")
def golden():
    return load_golden("transnetv2")


@contextlib.contextmanager
def torch_default_backends():
    """The precision the reference runs with: torch's defaults, TF32 cuDNN convolutions and fp32 matmuls.  Set explicitly,
    since an earlier test of the session may have left other values behind."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = False, True
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _windows(B, T, scale):
    x = torch.stack([torch.from_numpy(synth.shot_sequence(900 + b, T)).permute(0, 3, 1, 2).float() for b in range(B)])
    return x if scale == 255 else x / 255


def _tap(model, tap_id, x, nbytes, dtype):
    from nunif_b200 import _lib
    buf = torch.zeros(nbytes // torch.tensor([], dtype=dtype).element_size(), dtype=dtype, device=DEV)
    _lib.check(_lib.lib().nb200_debug_tap(tap_id, _lib.ptr(buf), nbytes))
    try:
        model(x)
    finally:
        _lib.lib().nb200_debug_tap(-1, None, 0)
    torch.cuda.synchronize()
    return buf


@pytest.mark.parametrize("scale", [1, 255])
@pytest.mark.parametrize("B,T", [(1, 100), (3, 100), (1, 37), (3, 37)])
def test_logits_within_gpu_reference_error(model, sd, B, T, scale):
    x = _windows(B, T, scale)
    one, extra = model(x.to(DEV))
    with torch.no_grad():
        want_one, want_many = otn.forward(sd, x)                       # fp32 on the CPU
        sdg = {k: v.to(DEV) for k, v in sd.items()}
        with torch_default_backends():
            ref_one, ref_many = otn.forward(sdg, x.to(DEV))           # torch's default GPU path (TF32 convolutions)
    assert one.shape == (B, T, 1) and extra["many_hot"].shape == (B, T, 1)
    for name, got, ref, want in (("one_hot", one[..., 0], ref_one, want_one), ("many_hot", extra["many_hot"][..., 0], ref_many, want_many)):
        e, r = stats(got.cpu(), want), stats(ref.cpu(), want)
        log_metric(f"transnetv2_{name}_B{B}_T{T}_s{scale}", engine_max=e["max"], engine_mean=e["mean"], engine_p999=e["p999"],
                   torch_gpu_max=r["max"], torch_gpu_mean=r["mean"], torch_gpu_p999=r["p999"])
        for k in ("max", "mean", "p999"):
            assert e[k] <= 4 * r[k] + 2e-3, (name, k, e, r)


@pytest.mark.parametrize("scale", [1, 255])
def test_histogram_taps_exact(model, scale):
    B, T = 2, 37
    x = _windows(B, T, scale)
    n = B * T
    counts = _tap(model, 200, x.to(DEV), n * 512 * 4, torch.int32).view(B, T, 512).cpu()
    want = otn.color_histograms(x)
    assert torch.equal(counts.long(), want)
    # the band: the cosine similarity of the exact counts, correctly rounded (torch's fp32 bmm differs by a few ulp)
    band = _tap(model, 201, x.to(DEV), n * 101 * 4, torch.float32).view(B, T, 101).cpu()
    c = want.double()
    exact = otn.band(c / c.norm(dim=2, keepdim=True)).float()
    assert float((band - exact).abs().max()) < 1e-6
    if scale == 1:
        assert torch.equal(band, otn.hist_band(x))   # every pixel in bin 0: the band is exactly 1 inside the window, 0 outside


def test_stack_and_fc1_taps(model, sd):
    B, T = 1, 37
    x = _windows(B, T, 1)
    feats = otn.stacks(sd, x)
    row = otn.fc1_input(sd, x)
    for tap_id, want in ((203, feats[0].permute(0, 2, 3, 4, 1)), (204, feats[1].permute(0, 2, 3, 4, 1)), (205, row)):
        got = _tap(model, tap_id, x.to(DEV), want.numel() * 2, torch.float16).view(want.shape).float().cpu()
        s = stats(got, want)
        log_metric(f"transnetv2_tap{tap_id}", **s)
        assert s["max"] < 2e-2 * (1 + float(want.abs().max())), (tap_id, s)


def test_batch_invariance(model):
    x = _windows(3, 100, 1).to(DEV)
    alone = model(x[1])[0]
    batched = model(x)[0]
    assert torch.equal(alone[0], batched[1])
    short = model(x[1, :37])[0]
    assert torch.equal(short[0], model(x[:, :37])[0][1])


def _golden_probs(golden, tag, n):
    pts = golden[f"{tag}_win_pts"][:, 25:75].flatten()[:n]
    prob = golden[f"{tag}_win_prob"][:, 25:75].flatten()[:n]
    return pts, prob


def _logit_bound(model, golden):
    """max |engine logit - reference logit| over the windows of the golden sequences"""
    e = 0.0
    for tag, seed, n, u16 in CASES:
        a = synth.shot_sequence(seed, n, u16)
        x = torch.from_numpy(a.astype(np.float32)).permute(0, 3, 1, 2) / (65535.0 if u16 else 255.0)
        idx = {p: i for i, p in enumerate(pts_of(n))}
        w = torch.tensor([[idx[p] for p in row] for row in golden[f"{tag}_win_pts"]])
        got = model(x[w].to(DEV))[0][..., 0].cpu()
        want = torch.logit(torch.from_numpy(golden[f"{tag}_win_prob"]).double()).float()
        e = max(e, float((got - want).abs().max()))
    return e


@pytest.mark.parametrize("batch", [1, 8])
def test_segment_sets_match_reference(model, golden, monkeypatch, batch):
    from nunif_b200.nunif import shot_boundary_detection as sbd
    monkeypatch.setattr(sbd, "WINDOW_BATCH", batch)
    bound = _logit_bound(model, golden)
    delta = 0.5 * bound   # sigmoid' <= 1/4: a probability moves by at most bound / 4; twice that as margin
    assert bound < 0.1, bound
    excluded = 0
    for tag, seed, n, u16 in CASES:
        frames = synth.shot_sequence(seed, n, u16)
        seg = sbd.detect_boundary(zip(frames, pts_of(n)), device=DEV, model=model)
        pts, prob = _golden_probs(golden, tag, n)
        ambiguous = {int(p) for p, q in zip(pts, prob) if abs(q - 0.5) < delta}
        excluded += len(ambiguous)
        assert (seg ^ set(golden[f"{tag}_set"].tolist())) <= ambiguous, tag
    log_metric(f"transnetv2_sets_batch{batch}", logit_bound=bound, delta=delta, excluded_frames=excluded)


def test_no_host_sync_before_the_end(model, golden):
    from nunif_b200.nunif import shot_boundary_detection as sbd
    n = 137
    frames = synth.shot_sequence(n, n)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        prob, kept = sbd._predict(zip(frames, pts_of(n)), torch.device(DEV), 100, 25, model)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    pts, want = _golden_probs(golden, f"len{n}", n)
    assert kept[:n] == pts.tolist() and prob.shape == (n,)
    assert float((prob.cpu() - torch.from_numpy(want)).abs().max()) < 0.05


def test_scene_flags_drive_minmax_flush(model, golden):
    """iw3/utils.py:748,805: reset_ema = [t in segment_pts for t in pts]; minmax_normalize flushes the EMA window at each."""
    from nunif_b200.nunif.shot_boundary_detection import detect_boundary
    from nunif_b200.iw3.base_depth_model import BaseDepthModel
    from nunif_b200.iw3.depth_scaler import EMAMinMaxScaler
    n = 137
    pts = pts_of(n)
    seg = detect_boundary(zip(synth.shot_sequence(n, n), pts), device=DEV, model=model)
    assert seg, "the sequence has boundaries"
    dm = BaseDepthModel.__new__(BaseDepthModel)
    dm.scaler = EMAMinMaxScaler(decay=0.9, buffer_size=3)
    depth = torch.rand(n, 1, 8, 12, generator=torch.Generator().manual_seed(5)).to(DEV)
    flags = [p in seg for p in pts]
    done, flushed_at = 0, []
    for i in range(0, n, 10):   # batches of 10 frames, as a video callback sees them
        out = dm.minmax_normalize(depth[i:i + 10], reset_ema=flags[i:i + 10])
        done += len(out)
        if any(flags[i:i + 10]):
            last = max(k for k in range(i, min(i + 10, n)) if flags[k])
            assert done >= last + 1   # every frame up to the scene end has come out
            flushed_at.append(last)
    assert flushed_at and {pts[k] for k in flushed_at} <= seg
    pts_g, prob = _golden_probs(golden, f"len{n}", n)
    assert seg == set(golden[f"len{n}_set"].tolist()) or all(abs(q - 0.5) < 0.05 for p, q in zip(pts_g, prob)
                                                             if (int(p) in seg) != (int(p) in set(golden[f"len{n}_set"].tolist())))
