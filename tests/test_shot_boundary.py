"""TransNetV2 and detect_boundary (iw3 --scene-detect) without a GPU: the oracle against the real reference's fp32 output
(tests/golden/transnetv2.npz), the detector's window plan against the windows the reference ran, the synthetic weights'
key names, and the host contract of the engine's TransNetV2 / detect_boundary."""
import numpy as np
import pytest
import torch

from tests.util import load_golden
from nunif_b200 import synth
from oracle import transnetv2 as otn
from oracle.gen_golden_transnetv2 import LENGTHS, WIN_SEED, U16_SEED, U16_LEN, pts_of

CASES = [(f"len{n}", n, n, False) for n in LENGTHS] + [("u16", U16_SEED, U16_LEN, True)]


@pytest.fixture(scope="module")
def golden():
    return load_golden("transnetv2")


def _frames01(seed, n, use_16bit=False):
    a = synth.shot_sequence(seed, n, use_16bit)
    return torch.from_numpy(a.astype(np.float32)).permute(0, 3, 1, 2) / (65535.0 if use_16bit else 255.0)


def test_synth_keys_match_reference_module(golden):
    assert list(golden["keys"]) == synth.transnetv2_keys() == list(synth.transnetv2_state_dict(0).keys())


@pytest.mark.parametrize("tag,seed,n,u16", CASES)
def test_sequences_regenerate(golden, tag, seed, n, u16):
    a = synth.shot_sequence(seed, n, u16)
    assert a.dtype == (np.uint16 if u16 else np.uint8) and a.shape == (n, 27, 48, 3)
    assert np.array_equal(a.reshape(n, -1).astype(np.int64).sum(1), golden[f"{tag}_sum"])


def test_oracle_window_logits(golden):
    sd = synth.transnetv2_state_dict(0)
    x = torch.from_numpy(synth.shot_sequence(WIN_SEED, 100)).permute(0, 3, 1, 2).float()
    assert np.array_equal(x.flatten(1).sum(1).long().numpy(), golden["win_sum"])
    for tag, xs in (("01", x / 255), ("255", x)):
        one, many = otn.forward(sd, xs)
        for k, v in (("one", one[0]), ("many", many[0])):
            want = torch.from_numpy(golden[f"win{tag}_{k}"])
            assert float((v - want).abs().max()) < 1e-4 * (1 + float(want.abs().max())), (tag, k)


def test_oracle_histograms_see_only_bin_zero_at_unit_scale():
    x = _frames01(3, 10).unsqueeze(0)
    h = otn.color_histograms(x)
    assert int(h[..., 0].min()) == 27 * 48 and int(h[..., 1:].sum()) == 0
    assert torch.equal(otn.hist_band(x)[0, 4], torch.cat([torch.zeros(46), torch.ones(10), torch.zeros(45)]))


@pytest.mark.parametrize("tag,seed,n,u16", CASES)
def test_window_plans_match_reference(golden, tag, seed, n, u16):
    from nunif_b200.nunif.shot_boundary_detection import window_plan
    pts = pts_of(n)
    want = golden[f"{tag}_win_pts"]
    plan, count = window_plan(pts)
    assert count == n
    assert [[pts[i] for i in w] for w in plan] == want.tolist()
    assert [[pts[i] for i in w] for w in otn.windows(pts)] == want.tolist()
    # what is kept: positions [25, 75) of every window, cut to the frame count, is every frame once and in order
    kept = want[:, 25:75].flatten()[:n]
    assert kept.tolist() == pts


@pytest.mark.parametrize("tag,seed,n,u16", [c for c in CASES if c[0] in ("len26", "len137", "u16")])
def test_oracle_detector_matches_reference(golden, tag, seed, n, u16):
    sd = synth.transnetv2_state_dict(0)
    pts = pts_of(n)
    seg, prob = otn.detect(_frames01(seed, n, u16), pts, lambda x: otn.forward(sd, x)[0])
    want = golden[f"{tag}_win_prob"][:, 25:75].flatten()[:n]
    assert float((prob - torch.from_numpy(want)).abs().max()) < 1e-5
    margin = np.abs(want - 0.5)
    ambiguous = {p for p, m in zip(pts, margin) if m < 1e-5}
    assert (seg ^ set(golden[f"{tag}_set"].tolist())) <= ambiguous


def test_window_queue_condition_and_empty_input():
    from nunif_b200.nunif.shot_boundary_detection import WindowQueue, detect_boundary
    with pytest.raises(AssertionError):
        WindowQueue(100, 30)
    with pytest.raises(AssertionError):
        WindowQueue(50, 25)
    with pytest.raises(ValueError):
        WindowQueue().finish()
    with pytest.raises(ValueError):
        detect_boundary([], model=object())   # no frames: the reference fails with an IndexError


def test_checkpoint_path_and_no_download(monkeypatch, tmp_path):
    import os
    from nunif_b200.iw3.base_depth_model import HUB_MODEL_DIR
    from nunif_b200.nunif import transnetv2 as tn

    def no_download(*a, **k):
        raise AssertionError("the engine must not download")
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", no_download)
    assert tn.checkpoint_path() == os.path.join(HUB_MODEL_DIR, "checkpoints", "transnetv2-pytorch-weights.pth")
    with pytest.raises(FileNotFoundError):
        tn.TransNetV2.load(path=str(tmp_path / "missing.pth"))


def test_no_cpu_path():
    from nunif_b200.nunif.transnetv2 import TransNetV2
    from nunif_b200.nunif.shot_boundary_detection import detect_boundary
    with pytest.raises(RuntimeError):
        TransNetV2(synth.transnetv2_state_dict(0), "cpu")
    with pytest.raises(RuntimeError):
        detect_boundary([(np.zeros((27, 48, 3), np.uint8), 0)], device="cpu", model=object())
