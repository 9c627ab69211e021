"""CPU: the oracle of `sbs.row_flow_v2` and of the symmetric row_flow_v3_sym driver against the real reference's fp32 output
(tests/golden/row_flow_v2.npz, oracle/gen_golden_row_flow_v2.py), and load_row_flow_model's method table and errors."""
import os
import re
import pytest
import torch

from tests.util import load_golden, t
from nunif_b200 import synth
from oracle import row_flow as orf, row_flow_v2 as orf2
from oracle.gen_golden_row_flow_v2 import LR_CASES, SYM_CASES, VIEWS, lr_inputs, sym_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_oracle_v2_delta_golden():
    g = load_golden("row_flow_v2")
    sd = synth.row_flow_v2_state_dict(0)
    for i in range(4):
        got = orf2.row_flow_v2_delta(sd, t(g[f"net{i}_x"]))
        assert got.shape == g[f"net{i}_delta"].shape
        assert float((got - t(g[f"net{i}_delta"])).abs().max()) < 1e-5, i


def test_oracle_v2_lr_golden():
    g = load_golden("row_flow_v2")
    sd = synth.row_flow_v2_state_dict(0)
    d, c = lr_inputs()
    assert torch.equal(d[..., :8, :8], t(g["v2_d_corner"])) and torch.equal(c[..., :8, :8], t(g["v2_c_corner"]))
    for i, (div, conv, view, steps, psb) in enumerate(LR_CASES):
        left, right = orf2.apply_divergence_nn_delta_LR(lambda x: orf2.row_flow_v2_delta(sd, x), c, d, div, conv, VIEWS[view],
                                                       steps=steps, preserve_screen_border=bool(psb))
        for tag, eye in (("left", left), ("right", right)):
            if f"v2lr{i}_{tag}" in g:
                assert float((eye - t(g[f"v2lr{i}_{tag}"])).abs().max()) < 1e-5, (i, tag)
            else:
                assert eye is c


def test_oracle_symmetric_golden():
    g = load_golden("row_flow_v2")
    sd = synth.row_flow_v3_state_dict(2)
    for i, (div, conv, view, h, w, H, W) in enumerate(SYM_CASES):
        d, c = sym_inputs(i, h, w, H, W)
        assert torch.equal(d[..., :8, :8], t(g[f"sym{i}_d"])) and torch.equal(c[..., :8, :8], t(g[f"sym{i}_c"]))
        left, right = orf2.apply_divergence_nn_symmetric(lambda x: orf.row_flow_delta(sd, x), c, d, div, conv, VIEWS[view])
        for tag, eye in (("left", left), ("right", right)):
            if f"sym{i}_{tag}" in g:
                assert float((eye - t(g[f"sym{i}_{tag}"])).abs().max()) < 1e-5, (i, tag)
            else:
                assert eye is c
    # the portrait case pins image_width = W: max(H, W) would double the divergence feature
    assert SYM_CASES[-1][3] > SYM_CASES[-1][4]


def test_load_row_flow_model_method_table():
    from nunif_b200.iw3 import RowFlowV2, RowFlowV3
    from nunif_b200.iw3.row_flow import ROW_FLOW_METHODS
    want = {"row_flow": (RowFlowV3, False, "iw3_row_flow_v3_20250627.pth"),
            "row_flow_v3": (RowFlowV3, False, "iw3_row_flow_v3_20250627.pth"),
            "row_flow_sym": (RowFlowV3, True, "iw3_row_flow_v3_sym_20250628.pth"),
            "row_flow_v3_sym": (RowFlowV3, True, "iw3_row_flow_v3_sym_20250628.pth"),
            "row_flow_v2": (RowFlowV2, False, "iw3_row_flow_v2_20240130.pth")}
    assert ROW_FLOW_METHODS == want
    assert RowFlowV2.name == "sbs.row_flow_v2" and RowFlowV2.symmetric is False and RowFlowV2.delta_output
    assert RowFlowV3.name == "sbs.row_flow_v3"


def test_load_row_flow_model_errors(tmp_path):
    from nunif_b200.iw3 import load_row_flow_model
    with pytest.raises(ValueError):
        load_row_flow_model("row_flow_v1", path=str(tmp_path / "x.pth"))
    with pytest.raises(FileNotFoundError, match="does not download"):
        load_row_flow_model("row_flow_v2", path=str(tmp_path / "missing.pth"))
    p = tmp_path / "v3.pth"
    torch.save({"name": "sbs.row_flow_v3", "state_dict": synth.row_flow_v3_state_dict(0)}, str(p))
    for m in ("row_flow_v2",):
        with pytest.raises(ValueError, match="sbs.row_flow_v3"):
            load_row_flow_model(m, path=str(p))
    p2 = tmp_path / "v2.pth"
    torch.save({"name": "sbs.row_flow_v2", "state_dict": synth.row_flow_v2_state_dict(0)}, str(p2))
    for m in ("row_flow", "row_flow_v3", "row_flow_sym", "row_flow_v3_sym"):
        with pytest.raises(ValueError, match="expected 'sbs.row_flow_v3'"):
            load_row_flow_model(m, path=str(p2))


def test_header_declares_row_flow_v2_entry_points():
    src = open(os.path.join(ROOT, "include", "nunif_b200.h")).read()
    assert re.search(r"NB200_MODEL_ROW_FLOW_V2\s*=\s*16", src)
    for s in ("nb200_row_flow_v2_delta", "nb200_backward_warp_delta_sym", "nb200_backward_warp_delta_f16"):
        assert re.search(r"\bint\s+" + s + r"\s*\(", src), s
