"""Generate tests/golden/null_depth.npz by running the REAL reference iw3/null_depth_model.py (NullDepthModel.load on the
CPU, then infer) on the seeded frames of oracle/null_depth.py, in fp32, with one intra-op thread (the last bits of ATen's
CPU bilinear resize depend on the thread count).

Run from the repository root, as a module:
    NUNIF_HOME=/tmp/nunif_home PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=<nunif checkout> python -m oracle.gen_golden_null_depth

  <case>/input_sum, input_corner    float64 sum and the [..., :8, :8] corner of the frames, so a change of the seeded
                                    frames shows
  <case>/t<tta>_d<dil>/shape        infer(frames, tta=bool(tta), edge_dilation=dil).shape
  <case>/t<tta>_d<dil>/sha256       SHA-256 of that output's fp32 bytes
  <case>/t<tta>_d<dil>/crop<i>      its null_depth.crops
"""
import os

import numpy as np
import torch

from oracle import null_depth as ond

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "null_depth.npz")


def main():
    from iw3.null_depth_model import NullDepthModel
    torch.set_num_threads(1)
    out = {}
    for case in ond.CASES:
        name, resolution = case[0], case[4]
        x = ond.frames(case)
        out[f"{name}/input_sum"] = np.array(float(x.double().sum()))
        out[f"{name}/input_corner"] = x[..., :8, :8].numpy()
        model = NullDepthModel("NULL")
        model.load(gpu=-1, resolution=resolution)
        for tta, dil in ond.VARIANTS:
            y = model.infer(x.clone(), tta=bool(tta), edge_dilation=dil)
            assert torch.equal(y, ond.infer(x.clone(), resolution, bool(tta), dil)), (name, tta, dil)
            key = f"{name}/t{tta}_d{dil}"
            out[f"{key}/shape"] = np.array(y.shape)
            out[f"{key}/sha256"] = ond.digest(y.numpy())
            for i, c in enumerate(ond.crops(y)):
                out[f"{key}/crop{i}"] = c.numpy()
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
