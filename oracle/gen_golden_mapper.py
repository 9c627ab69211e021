"""Generate tests/golden/mapper.npz by running the REAL reference iw3/mapper.py (and iw3/depth_scaler.py
minmax_normalize) on seeded inputs.  The reference's mapper module needs only torch and math.

Run from the repository root with a checkout of nagadomi/nunif on the path (nothing else of it is needed), as a module so
that oracle/iw3.py does not shadow the reference's iw3 package:
    PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=<nunif checkout> python -m oracle.gen_golden_mapper

Contents
  raw [2,1,48,80]     a seeded raw depth map          pts [1025]  linspace(0, 1) with both end points
  conv [3,1,1,1]      a seeded per-frame convergence
  names               every MAPPER_ALL name but "auto"
  pts/<name>, conv/<name>   get_mapper(name) of pts / conv
  mm/<name>           get_mapper(name)(minmax_normalize(frame, amin, amax)) per frame of raw
  cases, pts/<case>   blends and chains (one chain with two blends: the late-bound lambdas)
  ladder_names, ladder [n, 65]   get_mapper of every distinct name in the resolve table, on pts[::16]
  table_*             resolve_mapper_name(mapper, foreground_scale, metric_depth, mapper_type) -> name
  resolve_err_*, mapper_err_*   the exception type of each invalid call
"""
import os
import numpy as np
import torch

from iw3.mapper import get_mapper, resolve_mapper_name, MAPPER_ALL
from iw3.depth_scaler import minmax_normalize

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

OUT = os.path.join(ROOT, "tests", "golden", "mapper.npz")
torch.set_grad_enabled(False)

CASES = [
    "div_6+div_4=0.5", "div_25+div_10=0.35", "none+div_25=0.05", "div_2+div_1=", "mul_1+mul_2=0.5",
    "inv_mul_3+inv_mul_2=0.25", "inv_mul_1+none=0.7", "none+mul_1=0.68", "shift_045+shift_06=0.4",
    "shift_14+shift_20=0.85", "none+shift_14=0.01", "pow2+softplus=0.3", "softplus+softplus2=1.0", "mul_3+mul_2=0.0",
    "mul_1:div_6", "shift_20:pow2", "none:none", "div_6:div_6:div_6", "pow2:mul_1+mul_2=0.5:softplus",
    "mul_1+mul_2=0.5:div_6+div_1=0.25", "div_6+div_4=0.5:mul_2:inv_mul_1+inv_mul_2=0.75",
    "mul_1:mul_2:mul_3:none:div_6:shift_20:inv_mul_1:softplus",
]
SCALES = [round(-3 + 0.05 * i, 2) for i in range(121)] + [0.005, -0.005, 2.675, -2.675, -2.999, 2.999, 1e-9, -1e-9]
TYPES = {True: [None, "div"], False: [None, "mul", "shift"]}
RESOLVE_ERR = [(None, 1.5, True, "mul"), (None, 1.5, True, "shift"), (None, -0.5, False, "div"), (None, 2, True, "mul"),
               (None, 1, False, "div"), (None, 0.25, False, "foo")]
MAPPER_ERR = ["auto", "foo", "div_6+div_4", "div_6+div_4=1.5", "div_6+div_4=-0.1", "div_6+foo=0.5", "div_6:",
              "div_6+div_4+div_2=0.5", "div_6+div_4=abc", "div_6=0.5", "", "mul_1+mul_2=0.5=0.2", "foo+bar=2", "nan+x=nan"]


def exc_name(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001 - the type is what is recorded
        return type(e).__name__
    return ""


def main():
    g = torch.Generator().manual_seed(0)
    raw = (torch.randn(2, 1, 48, 80, generator=g) * torch.tensor([2.0, 0.3]).view(2, 1, 1, 1)
           + torch.tensor([5.0, -1.0]).view(2, 1, 1, 1))
    pts = torch.linspace(0, 1, 1025, dtype=torch.float32)
    assert pts[0] == 0 and pts[-1] == 1
    conv = torch.rand(3, 1, 1, 1, generator=g)
    out = dict(raw=raw, pts=pts, conv=conv)
    names = [n for n in MAPPER_ALL if n != "auto"]
    out["names"] = np.array(names)
    for n in names:
        f = get_mapper(n)
        out["pts/" + n] = f(pts)
        out["conv/" + n] = f(conv)
        out["mm/" + n] = torch.stack([f(minmax_normalize(d, d.amin(), d.amax())) for d in raw])
    out["cases"] = np.array(CASES)
    for c in CASES:
        out["pts/" + c] = get_mapper(c)(pts)

    rows = []
    for s in SCALES:
        for metric in (True, False):
            for t in TYPES[metric]:
                rows.append((None, s, metric, t))
    for metric in (True, False):
        rows += [("auto", 0.0, metric, None), ("mul_2", 1.5, metric, None), ("div_6+div_4=0.5", -2.0, metric, "shift")]
    out["table_mapper"] = np.array(["None" if r[0] is None else r[0] for r in rows])
    out["table_scale"] = np.array([r[1] for r in rows], dtype=np.float64)
    out["table_metric"] = np.array([r[2] for r in rows])
    out["table_type"] = np.array(["None" if r[3] is None else r[3] for r in rows])
    table = [resolve_mapper_name(mapper=r[0], foreground_scale=r[1], metric_depth=r[2], mapper_type=r[3]) for r in rows]
    out["table_name"] = np.array(table)
    ladder = sorted(set(table) - set(names))
    out["ladder_names"] = np.array(ladder)
    out["ladder"] = torch.stack([get_mapper(n)(pts[::16]) for n in ladder])

    out["resolve_err_args"] = np.array([[str(a) for a in r] for r in RESOLVE_ERR])
    out["resolve_err"] = np.array([exc_name(lambda r=r: resolve_mapper_name(*r)) for r in RESOLVE_ERR])
    out["mapper_err_names"] = np.array(MAPPER_ERR)
    out["mapper_err"] = np.array([exc_name(lambda n=n: get_mapper(n)) for n in MAPPER_ERR])
    assert all(out["resolve_err"]) and all(out["mapper_err"])

    np.savez_compressed(OUT, **{k: (v.numpy() if torch.is_tensor(v) else np.asarray(v)) for k, v in out.items()})
    print("wrote", OUT, os.path.getsize(OUT) // 1024, "KiB,", len(ladder), "ladder names")


if __name__ == "__main__":
    main()
