"""Generate tests/golden/zoedepth_any_infer.npz: the REAL iw3/zoedepth_model.py batch_infer and batch_preprocess with
prep_mod = 14 (the ZoeD_Any setting, :190-199) around a stand-in network - the third-party DepthAnythingMetricDepth module is
replaced by the oracle's restatement (oracle/zoedepth_any.py, reduced widths) behind the same `model(x)['metric_depth']`
interface - so the golden pins the reference's wrapper logic while the network stays pinned to transformers
(tests/test_zoedepth_any.py).  Also the mod-14 size rule and pads for common frame sizes.

Needs the reference (nagadomi/nunif) importable, as the other golden generators (oracle/gen_golden.py):
    NUNIF_HOME=/tmp/nunif_home PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=<nunif checkout>:. python oracle/gen_golden_zoedepth_any.py
"""
import os
import sys
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("NUNIF_HOME", "/tmp/nunif_home")
sys.path.insert(0, os.environ.get("NUNIF_REFERENCE", "/root/reference"))   # the location oracle/gen_golden.py uses

from nunif_b200 import synth  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
torch.set_grad_enabled(False)

# (H, W, h_height, v_height): 720p, 1080p, 4K, portrait 1080x1920, square, smaller than 392, resolution = 518
SIZES = [(720, 1280, 392, 518), (1080, 1920, 392, 518), (2160, 3840, 392, 518), (1920, 1080, 392, 518), (512, 512, 392, 518),
         (300, 200, 392, 518), (240, 320, 392, 518), (1080, 1920, 518, 518), (1920, 1080, 518, 518)]


def main():
    from iw3.zoedepth_model import batch_infer as ref_batch_infer, batch_preprocess as ref_batch_preprocess
    from oracle import zoedepth_any as oza
    out = {}
    rows = []
    for H, W, hh, vh in SIZES:
        y, pad_h, pad_w = ref_batch_preprocess(torch.rand(1, 3, H, W), h_height=hh, v_height=vh, ensure_multiple_of=14)
        rows.append([H, W, hh, vh, y.shape[2], y.shape[3], pad_h, pad_w])
    out["sizes"] = np.array(rows, dtype=np.int64)
    # the frames are regenerated from their seeds by the tests; a checksum and a corner of each detect a synth change
    land_seeds, land_hw, port_seed, port_hw = (81, 82), (54, 96), 83, (72, 48)
    land = torch.stack([synth.synth_image(s, 3, *land_hw, smooth=False) for s in land_seeds])
    port = synth.synth_image(port_seed, 3, *port_hw, smooth=False)
    out.update(land_seeds=np.array(land_seeds), land_hw=np.array(land_hw), port_seed=np.array(port_seed), port_hw=np.array(port_hw),
               land_sum=np.array(float(land.double().sum())), port_sum=np.array(float(port.double().sum())),
               land_corner=land[..., :8, :8], port_corner=port[..., :8, :8])
    for normed in (False, True):
        tag = "k" if normed else "n"
        sd = synth.zoedepth_any_state_dict(5, synth.ZOED_ANY_MINI, normed=normed)

        class Stub:
            device = torch.device("cpu")
            prep_h_height, prep_v_height, prep_mod = 56, 70, 14

            def __call__(self, x):
                return {"metric_depth": oza.zoedepth_any_forward(sd, x, oza.ZOED_ANY_MINI, normed)}

        for flip in (0, 1):
            for dil in (0, 2):
                out[f"{tag}_land_f{flip}_d{dil}"] = ref_batch_infer(Stub(), land.clone(), flip_aug=bool(flip), enable_amp=False, edge_dilation=dil)
                out[f"{tag}_port_f{flip}_d{dil}"] = ref_batch_infer(Stub(), port.clone(), flip_aug=bool(flip), enable_amp=False, edge_dilation=dil)
    path = os.path.join(OUT, "zoedepth_any_infer.npz")
    np.savez_compressed(path, **{k: (v.numpy() if torch.is_tensor(v) else np.asarray(v)) for k, v in out.items()})
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
