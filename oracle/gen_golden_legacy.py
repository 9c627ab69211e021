"""Generate tests/golden/upconv_7.npz and tests/golden/vgg_7.npz by running the REAL reference (nagadomi/nunif, a checkout
given by --reference or $NUNIF_REFERENCE, imported read-only) on seeded inputs.  Companion of oracle/gen_golden.py, which
it leaves untouched (its existing fixtures are not regenerated):
    python oracle/gen_golden_legacy.py --reference PATH/TO/nunif

The inputs are not stored: the tests regenerate them from nunif_b200.synth with the seeds kept in each file, and a
16 x 16 corner of every input pins them against synth drift.  Each file holds, for one model:
  x_seeds, x_corner, z          forward of 1 tile of 104 (noisy synthetic image)
  x_odd_seeds, x_odd_corner, z_odd  forward of 2 tiles of the odd size 61 (one smooth, one noisy)
  img_seed, img_hw, img_corner, render   tiled_render of a 96x112 image at tile 104, batch 3 (2 x 2 tiles for both
                                models: two batches, the second one ragged, and seams in both directions)
  cases, configs                SeamBlending.create_config over the size grid of seam_config.npz for (scale, offset, 0)
  query, tile                   find_valid_tile_size for 15 ... 600
"""
import argparse
import os
import sys
import tempfile
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nunif_b200 import synth  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")

TILES = (64, 112, 160, 256, 400)
SIZES = [(1, 1), (17, 33), (220, 220), (240, 240), (256, 256), (300, 420), (1080, 1920), (2160, 3840), (4320, 7680),
         (236, 237), (471, 12)]
# (seed, smooth) of the forward inputs and of the rendered image; the tests rebuild them with legacy_inputs()
X_SEEDS = [(13, False)]
X_ODD_SEEDS = [(14, True), (15, False)]
IMG_SEED, IMG_HW = 12, (96, 112)


def legacy_inputs(x_seeds, size):
    return torch.stack([synth.synth_image(int(s), 3, size, size, smooth=bool(sm)) for s, sm in x_seeds])


def save(name, **arrays):
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **{k: (v.numpy() if torch.is_tensor(v) else np.asarray(v)) for k, v in arrays.items()})
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


def gen_legacy():
    import waifu2x.models  # noqa
    from nunif.models import create_model
    from nunif.utils.render import tiled_render
    from nunif.utils.seam_blending import SeamBlending
    for name, sdf, tag in [("waifu2x.upconv_7", synth.upconv7_state_dict, "upconv_7"),
                           ("waifu2x.vgg_7", synth.vgg7_state_dict, "vgg_7")]:
        m = create_model(name).eval()
        m.load_state_dict(sdf(0), strict=True)
        x = legacy_inputs(X_SEEDS, 104)
        x_odd = legacy_inputs(X_ODD_SEEDS, 61)
        img = synth.synth_image(IMG_SEED, 3, *IMG_HW)
        y = tiled_render(img, m, tile_size=104, batch_size=3)
        scale, offset, blend = m.i2i_scale, m.i2i_offset, 0
        cases, rows = [], []
        for tile in TILES:
            for (h, w) in SIZES:
                p = SeamBlending.create_config((h, w), scale, offset, tile, blend)
                cases.append([h, w, scale, offset, tile, blend])
                rows.append([p["y_h"], p["y_w"], p["h_blocks"], p["w_blocks"], *p["pad"],
                             p["y_buffer_h"], p["y_buffer_w"], p["input_tile_step"], p["output_tile_step"]])
        q = np.arange(15, 601)
        save(tag, x_seeds=np.array(X_SEEDS, dtype=np.int64), x_corner=x[..., :16, :16], z=m(x),
             x_odd_seeds=np.array(X_ODD_SEEDS, dtype=np.int64), x_odd_corner=x_odd[..., :16, :16], z_odd=m(x_odd),
             img_seed=IMG_SEED, img_hw=np.array(IMG_HW), img_corner=img[..., :16, :16], render=y, tile_size=104, batch_size=3,
             scale=scale, offset=offset, cases=np.array(cases, dtype=np.int64), configs=np.array(rows, dtype=np.int64),
             query=q, tile=np.array([m.find_valid_tile_size(int(t)) for t in q]))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=os.environ.get("NUNIF_REFERENCE"), help="checkout of nagadomi/nunif")
    args = ap.parse_args()
    if not args.reference:
        ap.error("give the reference checkout with --reference or $NUNIF_REFERENCE")
    # the reference creates its home directory on import; keep it out of the (read-only) reference tree
    os.environ.setdefault("NUNIF_HOME", tempfile.mkdtemp(prefix="nunif_home_"))
    sys.path.insert(0, os.path.abspath(args.reference))
    torch.set_grad_enabled(False)
    torch.manual_seed(0)
    gen_legacy()
