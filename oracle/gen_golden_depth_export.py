"""Generate tests/golden/depth_export.npz from the reference's own export_images and process_config_images
(iw3/utils.py:1226-1347, :1831-1932), run from the source file via ast with their real globals where they import
(iw3/utils.py itself imports PyAV).  The depth model is the reference's NullDepthModel on the CPU.

Stored per export case: the NullDepthModel.infer outputs in call order, the 16-bit depth PNG pixels and text chunks, and
the iw3_export.yml without updated_at.  Per import case: the depth map as written (pixels, text), load_depth's output,
and the float SBS image process_config_images passes to to_pil_image.  Run: python oracle/gen_golden_depth_export.py"""
import ast
import json
import os
import sys
import tempfile
from fractions import Fraction
from argparse import Namespace
from os import path

import numpy as np
import torch
import yaml

ROOT = path.dirname(path.dirname(path.abspath(__file__)))
REF = "/root/reference"
sys.path.insert(0, REF)

import torch.nn.functional as F  # noqa: E402
from PIL import Image  # noqa: E402
from torchvision.transforms import functional as TF, InterpolationMode  # noqa: E402
from torchvision.transforms.functional import to_pil_image  # noqa: E402
from iw3 import export_config  # noqa: E402
from iw3.anaglyph import apply_anaglyph_redcyan  # noqa: E402
from iw3.base_depth_model import BaseDepthModel  # noqa: E402
from iw3.dilation import dilate_edge, edge_dilation_is_enabled  # noqa: E402
from iw3.forward_warp import apply_divergence_forward_warp  # noqa: E402
from iw3.mapper import get_mapper  # noqa: E402
from iw3.null_depth_model import NullDepthModel  # noqa: E402
from nunif.utils.image_loader import ImageLoader  # noqa: E402
from nunif.utils.pil_io import load_image_simple  # noqa: E402
from concurrent.futures import ThreadPoolExecutor  # noqa: E402

FUNCS = ("export_images", "process_config_images", "preprocess_image", "apply_divergence", "postprocess_padding",
         "postprocess_image", "make_output_filename", "get_image_ext")
IMAGE_SIZES = ((40, 56), (33, 47))     # (H, W); the second is odd in both axes
EXPORT_CASES = {
    # name: (resolution of NullDepth, export_disparity, mapper, export_depth_fit)
    "plain": (24, False, "none", False),
    "disparity_div6": (24, True, "div_6", False),
    "disparity_blend": (24, True, "mul_1+mul_2=0.5", False),
    "fit_up": (24, False, "none", True),
    "fit_down": (96, False, "none", True),
    "disparity_fit": (20, True, "div_6", True),
}
IMPORT_CASES = {
    # name: (export case whose output is converted, how the depth maps are rewritten)
    "u16": ("plain", None),
    "u16_skip": ("disparity_div6", None),
    "u8_rgb": ("plain", "u8_rgb"),
    "u16_range": ("plain", "range"),
    "u16_fit": ("fit_up", None),
}
DEPTH_RANGE = (0.125, 0.8125)


class _NoBar:
    def __init__(self, *a, **k):
        pass

    def update(self, n=1):
        pass

    def close(self):
        pass


def reference_functions(captured_sbs):
    src = open(path.join(REF, "iw3", "utils.py")).read()
    tree = ast.parse(src)
    nodes = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in FUNCS]
    consts = [n for n in tree.body if isinstance(n, ast.Assign) and isinstance(n.targets[0], ast.Name)
              and (n.targets[0].id.endswith("_SUFFIX") or n.targets[0].id in ("SMB_INVALID_CHARS", "IMAGE_IO_QUEUE_MAX"))]

    def capture_pil(x):
        captured_sbs.append(x.detach().clone())
        return to_pil_image(x)

    ns = {"torch": torch, "F": F, "TF": TF, "InterpolationMode": InterpolationMode, "path": path, "os": os,
          "PoolExecutor": ThreadPoolExecutor, "tqdm": _NoBar, "ImageLoader": ImageLoader, "load_image_simple": load_image_simple,
          "is_image": lambda f: path.splitext(f)[-1].lower() in (".png", ".jpg"), "export_config": export_config,
          "get_mapper": get_mapper, "dilate_edge": dilate_edge, "edge_dilation_is_enabled": edge_dilation_is_enabled,
          "apply_divergence_forward_warp": apply_divergence_forward_warp, "apply_anaglyph_redcyan": apply_anaglyph_redcyan,
          "equirectangular_projection": None, "BaseDepthModel": BaseDepthModel, "to_pil_image": capture_pil,
          "save_image": lambda im, filename, format="png", **kw: im.save(filename)}
    exec(compile(ast.Module(body=consts + nodes, type_ignores=[]), path.join(REF, "iw3", "utils.py"), "exec"), ns)
    return ns


def make_args(**kw):
    base = dict(export_disparity=False, export_depth_only=False, export_depth_fit=False, mapper="none", edge_dilation=2,
                depth_model="NULL", resume=False, disable_exif_transpose=False, max_workers=0, tta=False, low_vram=False,
                disable_amp=False, depth_aa=False, rotate_left=False, rotate_right=False, max_output_height=None,
                method="forward_fill", divergence=2.0, convergence=0.5, synthetic_view="both", ipd_offset=0, pad=None,
                pad_mode=None, vr180=False, half_sbs=False, tb=False, half_tb=False, cross_eyed=False, anaglyph=None,
                rgbd=False, half_rgbd=False, debug_depth=False, max_output_width=None, keep_aspect_ratio=False,
                metadata=None, format="png", resolution=None, preserve_screen_border=False)
    base.update(kw)
    return Namespace(**base)


def main():
    g = torch.Generator().manual_seed(20261018)
    out = {"meta": json.dumps({"image_sizes": IMAGE_SIZES, "export_cases": EXPORT_CASES, "import_cases": IMPORT_CASES,
                               "depth_range": DEPTH_RANGE})}
    captured = []
    ns = reference_functions(captured)
    with tempfile.TemporaryDirectory() as tmp:
        src = path.join(tmp, "src")
        os.makedirs(src)
        for i, (h, w) in enumerate(IMAGE_SIZES):
            px = (torch.rand((h, w, 3), generator=g) * 255).round().to(torch.uint8).numpy()
            Image.fromarray(px).save(path.join(src, f"im{i}.png"))
            out[f"rgb/{i}"] = px
        for name, (res, disparity, mapper, fit) in EXPORT_CASES.items():
            model = NullDepthModel("NULL")
            model.load(gpu=-1, resolution=res)
            infer = model.infer
            outs = []

            def recording_infer(x, _infer=infer, _outs=outs, **kw):
                y = _infer(x, **kw)
                _outs.append(y.clone())
                return y
            model.infer = recording_infer
            args = make_args(export_disparity=disparity, mapper=mapper, export_depth_fit=fit,
                             state={"depth_model": model, "device": torch.device("cpu"), "tqdm_fn": None,
                                    "stop_event": None, "suspend_event": None})
            dst = path.join(tmp, "export_" + name)
            ns["export_images"](src, dst, args)
            for i, y in enumerate(outs):
                out[f"export/{name}/infer/{i}"] = y.numpy()
                with Image.open(path.join(dst, "depth", f"im{i}.png")) as im:
                    out[f"export/{name}/depth/{i}"] = np.asarray(im)
                    out[f"export/{name}/text/{i}"] = np.array(json.dumps(dict(im.text)))
            with open(path.join(dst, export_config.FILENAME)) as f:
                yml = yaml.safe_load(f)
            yml.pop("updated_at")
            # the rgb_dir of an image export is relative; nothing in it depends on the temporary directory
            out[f"export/{name}/yml"] = np.array(json.dumps(yml))

        for name, (export_case, rewrite) in IMPORT_CASES.items():
            d = path.join(tmp, "export_" + export_case)
            depth_dir = path.join(d, "depth")
            for i in range(len(IMAGE_SIZES)):
                fn = path.join(depth_dir, f"im{i}.png")
                u16 = out[f"export/{export_case}/depth/{i}"]
                if rewrite == "u8_rgb":
                    px = np.stack([u16 >> 8, (u16 >> 4) & 0xff, u16 & 0xff], axis=2).astype(np.uint8)
                    Image.fromarray(px).save(fn)
                elif rewrite == "range":
                    BaseDepthModel.save_normalized_depth(torch.from_numpy(u16.astype(np.float32) / 0xffff).unsqueeze(0), fn,
                                                         png_info={}, min_depth_value=DEPTH_RANGE[0], max_depth_value=DEPTH_RANGE[1])
                with Image.open(fn) as im:
                    out[f"import/{name}/map/{i}"] = np.asarray(im)
                    out[f"import/{name}/text/{i}"] = np.array(json.dumps(dict(im.text)))
                out[f"import/{name}/decoded/{i}"] = BaseDepthModel.load_depth(fn)[0].numpy()
            captured.clear()
            args = make_args(mapper="div_6", input=path.join(d, export_config.FILENAME), output=path.join(tmp, "out_" + name),
                             state={"device": torch.device("cpu"), "tqdm_fn": None, "stop_event": None, "suspend_event": None,
                                    "convergence_model": None})
            ns["process_config_images"](export_config.ExportConfig.load(args.input), args, None)
            assert args.mapper == "div_6"
            for i, sbs in enumerate(captured):
                out[f"import/{name}/sbs/{i}"] = sbs.numpy()
            # restore the export's own maps for the next case that reads this directory
            for i in range(len(IMAGE_SIZES)):
                Image.fromarray(out[f"export/{export_case}/depth/{i}"]).save(path.join(depth_dir, f"im{i}.png"))
    # the yml text save() writes for a video config, without its updated_at line
    kw = dict(type="video", basename="clip", mapper="div_6", skip_mapper=False, skip_edge_dilation=True,
              user_data={"export_options": {"a": 1, "b": [1, 2]}, "scene_boundary": "00000012"},
              output_colorspace="bt709", source_color_range="tv")
    out["yml_kwargs"] = np.array(json.dumps(kw))
    for i, fps in enumerate(([30000, 1001], [30, 1], 24, 29.97)):
        with tempfile.TemporaryDirectory() as tmp:
            f = path.join(tmp, "c.yml")
            export_config.ExportConfig(**dict(kw, fps=Fraction(*fps) if isinstance(fps, list) else fps)).save(f)
            out[f"yml_text/{i}"] = np.array("".join(ln for ln in open(f).read().splitlines(True) if not ln.startswith("updated_at")))
            out[f"yml_fps/{i}"] = np.array(json.dumps(fps))
    dst = path.join(ROOT, "tests", "golden", "depth_export.npz")
    np.savez_compressed(dst, **out)
    print(dst, path.getsize(dst), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    main()
