"""GPU: depth export and import on the engine (csrc/depth_io.cu, nunif_b200/iw3/depth_io.py, nunif_b200/iw3/export.py)
against tests/golden/depth_export.npz (the reference's export_images / process_config_images with its NullDepthModel,
oracle/gen_golden_depth_export.py).  The depth model here is a stand-in whose infer returns the golden's recorded
NullDepthModel.infer outputs in call order; the engine does not build NULL."""
import json
import shutil
from argparse import Namespace

import numpy as np
import pytest
import torch
from PIL import Image
from PIL.PngImagePlugin import PngInfo

from tests.util import load_golden, log_metric
from oracle import depth_export as O
from oracle.mapper import mapper as oracle_mapper

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
G = load_golden("depth_export")
META = json.loads(str(G["meta"]))
N = len(META["image_sizes"])


class RecordedDepth:
    """infer returns the next recorded output; the normaliser is the engine's (BaseDepthModel)."""

    def __init__(self, outputs):
        from nunif_b200.iw3.base_depth_model import BaseDepthModel
        self.base = BaseDepthModel("NULL")
        self.outputs = list(outputs)

    def __getattr__(self, name):
        return getattr(self.base, name)

    def infer(self, x, **kw):
        return self.outputs.pop(0).to(x.device)


def _args(**kw):
    base = dict(export_disparity=False, export_depth_only=False, export_depth_fit=False, mapper="none", edge_dilation=2,
                depth_model="NULL", resume=False, disable_exif_transpose=False, max_workers=0, tta=False, low_vram=False,
                disable_amp=False, depth_aa=False, rotate_left=False, rotate_right=False, max_output_height=None,
                method="forward_fill", divergence=2.0, convergence=0.5, synthetic_view="both", ipd_offset=0, pad=None,
                pad_mode=None, vr180=False, half_sbs=False, tb=False, half_tb=False, cross_eyed=False, anaglyph=None,
                rgbd=False, half_rgbd=False, debug_depth=False, max_output_width=None, keep_aspect_ratio=False,
                metadata=None, format="png", resolution=None, preserve_screen_border=False)
    base.update(kw)
    return Namespace(**base)


def _normalized(case, i):
    d = torch.from_numpy(G[f"export/{case}/infer/{i}"])
    return (d - d.min()) / (d.max() - d.min())


def _torch_export(depth, mapper, size, align_corners):
    """The reference's export ops run with torch on the GPU."""
    if mapper is not None:
        depth = oracle_mapper(depth, mapper)
    if size is not None:
        depth = torch.nn.functional.interpolate(depth.unsqueeze(0), size=tuple(size), mode="bilinear", antialias=True,
                                                align_corners=align_corners).squeeze(0)
    return (0xffff * torch.clamp(depth, 0, 1)).to(torch.uint16).squeeze(0)


def test_export_plain_bit_exact():
    from nunif_b200.iw3.depth_io import export_depth_u16
    for i in range(N):
        got = export_depth_u16(_normalized("plain", i).to(DEV).contiguous())
        np.testing.assert_array_equal(got.cpu().numpy(), G[f"export/plain/depth/{i}"])


@pytest.mark.parametrize("case", [c for c, v in META["export_cases"].items() if v[1] or v[3]])
@pytest.mark.parametrize("align_corners", [True, False])
def test_export_mapper_fit_within_one_code(case, align_corners):
    from nunif_b200.iw3.depth_io import export_depth_u16
    _res, disparity, mapper, fit = META["export_cases"][case]
    mapper = mapper if disparity else None
    for i in range(N):
        size = META["image_sizes"][i] if fit else None
        d = _normalized(case, i).to(DEV)
        got = export_depth_u16(d, mapper=mapper, size=size, align_corners=align_corners).cpu().numpy().astype(np.int64)
        want = _torch_export(d, mapper, size, align_corners).cpu().numpy().astype(np.int64)
        diff = np.abs(got - want)
        log_metric(f"depth_export_{case}_ac{int(align_corners)}_{i}", max=int(diff.max()), frac=float((diff > 0).mean()))
        # measured on an H100: at most 0.72 % of the codes differ, each by one
        assert diff.max() <= 1 and (diff > 0).mean() <= 0.01, (case, i, diff.max(), (diff > 0).mean())
        if align_corners:
            # the reference's CPU ops for the same case
            golden = G[f"export/{case}/depth/{i}"].astype(np.int64)
            assert np.abs(got - golden).max() <= 1


@pytest.mark.parametrize("case", list(META["import_cases"]))
def test_import_decode(case):
    from nunif_b200.iw3.depth_io import import_depth
    for i in range(N):
        text = json.loads(str(G[f"import/{case}/text/{i}"]))
        rng = (float(text["iw3_min_depth_value"]), float(text["iw3_max_depth_value"])) if "iw3_min_depth_value" in text else None
        m = G[f"import/{case}/map/{i}"]
        got = import_depth(m, DEV, rng).cpu()
        want = torch.from_numpy(G[f"import/{case}/decoded/{i}"])
        if m.ndim == 2:
            assert torch.equal(got, want), case
        else:
            ulp = (got.view(torch.int32).long() - want.view(torch.int32).long()).abs().max().item()
            log_metric(f"depth_import_{case}_{i}_ulp", ulp=ulp)
            assert ulp <= 1


def test_image_round_trip(tmp_path):
    """export_images then process_config_images on the engine, for every export case and every import case."""
    from nunif_b200.iw3 import export_config as EC
    from nunif_b200.iw3.utils import export_images, process_config_images
    src = tmp_path / "src"
    src.mkdir()
    for i in range(N):
        Image.fromarray(G[f"rgb/{i}"]).save(src / f"im{i}.png")
    for case, (_res, disparity, mapper, fit) in META["export_cases"].items():
        model = RecordedDepth(torch.from_numpy(G[f"export/{case}/infer/{i}"]) for i in range(N))
        args = _args(export_disparity=disparity, mapper=mapper, export_depth_fit=fit,
                     state={"depth_model": model, "device": DEV})
        dst = tmp_path / ("export_" + case)
        export_images(str(src), str(dst), args)
        for i in range(N):
            with Image.open(dst / "depth" / f"im{i}.png") as im:
                got = np.asarray(im).astype(np.int64)
            want = G[f"export/{case}/depth/{i}"].astype(np.int64)
            assert np.abs(got - want).max() <= (0 if (mapper == "none" or not disparity) and not fit else 1), case
            np.testing.assert_array_equal(np.asarray(Image.open(dst / "rgb" / f"im{i}.png")), G[f"rgb/{i}"])
        cfg = EC.ExportConfig.load(str(dst / EC.FILENAME))
        cfg.fps, cfg.audio_file = 1, None
        yml = cfg.to_yaml_dict("x")
        yml.pop("updated_at")
        assert yml == json.loads(str(G[f"export/{case}/yml"])), case

    for case, (export_case, rewrite) in META["import_cases"].items():
        d = tmp_path / ("export_" + export_case)
        if rewrite is not None:
            # the same export with its depth maps replaced by the golden's 8-bit RGB / min-max maps
            d = tmp_path / ("import_" + case)
            shutil.copytree(tmp_path / ("export_" + export_case), d)
            for i in range(N):
                meta = PngInfo()
                for k, v in json.loads(str(G[f"import/{case}/text/{i}"])).items():
                    meta.add_text(k, v)
                Image.fromarray(G[f"import/{case}/map/{i}"]).save(d / "depth" / f"im{i}.png", pnginfo=meta)
        out = tmp_path / ("out_" + case)
        args = _args(mapper="div_6", input=str(d / EC.FILENAME), output=str(out),
                     state={"device": DEV, "convergence_model": None})
        process_config_images(EC.ExportConfig.load(args.input), args, None)
        assert args.mapper == "div_6"
        if case == "u16":
            # --format webp is written lossless: it decodes to the PNG's pixels
            webp = tmp_path / "out_webp"
            process_config_images(EC.ExportConfig.load(args.input), _args(mapper="div_6", input=args.input, output=str(webp),
                                  format="webp", state={"device": DEV, "convergence_model": None}), None)
            for i in range(N):
                np.testing.assert_array_equal(np.asarray(Image.open(webp / f"im{i}_LRF_Full_SBS.webp").convert("RGB")),
                                              np.asarray(Image.open(out / f"im{i}_LRF_Full_SBS.png")))
        for i in range(N):
            with Image.open(out / f"im{i}_LRF_Full_SBS.png") as im:
                got = torch.from_numpy(np.asarray(im).astype(np.float32) / 255).permute(2, 0, 1)
            want = torch.from_numpy(G[f"import/{case}/sbs/{i}"])
            err = (got - want).abs()
            log_metric(f"depth_import_sbs_{case}_{i}", max=float(err.max()), mean=float(err.mean()))
            # the PNG's rounding to 8 bits (half a code); the warp itself matched exactly on an H100
            assert float(err.max()) <= 0.5 / 255 + 1e-6, case


def test_video_export_callback_matches_oracle():
    """EMA on, a scene boundary inside the sequence, fit and a mapper: the emitted maps equal the oracle frame by frame
    within one code (the fit and mapper bound above)."""
    from nunif_b200.iw3.export import bind_export_frame_callback
    g = torch.Generator().manual_seed(7)
    T, H, W, h, w = 9, 36, 50, 18, 24
    raw = [torch.rand((1, h, w), generator=g) * (1 + 0.3 * k) + 0.1 * k for k in range(T)]
    scene_end = [k == 3 for k in range(T)]
    frames = [(torch.rand((H, W, 3), generator=g) * 255).to(torch.uint8) for _ in range(T)]
    model = RecordedDepth(raw)
    model.enable_ema(decay=0.75, buffer_size=3)
    args = _args(export_disparity=True, mapper="div_6", export_depth_fit=True, state={"device": DEV})
    cb = bind_export_frame_callback(model, args)
    got = []
    for f, end in zip(frames, scene_end):
        got += cb(f.to(DEV), end)
    got += cb(None)
    want = O.export_video_frames(raw, scene_end, 0.75, 3, lambda x: oracle_mapper(x, "div_6"), [(H, W)] * T)
    assert len(got) == len(want) == T
    for (frame, u16), (k, ref) in zip(got, want):
        assert torch.equal(frame.cpu(), frames[k])
        diff = (u16.cpu().long() - ref.long()).abs()
        assert int(diff.max()) <= 1, k


@pytest.mark.parametrize("skip_edge_dilation", [False, True])
def test_config_video_batch_callback_matches_oracle(skip_edge_dilation):
    """process_config_video's batch_callback frame by frame against oracle.depth_export.config_video_batch: the imported
    depths dilated (or not), the config's mapper instead of args.mapper, the forward_fill warp and the SBS compose."""
    from nunif_b200.iw3 import export_config as EC
    from nunif_b200.iw3.export import bind_config_video_batch_callback
    from tests.util import stats
    g = torch.Generator().manual_seed(9)
    x = torch.rand((3, 3, 40, 56), generator=g)
    depths = torch.rand((3, 1, 40, 56), generator=g)
    cfg = EC.ExportConfig(EC.VIDEO_TYPE, fps=30, mapper="div_6", skip_mapper=False, skip_edge_dilation=skip_edge_dilation)
    args = _args(mapper="none", state={"device": DEV, "convergence_model": None})
    got = bind_config_video_batch_callback(cfg, args, None)(x.to(DEV), depths.to(DEV), [False, True, False]).cpu()
    assert args.mapper == "none"
    want = O.config_video_batch(x, depths, 2, skip_edge_dilation, lambda d: oracle_mapper(d, "div_6"), 2.0, 0.5)
    assert got.shape == want.shape
    for i in range(3):
        s = stats(got[i], want[i])
        log_metric(f"depth_import_video_batch_skip{int(skip_edge_dilation)}_{i}", **s)
        assert s["frac_gt_1e3"] < 1e-3, (i, s)


def test_import_other_map_types(tmp_path):
    """32-bit integer ("I") and float ("F") maps decode on the device as load_depth decodes them on the host."""
    from nunif_b200.iw3.base_depth_model import BaseDepthModel
    g = np.random.default_rng(5)
    maps = {"i32.tif": g.integers(-1000, 70000, (13, 17)).astype(np.int32), "f32.tif": g.random((13, 17), np.float32) * 2 - 0.5}
    for name, m in maps.items():
        fn = str(tmp_path / name)
        Image.fromarray(m).save(fn)
        want, _ = BaseDepthModel.load_depth(fn)
        got, text = BaseDepthModel.load_depth(fn, device=DEV)
        assert text["filename"] == fn
        assert torch.equal(got.cpu(), want), name
    with pytest.raises(NotImplementedError):
        from nunif_b200.iw3.depth_io import import_depth
        import_depth(np.zeros((4, 4), np.float64), DEV)
