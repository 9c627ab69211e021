"""Depth export and import of iw3 on the engine: ``export_images`` (iw3/utils.py:1226-1347), ``process_config_images``
(:1831-1932), and the per-frame compute of the video export callback (``bind_export_single_frame_callback``,
:1366-1423) and of ``process_config_video``'s ``batch_callback`` (:1716-1738).

File I/O stays on the host as in the reference (PIL); every per-frame computation runs on the device and the host only
receives uint16 depth maps and uint8 images.  Video decoding, encoding, audio and the threaded writer stay with the
caller, as for every video path of the engine.  Differences that are deliberate:

* images are written from the device with round-half-even (``chw_float_to_hwc``, what video frames use), where the
  reference's ``to_pil_image`` truncates ``x * 255``; a frame the export did not resize or rotate round-trips exactly
  either way;
* ``--metadata filename`` output names raise ``NotImplementedError``.
"""
import contextlib
import os
from concurrent.futures import ThreadPoolExecutor
from os import path

import numpy as np
import torch

from . import export_config
from .depth_io import export_depth_u16
from .dilation import dilate_edge, edge_dilation_is_enabled
from .frames import chw_float_to_hwc, hwc_to_chw_float
from .postprocess import postprocess_image

IMAGE_IO_QUEUE_MAX = 100
IMG_EXTENSIONS = (".jpg", ".jpeg", ".png", ".ppm", ".bmp", ".pgm", ".tif", ".tiff", ".webp", ".dds")
_SUFFIXES = (("vr180", "_180x180_LR"), ("half_sbs", "_LR"), ("tb", "_TBF_fulltb"), ("half_tb", "_TB"),
             ("cross_eyed", "_RLF_cross"))
_IMAGE_EXT = {"png": ".png", "webp": ".webp", "jpeg": ".jpg"}


def _arg(args, name, default=None):
    return getattr(args, name, default)


def list_images(directory):
    """ImageLoader.listdir: the image files of ``directory``, sorted by path."""
    return sorted(path.join(directory, f) for f in os.listdir(directory) if path.splitext(f)[-1].lower() in IMG_EXTENSIONS)


def make_output_filename(input_filename, args):
    """iw3/utils.py:111-169 for an image without ``--metadata filename``: basename with SMB-invalid characters replaced,
    the layout suffix and the format's extension."""
    if _arg(args, "metadata", None) == "filename":
        raise NotImplementedError("--metadata filename output names are not implemented on the engine")
    if _arg(args, "rgbd", False) or _arg(args, "half_rgbd", False) or _arg(args, "debug_depth", False):
        raise NotImplementedError("an iw3_export.yml input makes stereo images; --rgbd / --half-rgbd / --debug-depth do not apply")
    basename = path.splitext(path.basename(input_filename))[0].translate({ord(c): ord("_") for c in '\\/:*?"<>|'})
    suffix = next((s for name, s in _SUFFIXES if _arg(args, name, False)), None)
    if suffix is None:
        anaglyph = _arg(args, "anaglyph", None)
        suffix = f"_redcyan_{anaglyph}" if anaglyph else "_LRF_Full_SBS"
    fmt = _arg(args, "format", "png")
    if fmt not in _IMAGE_EXT:
        raise NotImplementedError(fmt)
    return basename + suffix + _IMAGE_EXT[fmt]


def _load_rgb(filename, exif_transpose):
    """load_image_simple(filename, color="rgb") as an HWC uint8 array: transparency (an alpha channel, or a transparent
    palette / grey / RGB colour) is composited onto white, 32- and 16-bit grey images are scaled by 1/255 to 8 bits, and a
    file that cannot be decoded gives None, so that the caller skips it."""
    from PIL import Image, ImageOps
    try:
        with Image.open(filename) as im:
            im.load()
            if exif_transpose:
                im = ImageOps.exif_transpose(im)
            if isinstance(im.info.get("transparency"), (bytes, int)):
                if im.mode in ("RGB", "P"):
                    im = im.convert("RGBA")
                elif im.mode == "L":
                    im = im.convert("LA")
            if im.mode in ("LA", "RGBA"):
                opaque = Image.new(im.mode[:-1], im.size, (255,) * (len(im.mode) - 1))
                opaque.paste(im, mask=im.getchannel("A"))
                im = opaque
            if im.mode in ("I", "I;16"):
                im = im.point(lambda v: v / 255).convert("L")   # Pillow's I -> L conversion clips instead of scaling
            return np.array(im.convert("RGB"))
    except (OSError, ValueError, SyntaxError, Image.DecompressionBombError):
        # unreadable, truncated or oversized files are skipped, as load_image_simple does (UnidentifiedImageError is an
        # OSError; a broken PNG raises SyntaxError)
        return None


# the encoder options iw3 writes each output format with: lossless WebP, JPEG at quality 95 with 4:2:0 chroma
_SAVE_OPTIONS = {"png": dict(format="PNG", compress_level=6), "webp": dict(format="WEBP", quality=95, method=4, lossless=True),
                 "jpeg": dict(format="JPEG", quality=95, subsampling="4:2:0")}


def _save_rgb(hwc, filename, format="png"):
    from PIL import Image
    if format not in _SAVE_OPTIONS:
        raise NotImplementedError(format)
    Image.fromarray(hwc.cpu().numpy()).save(filename, **_SAVE_OPTIONS[format])


def _resume(files, done):
    """--resume: skip the files whose output exists, but redo the first of them in ``files`` order, as the reference's code
    does (its comment says "the last file", which it may have meant as the most recently written one)."""
    remaining = [fn for fn in files if not path.exists(done(fn))]
    existing = [fn for fn in files if path.exists(done(fn))]
    return ([existing[0]] if existing else []) + remaining


@contextlib.contextmanager
def config_mapper(config, args):
    """args.mapper while converting an export (:1802-1828, :1885-1932): "none" with skip_mapper, else the config's
    mapper when it has one; restored afterwards."""
    original = args.mapper
    try:
        if config.skip_mapper:
            args.mapper = "none"
        elif config.mapper is not None:
            args.mapper = config.mapper
        yield
    finally:
        args.mapper = original


def _progress(args, total, desc):
    tqdm_fn = (_arg(args, "state", None) or {}).get("tqdm_fn")
    return tqdm_fn(ncols=80, total=total, desc=desc) if tqdm_fn is not None else None


def _export_depth(depth, frame_size, args, align_corners):
    """The export step between minmax_normalize and save_normalized_depth: --export-disparity's mapper, the
    --export-depth-fit resize and the 16-bit quantisation, in one kernel."""
    return export_depth_u16(depth, mapper=args.mapper if args.export_disparity else None,
                            size=frame_size if args.export_depth_fit else None, align_corners=align_corners)


def export_images(input_path, output_dir, args, title=None):
    """--export of an image file or directory (iw3/utils.py:1226-1347): depth/<name>.png (16 bit), rgb/<name>.png and
    iw3_export.yml under ``output_dir``."""
    from .utils import preprocess_image
    if path.isdir(input_path):
        files = list_images(input_path)
        src_rgb_dir = path.normpath(path.abspath(input_path))
    else:
        files = [input_path]
        src_rgb_dir = path.normpath(path.abspath(path.dirname(input_path)))
    if not files:
        return
    disparity = bool(args.export_disparity)
    edge_dilation = args.edge_dilation if disparity else 0
    config = export_config.ExportConfig(
        type=export_config.IMAGE_TYPE, fps=1, mapper="none" if disparity else args.mapper,
        skip_mapper=disparity, skip_edge_dilation=disparity,
        user_data={"export_options": {"depth_model": args.depth_model, "export_disparity": args.export_disparity,
                                      "mapper": args.mapper, "edge_dilation": args.edge_dilation, "ema_normalize": False}})
    config.audio_file = None
    if args.export_depth_only:
        config.rgb_dir = rgb_dir = src_rgb_dir
    else:
        rgb_dir = path.join(output_dir, config.rgb_dir)
    depth_dir = path.join(output_dir, config.depth_dir)
    os.makedirs(depth_dir, exist_ok=True)
    os.makedirs(rgb_dir, exist_ok=True)
    state = args.state
    depth_model = state["depth_model"]
    depth_model.disable_ema()
    png_name = lambda fn: path.splitext(path.basename(fn))[0] + ".png"  # noqa: E731
    if args.resume:
        files = _resume(files, lambda fn: path.join(depth_dir, png_name(fn)))

    pbar = _progress(args, len(files), title or "Images")
    stop_event, suspend_event = state.get("stop_event"), state.get("suspend_event")
    with ThreadPoolExecutor(max_workers=max(args.max_workers, 8)) as pool, torch.inference_mode():
        futures = []
        for fn in files:
            rgb = _load_rgb(fn, not args.disable_exif_transpose)
            if rgb is not None:
                x = preprocess_image(hwc_to_chw_float(torch.from_numpy(rgb), state["device"]), args)
                depth = depth_model.infer(x, tta=args.tta, low_vram=args.low_vram, enable_amp=not args.disable_amp,
                                          edge_dilation=edge_dilation, depth_aa=args.depth_aa)
                depth = depth_model.minmax_normalize_chw(depth)
                depth_u16 = _export_depth(depth, x.shape[-2:], args, align_corners=True)
                futures.append(pool.submit(depth_model.save_normalized_depth, depth_u16, path.join(depth_dir, png_name(fn))))
                if not args.export_depth_only:
                    futures.append(pool.submit(_save_rgb, chw_float_to_hwc(x), path.join(rgb_dir, png_name(fn))))
            if pbar is not None:
                pbar.update(1)
            if suspend_event is not None:
                suspend_event.wait()
            if stop_event is not None and stop_event.is_set():
                break
            if len(futures) > IMAGE_IO_QUEUE_MAX:
                for f in futures:
                    f.result()
                futures = []
        for f in futures:
            f.result()
    if pbar is not None:
        pbar.close()
    config.save(path.join(output_dir, export_config.FILENAME))


def _import_depth_dilation(depth, config, args):
    """--edge-dilation on an imported map (:1717-1720, :1907-1908): the inverted dilation, unless the export already
    dilated it.  depth: B,1,H,W."""
    if not config.skip_edge_dilation and edge_dilation_is_enabled(args.edge_dilation):
        return -dilate_edge(-depth, args.edge_dilation)
    return depth


def process_config_images(config, args, side_model):
    """An iw3_export.yml of images as input (iw3/utils.py:1831-1932): each rgb/depth pair -> an SBS image under
    args.output, the depth read from its 16-bit file instead of a depth model."""
    from .base_depth_model import BaseDepthModel
    from .utils import apply_divergence
    state = args.state
    device = state["device"]
    rgb_dir, depth_dir, _ = config.resolve_paths(path.dirname(args.input))
    if side_model is not None and hasattr(side_model, "set_mode"):
        side_model.set_mode("image")
        side_model.reset()
    if state.get("convergence_model") is not None:
        state["convergence_model"].reset(enable_ema=False)
    output_dir = args.output
    os.makedirs(output_dir, exist_ok=True)
    rgb_files, depth_files = list_images(rgb_dir), list_images(depth_dir)
    out_name = lambda fn: path.join(output_dir, make_output_filename(path.basename(fn), args))  # noqa: E731
    if args.resume:
        rgb_files = _resume(rgb_files, out_name)
    key = lambda fn: path.splitext(path.basename(fn))[0]  # noqa: E731
    rgb_db, depth_db = {key(fn): fn for fn in rgb_files}, {key(fn): fn for fn in depth_files}
    keys = sorted(rgb_db.keys() & depth_db.keys())
    if not keys:
        raise ValueError(f"{rgb_dir} is empty")

    pbar = _progress(args, len(keys), "Images")
    stop_event, suspend_event = state.get("stop_event"), state.get("suspend_event")
    with config_mapper(config, args), ThreadPoolExecutor(max_workers=4) as pool, torch.inference_mode():
        futures = []
        for k in keys:
            rgb = _load_rgb(rgb_db[k], False)
            if rgb is None:
                raise ValueError(f"cannot read {rgb_db[k]}")
            x = hwc_to_chw_float(torch.from_numpy(rgb), device)
            depth = BaseDepthModel.load_depth(depth_db[k], device=device)[0]
            depth = _import_depth_dilation(depth.unsqueeze(0), config, args).squeeze(0)
            left_eye, right_eye = apply_divergence(depth, x, args, side_model)
            sbs = postprocess_image(left_eye, right_eye, args)
            futures.append(pool.submit(_save_rgb, chw_float_to_hwc(sbs), out_name(k), _arg(args, "format", "png")))
            if pbar is not None:
                pbar.update(1)
            if suspend_event is not None:
                suspend_event.wait()
            if stop_event is not None and stop_event.is_set():
                break
            if len(futures) > IMAGE_IO_QUEUE_MAX:
                for f in futures:
                    f.result()
                futures = []
        for f in futures:
            f.result()
    if pbar is not None:
        pbar.close()


def bind_export_frame_callback(depth_model, args):
    """The per-frame compute of the video export (bind_export_single_frame_callback, :1366-1423).

    Returns ``callback(frame, scene_end=False)``: ``frame`` is one HWC uint8 frame (any device), ``scene_end`` whether
    its pts is a scene boundary; ``callback(None)`` flushes at the end of the video.  Each call returns the
    ``(frame, depth_u16)`` pairs the EMA look-ahead releases, in order: the frame as given and its uint16 depth map on
    the device, ready for the caller's writer."""
    edge_dilation = args.edge_dilation if args.export_disparity else 0
    device = args.state["device"]
    src_queue = []

    def emit(depths):
        out = []
        for depth in depths:
            frame = src_queue.pop(0)
            out.append((frame, _export_depth(depth, tuple(frame.shape[:2]), args, align_corners=False)))
        return out

    @torch.inference_mode()
    def callback(frame, scene_end=False):
        from .utils import preprocess_image
        if frame is None:
            return emit(depth_model.flush_minmax_normalize())
        src_queue.append(frame)
        x = preprocess_image(hwc_to_chw_float(frame, device), args)
        depth = depth_model.infer(x, tta=args.tta, low_vram=args.low_vram, enable_amp=not args.disable_amp,
                                  edge_dilation=edge_dilation, depth_aa=args.depth_aa)
        depth = depth_model.minmax_normalize_chw(depth)
        depths = [depth] if depth is not None else []
        if scene_end:
            depths += depth_model.flush_minmax_normalize()
            depth_model.reset_state()
        return emit(depths)

    return callback


def bind_config_video_batch_callback(config, args, side_model):
    """process_config_video's batch_callback (:1716-1738): ``callback(x, depths, reset_pts)`` with frames x (B,3,H,W)
    and imported depths (B,1,H,W) on the device -> the B postprocessed frames (B,3,H',W'), with the config's mapper."""
    from .utils import apply_divergence

    @torch.inference_mode()
    def callback(x, depths, reset_pts):
        depths = _import_depth_dilation(depths, config, args)
        with config_mapper(config, args):
            left_eyes, right_eyes = apply_divergence(depths, x, args, side_model, reset_pts=reset_pts)
            return torch.stack([postprocess_image(left_eyes[i], right_eyes[i], args) for i in range(left_eyes.shape[0])])

    return callback
