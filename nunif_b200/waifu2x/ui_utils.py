"""Tensor side of waifu2x/ui_utils.py: ``process_image`` (:42-71) and the video ``frame_callback`` (:150-178), with
``--rotate-left`` / ``--rotate-right``, ``ctx.convert`` and ``--grain`` on the engine.  Image decoding and saving (PIL / wand),
PyAV and the CLI stay with the caller.

``args`` carries the reference's CLI attributes: rotate_left, rotate_right, method, noise_level, tile_size, batch_size, tta,
disable_amp, grain, grain_strength, grain_speed and state["device"]."""
import torch

from ..iw3.postprocess import rot90
from ..nunif.rgb_noise import apply_rgb_noise_like
from ..nunif.video import FrameBatchPipeline


def _rotate(x, args):
    # PIL's ROTATE_90 / ROTATE_270 of the image are rot90 k = 1 / 3 of its tensor (ui_utils.py:44-47, :157-160)
    if args.rotate_left:
        return rot90(x, 1)
    if args.rotate_right:
        return rot90(x, 3)
    return x


@torch.inference_mode()
def process_image(ctx, rgb, alpha, args, seed=None):
    """ui_utils.py:42-61 from ``IL.to_tensor(im, return_alpha=True)`` on: rgb (1 or 3, H, W) float and alpha (1, H, W) or
    None, rotated, converted, and with grain at ``grain_strength * 0.5``.  Returns (rgb, alpha) for ``IL.to_image``."""
    rgb = _rotate(rgb.to(args.state["device"]), args)
    if alpha is not None:
        alpha = _rotate(alpha.to(args.state["device"]), args)
    if rgb.shape[0] == 1:
        rgb = rgb.repeat(3, 1, 1)
    rgb, alpha = ctx.convert(
        rgb, alpha, args.method, args.noise_level,
        args.tile_size, args.batch_size,
        args.tta, enable_amp=not args.disable_amp,
        output_device=args.state["device"],
    )
    if args.grain:
        # grain_strength = 1/2 for image
        rgb = apply_rgb_noise_like(rgb, strength=args.grain_strength * 0.5, seed=seed)
    return rgb, alpha


def make_frame_callback(ctx, args):
    """ui_utils.py:150-166 as a FrameBatchPipeline callback: each frame of the (B, 3, H, W) batch rotated and converted."""
    @torch.inference_mode()
    def frame_callback(x):
        outs = []
        for rgb in x:
            out, _ = ctx.convert(
                _rotate(rgb, args), None, args.method, args.noise_level,
                args.tile_size, args.batch_size,
                args.tta, enable_amp=not args.disable_amp,
                output_device=rgb.device)
            outs.append(out)
        return torch.stack(outs)
    return frame_callback


def make_video_pipeline(ctx, args, batch_size, use_16bit=False, depth=3, seed=None, source=None, target=None):
    """The video path of ui_utils.py:150-178 on the engine: make_frame_callback in a FrameBatchPipeline whose output stage
    adds the temporal grain (``grain_strength``, ``grain_speed``) when ``args.grain`` is set and quantises for the encoder.
    ``source`` / ``target``: the (pix_fmt, colorspace, color_range) of the decoded and the encoded frames
    (nunif_b200.nunif.video.configure_colorspace), so that the pipeline takes and returns plane arrays."""
    grain = (args.grain_strength, args.grain_speed, seed) if args.grain else None
    return FrameBatchPipeline(make_frame_callback(ctx, args), batch_size, device=args.state["device"], depth=depth,
                              use_16bit=use_16bit, grain=grain, source=source, target=target)
