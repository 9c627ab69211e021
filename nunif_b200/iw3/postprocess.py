"""Mirror of iw3/utils.py:394-487 (postprocess_padding, postprocess_image): IPD / letterbox padding, half-SBS and
half-TB squeeze, VR180 equirectangular projection (iw3/equirectangular.py:7-40), anaglyph, SBS / top-bottom / cross-eyed
layout, max-output-size resize."""
import ctypes
import torch
import torch.nn.functional as F
from .. import _lib
from .anaglyph import apply_anaglyph_redcyan


def resize_bicubic_aa(x, size, clamp=False, align_corners=False):
    """TF.resize(x, size, interpolation=BICUBIC, antialias=True) for a CHW / BCHW float tensor (csrc/postprocess.cu);
    ``align_corners=True`` is F.interpolate(..., mode="bicubic", antialias=True, align_corners=True)."""
    _lib.require_cuda(x, "x")
    xf = x.float().contiguous()
    H, W = xf.shape[-2:]
    oh, ow = int(size[0]), int(size[1])
    planes = xf.numel() // (H * W)
    out = torch.empty(xf.shape[:-2] + (oh, ow), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().nb200_resize_bicubic_aa_ac(_lib.ptr(xf), planes, H, W, oh, ow, 1 if clamp else 0,
                                                         1 if align_corners else 0, _lib.ptr(out), _lib.stream_ptr(x.device)))
    return out


def rot90(x, k):
    """torch.rot90(x, k, (-2, -1)) for k = 1 or 3 on a CHW / BCHW float tensor (csrc/frame_ops.cu), bit-exact."""
    _lib.require_cuda(x, "x")
    xf = x.float().contiguous()
    H, W = xf.shape[-2:]
    out = torch.empty(xf.shape[:-2] + (W, H), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().nb200_rot90(_lib.ptr(xf), xf.numel() // (H * W), H, W, k, _lib.ptr(out), _lib.stream_ptr(x.device)))
    return out


def equirectangular_projection(c, device=None):
    """iw3/equirectangular.py:7-40: CHW float CUDA tensor -> VR180 view (csrc/postprocess.cu equirect_kernel)."""
    _lib.require_cuda(c, "c")
    cf = c.float().contiguous()
    C, H, W = cf.shape
    oh, ow = ctypes.c_int(), ctypes.c_int()
    _lib.check(_lib.lib().nb200_equirectangular_size(H, W, ctypes.byref(oh), ctypes.byref(ow)))
    out = torch.empty((C, oh.value, ow.value), dtype=torch.float32, device=c.device)
    with torch.cuda.device(c.device):
        _lib.check(_lib.lib().nb200_equirectangular(_lib.ptr(cf), C, H, W, _lib.ptr(out), _lib.stream_ptr(c.device)))
    return out


def _pad(x, left, top, right, bottom, value=0.0):
    # TF.pad(..., padding_mode="constant"): a constant-filled copy (layout plumbing, only with --ipd-offset / --pad options and
    # the autocrop uncrop)
    return F.pad(x, (left, right, top, bottom), mode="constant", value=value)


def postprocess_padding(left_eye, right_eye, pad, pad_mode):
    """iw3/utils.py:394-427."""
    assert pad_mode in {"tblr", "tb", "lr", "16:9", "top"}
    if pad_mode in {"tblr", "tb", "lr"}:
        pad_h = round(left_eye.shape[1] * pad) // 2 if "tb" in pad_mode else 0
        pad_w = round(left_eye.shape[2] * pad) // 2 if "lr" in pad_mode else 0
        return _pad(left_eye, pad_w, pad_h, pad_w, pad_h), _pad(right_eye, pad_w, pad_h, pad_w, pad_h)
    if pad_mode == "top":
        pad_top = round(left_eye.shape[1] * pad)
        return _pad(left_eye, 0, pad_top, 0, 0), _pad(right_eye, 0, pad_top, 0, 0)
    height, width = left_eye.shape[1:]
    target_ratio, current_ratio = 16 / 9, width / height
    if abs(target_ratio - current_ratio) > 1e-3:
        pad_h = pad_w = 0
        if current_ratio > target_ratio:
            pad_h = (round(width / target_ratio) - height) // 2
        else:
            pad_w = (round(height * target_ratio) - width) // 2
        return _pad(left_eye, pad_w, pad_h, pad_w, pad_h), _pad(right_eye, pad_w, pad_h, pad_w, pad_h)
    return left_eye, right_eye


def postprocess_image(left_eye, right_eye, args):
    """iw3/utils.py:430-487.  left_eye, right_eye: CHW float CUDA tensors; args: the iw3 argument namespace (fields
    ipd_offset, rgbd, half_rgbd, pad, pad_mode, vr180, half_sbs, half_tb, tb, cross_eyed, anaglyph, max_output_height,
    max_output_width, keep_aspect_ratio)."""
    _lib.require_cuda(left_eye, "left_eye")
    _lib.require_cuda(right_eye, "right_eye")
    g = lambda name, default=None: getattr(args, name, default)   # noqa: E731
    ipd_pad = int(abs(g("ipd_offset", 0)) * 0.01 * max(left_eye.shape[-2:]))
    ipd_pad -= ipd_pad % 2
    if ipd_pad > 0 and not (g("rgbd", False) or g("half_rgbd", False)):
        pad_o, pad_i = (ipd_pad * 2, ipd_pad) if g("ipd_offset", 0) > 0 else (ipd_pad, ipd_pad * 2)
        left_eye = _pad(left_eye, pad_o, 0, pad_i, 0)
        right_eye = _pad(right_eye, pad_i, 0, pad_o, 0)
    if g("pad") is not None or g("pad_mode") == "16:9":
        left_eye, right_eye = postprocess_padding(left_eye, right_eye, pad=g("pad"), pad_mode=g("pad_mode"))
    if g("vr180", False):
        left_eye = equirectangular_projection(left_eye)
        right_eye = equirectangular_projection(right_eye)
    elif g("half_sbs", False) or g("half_rgbd", False):
        left_eye = resize_bicubic_aa(left_eye, (left_eye.shape[1], left_eye.shape[2] // 2))
        right_eye = resize_bicubic_aa(right_eye, (right_eye.shape[1], right_eye.shape[2] // 2))
    elif g("half_tb", False):
        left_eye = resize_bicubic_aa(left_eye, (left_eye.shape[1] // 2, left_eye.shape[2]))
        right_eye = resize_bicubic_aa(right_eye, (right_eye.shape[1] // 2, right_eye.shape[2]))
    if g("anaglyph") is not None:
        sbs = apply_anaglyph_redcyan(left_eye, right_eye, g("anaglyph"))
    elif g("tb", False) or g("half_tb", False):
        sbs = torch.cat([left_eye, right_eye], dim=1).clamp_(0., 1.)
    elif g("cross_eyed", False):
        sbs = torch.cat([right_eye, left_eye], dim=2).clamp_(0., 1.)
    else:
        sbs = torch.cat([left_eye, right_eye], dim=2).clamp_(0., 1.)
    h, w = sbs.shape[1:]
    new_w, new_h = w, h
    if g("max_output_height") is not None and new_h > g("max_output_height"):
        if g("keep_aspect_ratio", False):
            new_w = int(g("max_output_height") / new_h * new_w)
        new_h = g("max_output_height")
    if g("max_output_width") is not None and new_w > g("max_output_width"):
        if g("keep_aspect_ratio", False):
            new_h = int(g("max_output_width") / new_w * new_h)
        new_w = g("max_output_width")
    if new_w != w or new_h != h:
        new_h -= new_h % 2
        new_w -= new_w % 2
        sbs = resize_bicubic_aa(sbs, (new_h, new_w), clamp=True)
    return sbs
