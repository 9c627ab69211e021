"""What the float64 kernel-replay modules (tests/test_gpu_kernel_replay*.py) share: the launch recorder's reader, the networks
whose launches they record, the deduplication of recorded and synthetic configurations, guarded buffers, the error tally and
the replay loop; and the float64 references of the fused Swin block's head and tail, which the persistent-schedule tests
(tests/test_gpu_swin_head_persistent.py) use too.

A recorded line is `kind,name=value,...`, named where the library's host code writes it (include/nunif_b200.h), so a
configuration here is the dict {name: value} of one line, in the order the line gives.
"""
import ctypes
import math
import time
import zlib

import torch
import torch.nn.functional as F

from tests.util import log_metric
from nunif_b200 import _lib, synth

DEV = "cuda:0"
U = 2.0 ** -24                 # fp32 unit roundoff
SENTINEL = 0x7E5B              # an fp16 NaN payload: fp16 guards keep exactly this bit pattern
SENTINEL32 = 0x7FC05B5B        # an fp32 NaN payload: fp32 guards keep exactly this bit pattern
GUARD = 4096                   # guard elements before and after every buffer
# the host code's choices for a launch (gemm's tile width, K step and grid, the conv kinds' kernel path): recorded, but not
# part of what identifies a configuration
HOST_CHOICES = ("block_n", "bk", "grid", "path")


# ------------------------------------------------------------------------------------------------------------ recorder
def _num(v):
    return int(v) if v.lstrip("-").isdigit() else float(v)


def recorded(mask, fn):
    """Run fn() with the recorder on for the kinds of `mask` (nb200_record_launches bits); -> [(kind, {name: value})] of its
    launches."""
    lib = _lib.lib()
    _lib.check(lib.nb200_record_launches(mask))
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        lib.nb200_record_launches(0)
    cap = 1 << 20
    while True:
        buf = ctypes.create_string_buffer(cap)
        if lib.nb200_recorded_launches_named(buf, cap) == 0:
            break
        if b"buffer too small" not in lib.nb200_last_error():
            _lib.check(1)
        cap *= 4
    recs = []
    for line in buf.value.decode().splitlines():
        kind, *fields = line.split(",")
        recs.append((kind, {name: _num(v) for name, v in (f.split("=") for f in fields)}))
    return recs


def record_networks(mask, networks, unique=True):
    """name -> [(kind, config)] of one forward of each (name, run) of `networks` under the recorder; with `unique`, each
    recorded (kind, config) once, in the order first recorded."""
    out = {}
    for name, fn in networks:
        t0 = time.time()
        recs = recorded(mask, fn)
        torch.cuda.empty_cache()
        print(f"{name}: {len(recs)} launches recorded in {time.time() - t0:.1f} s")
        if unique:
            first = {}
            for kind, r in recs:
                first.setdefault((kind, tuple(r.items())), (kind, r))
            recs = list(first.values())
        out[name] = recs
    return out


def _key_fields(r):
    return [f for f in r if f not in HOST_CHOICES]


def configurations(production, kind, synthetic=()):
    """-> [(network or "synthetic", config)] of `kind`: the recorded configurations, then the synthetic ones, each once.  A
    configuration is identified by every field but the host's choices, in the order of the first one (a recorded one, when
    any is), so a synthetic dict may list its fields in any order."""
    configs = [(n, r) for n, recs in production.items() for k, r in recs if k == kind] + [("synthetic", r) for r in synthetic]
    fields = _key_fields(configs[0][1]) if configs else []
    seen, out = set(), []
    for name, r in configs:
        key = tuple(r[f] for f in fields)
        if key not in seen:
            seen.add(key)
            out.append((name, r))
    return out


def _seed(*parts):
    return zlib.crc32(repr(parts).encode())


# ------------------------------------------------------------------------------------------------------------ networks
def _gen(seed):
    return torch.Generator().manual_seed(seed)


def waifu2x(name, sd_fn, T=256, n=16, view=None, seed=1):
    """One batch of n T x T tiles through the waifu2x model `name` (or its to_2x / to_1x view)."""
    def run():
        from nunif_b200.nunif.models import create_model
        m = create_model(name, sd_fn(), DEV)
        if view:
            m = getattr(m, view)()
        m(torch.rand(n, 3, T, T, generator=_gen(seed)).to(DEV))
    return run


def _depth_anything(encoder, v1=False):
    def run():
        from nunif_b200.iw3 import DepthAnythingNet
        from nunif_b200.iw3.depth_anything_preprocess import preprocess_size
        h, w = preprocess_size(1080, 1920)
        net = DepthAnythingNet(synth.depth_anything_v2_state_dict(0, encoder=encoder), DEV, encoder=encoder, v1=v1)
        net(torch.randn(4, 3, h, w, generator=_gen(2)).to(DEV))
    return run


def _zoe_n():
    from nunif_b200.iw3 import ZoeDepthNet
    from nunif_b200.iw3.zoedepth_preprocess import preprocess_size
    _, _, ph, pw, fh, fw = preprocess_size(2160, 3840)
    ZoeDepthNet(synth.zoedepth_state_dict(0), DEV)(torch.randn(2, 3, fh + 2 * ph, fw + 2 * pw, generator=_gen(3)).clamp_(-1, 1).to(DEV))


def zoe_any(kitti, model, seed):
    """ZoeD_Any_N / ZoeD_Any_K on a 1080p landscape and a portrait frame."""
    def run():
        from nunif_b200.iw3 import ZoeDepthAnythingNet
        from nunif_b200.iw3.zoedepth_preprocess import preprocess_size
        net = ZoeDepthAnythingNet(synth.zoedepth_any_state_dict(0, None, kitti), DEV, model)
        for H, W in ((1080, 1920), (1920, 1080)):
            _, _, ph, pw, fh, fw = preprocess_size(H, W, h_height=392, v_height=518, ensure_multiple_of=14)
            net(torch.randn(1, 3, fh + 2 * ph, fw + 2 * pw, generator=_gen(seed)).clamp_(-1, 1).to(DEV))
    return run


def _depth_input(B, h, w):
    from oracle.row_flow import make_input
    return make_input(synth.synth_depth(7, B, h, w), 2.5, 0.4).to(DEV)


def _row_flow_v3():
    from nunif_b200.iw3 import RowFlowV3
    RowFlowV3(synth.row_flow_v3_state_dict(0), DEV)(_depth_input(1, 1080, 1920))


def _mlbw(layers):
    def run():
        from nunif_b200.iw3 import MLBW
        MLBW(synth.mlbw_state_dict(0, num_layers=layers), DEV)(_depth_input(1, 1080, 1920))
    return run


def _depth_aa():
    from nunif_b200.iw3.depth_aa import DepthAA
    from nunif_b200.iw3.depth_anything_preprocess import preprocess_size
    h, w = preprocess_size(1080, 1920)
    DepthAA(synth.depth_aa_state_dict(0), DEV)(synth.synth_depth(8, 4, h, w).to(DEV))


def _light_inpaint():
    from nunif_b200.iw3 import LightInpaintV1
    x = torch.rand(1, 3, 1080, 1920, generator=_gen(5)).to(DEV)
    mask = (torch.rand(1, 1, 1080, 1920, generator=_gen(6)) < 0.05).float().to(DEV)
    LightInpaintV1(synth.light_inpaint_v1_state_dict(0), DEV).infer(x, mask)


def _transnet():
    from nunif_b200.nunif.transnetv2 import TransNetV2
    m = TransNetV2(synth.transnetv2_state_dict(0), DEV)
    for B in (1, 8):
        x = torch.stack([torch.from_numpy(synth.shot_sequence(900 + b, 100)).permute(0, 3, 1, 2).float() for b in range(B)])
        m(x.to(DEV))


def swin_sd(scale):
    return lambda: synth.swin_unet_state_dict(0, scale)


MODELS = [
    ("swin_unet_4x", waifu2x("waifu2x.swin_unet_4x", swin_sd(4))),   # bench swin4x_4k: tile 256, batch 16
    ("swin_unet_4x.to_2x", waifu2x("waifu2x.swin_unet_4x", swin_sd(4), view="to_2x")),   # bench swin2x_4k
    ("swin_unet_2x", waifu2x("waifu2x.swin_unet_2x", swin_sd(2))),   # tiled_render default: tile 256, batch 16
    ("swin_unet_1x", waifu2x("waifu2x.swin_unet_1x", swin_sd(1))),   # tiled_render default: tile 256, batch 16
    ("upcunet", waifu2x("waifu2x.upcunet", synth.upcunet_state_dict)),      # bench upcunet: tile 256, batch 16
    ("cunet", waifu2x("waifu2x.cunet", synth.cunet_state_dict)),            # tiled_render default: tile 256, batch 16
    ("upconv_7", waifu2x("waifu2x.upconv_7", synth.upconv7_state_dict)),    # tiled_render default: tile 256, batch 16
    ("vgg_7", waifu2x("waifu2x.vgg_7", synth.vgg7_state_dict)),             # tiled_render default: tile 256, batch 16
    ("depth_anything_v2_s", _depth_anything("vits")),        # bench iw3_1080p: 1080p frames -> 392 x 686, B = 4
    ("depth_anything_v2_b", _depth_anything("vitb")),        # iw3 Any_V2_B on the same 1080p batch
    ("depth_anything_v2_l", _depth_anything("vitl")),        # iw3 Any_V2_L on the same 1080p batch
    ("depth_anything_v1_s", _depth_anything("vits", True)),  # iw3 Any_S (V1) on the same 1080p batch
    ("zoed_n", _zoe_n),                                      # bench iw3_4k_zoe: 4K frames -> 384 x 704, B = 2
    ("zoed_any_n", zoe_any(False, "ZoeD_Any_N", 4)),         # iw3 default model: 1080p landscape (392 x 700) and portrait (v_height 518)
    ("row_flow_v3", _row_flow_v3),                           # iw3 row_flow_v3 on a 1080p depth map
    ("mlbw_l2", _mlbw(2)),                                   # iw3 mlbw_l2 on a 1080p depth map
    ("mlbw_l4", _mlbw(4)),                                   # iw3 mlbw_l4 on a 1080p depth map
    ("depth_aa", _depth_aa),                                 # iw3 depth_aa on the Depth-Anything output of a 1080p batch (392 x 686, B = 4)
    ("light_inpaint_v1", _light_inpaint),                    # iw3 forward_inpaint on a 1080p frame
    ("transnetv2", _transnet),                               # --scene-detect: 100-frame windows, one alone and 8 batched
]


# the learned stereo networks' own kernels (tests/test_gpu_kernel_replay_stereo.py): each on a 1080p landscape and a portrait
# depth map, one frame at a time as iw3 runs them
STEREO_FRAMES = ((1080, 1920), (1920, 1080))


def _stereo(build):
    def run():
        net = build()
        for h, w in STEREO_FRAMES:
            net(_depth_input(1, h, w))
    return run


def _mlbw_inpaint():
    """iw3 mlbw_l2_inpaint on a 1080p frame: the hole-mask MLBW warps each eye, the left one mirrored, then
    postprocess_hole_mask and light_inpaint_v1 fill the holes."""
    from nunif_b200.iw3 import MLBW, LightInpaintV1, MLBWInpaint
    net = MLBWInpaint(LightInpaintV1(synth.light_inpaint_v1_state_dict(0), DEV), MLBW(synth.mask_mlbw_state_dict(0), DEV), DEV)
    x = torch.rand(1, 3, 1080, 1920, generator=_gen(10)).to(DEV)
    net.infer(x, synth.synth_depth(11, 1, 1080, 1920).to(DEV), 2.5, 0.4)


def _depth_aa_infer():
    from nunif_b200.iw3.depth_aa import DepthAA
    from nunif_b200.iw3.depth_anything_preprocess import preprocess_size
    h, w = preprocess_size(1080, 1920)
    DepthAA(synth.depth_aa_state_dict(0), DEV).infer(synth.synth_depth(8, 4, h, w).to(DEV))


def _iw3(cls, sd):
    def build():
        from nunif_b200 import iw3
        return getattr(iw3, cls)(sd(), DEV)
    return build


STEREO_MODELS = [
    ("row_flow_v3", _stereo(_iw3("RowFlowV3", synth.row_flow_v3_state_dict))),          # iw3's default method
    ("row_flow_v2", _stereo(_iw3("RowFlowV2", synth.row_flow_v2_state_dict))),
    ("mlbw_l2", _stereo(_iw3("MLBW", lambda: synth.mlbw_state_dict(0, 2)))),
    ("mlbw_l4", _stereo(_iw3("MLBW", lambda: synth.mlbw_state_dict(0, 4)))),
    ("mask_mlbw_l2", _stereo(_iw3("MLBW", synth.mask_mlbw_state_dict))),                # the hole head
    ("mlbw_l2_inpaint", _mlbw_inpaint),                     # postprocess_hole_mask with mirror 0 (right eye) and 1 (left eye)
    ("depth_aa", _depth_aa_infer),                          # DepthAA.infer, as Depth-Anything's batch_infer calls it (392 x 686, B = 4)
]


# the backward stereo warps and the AA depth resize (tests/test_gpu_kernel_replay_warp.py): production flows through the
# Python API, as bench.py and iw3.utils.apply_divergence call them, on seeded frames and depth maps at the sizes the depth
# models return (Depth-Anything's preprocess_size)
def _frames(seed, B, H, W):
    return torch.stack([synth.synth_image(seed + i, 3, H, W, smooth=False) for i in range(B)]).to(DEV)


def _bench_sbs(B, H, W, h, w, **kw):
    def run():
        from nunif_b200.iw3 import stereo_sbs
        stereo_sbs(_frames(50, B, H, W), synth.synth_depth(60, B, h, w).to(DEV), 2.0, 0.5, method="backward",
                   edge_dilation=[2, 1], **kw)
    return run


def _args(method, view="both", convergence=0.5, **kw):
    from types import SimpleNamespace
    return SimpleNamespace(method=method, mapper="none", divergence=2.0, convergence=convergence, synthetic_view=view,
                           **{**dict(warp_steps=None, preserve_screen_border=False, stereo_width=None, disable_amp=False,
                                     state=None), **kw})


def _grid_sample_views():
    """A 1080p landscape frame, a portrait frame and a 240 x 320 frame (whose 392 x 518 depth is larger than the frame),
    each with synthetic_view both, left and right."""
    from nunif_b200.iw3.utils import apply_divergence
    from nunif_b200.iw3.depth_anything_preprocess import preprocess_size
    for k, (H, W) in enumerate(((1080, 1920), (1920, 1080), (240, 320))):
        h, w = preprocess_size(H, W)
        for view in ("both", "left", "right"):
            apply_divergence(synth.synth_depth(70 + k, 1, h, w).to(DEV), _frames(80 + k, 1, H, W), _args("grid_sample", view), None)


def _grid_sample_conv_tensor():
    """Auto-convergence's B,1,1,1 convergence tensor on a batch of four 1080p frames."""
    from nunif_b200.iw3.utils import apply_divergence
    conv = torch.tensor([0.5, 0.0, 0.9, 0.25], device=DEV).view(4, 1, 1, 1)
    apply_divergence(synth.synth_depth(73, 4, 392, 686).to(DEV), _frames(83, 4, 1080, 1920), _args("grid_sample", convergence=conv), None)


def _learned(method, build, H=1080, W=1920, views=("both",), **kw):
    """A learned warp (apply_divergence's side-model branch) on a frame with the Depth-Anything-sized depth of a 1080p frame."""
    def run():
        from nunif_b200.iw3.utils import apply_divergence
        model = build()
        for view in views:
            apply_divergence(synth.synth_depth(74, 1, 392, 686).to(DEV), _frames(84, 1, H, W), _args(method, view, **kw), model)
    return run


def _rf_sym():
    from nunif_b200.iw3 import RowFlowV3
    return RowFlowV3(synth.row_flow_v3_state_dict(0), DEV, symmetric=True)


WARP_FLOWS = [
    ("stereo_sbs_1080p", _bench_sbs(4, 1080, 1920, 392, 686)),                                 # bench configs[2]
    ("stereo_sbs_4k_dubois", _bench_sbs(2, 2160, 3840, 384, 704, mapper="div_6", anaglyph="dubois")),   # bench configs[4]
    ("grid_sample_views", _grid_sample_views),
    ("grid_sample_conv_tensor", _grid_sample_conv_tensor),
    ("row_flow_v3", _learned("row_flow_v3", _iw3("RowFlowV3", synth.row_flow_v3_state_dict), warp_steps=1)),
    ("row_flow_v3_steps2", _learned("row_flow_v3", _iw3("RowFlowV3", synth.row_flow_v3_state_dict), warp_steps=2)),
    ("row_flow_v2", _learned("row_flow_v2", _iw3("RowFlowV2", synth.row_flow_v2_state_dict))),
    ("row_flow_v3_sym", _learned("row_flow_v3_sym", _rf_sym, views=("both", "left"))),
    ("mlbw_l2", _learned("mlbw_l2", _iw3("MLBW", lambda: synth.mlbw_state_dict(0, 2)))),
    ("mlbw_l4", _learned("mlbw_l4", _iw3("MLBW", lambda: synth.mlbw_state_dict(0, 4)))),
    ("mask_mlbw_l2", _learned("mask_mlbw_l2", _iw3("MLBW", synth.mask_mlbw_state_dict))),
    ("row_flow_v3_stereo_width", _learned("row_flow_v3", _iw3("RowFlowV3", synth.row_flow_v3_state_dict), 2160, 3840, stereo_width=1920)),
]


# the forward stereo warp (tests/test_gpu_kernel_replay_forward_warp.py): production flows through the Python API, on seeded
# frames and depth maps at the sizes the depth models return
def _fwd_sbs(B, H, W, h, w, method="forward_fill", **kw):
    def run():
        from nunif_b200.iw3 import stereo_sbs
        stereo_sbs(_frames(50, B, H, W), synth.synth_depth(60, B, h, w).to(DEV), 2.0, 0.5, method=method, edge_dilation=[2, 1], **kw)
    return run


def _forward_views():
    """forward_fill and forward in every synthetic_view on a 1080p landscape frame, a portrait frame and a 240 x 320 frame
    (whose 392 x 518 Depth-Anything depth is larger than the frame)."""
    from nunif_b200.iw3.utils import apply_divergence
    from nunif_b200.iw3.depth_anything_preprocess import preprocess_size
    for k, (H, W) in enumerate(((1080, 1920), (1920, 1080), (240, 320))):
        h, w = preprocess_size(H, W)
        for method in ("forward_fill", "forward"):
            for view in ("both", "left", "right"):
                apply_divergence(synth.synth_depth(90 + k, 1, h, w).to(DEV), _frames(95 + k, 1, H, W), _args(method, view), None)


def _forward_conv_tensor():
    """Auto-convergence's B,1,1,1 convergence tensor on a batch of four 1080p frames."""
    from nunif_b200.iw3.utils import apply_divergence
    conv = torch.tensor([0.5, 0.0, 0.9, 0.25], device=DEV).view(4, 1, 1, 1)
    apply_divergence(synth.synth_depth(93, 4, 392, 686).to(DEV), _frames(98, 4, 1080, 1920), _args("forward_fill", convergence=conv), None)


def _forward_inpaint(max_width):
    """forward_inpaint (synthetic light_inpaint_v1 weights) on a 1080p frame, at full width or resized to max_width."""
    def run():
        from nunif_b200.iw3.utils import apply_divergence
        from nunif_b200.iw3 import ForwardInpaint
        model = ForwardInpaint(synth.light_inpaint_v1_state_dict(0), DEV)
        apply_divergence(synth.synth_depth(94, 1, 392, 686).to(DEV), _frames(99, 1, 1080, 1920),
                         _args("forward_inpaint", inpaint_max_width=max_width), model)
    return run


def _forward_null_depth():
    """The NULL depth model at the frame's own size (a square frame): the warp's resize-free path."""
    from nunif_b200.iw3.null_depth_model import NullDepthNet
    from nunif_b200.iw3 import stereo_sbs
    x = _frames(100, 1, 512, 512)
    stereo_sbs(x, NullDepthNet(512)(x), 2.0, 0.5, method="forward_fill")


FWARP_FLOWS = [
    ("stereo_sbs_1080p", _fwd_sbs(4, 1080, 1920, 392, 686)),                                    # bench configs[2]
    ("stereo_anaglyph", _fwd_sbs(1, 1080, 1920, 392, 686, method="forward", anaglyph="dubois")),   # both eyes, compose NONE
    ("forward_views", _forward_views),
    ("forward_conv_tensor", _forward_conv_tensor),
    ("forward_inpaint", _forward_inpaint(None)),
    ("forward_inpaint_max_width", _forward_inpaint(640)),
    ("null_depth", _forward_null_depth),
]


# ------------------------------------------------------------------------------------------------------------ AA resize bound
DW = 10.5 * U   # one tap weight tri(((j + min) - centre + 0.5) * inv) at a given centre: the subtraction, + 0.5 and * inv
                # rounded, inv = 1 / scale within 2U / scale of the exact (|t| <= support + 1.5): (5 + 4.5 / scale) U <= 9.5U
                # downsampling, 5.5U upsampling; then 1 - |arg| rounded (U)


def aa_axis(n_in, n_out):
    """One axis of ATen's antialiased bilinear resize with align_corners=True (csrc/aa_resize.cuh): per output index the
    exact centre c = s (i + 0.5), s = (n_in - 1) / (n_out - 1), its taps [lo, hi) and their weight sum S.  -> (window start,
    window length, centre term, weight term, taps) where
      the centre term = slope * E_c: E_c = 2U c (the fp32 scale and the product rounded); the taps that enter or leave as
        the centre moves weigh zero there, so the sample is continuous in c, and |dv/dc| = |sum_j (w'_j / S)(x_j - v)|
        <= (taps + 2) inv / S * (max - min of x over the window), |w'_j| <= inv
      the weight term = 2 taps DW / S + (taps + 1) U: each weight's DW, the sum S (taps DW + taps U S) and the division
    The window [lo - 1, hi] holds every tap a centre within E_c of c can use."""
    s = (n_in - 1) / (n_out - 1) if n_out > 1 else 0.0
    support, inv = (s, 1 / s) if s >= 1 else (1.0, 1.0)
    c = s * (torch.arange(n_out, dtype=torch.float64) + 0.5)
    lo = (c - support + 0.5).trunc().clamp(min=0)
    hi = (c + support + 0.5).trunc().clamp(max=n_in)
    size = hi - lo
    K = int(size.max()) + 2
    j = lo.view(-1, 1) + torch.arange(K, dtype=torch.float64).view(1, -1)
    wts = ((1 - ((j - c.view(-1, 1) + 0.5) * inv).abs()).clamp(min=0) * (j < hi.view(-1, 1))).sum(1)
    slope = (size + 2) * inv / wts
    start = (lo - 1).clamp(min=0).long()
    to = lambda t: t.to(DEV)
    return to(start), K, to(slope * 2 * U * c), to(2 * size * DW / wts + (size + 1) * U), to(size)


def aa_resize_reference(x64, H, W):
    """F.interpolate(x64, (H, W), bilinear, align_corners=True, antialias=True) in float64 and the bound on the kernels' fp32
    sample (csrc/aa_resize.cuh) of x64 [B][C][h][w]:
      R (cterm_y + cterm_x) + M (wterm_y + wterm_x + (taps_y + taps_x) U)
    with aa_axis's terms, M the largest |x| and R the range of x over the window, and the two fp32 accumulations
    (taps - 1 sums each, first order).  -> (reference, bound), the bound without SECOND_ORDER's margin."""
    h, w = x64.shape[-2:]
    ref = F.interpolate(x64, size=(H, W), mode="bilinear", align_corners=True, antialias=True)
    ys, Ky, cy, wy, ny = aa_axis(h, H)
    xs, Kx, cx, wx, nx = aa_axis(w, W)
    xp = F.pad(x64, (0, Kx, 0, Ky), mode="replicate")
    win = lambda m: F.max_pool2d(m, (Ky, Kx), 1)[:, :, ys][:, :, :, xs]
    hi, lo = win(xp), -win(-xp)
    M, R = torch.maximum(hi.abs(), lo.abs()), hi - lo
    return ref, R * (cy.view(H, 1) + cx.view(1, W)) + M * (wy.view(H, 1) + wx.view(1, W) + (ny.view(H, 1) + nx.view(1, W)) * U)


# ------------------------------------------------------------------------------------------------------------ guarded buffers
def guarded(n):
    """fp16 buffer of GUARD + n + GUARD elements, all SENTINEL."""
    return torch.full((n + 2 * GUARD,), SENTINEL, dtype=torch.int16, device=DEV).view(torch.float16)


def guarded32(n):
    """fp32 buffer of GUARD + n + GUARD elements, all SENTINEL32."""
    return torch.full((n + 2 * GUARD,), SENTINEL32, dtype=torch.int32, device=DEV).view(torch.float32)


def body(buf, n):
    """The n elements between the guards (a view whose data_ptr is what the kernel gets)."""
    return buf[GUARD:GUARD + n]


def guards_ok(buf, n):
    if buf.dtype == torch.float16:
        b, s = bits(buf), SENTINEL
    else:
        b, s = buf.view(torch.int32), SENTINEL32
    return bool((b[:GUARD] == s).all() and (b[GUARD + n:] == s).all())


def bits(t):
    return t.view(torch.int16)


def view(buf, shape, strides, offset=0):
    return buf.as_strided(shape, strides, GUARD + offset)


def extent(shape, strides, offset=0):
    return offset + sum((s - 1) * st for s, st in zip(shape, strides)) + 1


# ------------------------------------------------------------------------------------------------------------ error bounds
def ulp16(x):
    """fp16 spacing at |x| (float64), floored at 2^-24 (the subnormal spacing)."""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 10).clamp_min(2.0 ** -24)


def rounded(v, E):
    """An fp16 rounding point: the kernel rounds a value within E of the float64 v.  Rounding is monotone, so its result lies
    between the roundings of v - E and v + E: -> (v rounded, bound on |kernel's rounded value - v rounded|).  The bound is 0
    wherever no rounding boundary lies within E, so only those few elements carry an error forward."""
    r = v.half().double()
    return r, torch.maximum((v + E).half().double() - r, r - (v - E).half().double())


def round16_bound(ref, E):
    """Bound on |fp16(v) - ref| for a value v the kernel computes within E of ref: half an fp16 ulp at |ref| + E, plus E."""
    return 0.5 * ulp16(ref.abs() + E) + E


class Tally:
    """Worst err / bound, elements over their bound, and the other problems of one replayed configuration."""

    def __init__(self):
        self.worst, self.over, self.bad = 0.0, 0, []

    def add(self, got, ref, bound):
        ratio = torch.nan_to_num((got.double() - ref).abs() / bound, nan=math.inf)
        self.worst = max(self.worst, float(ratio.max()))
        self.over += int((ratio > 1).sum())

    def exact(self, what, got, want):
        """Bit-identical (int views of the same dtype)."""
        if not torch.equal(got, want):
            self.bad.append(f"{what}: {int((got != want).sum())} elements differ")

    def guards(self, what, buf, n):
        if not guards_ok(buf, n):
            self.bad.append(f"{what}: guard changed")

    def no_nan(self, what, t):
        if bool(torch.isnan(t).any()):
            self.bad.append(f"NaN in {what}")

    def result(self):
        return self.worst, self.over, self.bad


# ------------------------------------------------------------------------------------------------------------ replay
def replay(kind, cases, check, variant=None):
    """Replay each configuration of `cases` (configurations()) through check(r, seed) -> Tally.result(), or, with variant =
    (name, values), through check(r, seed, value) for each value.  Logs each result and the summary, and fails if any
    configuration has a problem or an element over its bound.  The seed is _seed(network, kind, configuration key)."""
    values = variant[1] if variant else (None,)
    fields = _key_fields(cases[0][1])
    t0, worst, fails = time.time(), 0.0, []
    for name, r in cases:
        key = tuple(r[f] for f in fields)
        cfg = ",".join(f"{f}={v}" for f, v in zip(fields, key))
        for value in values:
            extra = {variant[0]: int(value)} if variant else {}
            ratio, over, bad = check(r, _seed(name, kind, key), *((value,) if variant else ()))
            log_metric(f"replay_{kind}", model=name, cfg=cfg, **extra, err_over_bound=f"{ratio:.3g}")
            worst = max(worst, ratio)
            if bad or over:
                fails.append(f"{name} {cfg} {extra}: {bad} max err/bound {ratio:.3g}, {over} elements over")
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    n_prod = sum(1 for n, _ in cases if n != "synthetic")
    count = {f"{variant[0]}s": len(values)} if variant else {}
    times = "".join(f" x {n} {k}" for k, n in count.items())
    print(f"\n{kind}: {len(cases)} configurations ({n_prod} recorded, {len(cases) - n_prod} synthetic){times}, worst err/bound "
          f"{worst:.3g}, {time.time() - t0:.1f} s, peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")
    log_metric(f"replay_{kind}_summary", configs=len(cases), **count, worst=worst)
    assert not fails, "\n".join(fails[:20])


# ------------------------------------------------------------------------------------------------------------ Swin block references
def gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def window_attention64(qkv, table, C, shift, eqkv=None, ws=6, heads=6):
    """float64 torchvision shifted_window_attention body (swin_transformer.py:166-221) without the Linears.  qkv [B][H][W][3C]
    -> output, sum_j p_j |v_j|, max_j p_j sum_j |v_j|, and with eqkv (a bound on the error of each q|k|v element) the first-order bound on the
    output error they cause: sum_j p_j (|ds_j| |v_j - o| + ev_j), ds_j the score error.  As torchvision (:151-155), an axis the
    window covers is not shifted, each axis on its own."""
    from nunif_b200.synth import relative_position_index
    B, H, W, _ = qkv.shape
    d = C // heads
    sh, sw = (shift if ws < H else 0), (shift if ws < W else 0)
    nh, nw = H // ws, W // ws

    def windows(t):
        t = torch.roll(t, shifts=(-sh, -sw), dims=(1, 2)) if sh + sw > 0 else t
        return t.view(B, nh, ws, nw, ws, 3 * C).permute(0, 1, 3, 2, 4, 5).reshape(B * nh * nw, ws * ws, 3, heads, d).permute(2, 0, 3, 1, 4)
    xw = windows(qkv)
    q, k, v = xw[0] * d ** -0.5, xw[1], xw[2]
    attn = q @ k.transpose(-2, -1)
    idx = relative_position_index(ws).to(qkv.device)
    attn = attn + table[idx].view(ws * ws, ws * ws, -1).permute(2, 0, 1).unsqueeze(0)
    if sh + sw > 0:
        # torchvision's slices as written: with a zero shift, (-ws, -0) is empty and (-0, None) the whole axis
        m = torch.zeros((H, W), device=qkv.device, dtype=qkv.dtype)
        cnt = 0
        for hs in ((0, -ws), (-ws, -sh), (-sh, None)):
            for ws_ in ((0, -ws), (-ws, -sw), (-sw, None)):
                m[hs[0]:hs[1], ws_[0]:ws_[1]] = cnt
                cnt += 1
        m = m.view(nh, ws, nw, ws).permute(0, 2, 1, 3).reshape(nh * nw, ws * ws)
        m = m.unsqueeze(1) - m.unsqueeze(2)
        m = m.masked_fill(m != 0, -100.0).masked_fill(m == 0, 0.0)
        attn = (attn.view(B, nh * nw, heads, ws * ws, ws * ws) + m.unsqueeze(1).unsqueeze(0)).view(-1, heads, ws * ws, ws * ws)
    p = attn.softmax(-1)
    o = p @ v
    outs = [o, p @ v.abs(), p.amax(-1, keepdim=True) * v.abs().sum(-2, keepdim=True)]
    if eqkv is not None:
        ew = windows(eqkv)
        eq, ek, ev = ew[0] * d ** -0.5, ew[1], ew[2]
        ds = eq @ (k.abs() + ek).transpose(-2, -1) + q.abs() @ ek.transpose(-2, -1)
        pd = p * ds
        # exp(ds) - 1 <= 1.1 ds for the ds << 0.1 seen here: first order with a margin
        outs.append(1.1 * (pd @ v.abs() + pd.sum(-1, keepdim=True) * o.abs()) + p @ ev)
    res = []
    for o in outs:
        o = o.transpose(1, 2).reshape(-1, ws * ws, C).view(B, nh, nw, ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, C)
        res.append(torch.roll(o, shifts=(sh, sw), dims=(1, 2)) if sh + sw > 0 else o)
    return res


def swin_attn_check(r, seed):
    """One call of nb200_swin_attn_fused_f16 (the fused block head) on seeded data against window_attention64, per element
    within ulp16 + 2^-9 sum_j p_j |v_j| + 2^-25 max_j p_j sum_j |v_j| + the propagated q|k|v rounding differences; the output's
    guards and x's bits must not change.  -> Tally.result()."""
    B, H, W, C, shift = r["B"], r["H"], r["W"], r["C"], r["shift"]
    g = torch.Generator(device=DEV).manual_seed(seed)
    rn = lambda *shape: torch.randn(*shape, generator=g, device=DEV)
    x = rn(B, H, W, C).half()
    wqkv = (rn(3 * C, C) / C ** 0.5).half()
    bqkv = 0.1 * rn(3 * C)
    table = 0.5 * rn(121, 6)
    n = B * H * W * C
    att = guarded(n)
    x0 = x.clone()
    _lib.check(_lib.lib().nb200_swin_attn_fused_f16(_lib.ptr(x), _lib.ptr(wqkv), _lib.ptr(bqkv), _lib.ptr(table),
                                                    ctypes.c_void_p(att.data_ptr() + 2 * GUARD), B, H, W, C, shift, _lib.stream_ptr()))
    torch.cuda.synchronize()
    tally = Tally()
    got = body(att, n).view(B, H, W, C)
    tally.no_nan("the output", got)
    tally.guards("output", att, n)
    tally.exact("x", bits(x), bits(x0))
    for b in range(B):
        # q|k|v are rounded to fp16 after the bias, as the kernel stores them; before that the kernel's fp32 GEMM is within
        # 2^-20 sum|x w| (+ the bias add) of the float64 one
        xb = x[b:b + 1].double()
        v = xb @ wqkv.double().t() + bqkv.double()
        qkv, eqkv = rounded(v, 2.0 ** -20 * (xb.abs() @ wqkv.double().abs().t()) + 2.0 ** -22 * v.abs())
        ref, spv, sub, eprop = window_attention64(qkv, table.double(), C, shift, eqkv)
        # fp16 P, its fp32 row sum and ex2.approx as in the ViT attention; plus the q|k|v rounding differences
        bound = ulp16(ref) + 2.0 ** -9 * spv + 2.0 ** -25 * sub + eprop
        tally.add(got[b:b + 1], ref, bound)
    return tally.result()


def mlp_reference(x, att, wp, bp, w1, b1, w2, b2, wy, by):
    """float64 block tail with the kernel's fp16 rounding points (x1, hidden, and with wy the block output) -> (reference,
    bound per element).  Before each rounding point, the kernel's fp32 value differs from the float64 one by at most: 2^-20
    sum|a w| per GEMM (wgmma fp32 accumulation), 2^-21 |v| for the fp32 bias / residual adds and the GELU evaluation, 1e-6 for
    the GELU polynomial, and the differences carried from the previous rounding point through the GEMM (GELU's slope is at
    most 1.13).  rounded() turns that into the difference after rounding."""
    acc = 2.0 ** -20
    x = x.double()
    if att is not None:
        a = att.double()
        v = x + a @ wp.double().t() + bp.double()
        x1, e1 = rounded(v, acc * (a.abs() @ wp.double().abs().t()) + 2.0 ** -21 * (x.abs() + v.abs()))
    else:
        x1, e1 = x, torch.zeros_like(x)
    w1a = w1.double().abs()
    pre = x1 @ w1.double().t() + b1.double()
    h, eh = rounded(gelu64(pre), 1.13 * (acc * (x1.abs() @ w1a.t()) + e1 @ w1a.t()) + 2.0 ** -21 * pre.abs() + 1e-6)
    w2a = w2.double().abs()
    o = x1 + h @ w2.double().t() + b2.double()
    eo = e1 + acc * (h.abs() @ w2a.t()) + eh @ w2a.t() + 2.0 ** -21 * (x1.abs() + o.abs())
    if wy is None:
        return o, ulp16(o) + eo
    o, eo = rounded(o, eo)
    wya = wy.double().abs()
    y = o @ wy.double().t() + by.double()
    return y, ulp16(y) + acc * (o.abs() @ wya.t()) + eo @ wya.t()
