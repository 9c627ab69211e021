"""Mirror of iw3's learned stereo warp: the `sbs.row_flow_v3` model (iw3/models/row_flow_v3.py) in delta_output mode and
its driver apply_divergence_nn_LR / apply_divergence_nn_delta (iw3/backward_warp.py:124-232).

The delta network runs as wgmma GEMMs + the kernels in csrc/rowflow_kernels.cu; the warp is the fused grid-sample kernel
(csrc/warp_backward.cu, nb200_backward_warp_delta).  steps > 1 (iterative re-warping of the depth, :205-226) and
preserve_screen_border (:33-47) run the same kernels once per step.
"""
import ctypes
import torch
from .. import _lib

KIND_ROW_FLOW_V3 = 7     # NB200_MODEL_ROW_FLOW_V3
KIND_MLBW = 11           # NB200_MODEL_MLBW


def _create(kind, state_dict, device):
    items = [(k, v.detach().to("cpu", torch.float32).contiguous()) for k, v in state_dict.items()]
    n = len(items)
    names = (ctypes.c_char_p * n)(*[k.encode() for k, _ in items])
    datas = (ctypes.c_void_p * n)(*[v.data_ptr() for _, v in items])
    numels = (ctypes.c_int64 * n)(*[v.numel() for _, v in items])
    h = ctypes.c_void_p()
    with torch.cuda.device(device):
        _lib.check(_lib.lib().nb200_model_create(kind, n, names, datas, numels, 0, ctypes.byref(h)))
    return h


class MLBW:
    """Packed `sbs.mlbw` (iw3/models/mlbw.py; methods mlbw_l2 / mlbw_l4 and their `s` variants, hole_mask=False) in delta_output
    mode: ``model(x)`` with x = B,3,h,w returns ``(delta B,L,h,w, layer_weight B,L,h,w)`` (:237-245 without the y interleave)."""
    name = "sbs.mlbw"
    symmetric = False
    delta_output = True
    hole_mask = False

    def __init__(self, state_dict, device="cuda:0"):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("nunif_b200 models live on a CUDA (sm_90) device; there is no CPU path")
        self._h = _create(KIND_MLBW, state_dict, self.device)
        self.num_layers = int(_lib.lib().nb200_mlbw_num_layers(self._h))

    def __del__(self):
        try:
            if self._h:
                _lib.lib().nb200_model_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def __call__(self, x):
        _lib.require_cuda(x, "x")
        assert x.ndim == 4 and x.shape[1] == 3
        B, _, h, w = x.shape
        xf = x.float().contiguous()
        delta = torch.empty((B, self.num_layers, h, w), dtype=torch.float32, device=x.device)
        lw = torch.empty_like(delta)
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().nb200_mlbw_delta(self._h, _lib.ptr(xf), B, h, w, _lib.ptr(delta), _lib.ptr(lw), _lib.stream_ptr(x.device)))
        return delta, lw


class RowFlowV3:
    """Packed `sbs.row_flow_v3`; ``model(x)`` with x = B,3,h,w (depth, divergence feature, convergence feature) returns the
    delta B,2,h,w (x component, zero y component) like the reference with ``delta_output=True`` (row_flow_v3.py:111-116)."""
    name = "sbs.row_flow_v3"
    symmetric = False
    delta_output = True

    def __init__(self, state_dict, device="cuda:0"):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("nunif_b200 models live on a CUDA (sm_90) device; there is no CPU path")
        self._h = _create(KIND_ROW_FLOW_V3, state_dict, self.device)

    def __del__(self):
        try:
            if self._h:
                _lib.lib().nb200_model_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def delta_x(self, x):
        _lib.require_cuda(x, "x")
        assert x.ndim == 4 and x.shape[1] == 3
        B, _, h, w = x.shape
        xf = x.float().contiguous()
        out = torch.empty((B, 1, h, w), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().nb200_row_flow_delta(self._h, _lib.ptr(xf), B, h, w, _lib.ptr(out), _lib.stream_ptr(x.device)))
        return out

    def __call__(self, x):
        d = self.delta_x(x)
        return torch.cat([d, torch.zeros_like(d)], dim=1)


def make_divergence_feature_value(divergence, convergence, image_width):
    """iw3/backward_warp.py:8-15."""
    divergence_pix = divergence * 0.5 * 0.01 * image_width
    return divergence_pix / 32.0, (-divergence_pix * convergence) / 32.0


def _warp_delta(c, delta, delta_scale):
    B, _, H, W = c.shape
    h, w = delta.shape[-2:]
    out = torch.empty_like(c)
    with torch.cuda.device(c.device):
        _lib.check(_lib.lib().nb200_backward_warp_delta(_lib.ptr(c), _lib.ptr(delta), B, H, W, h, w, float(delta_scale), _lib.ptr(out),
                                                        _lib.stream_ptr(c.device)))
    return out


def make_input(depth, divergence, convergence, preserve_screen_border=False):
    """make_input_tensor(None, depth, ...) for a batch (iw3/backward_warp.py:18-63): depth, divergence feature, convergence
    feature; with preserve_screen_border the two features fade linearly to zero over `border_pix` columns at both edges."""
    B, _, H, W = depth.shape
    base = max(H, W)
    dv, cv = make_divergence_feature_value(divergence, convergence, base)
    df, cf = torch.full_like(depth, dv), torch.full_like(depth, cv)
    if preserve_screen_border:
        bp = round(divergence * 0.75 * 0.01 * base * (W / base))                               # :36
        if bp > 0:
            wl = torch.linspace(0.0, 1.0, bp, device=depth.device)
            wr = torch.linspace(1.0, 0.0, bp, device=depth.device)
            for f in (df, cf):
                f[..., :bp] = wl * f[..., :bp]
                f[..., -bp:] = wr * f[..., -bp:]
    return torch.cat([depth, df, cf], dim=1)


def apply_divergence_nn_delta(model, c, depth, divergence, convergence, steps, shift, preserve_screen_border=False, enable_amp=True):
    """iw3/backward_warp.py:185-232."""
    steps = 1 if steps is None else int(steps)
    assert steps >= 1
    if not enable_amp:
        raise NotImplementedError("nunif_b200 implements the reference's CUDA autocast (fp16) forward only")
    _lib.require_cuda(c, "c")
    _lib.require_cuda(depth, "depth")
    c, depth = c.float().contiguous(), depth.float().contiguous()
    if shift > 0:
        c, depth = torch.flip(c, (3,)), torch.flip(depth, (3,))
    B, _, H, W = depth.shape
    delta_scale = 1.0 / (W // 2 - 1)                                                           # :201
    depth_warp, deltas = depth, []
    for j in range(steps):
        deltas.append(model.delta_x(make_input(depth_warp, divergence / steps, convergence, preserve_screen_border)))
        if j + 1 < steps:
            # backward_warp(depth_warp, grid, delta, delta_scale) :220-221 (the warp kernel takes 3-channel frames)
            depth_warp = _warp_delta(depth_warp.expand(-1, 3, -1, -1).contiguous(), deltas[-1], delta_scale)[:, :1].contiguous()
    z = c
    for delta in deltas:                                                                       # :223-226
        z = _warp_delta(z, delta, delta_scale)
    return torch.flip(z, (3,)) if shift > 0 else z


def apply_divergence_nn_delta_weight(model, c, depth, divergence, convergence, steps, shift, preserve_screen_border=False, enable_amp=True):
    """iw3/backward_warp.py:262-329 for sbs.mlbw without a hole mask: every flow layer warps the frame, the warps are blended with
    the (antialias-bilinear resized) layer weights.  ``steps`` is ignored by the reference for this model."""
    if not enable_amp:
        raise NotImplementedError("nunif_b200 implements the reference's CUDA autocast (fp16) forward only")
    _lib.require_cuda(c, "c")
    _lib.require_cuda(depth, "depth")
    c, depth = c.float().contiguous(), depth.float().contiguous()
    if shift > 0:
        c, depth = torch.flip(c, (3,)), torch.flip(depth, (3,))
    B, _, H, W = depth.shape
    delta, lw = model(make_input(depth, divergence, convergence, preserve_screen_border))
    if c.shape[2:] != lw.shape[2:]:                                                            # :296-298
        L = lw.shape[1]
        lw_full = torch.empty((B, L, c.shape[2], c.shape[3]), dtype=torch.float32, device=c.device)
        with torch.cuda.device(c.device):
            _lib.check(_lib.lib().nb200_depth_resize_aa(_lib.ptr(lw.contiguous()), B * L, H, W, c.shape[2], c.shape[3], _lib.ptr(lw_full),
                                                        _lib.stream_ptr(c.device)))
        lw = lw_full
    delta_scale = 1.0 / (W // 2 - 1)
    z = torch.zeros_like(c)
    for i in range(model.num_layers):                                                          # :304-309
        z += _warp_delta(c, delta[:, i:i + 1].contiguous(), delta_scale) * lw[:, i:i + 1]
    z = z.clamp_(0, 1)
    return torch.flip(z, (3,)) if shift > 0 else z


def apply_divergence_nn(model, c, depth, divergence, convergence, steps, shift, preserve_screen_border=False, enable_amp=True):
    """iw3/backward_warp.py:163-182."""
    fn = apply_divergence_nn_delta_weight if getattr(model, "name", "") == "sbs.mlbw" else apply_divergence_nn_delta
    return fn(model, c, depth, divergence, convergence, steps, shift, preserve_screen_border=preserve_screen_border, enable_amp=enable_amp)


def apply_divergence_nn_LR(model, c, depth, divergence, convergence, steps=None, synthetic_view="both",
                           preserve_screen_border=False, enable_amp=True):
    """iw3/backward_warp.py:124-160 for the non-symmetric delta models (sbs.row_flow_v3, sbs.mlbw)."""
    assert synthetic_view in {"both", "right", "left"}
    if getattr(model, "symmetric", False):
        raise NotImplementedError("symmetric side models (row_flow_v2) are not implemented by the H100 engine")
    kw = dict(steps=steps, preserve_screen_border=preserve_screen_border, enable_amp=enable_amp)
    if synthetic_view == "both":
        return (apply_divergence_nn(model, c, depth, divergence, convergence, shift=-1, **kw),
                apply_divergence_nn(model, c, depth, divergence, convergence, shift=1, **kw))
    if synthetic_view == "right":
        return c, apply_divergence_nn(model, c, depth, divergence * 2, convergence, shift=1, **kw)
    return apply_divergence_nn(model, c, depth, divergence * 2, convergence, shift=-1, **kw), c
