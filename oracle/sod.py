"""Functional restatement of iw3's auto-convergence for tests: the `iw3.sod_v1` network (SODV1.infer, iw3/models/sod_v1.py;
U2NETP with fused BatchNorm, nunif/utils/u2netp.py), ConvergenceEstimator.depth_position_from_ratio and its EMA
(iw3/convergence_estimator.py), and the convergence-tensor terms the warps receive.

``sod_infer(sd, rgb, depth)`` runs in the dtype of its inputs; called on CUDA inside ``torch.autocast("cuda")`` it gives the
reference's autocast numerics (fp16 convs, upsampling and sigmoid)."""
import torch
import torch.nn.functional as F
from nunif_b200.synth import SOD_STAGES

SOD_SIZE = 192


def fold(sd, name, eps=1e-5):
    """torch.nn.utils.fuse_conv_bn_eval of one REBNCONV: (weight, bias) in fp32."""
    w, b = sd[name + ".conv_s1.weight"].float(), sd[name + ".conv_s1.bias"].float()
    rs = torch.rsqrt(sd[name + ".bn_s1.running_var"].float() + eps)
    gamma, beta, mean = sd[name + ".bn_s1.weight"].float(), sd[name + ".bn_s1.bias"].float(), sd[name + ".bn_s1.running_mean"].float()
    return w * (gamma * rs).reshape(-1, 1, 1, 1), (b - mean) * rs * gamma + beta


def _conv(sd, x, name, dil):
    w, b = fold(sd, name)
    w, b = w.to(x.device), b.to(x.device)
    return F.relu(F.conv2d(x, w, b, padding=dil, dilation=dil))


def _up(x, ref):
    return F.interpolate(x, size=ref.shape[2:], mode="bilinear", align_corners=False)


def _pool(x):
    return F.max_pool2d(x, 2, 2, ceil_mode=True)


def rsu(sd, prefix, n, x):
    """RSU7/6/5/4 (n) or RSU4F (n = 0) of u2netp.py."""
    p = prefix + ".rebnconv"
    hxin = _conv(sd, x, p + "in", 1)
    if n == 0:
        hx1 = _conv(sd, hxin, p + "1", 1)
        hx2 = _conv(sd, hx1, p + "2", 2)
        hx3 = _conv(sd, hx2, p + "3", 4)
        hx4 = _conv(sd, hx3, p + "4", 8)
        hx3d = _conv(sd, torch.cat((hx4, hx3), 1), p + "3d", 4)
        hx2d = _conv(sd, torch.cat((hx3d, hx2), 1), p + "2d", 2)
        return _conv(sd, torch.cat((hx2d, hx1), 1), p + "1d", 1) + hxin
    hx = [_conv(sd, hxin, p + "1", 1)]
    for k in range(2, n):
        hx.append(_conv(sd, _pool(hx[-1]), p + str(k), 1))
    d = _conv(sd, hx[-1], p + str(n), 2)
    for k in range(n - 1, 1, -1):
        d = _up(_conv(sd, torch.cat((d, hx[k - 1]), 1), p + f"{k}d", 1), hx[k - 2])
    return _conv(sd, torch.cat((d, hx[0]), 1), p + "1d", 1) + hxin


def u2netp(sd, x):
    """U2NETP.forward in eval mode: sigmoid(d0)."""
    kinds = {s: n for s, n, _ in SOD_STAGES}
    enc = []
    hx = x
    for s in ("stage1", "stage2", "stage3", "stage4", "stage5"):
        enc.append(rsu(sd, "u2netp." + s, kinds[s], hx))
        hx = _pool(enc[-1])
    hx6 = rsu(sd, "u2netp.stage6", 0, hx)
    dec = [hx6]
    d = hx6
    for s, skip in zip(("stage5d", "stage4d", "stage3d", "stage2d", "stage1d"), reversed(enc)):
        d = rsu(sd, "u2netp." + s, kinds[s], torch.cat((_up(d, skip), skip), 1))
        dec.append(d)
    hxd = list(reversed(dec))     # hx1d, hx2d, hx3d, hx4d, hx5d, hx6
    side = []
    for k in range(6):
        w, b = sd[f"u2netp.side{k + 1}.weight"].to(x.device), sd[f"u2netp.side{k + 1}.bias"].to(x.device)
        s = F.conv2d(hxd[k], w, b, padding=1)
        side.append(s if k == 0 else _up(s, side[0]))
    d0 = F.conv2d(torch.cat(side, 1), sd["u2netp.outconv.weight"].to(x.device), sd["u2netp.outconv.bias"].to(x.device))
    return torch.sigmoid(d0)


def sod_infer(sd, rgb, depth):
    """SODV1.infer: (saliency, depth_192)."""
    s = (SOD_SIZE, SOD_SIZE)
    rgb = F.interpolate(rgb, s, mode="bilinear", antialias=False, align_corners=False)
    depth = F.interpolate(depth, s, mode="bilinear", antialias=False, align_corners=False)
    x = torch.cat((rgb, depth, depth ** 0.5, depth ** 2), dim=1)
    return u2netp(sd, x), depth


def position_one(d, mask, pos):
    """The rule of depth_position_from_ratio for one image: d, mask flat tensors -> 0-dim fp32 (before the clamp)."""
    d = d[mask]
    if d.numel() == 0:
        return torch.tensor(0.5, dtype=torch.float32, device=d.device)
    q01, q09 = d.quantile(0.1), d.quantile(0.9)
    r = q09 - q01
    if r < 1e-6:
        return q01
    return (q01 + q09) / 2 + (pos - 0.5) * (r * 3.0)


def depth_position(saliency, depth, pos):
    """ConvergenceEstimator.depth_position_from_ratio -> B,1,1,1 fp32."""
    B = depth.shape[0]
    res = [position_one(depth[i].flatten().float(), saliency[i].flatten() > 0.5, pos).float() for i in range(B)]
    return torch.stack(res).reshape(B, 1, 1, 1).clamp(0, 1)


class EMA:
    """The EMA state of ConvergenceEstimator.__call__."""

    def __init__(self, decay=0.9):
        self.decay, self.value = decay, None

    def reset(self):
        self.value = None

    def __call__(self, z_pos, reset_pts=None):
        reset_pts = reset_pts if reset_pts is not None else [False] * z_pos.shape[0]
        out = []
        for i in range(z_pos.shape[0]):
            p = z_pos[i]
            self.value = p.clone() if self.value is None else self.decay * self.value + (1.0 - self.decay) * p
            out.append(self.value.clone())
            if reset_pts[i]:
                self.reset()
        return torch.stack(out, 0)


def backward_index_shift(depth, divergence, convergence, synthetic_view="both"):
    """index_shift of apply_divergence_grid_sample (backward_warp.py:104-106) for a float or B,1,1,1 convergence."""
    if synthetic_view != "both":
        divergence = divergence * 2
    shift_size = divergence * 0.01
    return depth * shift_size - (shift_size * convergence)


def convergence_feature(divergence, convergence, image_width):
    """make_divergence_feature_value's convergence feature (backward_warp.py:8-13) for a float or a tensor."""
    return (-(divergence * 0.5 * 0.01 * image_width) * convergence) / 32.0
