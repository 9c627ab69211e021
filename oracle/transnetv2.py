"""TransNetV2 and its sliding-window detector, restated from the module and driver code (nunif/utils/transnetv2.py,
nunif/utils/shot_boundary_detection.py) as plain torch-CPU functions of the state_dict.

Network: three stacks of two (2+1)-D dilated blocks, two similarity branches and the fc head; x [B][T][3][27][48] ->
(one_hot [B][T], many_hot [B][T]) logits.  Detector: the windows as a closed form over the padded frame stream
S = [first] * pad + frames + [last] * inf: window k is S[k * step : k * step + window], step = window - 2 * pad, it keeps
positions [pad, window - pad), and windows run until the last kept pts is the last frame's.
"""
import torch
import torch.nn.functional as F

DILATIONS = (1, 2, 4, 8)
BAND = 101


def _block(sd, p, x, relu):
    outs = []
    for d in DILATIONS:
        c = f"{p}.Conv3D_{d}.layers."
        y = F.conv3d(x, sd[c + "0.weight"], padding=(0, 1, 1))
        outs.append(F.conv3d(y, sd[c + "1.weight"], padding=(d, 0, 0), dilation=(d, 1, 1)))
    y = torch.cat(outs, 1)
    y = F.batch_norm(y, sd[p + ".bn.running_mean"], sd[p + ".bn.running_var"], sd[p + ".bn.weight"], sd[p + ".bn.bias"],
                     training=False, eps=1e-3)
    return F.relu(y) if relu else y


def stacks(sd, x):
    """The three stack outputs [B][C][T][h][w] of x [B][T][3][27][48]."""
    h = x.permute(0, 2, 1, 3, 4)
    out = []
    for s in range(3):
        b1 = _block(sd, f"SDDCNN.{s}.DDCNN.0", h, True)
        b2 = _block(sd, f"SDDCNN.{s}.DDCNN.1", b1, False)
        h = F.avg_pool3d(F.relu(b2) + b1, (1, 2, 2))
        out.append(h)
    return out


def band(e):
    """[B][T][D] unit vectors -> [B][T][101]: entry j of frame t is <e_t, e_{t+j-50}>, zero outside the window."""
    B, T, _ = e.shape
    sim = e @ e.transpose(1, 2)
    out = torch.zeros(B, T, BAND, dtype=sim.dtype, device=sim.device)
    for j in range(BAND):
        o = j - BAND // 2
        lo, hi = max(0, -o), min(T, T - o)
        if lo < hi:
            i = torch.arange(lo, hi, device=sim.device)
            out[:, lo:hi, j] = sim[:, i, i + o]
    return out


def color_histograms(x):
    """x [B][T][3][27][48] -> int64 counts [B][T][512] of bin (R >> 5) * 64 + (G >> 5) * 8 + (B >> 5) of x.int()."""
    q = x.to(torch.int32) >> 5
    bins = (q[:, :, 0] * 64 + q[:, :, 1] * 8 + q[:, :, 2]).flatten(2).long()
    return F.one_hot(bins, 512).sum(2)


def hist_band(x):
    h = color_histograms(x).float()
    return band(F.normalize(h, p=2, dim=2))


def sim_band(sd, feats):
    m = torch.cat([f.mean(dim=(3, 4)) for f in feats], 1).transpose(1, 2)
    e = F.linear(m, sd["frame_sim_layer.projection.weight"], sd["frame_sim_layer.projection.bias"])
    return band(F.normalize(e, p=2, dim=2))


def fc1_input(sd, x):
    feats = stacks(sd, x)
    hb = F.relu(F.linear(hist_band(x), sd["color_hist_layer.fc.weight"], sd["color_hist_layer.fc.bias"]))
    sb = F.relu(F.linear(sim_band(sd, feats), sd["frame_sim_layer.fc.weight"], sd["frame_sim_layer.fc.bias"]))
    last = feats[-1].permute(0, 2, 3, 4, 1).flatten(2)   # (h, w, c)
    return torch.cat([hb, sb, last], 2)


def forward(sd, x):
    """x [B][T][3][27][48] (or [T][3][27][48]) -> (one_hot, many_hot) [B][T]."""
    if x.ndim == 4:
        x = x.unsqueeze(0)
    h = F.relu(F.linear(fc1_input(sd, x), sd["fc1.weight"], sd["fc1.bias"]))
    one = F.linear(h, sd["cls_layer1.weight"], sd["cls_layer1.bias"])[..., 0]
    many = F.linear(h, sd["cls_layer2.weight"], sd["cls_layer2.bias"])[..., 0]
    return one, many


def windows(pts, window_size=100, padding_size=25):
    """Frame indices of every window detect_boundary runs for frames with these pts (closed form, see the module doc)."""
    n = len(pts)
    if n == 0:
        raise ValueError("no frames")
    step = window_size - 2 * padding_size

    def s(i):
        return min(max(i - padding_size, 0), n - 1)

    out, k = [], 0
    while True:
        out.append([s(k * step + i) for i in range(window_size)])
        k += 1
        if pts[out[-1][window_size - padding_size - 1]] == pts[-1]:
            return out


def detect(frames01, pts, predict, window_size=100, padding_size=25, threshold=0.5):
    """The segment set for frames [N][3][27][48] in [0, 1] and their pts; predict(x [B][T][3][27][48]) -> one_hot [B][T]."""
    ws = windows(pts, window_size, padding_size)
    probs, kept = [], []
    for w in ws:
        p = torch.sigmoid(predict(frames01[w].unsqueeze(0))[0])
        probs.append(p[padding_size:window_size - padding_size])
        kept += [pts[i] for i in w[padding_size:window_size - padding_size]]
    prob = torch.cat(probs)[:len(pts)]
    return set(p for p, q in zip(kept[:len(pts)], (prob > threshold).tolist()) if q), prob
