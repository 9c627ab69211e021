"""ORACLE (test infrastructure only - never imported by nunif_b200/): CPU/torch restatement of the window-attention block
`WABlock` that sbs.row_flow_v3, sbs.mlbw and iw3.depth_aa are built from (iw3/models/row_flow_v3.py:13-29, mlbw.py:18-34,
depth_aa.py:11-26): x + WindowMHA2d(x, attn_mask=WindowScoreBias()), then x + act(conv3x3(reppad(gelu(conv1x1(x))))).
Functional style (state_dict in); `p` is the block's prefix, e.g. "blocks.1.".
"""
import torch.nn.functional as F


def window_bias(sd, p, ws):
    """WindowScoreBias.forward (nunif/modules/attention.py:408-420): (N, N) additive attention bias."""
    N = ws * ws
    b = F.linear(F.gelu(F.linear(sd[p + "delta"], sd[p + "to_bias.0.weight"], sd[p + "to_bias.0.bias"])),
                 sd[p + "to_bias.2.weight"], sd[p + "to_bias.2.bias"])
    return b[sd[p + "index"]].reshape(N, N)


def window_mha2d(sd, p, x, ws, heads, shift):
    """The block's self.mha(x, attn_mask=self.bias()): WindowMHA2d (nunif/modules/attention.py:118-161), i.e. zero padding by
    ws/2 in the shifted directions, window attention, crop.  shift = bool (both directions) or (shift_h, shift_w); x: B,C,H,W."""
    sh, sw = shift if isinstance(shift, tuple) else (shift, shift)
    ph, pw = (ws // 2 if sh else 0), (ws // 2 if sw else 0)
    if ph or pw:
        x = F.pad(x, (pw, pw, ph, ph), mode="constant", value=0)
    B, C, H, W = x.shape
    oh, ow = H // ws, W // ws
    t = x.reshape(B, C, oh, ws, ow, ws).permute(0, 2, 4, 3, 5, 1).reshape(B * oh * ow, ws * ws, C)     # bchw_to_bnc
    qkv = F.linear(t, sd[p + "mha.mha.qkv_proj.weight"], sd[p + "mha.mha.qkv_proj.bias"])
    q, k, v = qkv.split(C, dim=-1)
    d = C // heads
    q, k, v = [a.reshape(-1, ws * ws, heads, d).permute(0, 2, 1, 3) for a in (q, k, v)]
    a = F.scaled_dot_product_attention(q, k, v, attn_mask=window_bias(sd, p + "bias.", ws).to(q.dtype))
    a = a.permute(0, 2, 1, 3).reshape(-1, ws * ws, C)
    a = F.linear(a, sd[p + "mha.mha.head_proj.weight"], sd[p + "mha.mha.head_proj.bias"])
    a = a.reshape(B, oh, ow, ws, ws, C).permute(0, 5, 1, 3, 2, 4).reshape(B, C, H, W)                    # bnc_to_bchw
    return a[:, :, ph:H - ph, pw:W - pw]


def wa_block(sd, p, x, ws, heads, shift, act):
    """WABlock.forward; act: LeakyReLU(0.1) after the 3x3 (row_flow_v3, depth_aa) or none (mlbw)."""
    x = x + window_mha2d(sd, p, x, ws, heads, shift)
    m = F.gelu(F.conv2d(x, sd[p + "conv_mlp.0.weight"], sd[p + "conv_mlp.0.bias"]))
    m = F.conv2d(F.pad(m, (1, 1, 1, 1), mode="replicate"), sd[p + "conv_mlp.3.weight"], sd[p + "conv_mlp.3.bias"])
    if act:
        m = F.leaky_relu(m, 0.1)
    return x + m
