"""Oracle: overlapping-tile render with seam blending (TEST INFRASTRUCTURE).

Restates nunif/utils/seam_blending.py (reference) in plain torch-CPU fp32.
Integer planning must be bit-exact; the float blend follows the reference's
raster-order running weighted average so the oracle itself is bit-identical to
the reference on CPU.
"""
import math
import torch
import torch.nn.functional as F


def create_config(x_h, x_w, scale, offset, tile_size, blend_size):
    """seam_blending.py:109-143 (SeamBlending.create_config)."""
    input_offset = math.ceil(offset / scale)
    input_blend_size = math.ceil(blend_size / scale)
    input_tile_step = tile_size - (input_offset * 2 + input_blend_size)
    h_blocks = w_blocks = input_h = input_w = 0
    while input_h < x_h + input_offset * 2:
        input_h = h_blocks * input_tile_step + tile_size
        h_blocks += 1
    while input_w < x_w + input_offset * 2:
        input_w = w_blocks * input_tile_step + tile_size
        w_blocks += 1
    return {
        "y_h": math.floor(x_h * scale),
        "y_w": math.floor(x_w * scale),
        "h_blocks": h_blocks,
        "w_blocks": w_blocks,
        "pad": (input_offset, input_w - (x_w + input_offset),
                input_offset, input_h - (x_h + input_offset)),
        "y_buffer_h": input_h * scale,
        "y_buffer_w": input_w * scale,
        "input_tile_step": input_tile_step,
        "output_tile_step": input_tile_step * scale,
    }


def create_blend_filter(scale, offset, tile_size, blend_size, out_channels):
    """seam_blending.py:146-153: inner ones + ``blend_size`` rings of
    1 - (i+1)/(blend_size+1), growing outward."""
    model_output_size = tile_size * scale - offset * 2
    inner = model_output_size - blend_size * 2
    x = torch.ones((out_channels, inner, inner), dtype=torch.float32)
    for i in range(blend_size):
        value = 1 - (1 / (blend_size + 1)) * (i + 1)
        x = F.pad(x, (1, 1, 1, 1), mode="constant", value=value)
    return x


def find_valid_tile_size(validator, base_tile_size):
    """nunif/models/model.py:51-62."""
    t = int(base_tile_size)
    while t > 0:
        if validator is None or validator(t):
            return t
        t -= 1
    raise ValueError(f"Could not find valid tile size: tile_size={base_tile_size}")


def cunet_tile_validator(size):
    """waifu2x/models/cunet.py:124-125."""
    return size % 4 == 0


def swin_tile_validator(size):
    """waifu2x/models/swin_unet.py:202-205."""
    return size > 16 and (size - 16) % 12 == 0 and (size - 16) % 16 == 0


def tiled_render(x, model_fn, scale, offset, blend_size, tile_size, batch_size):
    """seam_blending.py:48-106 + update :156-174 + get_output :39-40.

    x: C,H,W fp32.  model_fn: (B,C,T,T) -> (B,C,T*scale-2*offset, ...).
    """
    C, H, W = x.shape
    blend_size = blend_size or 0
    cfg = create_config(H, W, scale, offset, tile_size, blend_size)
    pixels = torch.zeros((C, cfg["y_buffer_h"], cfg["y_buffer_w"]), dtype=torch.float32, device=x.device)   # (the reference keeps
    if blend_size > 0:                                                                                      #  its buffers on the frame's device)
        weights = torch.zeros_like(pixels)
        blend_filter = create_blend_filter(scale, offset, tile_size, blend_size, C).to(x.device)
    step_in = cfg["input_tile_step"]
    step_out = cfg["output_tile_step"]
    xp = F.pad(x.unsqueeze(0), cfg["pad"], mode="replicate")[0]

    def flush(tiles, idx):
        z = model_fn(torch.stack(tiles))
        for k, (hi, wi) in enumerate(idx):
            zk = z[k].float()
            _, oh, ow = zk.shape
            sl = (slice(None), slice(step_out * hi, step_out * hi + oh),
                  slice(step_out * wi, step_out * wi + ow))
            if blend_size > 0:
                old_w = weights[sl]
                next_w = old_w + blend_filter
                old_w = old_w / next_w
                new_w = 1 - old_w
                pixels[sl] = pixels[sl] * old_w + zk * new_w
                weights[sl] += blend_filter
            else:
                pixels[sl] = zk

    tiles, idx = [], []
    for hi in range(cfg["h_blocks"]):
        for wi in range(cfg["w_blocks"]):
            i, j = hi * step_in, wi * step_in
            tiles.append(xp[:, i:i + tile_size, j:j + tile_size])
            idx.append((hi, wi))
            if len(tiles) == batch_size:
                flush(tiles, idx)
                tiles, idx = [], []
    if tiles:
        flush(tiles, idx)
    return torch.clamp(pixels[:, 0:cfg["y_h"], 0:cfg["y_w"]], 0., 1.).contiguous()


def tiled_render_closed_form(x, model_fn, scale, offset, blend_size, tile_size, batch_size):
    """Order-independent statement of the same blend: sum(w*z)/sum(w).

    This is what the H100 engine computes (DESIGN.md); SURVEY.md section 7
    hard-part 2 measured it within 4.2e-7 of the raster-order reference.
    """
    C, H, W = x.shape
    blend_size = blend_size or 0
    cfg = create_config(H, W, scale, offset, tile_size, blend_size)
    num = torch.zeros((C, cfg["y_buffer_h"], cfg["y_buffer_w"]), dtype=torch.float64)
    den = torch.zeros_like(num)
    S = tile_size * scale - 2 * offset
    bf = (create_blend_filter(scale, offset, tile_size, blend_size, C).double()
          if blend_size > 0 else torch.ones((C, S, S), dtype=torch.float64))
    xp = F.pad(x.unsqueeze(0), cfg["pad"], mode="replicate")[0]
    step_in, step_out = cfg["input_tile_step"], cfg["output_tile_step"]
    tiles, idx = [], []
    for hi in range(cfg["h_blocks"]):
        for wi in range(cfg["w_blocks"]):
            tiles.append(xp[:, hi * step_in:hi * step_in + tile_size, wi * step_in:wi * step_in + tile_size])
            idx.append((hi, wi))
    for b0 in range(0, len(tiles), batch_size):
        z = model_fn(torch.stack(tiles[b0:b0 + batch_size])).double()
        for k, (hi, wi) in enumerate(idx[b0:b0 + batch_size]):
            sl = (slice(None), slice(step_out * hi, step_out * hi + S), slice(step_out * wi, step_out * wi + S))
            if blend_size > 0:
                num[sl] += z[k] * bf
                den[sl] += bf
            else:
                num[sl] = z[k]
                den[sl] = 1
    out = num / den.clamp_min(1e-30)
    return torch.clamp(out[:, 0:cfg["y_h"], 0:cfg["y_w"]], 0., 1.).float().contiguous()
