"""ORACLE (test infrastructure only): steps 1-6 of nunif/utils/video.py:309-416 ``hdr2sdr`` - PQ (HDR10) / HLG BT.2020 ->
BT.709 / BT.601 SDR with the Hable tone map - restated as a function of a uint16 HWC tensor instead of a PyAV frame.

The ops, their order, the dtypes and the layouts (the permuted CHW view of the HWC frame, the reshape before torch.mm) are
the reference's, so that on the CPU the result is the reference's bit for bit (tests/golden/hdr2sdr.npz, made by
oracle/gen_golden_hdr2sdr.py from the real function), and on CUDA it is what the reference computes with ``device=`` a GPU.

``golden_inputs()`` regenerates the frames the golden was made from; ``encode_output`` / ``reference_output`` are the
golden's storage of the reference's outputs.
"""
import hashlib

import numpy as np
import torch

PQ, HLG = 16, 18                       # color_trc: AVCOL_TRC_SMPTE2084, AVCOL_TRC_ARIB_STD_B67

MATRIX = {
    "bt709": [[1.6605, -0.5876, -0.0728],
              [-0.1246, 1.1329, -0.0083],
              [-0.0182, -0.1006, 1.1187]],
    "bt601": [[1.5540, -0.5143, -0.0397],
              [-0.1017, 1.1147, -0.0130],
              [-0.0163, -0.0886, 1.1049]],
}


def hdr2sdr(x, color_trc, output_colorspace, pq_exposure=110.0, pq_white_point=5.0, hlg_exposure=1.2, hlg_white_point=0.8,
            hlg_saturation_gain=0.9, device="cpu", taps=None):
    """x: uint16 [H][W][3] rgb48, full range -> uint16 [H][W][3] on ``device`` (video.py:321-398).
    ``taps``, a dict, receives [3][H][W] fp32 intermediates: "sdr" (the BT.2020 input of the colour matrix), "linear" (its
    clamped output, the OETF's input) and "scaled" (the value the final cast truncates)."""
    assert output_colorspace in {"bt709", "bt601"} and color_trc in {PQ, HLG}
    assert x.dtype == torch.uint16 and x.ndim == 3 and x.shape[2] == 3
    x = x.contiguous().to(device).permute(2, 0, 1) / 65535.0
    if color_trc == PQ:
        m1, m2 = 2610 / 16384, 2523 / 4096 * 128
        c1, c2, c3 = 3424 / 4096, 2413 / 4096 * 32, 2392 / 4096 * 32
        x_pow = torch.pow(x, 1.0 / m2)
        linear_2020 = torch.pow(torch.clamp(x_pow - c1, min=0) / (c2 - c3 * x_pow), 1.0 / m1)
        current_exposure, current_white = pq_exposure, pq_white_point
    else:
        a, b, c = 0.17883277, 0.28466892, 0.55991073
        linear_2020 = torch.where(x <= 0.5, torch.pow(x, 2.0) / 3.0, (torch.exp((x - c) / a) + b) / 12.0)
        current_exposure, current_white = hlg_exposure, hlg_white_point
    x_lin = linear_2020 * current_exposure

    def hable_map(v, E=0.02):
        A, B, C, D, E, F = 0.15, 0.50, 0.10, 0.20, E, 0.30
        return ((v * (A * v + C * B) + D * E) / (v * (A * v + B) + D * F)) - E / F

    white = torch.tensor(current_white, dtype=x.dtype, device=x.device)
    if color_trc == HLG:
        sdr = hable_map(x_lin, E=0.01) / hable_map(white, E=0.01)
        if hlg_saturation_gain < 1.0:
            luma = sdr[0] * 0.2126 + sdr[1] * 0.7152 + sdr[2] * 0.0722
            sdr = (sdr * hlg_saturation_gain) + (luma * (1.0 - hlg_saturation_gain))
    else:
        sdr = hable_map(x_lin) / hable_map(white)
    matrix = torch.tensor(MATRIX[output_colorspace], dtype=x.dtype, device=x.device)
    c, h, w = sdr.shape
    sd = torch.mm(matrix, sdr.reshape(c, -1)).reshape(c, h, w)
    sd = torch.clamp(sd, 0, 1)
    gamma = torch.where(sd < 0.018, sd * 4.5, 1.099 * torch.pow(sd, 0.45) - 0.099)
    scaled = gamma.clamp(0, 1) * 65535
    if taps is not None:
        taps.update(sdr=sdr, linear=sd, scaled=scaled)
    return scaled.to(torch.uint16).permute(1, 2, 0).contiguous()


# ---- golden inputs (oracle/gen_golden_hdr2sdr.py, tests/test_hdr2sdr.py, tests/test_gpu_hdr2sdr.py)

# name, color_trc, output_colorspace, keyword arguments that differ from hdr2sdr's defaults
CONFIGS = (
    ("pq_bt709", PQ, "bt709", {}),
    ("pq_bt601", PQ, "bt601", {}),
    ("hlg_bt709", HLG, "bt709", {}),
    ("hlg_bt601", HLG, "bt601", {}),
    ("hlg_bt709_nosat", HLG, "bt709", dict(hlg_saturation_gain=1.0, hlg_exposure=1.5, hlg_white_point=1.1)),
    ("hlg_bt601_sat05", HLG, "bt601", dict(hlg_saturation_gain=0.5, hlg_exposure=0.9, hlg_white_point=0.6)),
    ("pq_bt709_exp", PQ, "bt709", dict(pq_exposure=60.0, pq_white_point=9.5)),
)
PERM_SEEDS = (11, 12, 13)
# every code on either side of a branch edge: 0 / 65535, HLG x <= 0.5 (32767 | 32768), the PQ clamp x^(1/m2) < c1 (code 0 only)
EDGE_CODES = (0, 1, 2, 3, 255, 256, 4096, 16384, 32766, 32767, 32768, 32769, 49152, 65533, 65534, 65535)


def golden_inputs():
    """name -> uint16 [H][W][3] frame:
    perm  256 x 256: R, G, B are three different permutations of 0..65535 (every code in every channel)
    gray  256 x 256: R = G = B = 0..65535 in raster order (every neutral level: each OETF switch at 0.018 of a grey)
    edges 16 x 256: every (R, G, B) of EDGE_CODES^3, in raster order"""
    perm = np.stack([np.random.default_rng(s).permutation(65536) for s in PERM_SEEDS], -1).reshape(256, 256, 3)
    gray = np.repeat(np.arange(65536).reshape(256, 256, 1), 3, -1)
    e = np.asarray(EDGE_CODES)
    edges = np.stack(np.meshgrid(e, e, e, indexing="ij"), -1).reshape(16, 256, 3)
    return {k: torch.from_numpy(v.astype(np.uint16)) for k, v in (("perm", perm), ("gray", gray), ("edges", edges))}


def input_checksum(x):
    """int64 sum of code * (1 + flat index mod 65521): catches a reordered or altered regenerated input."""
    v = x.reshape(-1).to(torch.int64)
    return int((v * (1 + torch.arange(v.numel()) % 65521)).sum())


# The golden keeps the gray and edge outputs whole, each channel delta-coded along the raster (int32, mostly small steps),
# and the perm outputs (noise-like: about 300 KB per configuration compressed) as their SHA-256 plus a seeded sample of
# PERM_SAMPLE pixels.
FULL_FRAMES = ("gray", "edges")
PERM_SAMPLE_SEED, PERM_SAMPLE = 14, 1024


def perm_sample_index():
    return np.sort(np.random.default_rng(PERM_SAMPLE_SEED).choice(65536, PERM_SAMPLE, replace=False))


def digest(y):
    """SHA-256 of a uint16 [H][W][3] frame's little-endian bytes, as uint8 [32]."""
    b = np.ascontiguousarray(np.asarray(y), dtype="<u2").tobytes()
    return np.frombuffer(hashlib.sha256(b).digest(), dtype=np.uint8).copy()


def encode_output(name, y):
    """The golden entries (suffix -> array) of the reference's uint16 [H][W][3] output ``y`` for input frame ``name``."""
    y = np.asarray(y)
    if name in FULL_FRAMES:
        return {"delta": np.diff(y.reshape(-1, 3).astype(np.int32), axis=0, prepend=0)}
    return {"sha256": digest(y), "sample": y.reshape(-1, 3)[perm_sample_index()]}


def reference_output(golden, config, name, x):
    """The reference's uint16 [H][W][3] output for ``config`` (a CONFIGS entry) on golden input ``name`` (= ``x``).  A perm
    output is recomputed by this oracle on the CPU and must match the stored digest and sample; it raises otherwise."""
    cname, trc, cs, kw = config
    key = f"out/{cname}/{name}/"
    if name in FULL_FRAMES:
        return np.cumsum(golden[key + "delta"], axis=0).astype(np.uint16).reshape(tuple(x.shape))
    y = hdr2sdr(x, trc, cs, **kw).numpy()
    if not (np.array_equal(y.reshape(-1, 3)[perm_sample_index()], golden[key + "sample"])
            and np.array_equal(digest(y), golden[key + "sha256"])):
        raise AssertionError(f"{cname}/{name}: the CPU oracle no longer reproduces the reference's output")
    return y
