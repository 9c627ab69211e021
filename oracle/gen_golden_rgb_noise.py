"""Generate tests/golden/rgb_noise.npz by running the REAL reference nunif/utils/rgb_noise.py (rgb_noise_like,
apply_rgb_noise) on the CPU, in fp32, on seeded inputs (oracle/rgb_noise.py lists them).

Run from the repository root, as a module:
    PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=<nunif checkout> python -m oracle.gen_golden_rgb_noise

  noise/<case>                       rgb_noise_like(torch.zeros(shape), level) after torch.manual_seed(seed)
  noise/<case>/sha256, crop<i>       for the FULL_NOISE cases: its SHA-256 and the CROPS of its last frame
  apply/<case>/<params>              apply_rgb_noise(golden_rgb(shape, 100 + i), rgb_noise_like(...) after
                                     torch.manual_seed(200 + i), **PARAMS[params])
  temporal/noise<t>, buffer<t>, out<t>, u8_<t>, u16_<t>
                                     the video path (ui_utils.py:167-175) over TEMPORAL_SHAPES: frame t is
                                     golden_rgb(shape, 300 + t), its noise rgb_noise_like after torch.manual_seed(400 + t);
                                     the buffer after the frame, apply_rgb_noise of it, and from_tensor's 8 / 16-bit frames
"""
import os

import numpy as np
import torch

from oracle import rgb_noise as orn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "rgb_noise.npz")


def main():
    from nunif.utils.rgb_noise import rgb_noise_like, apply_rgb_noise
    torch.set_num_threads(1)
    out = {}
    for name, shape, level, seed in orn.NOISE_CASES:
        torch.manual_seed(seed)
        n = rgb_noise_like(torch.zeros(shape), level).numpy()
        torch.manual_seed(seed)
        assert np.array_equal(n, orn.rgb_noise_like(torch.zeros(shape), level).numpy()), name
        if name in orn.FULL_NOISE:
            out[f"noise/{name}/sha256"] = orn.digest(n)
            for i, (sy, sx) in enumerate(orn.CROPS):
                out[f"noise/{name}/crop{i}"] = n[..., sy, sx]
        else:
            out[f"noise/{name}"] = n
    for i, (name, shape) in enumerate(orn.APPLY_CASES):
        rgb = orn.golden_rgb(shape, 100 + i)
        torch.manual_seed(200 + i)
        noise = rgb_noise_like(rgb) * 3.0       # wide enough that the clamp bites at both ends
        out[f"apply/{name}/noise"] = noise.numpy()
        for pname, kw in orn.PARAMS.items():
            y = apply_rgb_noise(rgb.clone(), noise.clone(), **kw)
            assert np.array_equal(y.numpy(), orn.apply_rgb_noise(rgb.clone(), noise.clone(), **kw).numpy()), (name, pname)
            out[f"apply/{name}/{pname}"] = y.numpy()
    # ui_utils.py:166-177 with the reference's own state: noise_buffer starts as an empty tensor
    noise_buffer = torch.zeros((0,))
    for t, shape in enumerate(orn.TEMPORAL_SHAPES):
        rgb = orn.golden_rgb(shape, 300 + t)
        torch.manual_seed(400 + t)
        noise = rgb_noise_like(rgb)
        out[f"temporal/noise{t}"] = noise.numpy().copy()       # the reference scales noise in place below
        if noise.shape != noise_buffer.shape:
            noise_buffer.resize_(noise.shape)
            noise_buffer.copy_(noise)
        else:
            noise_buffer.mul_((1.0 - orn.TEMPORAL_SPEED))
            noise_buffer.add_(noise.mul_(orn.TEMPORAL_SPEED))
        y = apply_rgb_noise(rgb, noise_buffer, strength=orn.TEMPORAL_STRENGTH)
        out[f"temporal/buffer{t}"] = noise_buffer.numpy().copy()
        out[f"temporal/out{t}"] = y.numpy()
        out[f"temporal/u8_{t}"] = orn.from_tensor(y, 8).numpy()
        out[f"temporal/u16_{t}"] = orn.from_tensor(y, 16).numpy()
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
