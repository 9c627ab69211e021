"""CPU: the depth export / import restatement (oracle/depth_export.py) against tests/golden/depth_export.npz, generated
from the reference's export_images and process_config_images (oracle/gen_golden_depth_export.py), and the engine's
iw3_export.yml mirror (nunif_b200/iw3/export_config.py)."""
import json
from fractions import Fraction

import numpy as np
import pytest
import torch
import yaml

from nunif_b200.iw3 import export_config as EC
from oracle import depth_export as O
from oracle.mapper import mapper as oracle_mapper
from tests.util import load_golden

G = load_golden("depth_export")
META = json.loads(str(G["meta"]))
N = len(META["image_sizes"])


@pytest.mark.parametrize("case", list(META["export_cases"]))
def test_oracle_export_equals_golden(case):
    _res, disparity, mapper, fit = META["export_cases"][case]
    for i in range(N):
        depth = torch.from_numpy(G[f"export/{case}/infer/{i}"])
        mn, mx = depth.min(), depth.max()
        depth = (depth - mn) / (mx - mn)   # minmax_normalize_chw without EMA
        got = O.export_frame(depth, (lambda x: oracle_mapper(x, mapper)) if disparity else None,
                             META["image_sizes"][i] if fit else None, align_corners=True)
        np.testing.assert_array_equal(got.numpy(), G[f"export/{case}/depth/{i}"])
        assert json.loads(str(G[f"export/{case}/text/{i}"])) == {}


@pytest.mark.parametrize("case", list(META["import_cases"]))
def test_oracle_import_equals_load_depth(case):
    for i in range(N):
        text = json.loads(str(G[f"import/{case}/text/{i}"]))
        rng = (float(text["iw3_min_depth_value"]), float(text["iw3_max_depth_value"])) if "iw3_min_depth_value" in text else None
        got = O.import_frame(G[f"import/{case}/map/{i}"], rng)
        np.testing.assert_array_equal(got.numpy(), G[f"import/{case}/decoded/{i}"])
        assert f"import/{case}/sbs/{i}" in G


@pytest.mark.parametrize("case", list(META["export_cases"]))
def test_export_config_round_trips_golden(case, tmp_path):
    want = json.loads(str(G[f"export/{case}/yml"]))
    f = tmp_path / EC.FILENAME
    with open(f, "w") as fh:
        yaml.dump(dict(want, updated_at="2026-01-02T03:04:05"), fh, default_flow_style=False, sort_keys=False)
    cfg = EC.ExportConfig.load(str(f))
    assert cfg.type == EC.IMAGE_TYPE and cfg.fps is None
    assert cfg.updated_at.year == 2026
    # an image config is written with fps 1 and no audio file, as export_images does
    cfg.fps, cfg.audio_file = 1, None
    got = cfg.to_yaml_dict(updated_at="x")
    got.pop("updated_at")
    assert got == want and list(got) == list(want)


def test_export_config_yaml_matches_reference_bytes(tmp_path):
    """The mirror writes the reference's yml byte for byte apart from updated_at (the golden's yml_text/* entries)."""
    kw = dict(json.loads(str(G["yml_kwargs"])))
    for key in sorted(k for k in G if k.startswith("yml_text/")):
        fps = json.loads(str(G[key.replace("yml_text/", "yml_fps/")]))
        fps = Fraction(*fps) if isinstance(fps, list) else fps
        EC.ExportConfig(**dict(kw, fps=fps)).save(str(tmp_path / "e.yml"))
        got = "".join(ln for ln in open(tmp_path / "e.yml").read().splitlines(True) if not ln.startswith("updated_at"))
        assert got == str(G[key])


@pytest.mark.parametrize("fps,want", [("30000/1001", Fraction(30000, 1001)), (30, 30), (29.97, 29.97), ("25", 25.0)])
def test_export_config_video_fps(fps, want, tmp_path):
    f = tmp_path / EC.FILENAME
    f.write_text(yaml.dump({"type": "video", "fps": fps}))
    got = EC.ExportConfig.load(str(f)).fps
    assert got == want and type(got) is type(want)


@pytest.mark.parametrize("doc", [{"type": "movie", "fps": 30}, {"fps": 30}, {"type": "video", "fps": "abc"},
                                 {"type": "video", "fps": None}, {"type": "video", "fps": "30/"}])
def test_export_config_refuses(doc, tmp_path):
    f = tmp_path / EC.FILENAME
    f.write_text(yaml.dump(doc))
    with pytest.raises(ValueError):
        EC.ExportConfig.load(str(f))


def test_export_config_resolve_paths(tmp_path):
    (tmp_path / "rgb").mkdir()
    (tmp_path / "depth").mkdir()
    cfg = EC.ExportConfig(EC.VIDEO_TYPE, fps=30)
    rgb, depth, audio = cfg.resolve_paths(str(tmp_path))
    assert (rgb, depth, audio) == (str(tmp_path / "rgb"), str(tmp_path / "depth"), None)
    (tmp_path / "audio.m4a").write_bytes(b"")
    assert cfg.resolve_paths(str(tmp_path))[2] == str(tmp_path / "audio.m4a")
    cfg.depth_dir = "missing"
    with pytest.raises(ValueError):
        cfg.resolve_paths(str(tmp_path))


def test_oracle_video_export_resets_at_scene_end():
    """Frames after a scene boundary are normalised as a fresh sequence, and differ from a run without the boundary."""
    g = torch.Generator().manual_seed(3)
    depths = [torch.rand((1, 6, 8), generator=g) * (i + 1) + 0.5 * i for i in range(7)]
    split = O.export_video_frames(depths, [False, False, True, False, False, False, False], decay=0.75, buffer_size=2)
    assert [i for i, _ in split] == list(range(7))
    first = O.export_video_frames(depths[:3], [False] * 3, decay=0.75, buffer_size=2)
    second = O.export_video_frames(depths[3:], [False] * 4, decay=0.75, buffer_size=2)
    for (_, got), (_, want) in zip(split, first + second):
        assert torch.equal(got, want)
    whole = O.export_video_frames(depths, [False] * 7, decay=0.75, buffer_size=2)
    assert not all(torch.equal(a, b) for (_, a), (_, b) in zip(split[3:], whole[3:]))
