"""``iw3_export.yml``, the file ``--export`` writes beside the depth maps and that an ``iw3_export.yml`` input reads back
(iw3/export_config.py).  Host only.  The keys, their order and the ``fps`` forms are the reference's:

* ``fps`` is saved as an int, as ``"num/den"`` for a non-integral Fraction, else as a float; on load a video's ``fps``
  becomes a Fraction (``"num/den"``), stays an int, or becomes a float, and anything else raises ``ValueError``;
* an image export has no ``fps`` and no audio file on load;
* ``type`` must be ``images`` or ``video`` (``ValueError`` on load).
"""
from datetime import datetime
from fractions import Fraction
from os import path

import yaml

FILENAME = "iw3_export.yml"
RGB_DIR = "rgb"
DEPTH_DIR = "depth"
AUDIO_FILE = "audio.m4a"
IMAGE_TYPE = "images"
VIDEO_TYPE = "video"
_TYPES = (IMAGE_TYPE, VIDEO_TYPE)


def _fps_to_yaml(fps):
    if isinstance(fps, Fraction):
        return fps.numerator if fps.denominator == 1 else f"{fps.numerator}/{fps.denominator}"
    if type(fps) is int:
        return fps
    return float(fps)


def _fps_from_yaml(fps, file_path):
    try:
        if isinstance(fps, str) and "/" in fps:
            parts = fps.split("/")
            return Fraction(int(parts[0]), int(parts[1]))
        if type(fps) is int:
            return fps
        return float(fps)
    except (ValueError, TypeError, IndexError, ZeroDivisionError):
        raise ValueError(f"Invalid fps={fps} in {file_path}")


def resolve_path(base_dir, entry):
    """``entry`` relative to ``base_dir`` unless it is absolute or None."""
    if entry is None or path.isabs(entry):
        return entry
    return path.join(base_dir, entry)


class ExportConfig:
    def __init__(self, type, basename=None, fps=None, mapper=None, skip_mapper=None, skip_edge_dilation=None,
                 rgb_dir=None, depth_dir=None, audio_file=None, user_data=None, updated_at=None,
                 output_colorspace=None, source_color_range=None):
        assert type in _TYPES
        self.type = type
        self.basename = basename
        self.fps = fps
        self.mapper = mapper
        self.skip_mapper = skip_mapper
        self.skip_edge_dilation = skip_edge_dilation
        self.rgb_dir = rgb_dir or RGB_DIR
        self.depth_dir = depth_dir or DEPTH_DIR
        self.audio_file = audio_file or AUDIO_FILE
        self.output_colorspace = output_colorspace
        self.source_color_range = source_color_range
        self.user_data = {} if user_data is None else user_data
        self.updated_at = updated_at

    def to_yaml_dict(self, updated_at=None):
        """The mapping ``save`` writes, in its key order; ``updated_at`` defaults to now (local time, ISO format)."""
        config = {"type": self.type}
        if self.basename:
            config["basename"] = self.basename
        config["fps"] = _fps_to_yaml(self.fps)
        config["rgb_dir"] = self.rgb_dir
        config["depth_dir"] = self.depth_dir
        if self.audio_file:
            config["audio_file"] = self.audio_file
        for key in ("mapper", "skip_mapper", "skip_edge_dilation", "source_color_range", "output_colorspace"):
            if getattr(self, key) is not None:
                config[key] = getattr(self, key)
        config["updated_at"] = updated_at if updated_at is not None else datetime.now().isoformat()
        config["user_data"] = self.user_data
        return config

    def save(self, file_path, updated_at=None):
        with open(file_path, mode="w", encoding="utf-8") as f:
            yaml.dump(self.to_yaml_dict(updated_at), f, encoding="utf-8", default_flow_style=False, sort_keys=False)

    @staticmethod
    def load(file_path):
        with open(file_path, mode="r", encoding="utf-8") as f:
            config = yaml.safe_load(f)
        export_type = config.get("type")
        if export_type not in _TYPES:
            raise ValueError(f"Unsupported type={export_type} in {file_path}")
        video = export_type == VIDEO_TYPE
        updated_at = config.get("updated_at")
        if updated_at is not None:
            try:
                updated_at = datetime.fromisoformat(updated_at)
            except (TypeError, ValueError):
                updated_at = None
        return ExportConfig(export_type, basename=config.get("basename"),
                            fps=_fps_from_yaml(config.get("fps"), file_path) if video else None,
                            mapper=str(config.get("mapper", "none")),
                            skip_mapper=config.get("skip_mapper", False),
                            skip_edge_dilation=config.get("skip_edge_dilation", False),
                            rgb_dir=config.get("rgb_dir"), depth_dir=config.get("depth_dir"),
                            audio_file=config.get("audio_file") if video else None,
                            user_data=config.get("user_data", {}), updated_at=updated_at,
                            source_color_range=config.get("source_color_range"),
                            output_colorspace=config.get("output_colorspace"))

    def to_dict(self):
        return dict(type=self.type, basename=self.basename, fps=self.fps, mapper=self.mapper, skip_mapper=self.skip_mapper,
                    skip_edge_dilation=self.skip_edge_dilation, rgb_dir=self.rgb_dir, depth_dir=self.depth_dir,
                    audio_file=self.audio_file, user_data=self.user_data, updated_at=self.updated_at)

    def __repr__(self):
        return repr(self.to_dict())

    def resolve_paths(self, base_dir):
        """(rgb_dir, depth_dir, audio_file) under ``base_dir``; raises ``ValueError`` if a directory is missing.  The
        audio file is None for images or when it does not exist."""
        rgb_dir = resolve_path(base_dir, self.rgb_dir or "rgb_dir")
        depth_dir = resolve_path(base_dir, self.depth_dir or "depth_dir")
        audio_file = resolve_path(base_dir, self.audio_file)
        if not path.exists(rgb_dir):
            raise ValueError(f"ExportConfig: rgb_dir={rgb_dir} not found")
        if not path.exists(depth_dir):
            raise ValueError(f"ExportConfig: depth_dir={depth_dir} not found")
        if self.type != VIDEO_TYPE or (audio_file is not None and not path.exists(audio_file)):
            audio_file = None
        return rgb_dir, depth_dir, audio_file
