"""H100-native mirror of waifu2x.hub / waifu2x.utils (reference: waifu2x/hub.py, waifu2x/utils.py)."""
from .utils import Waifu2x  # noqa: F401
from .hub import Waifu2xImageModel, waifu2x, MODEL_TYPES, METHODS  # noqa: F401
