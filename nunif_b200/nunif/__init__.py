"""H100-native mirror of the nunif pieces on the waifu2x hot path
(nunif/models/model.py, nunif/models/utils.py, nunif/utils/render.py)."""
