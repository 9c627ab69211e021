"""Mirror of iw3/depth_model_factory.py:10-33: ``create_depth_model(model_type)``, the call iw3 makes for ``--depth-model``
(iw3/utils.py:2191).  Routes to the engine's depth models; a model type iw3 knows but the engine does not build raises
NotImplementedError naming it, an unknown one ValueError as in the reference."""
from .zoedepth_model import ZoeDepthModel
from .zoedepth_any_model import ZoeDepthAnythingModel
from .depth_anything_model import DepthAnythingModel
from .null_depth_model import NullDepthModel

# model types of iw3's other depth models (depth_anything_model.py:12-35, zoedepth_model.py:12-20, depth_pro_model.py,
# video_depth_anything*_model.py, depth_anything_v3_model.py) that the engine does not build
NOT_BUILT = (
    ["ZoeD_K", "ZoeD_NK"]
    + [f"Any_V2_{d}_{s}" for d in "NK" for s in "SBL"] + ["Any_V2_N", "Any_V2_K"]
    + [f"Distill_Any_{s}" for s in "SBL"]
    + ["DepthPro", "DepthPro_S"]
    + [f"VDA_{s}" for s in "SBL"] + ["VDA_Metric"] + [f"VDA_Metric_{s}" for s in "SBL"]
    + [f"VDA_Stream_{s}" for s in "SBL"] + [f"VDA_Stream_Metric_{s}" for s in "SBL"]
    + ["Any_V3_Mono", "Any_V3_Mono_01"]
)


def create_depth_model(model_type):
    for cls in (ZoeDepthModel, ZoeDepthAnythingModel, DepthAnythingModel, NullDepthModel):
        if cls.supported(model_type):
            return cls(model_type)
    if model_type in NOT_BUILT:
        raise NotImplementedError(f"depth model {model_type} is not built on the H100 engine")
    raise ValueError(f"{model_type} is not supported")
