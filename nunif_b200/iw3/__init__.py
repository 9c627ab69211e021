"""H100-native mirror of the iw3 hot-path callables (reference: iw3/*.py).

Same names, argument meaning and error behaviour as the reference functions so
that ``iw3.utils.apply_divergence`` / ``postprocess_image`` can import these in
place of the originals (INTEGRATION.md).  Every function requires CUDA tensors
and dispatches to hand-written sm_90a kernels through the C ABI; there is no
CPU path.
"""
from .backward_warp import apply_divergence_grid_sample  # noqa: F401
from .forward_warp import apply_divergence_forward_warp  # noqa: F401
from .dilation import dilate_edge, edge_dilation_parse, edge_dilation_is_enabled, mask_closing, dilate_outer, dilate_inner  # noqa: F401
from .depth_scaler import minmax_normalize, depth_mapper, EMAMinMaxScaler  # noqa: F401
from .mapper import get_mapper, resolve_mapper_name, get_mapper_levels  # noqa: F401
from .mapper import METRIC_DIV_MAPPER, RELATIVE_MUL_MAPPER, RELATIVE_SHIFT_MAPPER, LEGACY_MAPPER, MAPPER_ALL  # noqa: F401
from .base_depth_model import BaseDepthModel  # noqa: F401
from .anaglyph import apply_anaglyph_redcyan  # noqa: F401
from .stereo import stereo_sbs  # noqa: F401
from .frames import hwc_to_chw_float, chw_float_to_hwc  # noqa: F401
from .depth_anything_preprocess import batch_preprocess, preprocess_size  # noqa: F401
from .depth_anything_model import DepthAnythingModel, DepthAnythingNet, batch_infer  # noqa: F401
from . import zoedepth_preprocess  # noqa: F401
from .zoedepth_model import ZoeDepthModel, ZoeDepthNet  # noqa: F401
from .zoedepth_any_model import ZoeDepthAnythingModel, ZoeDepthAnythingNet  # noqa: F401
from .null_depth_model import NullDepthModel, NullDepthNet  # noqa: F401
from .depth_model_factory import create_depth_model  # noqa: F401
from .row_flow import RowFlowV3, MLBW, apply_divergence_nn_LR, apply_divergence_nn_delta, apply_divergence_nn_delta_weight  # noqa: F401
from .row_flow import RowFlowV2, apply_divergence_nn_symmetric, load_row_flow_model  # noqa: F401
from .row_flow import postprocess_hole_mask  # noqa: F401
from .depth_aa import DepthAA  # noqa: F401
from .postprocess import postprocess_image, postprocess_padding, resize_bicubic_aa, rot90, equirectangular_projection  # noqa: F401
from .forward_inpaint import ForwardInpaint, LightInpaintV1  # noqa: F401
from .mlbw_inpaint import MLBWInpaint  # noqa: F401
from .convergence_estimator import ConvergenceEstimator, SODV1  # noqa: F401
from .utils import apply_divergence, process_image, preprocess_image, apply_rgbd, debug_depth_image  # noqa: F401
from .video import bind_single_frame_callback, bind_batch_frame_callback  # noqa: F401
