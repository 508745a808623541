"""config_*.yml -> plain parameter structs.  The reference reads one shared YAML::Node at call time
(SURVEY.md §5); the yml files stay UNCHANGED — this module only maps the keys the hot path reads onto the C-ABI
structs.  Keys and their readers in the reference:

  bundle.num_iter_outter / num_iter_inner / robust_delta   Solver/CUDASolverBundling.cpp:193,210,214
  bundle.image_downscale                                    LossGPU.cu:55
  p2p.max_dist / p2p.max_normal_angle                       Solver/CUDASolverBundling.cpp:93-94
  feature_corres.max_dist_*/max_normal_*                    FeatureManager.cpp:292-295
  ransac.max_iter / ransac.inlier_dist                      FeatureManager.cpp:663-670,713
  bundle.max_BA_frames / min_fm_edges_newframe              Bundler.cpp:222-274,343
"""
from __future__ import annotations

import copy
import math
from typing import Any, Mapping, Union

from ._lib import SolverParams

# Values of the reference's config_nocs.yml for the keys above (used when no yml is supplied, e.g. synthetic benches).
NOCS_DEFAULTS = {
    "bundle": {"num_iter_outter": 7, "num_iter_inner": 5, "window_size": 2, "max_BA_frames": 15,
               "subset_selection_method": "greedy_rot", "robust_delta": 0.005, "min_fm_edges_newframe": 10,
               "image_downscale": 4},
    "keyframe": {"min_interval": 1, "min_feat_num": 0, "min_rot": 10},
    "feature_corres": {"mutual": True, "max_dist_no_neighbor": 0.02, "max_normal_no_neighbor": 45,
                       "max_dist_neighbor": 10000, "max_normal_neighbor": 180},
    "ransac": {"max_iter": 2000, "num_sample": 3, "inlier_dist": 0.005, "inlier_normal_angle": 45,
               "max_trans_neighbor": 0.2, "max_rot_deg_neighbor": 25, "max_trans_no_neighbor": 0.02,
               "max_rot_no_neighbor": 10},
    "p2p": {"max_dist": 0.02, "max_normal_angle": 45},
    "depth_processing": {"erode": {"radius": 1, "diff": 0.001, "ratio": 0.8},
                         "bilateral_filter": {"radius": 2, "sigma_D": 2, "sigma_R": 100000}},
}


def load_yml(yml: Union[None, str, Mapping[str, Any]]) -> dict:
    """Accepts a path to a config_*.yml, an already-parsed mapping, or None (NOCS defaults)."""
    if yml is None:
        return copy.deepcopy(NOCS_DEFAULTS)
    if isinstance(yml, str):
        import yaml
        with open(yml) as f:
            return yaml.safe_load(f)
    return dict(yml)


def solver_params(yml: Union[None, str, Mapping[str, Any]] = None) -> SolverParams:
    y = load_yml(yml)
    b, p2p = y["bundle"], y["p2p"]
    return SolverParams(
        int(b["num_iter_outter"]), int(b["num_iter_inner"]), float(b["robust_delta"]), float(b["image_downscale"]),
        float(p2p["max_dist"]), float(math.cos(float(p2p["max_normal_angle"]) / 180.0 * math.pi)),
        0.1, 9999.0,   # denseDepthMin / denseDepthMax, hard-wired (CUDASolverBundling.cpp:97-98)
        1.0, 1.0,      # m_localWeightsSparse / m_localWeightsDenseDepth (SBA.cpp:28-30)
    )


def depth_params(yml: Union[None, str, Mapping[str, Any]] = None):
    """config "depth_processing" -> bt_depth_params (read where Frame::processDepth reads it, Frame.cpp:160-165)."""
    from ._lib import DepthParams
    y = load_yml(yml)
    dp = y.get("depth_processing", NOCS_DEFAULTS["depth_processing"])
    e, b = dp["erode"], dp["bilateral_filter"]
    return DepthParams(int(e["radius"]), float(e["diff"]), float(e["ratio"]), int(b["radius"]), float(b["sigma_D"]), float(b["sigma_R"]))


def mask_mode(yml: Union[None, str, Mapping[str, Any]] = None) -> int:
    """config "data_dir" -> bt_frames_preprocess_masked's mask_mode.  The reference keeps only the convex hull of the mask's largest
    component when data_dir contains "NOCS" and uses the mask as it is otherwise (Frame.cpp:251,267).  Without a yml: the NOCS
    defaults, i.e. largest-hull mode."""
    from ._lib import BT_MASK_AS_IS, BT_MASK_LARGEST_HULL
    if yml is None:
        return BT_MASK_LARGEST_HULL
    return BT_MASK_LARGEST_HULL if "NOCS" in str(load_yml(yml).get("data_dir", "")) else BT_MASK_AS_IS
