"""ctypes binding of libb200nerf.so (see include/b200nerf.h).  There is no fallback: if the library is missing or
fails to load, importing/using the backend raises."""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_uint8, c_void_p

from . import build as _build

MAX_LEVELS = 16
FIELD_MAIN, FIELD_PROP0, FIELD_PROP1 = 0, 1, 2


class GridDesc(ctypes.Structure):
    _fields_ = [
        ("num_levels", c_int32),
        ("features_per_level", c_int32),
        ("log2_hashmap_size", c_int32),
        ("scalings", c_float * MAX_LEVELS),
    ]


class TcnnGridDesc(ctypes.Structure):
    """b200nerf_tcnn_grid_desc: tiny-cuda-nn HashGrid layout (per-level constants from tcnn_compat.grid_layout)."""

    _fields_ = [
        ("num_levels", c_int32),
        ("features_per_level", c_int32),
        ("n_input_dims", c_int32),
        ("scale", c_float * MAX_LEVELS),
        ("resolution", ctypes.c_uint32 * MAX_LEVELS),
        ("offset", ctypes.c_uint32 * MAX_LEVELS),
        ("size", ctypes.c_uint32 * MAX_LEVELS),
        ("dense", c_uint8 * MAX_LEVELS),
        ("scalings", c_float * MAX_LEVELS),
    ]


class Rays(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in
                ("origins", "directions", "pixel_area", "times", "nears", "fars", "sensor_idx", "is_lidar")] + [("image_width", c_int32)]


class Outputs(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in
                ("features", "depth", "accumulation", "prop_depth_0", "prop_depth_1", "intensity", "ray_drop_logit")]


MAX_PEERS = 16


class PeerOutputs(ctypes.Structure):
    _fields_ = [("n_peers", c_int32), ("self_rank", c_int32), ("row_offset", c_int64),
                ("features", c_void_p * MAX_PEERS), ("depth", c_void_p * MAX_PEERS), ("accumulation", c_void_p * MAX_PEERS)]


TRACE_FIELDS = ("prop_weights_0", "prop_weights_1", "bins_s_1", "bins_e_1", "bins_s_2", "bins_e_2", "inds_1", "inds_2",
                "sdf", "alpha", "field_feature", "weights", "actor_id_0", "actor_id_1", "actor_id_main")


class Trace(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in TRACE_FIELDS]


# name -> (restype, argtypes); every symbol include/b200nerf.h declares
class ConvParams(ctypes.Structure):
    _fields_ = [("weight", c_void_p), ("bias", c_void_p)]


class ConvBnParams(ctypes.Structure):
    _fields_ = [("conv_weight", c_void_p), ("conv_bias", c_void_p), ("bn_weight", c_void_p), ("bn_bias", c_void_p),
                ("bn_running_mean", c_void_p), ("bn_running_var", c_void_p)]


class RgbDecoderParams(ctypes.Structure):
    _fields_ = [("in_dim", ctypes.c_int32), ("hidden_dim", ctypes.c_int32), ("upsample", ctypes.c_int32), ("bn_eps", c_float),
                ("in_conv", ConvParams), ("block", (ConvBnParams * 2) * 4), ("up_conv", ConvParams), ("out_conv", ConvParams)]


SIGNATURES = {
    "b200nerf_last_error": (c_char_p, []),
    "b200nerf_version": (c_int, []),
    "b200nerf_create": (c_int, [c_int, POINTER(c_void_p)]),
    "b200nerf_destroy": (c_int, [c_void_p]),
    "b200nerf_set_field_grids": (c_int, [c_void_p, c_int, POINTER(GridDesc), c_void_p, POINTER(GridDesc),
                                         POINTER(c_void_p), c_int, c_float, c_float]),
    "b200nerf_set_proposal_decoder": (c_int, [c_void_p, c_int, c_void_p, c_int]),
    "b200nerf_set_main_mlps": (c_int, [c_void_p] + [c_void_p] * 10 + [c_float]),
    "b200nerf_set_lidar_decoder": (c_int, [c_void_p] + [c_void_p] * 6),
    "b200nerf_set_appearance": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_float]),
    "b200nerf_set_appearance_per_sensor": (c_int, [c_void_p, c_void_p, c_int, c_int]),
    "b200nerf_set_actors": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    POINTER(c_float)]),
    "b200nerf_set_sampling": (c_int, [c_void_p, c_int, c_int, c_int, c_float, c_float, c_float, c_float,
                                      POINTER(c_float), POINTER(c_float), POINTER(c_int), c_float]),
    "b200nerf_nff_render_fwd": (c_int, [c_void_p, POINTER(Rays), c_int64, POINTER(Outputs), POINTER(Trace), c_void_p]),
    "b200nerf_set_param_stream": (c_int, [c_void_p, c_void_p]),
    "b200nerf_set_field_grids_tcnn": (c_int, [c_void_p, c_int, POINTER(TcnnGridDesc), c_void_p, POINTER(TcnnGridDesc), c_void_p, c_int,
                                              c_float, c_float]),
    "b200nerf_tcnn_hashgrid_fwd": (c_int, [c_void_p, POINTER(TcnnGridDesc), c_void_p, c_void_p, c_void_p, c_int64, c_void_p]),
    "b200nerf_hashgrid_fwd": (c_int, [c_void_p, POINTER(GridDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_int64,
                                      c_void_p]),
    "b200nerf_sh4_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_void_p]),
    "b200nerf_mlp_fwd": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, POINTER(c_void_p), POINTER(c_void_p),
                                 POINTER(c_int), c_void_p, c_void_p]),
    "b200nerf_mlp_fwd_train": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, POINTER(c_void_p), POINTER(c_void_p),
                                       POINTER(c_int), c_void_p, POINTER(c_void_p), c_void_p]),
    "b200nerf_mlp_dgrad": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "b200nerf_check_status": (c_int, [c_void_p]),
    "b200nerf_set_mlp_mode": (c_int, [c_void_p, c_int]),
    "b200nerf_set_peer_outputs": (c_int, [c_void_p, POINTER(PeerOutputs)]),
    "b200nerf_pdf_resample": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_void_p,
                                      c_void_p, c_void_p, c_void_p]),
    "b200nerf_density_to_weights": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "b200nerf_alpha_to_weights": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "b200nerf_spaced_sample": (c_int, [c_void_p, c_int, c_float, c_float, c_void_p, c_void_p, c_int64, c_int, c_void_p,
                                       c_void_p, c_void_p]),
    "b200nerf_isotropic_gaussian_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p,
                                                c_void_p, c_void_p]),
    "b200nerf_neurad_encoding_fwd": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int64,
                                             c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200nerf_neurad_encoding_bwd": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p,
                                             c_void_p, c_void_p, c_void_p, POINTER(c_void_p), c_void_p, c_void_p]),
    "b200nerf_neurad_encoding_pose_bwd": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p,
                                                  c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200nerf_neurad_encoding_mean_bwd": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p,
                                                  c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200nerf_isotropic_gaussian_bwd": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200nerf_hashgrid_bwd": (c_int, [c_void_p, POINTER(GridDesc), c_void_p, c_void_p, c_int64, c_void_p, c_void_p]),
    "b200nerf_alpha_to_weights_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p]),
    "b200nerf_density_to_weights_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p]),
    "b200nerf_composite_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                       c_int64, c_int, c_void_p, c_void_p, c_void_p]),
    "b200nerf_field_heads_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_float,
                                         c_void_p, c_void_p, c_void_p]),
    "b200nerf_linear_wgrad": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b200nerf_linear_wgrad_tc": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b200nerf_relu_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_void_p]),
    "b200nerf_field_mid_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p]),
    "b200nerf_field_tail_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_float, c_void_p, c_void_p, c_void_p,
                                        c_void_p]),
    "b200nerf_spacing_to_euclidean": (c_int, [c_void_p, c_int, c_float, c_float, c_void_p, c_void_p, c_void_p, c_int64, c_int,
                                              c_void_p, c_void_p]),
    "b200nerf_spaced_sample_stratified": (c_int, [c_void_p, c_int, c_float, c_float, c_void_p, c_void_p, c_void_p, c_int, c_int64,
                                                  c_int, c_void_p, c_void_p, c_void_p]),
    "b200nerf_pdf_resample_stratified": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                                 c_float, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200nerf_distortion_loss": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_void_p]),
    "b200nerf_zipnerf_interlevel_loss": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_float, c_int64,
                                                 c_void_p, c_void_p, c_void_p]),
    "b200nerf_lidar_carving_mask": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_float, c_int64, c_int,
                                            c_void_p, c_void_p]),
    "b200nerf_frustum_positions": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, POINTER(c_float),
                                           c_void_p, c_void_p]),
    "b200nerf_density_rgb_heads": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_void_p]),
    "b200nerf_composite": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(c_float), c_void_p, c_void_p,
                                   c_int, c_int64, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200nerf_set_rgb_decoder": (c_int, [c_void_p, POINTER(RgbDecoderParams)]),
    "b200nerf_rgb_decode_workspace_bytes": (c_int64, [c_int, c_int, c_int]),
    "b200nerf_rgb_decode_fwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int64, c_int,
                                        c_void_p]),
    "b200nerf_raygen_pinhole": (c_int, [c_void_p, POINTER(c_float), c_float, c_float, c_float, c_float, c_int, c_int,
                                        c_int, c_int, c_int, c_int, c_int, c_int, c_float, POINTER(c_float), c_float,
                                        c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200nerf_raygen_lidar_grid": (c_int, [c_void_p, POINTER(c_float), c_float, c_float, c_int, c_int, c_double, c_float,
                                           c_float, POINTER(c_float), c_float, c_float, c_void_p, c_void_p, c_void_p,
                                           c_void_p, c_void_p]),
    "b200nerf_raygen_lidar_points": (c_int, [c_void_p, POINTER(c_float), c_void_p, c_int, c_int64, c_float,
                                             POINTER(c_float), c_float, c_float, c_void_p, c_void_p, c_void_p,
                                             c_void_p, c_void_p, c_void_p]),
}

_LIB = None


def library_path() -> str:
    """The in-tree library; B200NERF_LIB selects an A/B build of the same sources (neurad-studio_b200/build.py
    build_variant) for GPU experiments."""
    return os.environ.get("B200NERF_LIB") or _build.LIB_PATH


def load(build_if_missing: bool = True) -> ctypes.CDLL:
    """Load (building first if the .so is absent and nvcc is available) and bind every exported symbol."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = library_path()
    if not os.path.exists(path):
        if not build_if_missing:
            raise RuntimeError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
        _build.build()
    lib = ctypes.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _LIB = lib
    return lib


class B200NerfError(RuntimeError):
    pass


def check(lib: ctypes.CDLL, rc: int) -> None:
    if rc != 0:
        raise B200NerfError(f"libb200nerf error {rc}: {lib.b200nerf_last_error().decode()}")
