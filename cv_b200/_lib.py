"""ctypes binding of cv_b200/libcvb200.so (the C ABI declared in include/cvb200.h, cvb200_sfm.h and cvb200_tri.h) and of its modules
cv_b200/libcvb200_opt.so (include/cvb200_opt.h), cv_b200/libcvb200_pinhole.so (include/cvb200_pinhole.h), cv_b200/libcvb200_image.so
(include/cvb200_image.h), cv_b200/libcvb200_filter.so (include/cvb200_filter.h), cv_b200/libcvb200_lsh.so (include/cvb200_lsh.h),
cv_b200/libcvb200_stages.so (include/cvb200_stages.h), cv_b200/libcvb200_batch.so (include/cvb200_batch.h), cv_b200/libcvb200_init.so
(include/cvb200_init.h), cv_b200/libcvb200_constraints.so (include/cvb200_constraints.h), cv_b200/libcvb200_reconstruction.so
(include/cvb200_reconstruction.h), cv_b200/libcvb200_export.so (include/cvb200_export.h) and
cv_b200/libcvb200_register.so (include/cvb200_register.h), cv_b200/libcvb200_incorporate.so (include/cvb200_incorporate.h),
cv_b200/libcvb200_merge.so (include/cvb200_merge.h) and cv_b200/libcvb200_try_init.so (include/cvb200_try_init.h)."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

CVB_OK, CVB_EINVAL, CVB_ENODEV, CVB_ECUDA, CVB_ENOMEM, CVB_ECAP, CVB_EUNSUPPORTED = 0, -1, -2, -3, -4, -5, -6
_ERRNAMES = {-1: "EINVAL", -2: "ENODEV", -3: "ECUDA", -4: "ENOMEM", -5: "ECAP", -6: "EUNSUPPORTED"}


class CvbError(RuntimeError):
    def __init__(self, code, msg=""):
        super().__init__(f"cvb200 error {_ERRNAMES.get(code, code)}: {msg}")
        self.code = code


class AkazeCfg(C.Structure):
    """cvb_akaze_cfg == akaze::Akaze (akaze/src/lib.rs:109-142)"""
    _fields_ = [
        ("maximum_features", C.c_int64),
        ("num_sublevels", C.c_uint32),
        ("max_octave_evolution", C.c_uint32),
        ("base_scale_offset", C.c_double),
        ("initial_contrast", C.c_double),
        ("contrast_percentile", C.c_double),
        ("contrast_factor_num_bins", C.c_uint64),
        ("derivative_factor", C.c_double),
        ("detector_threshold", C.c_double),
        ("descriptor_channels", C.c_uint64),
        ("descriptor_pattern_size", C.c_uint64),
    ]


# cvb_keypoint == akaze::KeyPoint (akaze/src/lib.rs:71-93)
KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("response", "<f4"), ("size", "<f4"), ("angle", "<f4"),
                     ("octave", "<u4"), ("class_id", "<u4")])

# every symbol include/cvb200.h declares (checked by tests/test_abi.py)
ABI_SYMBOLS = [
    "cvb_ctx_create", "cvb_ctx_create_on_stream", "cvb_ctx_destroy", "cvb_ctx_sync", "cvb_last_error", "cvb_version",
    "cvb_ctx_launch_count", "cvb_ctx_timer_begin", "cvb_ctx_timer_end", "cvb_ctx_profile", "cvb_ctx_profile_report",
    "cvb_akaze_default_cfg", "cvb_akaze_extract", "cvb_akaze_extract_batch", "cvb_akaze_extract_batch_dev", "cvb_akaze_dev_overflow",
    "cvb_akaze_debug_num_evolutions", "cvb_akaze_debug_evolution", "cvb_akaze_debug_plane", "cvb_akaze_debug_contrast",
    "cvb_akaze_debug_stage",
    "cvb_hamming_knn", "cvb_hamming_knn_dev", "cvb_hamming_knn_dev_counts", "cvb_match_symmetric", "cvb_match_symmetric_dev",
    "cvb_arrsac_default_cfg", "cvb_rng_seed_xoshiro256pp", "cvb_rng_seed_pcg64", "cvb_rng_next_u32",
    "cvb_eight_point_batch", "cvb_p3p_batch", "cvb_five_point_batch", "cvb_arrsac_five_point", "cvb_residuals_camera_to_camera", "cvb_residuals_world_to_camera",
    "cvb_triangulate_linear_eigen", "cvb_arrsac_eight_point", "cvb_arrsac_p3p",
    "cvb_hash_bag", "cvb_hash_bag_dev", "cvb_match_symmetric_pairs_dev", "cvb_pair_bearings_dev", "cvb_arrsac_eight_point_dev", "cvb_arrsac_p3p_dev", "cvb_arrsac_commit_rng",
    "cvb_two_view_pair_dev", "cvb_two_view_frames",
    "cvb_single_view_optimize_l2", "cvb_three_view_optimize_l2", "cvb_observation_losses", "cvb_tri_landmarks_robust",
]

# every symbol include/cvb200_sfm.h declares (the K1 camera and cv-sfm's frame ingestion; checked by tests/test_abi_sfm.py)
SFM_ABI_SYMBOLS = [
    "cvb_pair_bearings_k1_dev", "cvb_two_view_pair_k1_dev", "cvb_two_view_frames_k1", "cvb_frame_features_batch", "cvb_frame_features_batch_dev",
]

# every symbol include/cvb200_tri.h declares (cv-geom's triangulators; checked by tests/test_abi_tri.py)
TRI_ABI_SYMBOLS = [
    "cvb_triangulator_default", "cvb_triangulate_observations", "cvb_triangulate_relative", "cvb_observation_losses_tri",
    "cvb_tri_landmarks_robust_tri",
]

# every symbol include/cvb200_opt.h declares (cv-optimize's L1 optimizers), exported by libcvb200_opt.so; checked by tests/test_abi_opt.py
OPT_ABI_SYMBOLS = [
    "cvb_single_view_optimize_l1", "cvb_three_view_optimize_l1",
]

# every symbol include/cvb200_pinhole.h declares (cv-pinhole's reprojection error and EssentialMatrix), exported by libcvb200_pinhole.so;
# checked by tests/test_abi_pinhole.py
PINHOLE_ABI_SYMBOLS = [
    "cvb_pose_reprojection_error", "cvb_pose_reprojection_error_dev", "cvb_eight_point_essential_batch", "cvb_residuals_essential",
    "cvb_essential_recondition", "cvb_essential_decompose",
]

# every symbol include/cvb200_image.h declares (8- and 16-bit frames into the extractor), exported by libcvb200_image.so;
# checked by tests/test_abi_image.py
IMAGE_ABI_SYMBOLS = [
    "cvb_gray_float_from_dynamic_dev", "cvb_akaze_extract_dynamic_batch", "cvb_akaze_extract_dynamic_batch_dev",
    "cvb_frame_features_dynamic_batch", "cvb_two_view_frames_dynamic_k1",
]

# every symbol include/cvb200_filter.h declares (akaze::image: filters, Gaussian kernel and blur, half_size), exported by
# libcvb200_filter.so; checked by tests/test_abi_filter.py
FILTER_ABI_SYMBOLS = [
    "cvb_gaussian_kernel", "cvb_horizontal_filter", "cvb_horizontal_filter_dev", "cvb_vertical_filter", "cvb_vertical_filter_dev",
    "cvb_separable_filter", "cvb_separable_filter_dev", "cvb_gaussian_blur", "cvb_gaussian_blur_dev", "cvb_half_size", "cvb_half_size_dev",
]

# every symbol include/cvb200_lsh.h declares (exact Hamming k-NN over frame hashes: cv-sfm's similar-frame search), exported by
# libcvb200_lsh.so; checked by tests/test_abi_lsh.py
LSH_ABI_SYMBOLS = [
    "cvb_hash_knn", "cvb_hash_knn_dev",
]

# every symbol include/cvb200_stages.h declares (AKAZE's staged surface: scale space, find_image_keypoints, extract_descriptors),
# exported by libcvb200_stages.so; checked by tests/test_abi_stages.py
STAGES_ABI_SYMBOLS = [
    "cvb_akaze_scale_space", "cvb_akaze_scale_space_dev", "cvb_akaze_evolutions", "cvb_akaze_find_image_keypoints",
    "cvb_akaze_find_image_keypoints_dev", "cvb_akaze_extract_descriptors", "cvb_akaze_extract_descriptors_dev",
]

# every symbol include/cvb200_batch.h declares (B independent ARRSAC problems per launch), exported by libcvb200_batch.so; checked by
# tests/test_abi_batch.py
BATCH_ABI_SYMBOLS = [
    "cvb_arrsac_batch_dev", "cvb_arrsac_batch", "cvb_arrsac_commit_rng_batch", "cvb_two_view_options_dev",
]
# CVB_ARRSAC_BATCH_MAX of include/cvb200_batch.h
ARRSAC_BATCH_MAX = 64

# every symbol include/cvb200_init.h declares (cv-sfm's three-view initialisation), exported by libcvb200_init.so; checked by
# tests/test_abi_init.py
INIT_ABI_SYMBOLS = ["cvb_init_cfg_default", "cvb_init_reconstruction_dev"]

# every symbol include/cvb200_constraints.h declares (cv-sfm's three-view constraints), exported by libcvb200_constraints.so; checked by
# tests/test_abi_constraints.py
CONSTRAINTS_ABI_SYMBOLS = ["cvb_constraints_cfg_default", "cvb_view_constraints_check", "cvb_view_constraints_dev", "cvb_view_constraints",
                           "cvb_three_view_adaptive_optimize_l2_dev"]
# CVB_CONSTRAINTS_MAX_LANDMARKS of include/cvb200_constraints.h
CONSTRAINTS_MAX_LANDMARKS = 512

# every symbol include/cvb200_reconstruction.h declares (cv-sfm's reconstruction optimisation), exported by libcvb200_reconstruction.so;
# checked by tests/test_abi_reconstruction.py
RECONSTRUCTION_ABI_SYMBOLS = ["cvb_recon_cfg_default", "cvb_optimize_reconstruction_check", "cvb_optimize_reconstruction_dev",
                              "cvb_optimize_reconstruction"]

# every symbol include/cvb200_export.h declares (cv-sfm's reconstruction export), exported by libcvb200_export.so; checked by
# tests/test_abi_export.py
EXPORT_ABI_SYMBOLS = ["cvb_export_cfg_default", "cvb_export_check", "cvb_robust_landmarks_dev", "cvb_robust_landmarks",
                      "cvb_export_reconstruction_dev", "cvb_export_reconstruction", "cvb_normalize_reconstruction_dev",
                      "cvb_normalize_reconstruction"]
# every symbol include/cvb200_register.h declares (cv-sfm's frame registration), exported by libcvb200_register.so; checked by
# tests/test_abi_register.py
REGISTER_ABI_SYMBOLS = ["cvb_register_cfg_default", "cvb_register_check", "cvb_register_frame_dev", "cvb_register_frame"]
# every symbol include/cvb200_incorporate.h declares (cv-sfm's frame incorporation), exported by libcvb200_incorporate.so; checked by
# tests/test_abi_incorporate.py
INCORPORATE_ABI_SYMBOLS = ["cvb_incorporate_check", "cvb_add_view_dev", "cvb_add_view", "cvb_apply_optimization_dev", "cvb_apply_optimization",
                           "cvb_incorporate_frame_dev", "cvb_incorporate_frame"]
# every symbol include/cvb200_merge.h declares (cv-sfm's reconstruction merging), exported by libcvb200_merge.so; checked by
# tests/test_abi_merge.py
MERGE_ABI_SYMBOLS = ["cvb_merge_check", "cvb_incorporate_reconstruction_dev", "cvb_incorporate_reconstruction", "cvb_merge_reconstructions_dev",
                     "cvb_merge_reconstructions"]
# every symbol include/cvb200_try_init.h declares (cv-sfm's reconstruction creation), exported by libcvb200_try_init.so; checked by
# tests/test_abi_try_init.py
TRY_INIT_ABI_SYMBOLS = ["cvb_try_init_check", "cvb_add_reconstruction_dev", "cvb_add_reconstruction", "cvb_try_init_dev", "cvb_try_init"]

# cvb_akaze_evolution: the scalar fields of akaze's EvolutionStep (evolution.rs:8-44), level size and FED step count
EVOLUTION_DTYPE = np.dtype([("octave", "<u4"), ("sublevel", "<u4"), ("esigma", "<f8"), ("etime", "<f8"), ("sigma_size", "<u4"),
                            ("width", "<u4"), ("height", "<u4"), ("n_fed_steps", "<u4")])


def lib_path():
    return os.path.join(_HERE, "libcvb200.so")


def load_library():
    """Loads the CUDA extension. Fails loudly when it has not been built (no fallback)."""
    global _LIB
    if _LIB is not None:
        return _LIB
    p = lib_path()
    if not os.path.exists(p):
        raise CvbError(CVB_ENODEV, f"{p} not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                                   f"or `make -C cv_b200/csrc`")
    # one hardware queue per stream when many contexts are pipelined (effective only if CUDA is not initialised yet)
    os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
    L = C.CDLL(p)
    vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
    L.cvb_ctx_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.cvb_ctx_create_on_stream.argtypes = [C.c_int, vp, C.POINTER(vp)]
    L.cvb_ctx_destroy.argtypes = [vp]
    L.cvb_ctx_destroy.restype = None
    L.cvb_ctx_sync.argtypes = [vp]
    L.cvb_last_error.argtypes = [vp]
    L.cvb_last_error.restype = C.c_char_p
    L.cvb_version.restype = C.c_char_p
    L.cvb_ctx_launch_count.argtypes = [vp]
    L.cvb_ctx_launch_count.restype = u64
    L.cvb_ctx_timer_begin.argtypes = [vp]
    L.cvb_ctx_timer_end.argtypes = [vp, C.POINTER(C.c_float)]
    L.cvb_ctx_profile.argtypes = [vp, C.c_int]
    L.cvb_ctx_profile_report.argtypes = [vp, C.c_char_p, C.c_size_t]
    L.cvb_akaze_default_cfg.argtypes = [C.POINTER(AkazeCfg)]
    L.cvb_akaze_default_cfg.restype = None
    L.cvb_akaze_extract.argtypes = [vp, C.POINTER(AkazeCfg), vp, u32, u32, vp, vp, u32, C.POINTER(u32)]
    L.cvb_akaze_extract_batch.argtypes = [vp, C.POINTER(AkazeCfg), vp, u32, u32, u32, vp, vp, u32, vp]
    L.cvb_akaze_extract_batch_dev.argtypes = [vp, C.POINTER(AkazeCfg), vp, u32, u32, u32, vp, vp, u32, vp]
    L.cvb_akaze_dev_overflow.argtypes = [vp, C.POINTER(u32)]
    L.cvb_akaze_debug_num_evolutions.argtypes = [vp, C.POINTER(u32)]
    L.cvb_akaze_debug_evolution.argtypes = [vp, u32] + [C.POINTER(u32)] * 5
    L.cvb_akaze_debug_plane.argtypes = [vp, u32, u32, u32, vp]
    L.cvb_akaze_debug_contrast.argtypes = [vp, u32, C.POINTER(C.c_double)]
    L.cvb_akaze_debug_stage.argtypes = [vp, u32, u32, vp, u32, C.POINTER(u32)]
    L.cvb_hamming_knn.argtypes = [vp, vp, u32, vp, u32, u32, vp, vp]
    L.cvb_hamming_knn_dev.argtypes = [vp, vp, u32, vp, u32, u32, vp, vp]
    L.cvb_hamming_knn_dev_counts.argtypes = [vp, vp, vp, u32, vp, vp, u32, u32, vp, vp]
    L.cvb_match_symmetric.argtypes = [vp, vp, u32, vp, u32, u32, vp, u32, C.POINTER(u32)]
    L.cvb_match_symmetric_dev.argtypes = [vp, vp, u32, vp, u32, u32, vp]
    L.cvb_hash_bag.argtypes = [vp, vp, u32, vp, u32, vp]
    L.cvb_hash_bag_dev.argtypes = [vp, vp, vp, u32, vp, u32, vp]
    _LIB = L
    return L


_OPT_LIB = None


def opt_lib_path():
    return os.path.join(_HERE, "libcvb200_opt.so")


def load_opt_library():
    """Loads libcvb200_opt.so, the module of include/cvb200_opt.h over libcvb200.so (same contexts). Fails loudly when missing."""
    global _OPT_LIB
    if _OPT_LIB is None:
        load_library()
        p = opt_lib_path()
        if not os.path.exists(p):
            raise CvbError(CVB_ENODEV, f"{p} not built: run `make -C cv_b200/csrc`")
        _OPT_LIB = C.CDLL(p)
    return _OPT_LIB


_PINHOLE_LIB = None


def pinhole_lib_path():
    return os.path.join(_HERE, "libcvb200_pinhole.so")


def load_pinhole_library():
    """Loads libcvb200_pinhole.so, the module of include/cvb200_pinhole.h over libcvb200.so (same contexts). Fails loudly when missing."""
    global _PINHOLE_LIB
    if _PINHOLE_LIB is None:
        load_library()
        p = pinhole_lib_path()
        if not os.path.exists(p):
            raise CvbError(CVB_ENODEV, f"{p} not built: run `make -C cv_b200/csrc`")
        _PINHOLE_LIB = C.CDLL(p)
    return _PINHOLE_LIB


_IMAGE_LIB = None


def image_lib_path():
    return os.path.join(_HERE, "libcvb200_image.so")


def load_image_library():
    """Loads libcvb200_image.so, the module of include/cvb200_image.h over libcvb200.so (same contexts). Fails loudly when missing."""
    global _IMAGE_LIB
    if _IMAGE_LIB is None:
        load_library()
        p = image_lib_path()
        if not os.path.exists(p):
            raise CvbError(CVB_ENODEV, f"{p} not built: run `make -C cv_b200/csrc`")
        _IMAGE_LIB = C.CDLL(p)
    return _IMAGE_LIB


_FILTER_LIB = None


def filter_lib_path():
    return os.path.join(_HERE, "libcvb200_filter.so")


def load_filter_library():
    """Loads libcvb200_filter.so, the module of include/cvb200_filter.h over libcvb200.so (same contexts). Fails loudly when missing."""
    global _FILTER_LIB
    if _FILTER_LIB is None:
        load_library()
        p = filter_lib_path()
        if not os.path.exists(p):
            raise CvbError(CVB_ENODEV, f"{p} not built: run `make -C cv_b200/csrc`")
        _FILTER_LIB = C.CDLL(p)
    return _FILTER_LIB


_LSH_LIB = None


def lsh_lib_path():
    return os.path.join(_HERE, "libcvb200_lsh.so")


def load_lsh_library():
    """Loads libcvb200_lsh.so, the module of include/cvb200_lsh.h over libcvb200.so (same contexts). Fails loudly when missing."""
    global _LSH_LIB
    if _LSH_LIB is None:
        load_library()
        p = lsh_lib_path()
        if not os.path.exists(p):
            raise CvbError(CVB_ENODEV, f"{p} not built: run `make -C cv_b200/csrc`")
        _LSH_LIB = C.CDLL(p)
    return _LSH_LIB


_STAGES_LIB = None


def stages_lib_path():
    return os.path.join(_HERE, "libcvb200_stages.so")


def load_stages_library():
    """Loads libcvb200_stages.so, the module of include/cvb200_stages.h over libcvb200.so (same contexts). Fails loudly when missing."""
    global _STAGES_LIB
    if _STAGES_LIB is None:
        load_library()
        p = stages_lib_path()
        if not os.path.exists(p):
            raise CvbError(CVB_ENODEV, f"{p} not built: run `make -C cv_b200/csrc`")
        L = C.CDLL(p)
        vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        L.cvb_akaze_scale_space.argtypes = [vp, C.POINTER(AkazeCfg), vp, u32, u32, u32, C.POINTER(u64)]
        L.cvb_akaze_scale_space_dev.argtypes = [vp, C.POINTER(AkazeCfg), vp, u32, u32, u32, C.POINTER(u64)]
        L.cvb_akaze_evolutions.argtypes = [vp, u64, vp, u32, C.POINTER(u32)]
        L.cvb_akaze_find_image_keypoints.argtypes = [vp, u64, vp, u32, vp]
        L.cvb_akaze_find_image_keypoints_dev.argtypes = [vp, u64, vp, u32, vp]
        L.cvb_akaze_extract_descriptors.argtypes = [vp, C.POINTER(AkazeCfg), u64, vp, vp, vp, vp, vp]
        L.cvb_akaze_extract_descriptors_dev.argtypes = [vp, C.POINTER(AkazeCfg), u64, vp, vp, u32, vp, vp, vp]
        _STAGES_LIB = L
    return _STAGES_LIB


_BATCH_LIB = None


def batch_lib_path():
    return os.path.join(_HERE, "libcvb200_batch.so")


def load_batch_library():
    """Loads libcvb200_batch.so, the module of include/cvb200_batch.h over libcvb200.so (same contexts). Fails loudly when missing."""
    global _BATCH_LIB
    if _BATCH_LIB is None:
        load_library()
        p = batch_lib_path()
        if not os.path.exists(p):
            raise CvbError(CVB_ENODEV, f"{p} not built: run `make -C cv_b200/csrc`")
        L = C.CDLL(p)
        vp, u32, i32 = C.c_void_p, C.c_uint32, C.c_int32
        L.cvb_arrsac_batch_dev.argtypes = [vp, vp, i32, i32, vp, vp, vp, u32, u32, vp, vp, vp, u32, vp, vp]
        L.cvb_arrsac_batch.argtypes = [vp, vp, i32, i32, vp, vp, vp, u32, vp, vp, vp, vp, vp]
        L.cvb_arrsac_commit_rng_batch.argtypes = [vp, vp, u32, vp]
        L.cvb_two_view_options_dev.argtypes = [vp, vp, vp, vp, u32, u32, u32, vp, u32, u32, vp, vp, vp, vp, vp, vp, vp, vp]
        _BATCH_LIB = L
    return _BATCH_LIB


_INIT_LIB = None


def init_lib_path():
    return os.path.join(_HERE, "libcvb200_init.so")


def load_init_library():
    """Loads libcvb200_init.so, the module of include/cvb200_init.h over libcvb200.so (same contexts). Fails loudly when missing."""
    global _INIT_LIB
    if _INIT_LIB is None:
        load_library()
        p = init_lib_path()
        if not os.path.exists(p):
            raise CvbError(CVB_ENODEV, f"{p} not built: run `make -C cv_b200/csrc`")
        L = C.CDLL(p)
        vp, u32 = C.c_void_p, C.c_uint32
        L.cvb_init_cfg_default.argtypes = [vp]
        L.cvb_init_cfg_default.restype = None
        L.cvb_init_reconstruction_dev.argtypes = [vp, vp, vp, vp, u32, u32, u32, vp, u32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
        _INIT_LIB = L
    return _INIT_LIB


_CONSTRAINTS_LIB = None


def constraints_lib_path():
    return os.path.join(_HERE, "libcvb200_constraints.so")


def load_constraints_library():
    """Loads libcvb200_constraints.so, the module of include/cvb200_constraints.h over libcvb200.so (same contexts). Fails loudly when
    missing."""
    global _CONSTRAINTS_LIB
    if _CONSTRAINTS_LIB is None:
        load_library()
        p = constraints_lib_path()
        if not os.path.exists(p):
            raise CvbError(CVB_ENODEV, f"{p} not built: run `make -C cv_b200/csrc`")
        L = C.CDLL(p)
        vp, u32 = C.c_void_p, C.c_uint32
        L.cvb_constraints_cfg_default.argtypes = [vp]
        L.cvb_constraints_cfg_default.restype = None
        L.cvb_view_constraints_check.argtypes = [u32, vp, vp, u32, vp, vp, vp, u32]
        L.cvb_view_constraints_dev.argtypes = [vp, vp, vp, u32, vp, vp, vp, vp, u32, u32, vp, vp, u32, vp, u32, vp, vp, vp]
        L.cvb_view_constraints.argtypes = [vp, vp, vp, u32, vp, vp, vp, vp, u32, vp, vp, vp, u32, vp, vp, vp]
        L.cvb_three_view_adaptive_optimize_l2_dev.argtypes = [vp, vp, u32, vp, vp, u32, vp, vp]
        _CONSTRAINTS_LIB = L
    return _CONSTRAINTS_LIB


_RECONSTRUCTION_LIB = None


def reconstruction_lib_path():
    return os.path.join(_HERE, "libcvb200_reconstruction.so")


def load_reconstruction_library():
    """Loads libcvb200_reconstruction.so, the module of include/cvb200_reconstruction.h over libcvb200.so (same contexts). Fails loudly
    when missing."""
    global _RECONSTRUCTION_LIB
    if _RECONSTRUCTION_LIB is None:
        load_library()
        p = reconstruction_lib_path()
        if not os.path.exists(p):
            raise CvbError(CVB_ENODEV, f"{p} not built: run `make -C cv_b200/csrc`")
        L = C.CDLL(p)
        vp, u32 = C.c_void_p, C.c_uint32
        L.cvb_recon_cfg_default.argtypes = [vp]
        L.cvb_recon_cfg_default.restype = None
        L.cvb_optimize_reconstruction_check.argtypes = [u32, vp, vp, u32, vp, vp, vp, u32]
        L.cvb_optimize_reconstruction_dev.argtypes = [vp, vp, vp, u32, vp, vp, vp, vp, u32, u32, vp, vp, u32, vp, u32, vp, vp, vp, vp]
        L.cvb_optimize_reconstruction.argtypes = [vp, vp, vp, u32, vp, vp, vp, vp, u32, vp, vp, vp, u32, vp, vp, vp, vp]
        _RECONSTRUCTION_LIB = L
    return _RECONSTRUCTION_LIB


_EXPORT_LIB = None


def export_lib_path():
    return os.path.join(_HERE, "libcvb200_export.so")


def load_export_library():
    """Loads libcvb200_export.so, the module of include/cvb200_export.h over libcvb200.so (same contexts). Fails loudly when missing."""
    global _EXPORT_LIB
    if _EXPORT_LIB is None:
        load_library()
        p = export_lib_path()
        if not os.path.exists(p):
            raise CvbError(CVB_ENODEV, f"{p} not built: run `make -C cv_b200/csrc`")
        L = C.CDLL(p)
        vp, u32 = C.c_void_p, C.c_uint32
        L.cvb_export_cfg_default.argtypes = [vp]
        L.cvb_export_cfg_default.restype = None
        L.cvb_export_check.argtypes = [u32, vp, vp, u32, vp, vp, vp, u32, u32]
        L.cvb_robust_landmarks_dev.argtypes = [vp, vp, vp, u32, vp, vp, vp, vp, u32, u32, vp, vp, u32, vp, vp]
        L.cvb_robust_landmarks.argtypes = [vp, vp, vp, u32, vp, vp, vp, vp, u32, vp, vp, vp, vp]
        L.cvb_export_reconstruction_dev.argtypes = [vp, vp, vp, u32, vp, vp, vp, vp, vp, u32, u32, vp, vp, u32, vp, vp, vp, vp, vp]
        L.cvb_export_reconstruction.argtypes = [vp, vp, vp, u32, vp, vp, vp, vp, vp, u32, vp, vp, vp, vp, vp, vp, vp]
        L.cvb_normalize_reconstruction_dev.argtypes = [vp, vp, vp, u32, vp, vp, vp, vp, u32, u32, vp, vp, u32, vp, u32, u32, vp, vp, vp]
        L.cvb_normalize_reconstruction.argtypes = [vp, vp, vp, u32, vp, vp, vp, vp, u32, vp, vp, vp, u32, u32, vp, vp, vp]
        _EXPORT_LIB = L
    return _EXPORT_LIB


_REGISTER_LIB = None


def register_lib_path():
    return os.path.join(_HERE, "libcvb200_register.so")


def load_register_library():
    """Loads libcvb200_register.so, the module of include/cvb200_register.h over libcvb200.so (same contexts). Fails loudly when missing."""
    global _REGISTER_LIB
    if _REGISTER_LIB is None:
        load_library()
        p = register_lib_path()
        if not os.path.exists(p):
            raise CvbError(CVB_ENODEV, f"{p} not built: run `make -C cv_b200/csrc`")
        L = C.CDLL(p)
        vp, u32 = C.c_void_p, C.c_uint32
        L.cvb_register_cfg_default.argtypes = [vp]
        L.cvb_register_cfg_default.restype = None
        L.cvb_register_check.argtypes = [u32, vp, vp, u32, vp, vp, vp, u32]
        L.cvb_register_frame_dev.argtypes = [vp, vp, vp, vp, vp, u32, vp, vp, vp, vp, vp, u32, u32, vp, vp, u32, vp, vp, u32, vp, u32, vp, vp,
                                             vp, vp]
        L.cvb_register_frame.argtypes = [vp, vp, vp, vp, vp, u32, vp, vp, vp, vp, vp, u32, vp, vp, vp, vp, u32, vp, u32, vp, vp, vp, vp]
        _REGISTER_LIB = L
    return _REGISTER_LIB


_INCORPORATE_LIB = None


def incorporate_lib_path():
    return os.path.join(_HERE, "libcvb200_incorporate.so")


def load_incorporate_library():
    """Loads libcvb200_incorporate.so, the module of include/cvb200_incorporate.h over libcvb200.so (same contexts). Fails loudly when
    missing."""
    global _INCORPORATE_LIB
    if _INCORPORATE_LIB is None:
        load_library()
        p = incorporate_lib_path()
        if not os.path.exists(p):
            raise CvbError(CVB_ENODEV, f"{p} not built: run `make -C cv_b200/csrc`")
        L = C.CDLL(p)
        vp, u32 = C.c_void_p, C.c_uint32
        L.cvb_incorporate_check.argtypes = [u32, vp, vp, u32, vp, vp, vp, u32, u32, vp, u32, vp, u32, vp, u32]
        L.cvb_add_view_dev.argtypes = [vp, u32] + [vp] * 6 + [u32, u32, vp, vp, u32] + [vp] * 4 + [u32, vp, u32] + [vp] * 10
        L.cvb_add_view.argtypes = [vp, u32] + [vp] * 6 + [u32, vp, vp] + [vp] * 4 + [u32, vp, u32] + [vp] * 10
        L.cvb_apply_optimization_dev.argtypes = [vp, u32] + [vp] * 6 + [u32, u32, vp, vp, u32, vp, u32] + [vp] * 14
        L.cvb_apply_optimization.argtypes = [vp, u32] + [vp] * 6 + [u32, vp, vp, vp, u32] + [vp] * 14
        L.cvb_incorporate_frame_dev.argtypes = ([vp] * 7 + [u32] + [vp] * 6 + [u32, u32, vp, vp, u32, vp, u32, vp, vp, vp, u32, vp, u32] +
                                                [vp] * 13)
        L.cvb_incorporate_frame.argtypes = [vp] * 7 + [u32] + [vp] * 6 + [u32, vp, vp, vp, u32, vp, vp, vp, u32, vp, u32] + [vp] * 13
        _INCORPORATE_LIB = L
    return _INCORPORATE_LIB


_MERGE_LIB = None


def merge_lib_path():
    return os.path.join(_HERE, "libcvb200_merge.so")


def load_merge_library():
    """Loads libcvb200_merge.so, the module of include/cvb200_merge.h over libcvb200.so (same contexts). Fails loudly when missing."""
    global _MERGE_LIB
    if _MERGE_LIB is None:
        load_library()
        p = merge_lib_path()
        if not os.path.exists(p):
            raise CvbError(CVB_ENODEV, f"{p} not built: run `make -C cv_b200/csrc`")
        L = C.CDLL(p)
        vp, u32, i32 = C.c_void_p, C.c_uint32, C.c_int
        L.cvb_merge_check.argtypes = [u32, vp, vp, u32, vp, vp, vp, u32, u32, vp, vp, u32, vp, vp, u32, vp, i32, i32]
        L.cvb_incorporate_reconstruction_dev.argtypes = ([vp] * 3 + [u32] + [vp] * 6 + [u32, u32, vp, vp, u32, vp, u32, u32] + [vp] * 6 +
                                                         [u32, u32, vp, vp, u32, u32, vp, vp] + [vp] * 13)
        L.cvb_incorporate_reconstruction.argtypes = ([vp] * 3 + [u32] + [vp] * 6 + [u32, vp, vp, vp, u32, u32] + [vp] * 6 +
                                                     [u32, vp, vp, u32, vp, vp] + [vp] * 13)
        L.cvb_merge_reconstructions_dev.argtypes = ([vp] * 7 + [u32] + [vp] * 6 + [u32, u32, vp, vp, u32, vp, u32, u32] + [vp] * 6 +
                                                    [u32, u32, vp, vp, u32, u32, vp, u32] + [vp] * 15)
        L.cvb_merge_reconstructions.argtypes = ([vp] * 7 + [u32] + [vp] * 6 + [u32, vp, vp, vp, u32, u32] + [vp] * 6 +
                                                [u32, vp, vp, u32, vp, u32] + [vp] * 15)
        _MERGE_LIB = L
    return _MERGE_LIB


_TRY_INIT_LIB = None


def try_init_lib_path():
    return os.path.join(_HERE, "libcvb200_try_init.so")


def load_try_init_library():
    """Loads libcvb200_try_init.so, the module of include/cvb200_try_init.h over libcvb200.so (same contexts). Fails loudly when missing."""
    global _TRY_INIT_LIB
    if _TRY_INIT_LIB is None:
        load_library()
        p = try_init_lib_path()
        if not os.path.exists(p):
            raise CvbError(CVB_ENODEV, f"{p} not built: run `make -C cv_b200/csrc`")
        L = C.CDLL(p)
        vp, u32 = C.c_void_p, C.c_uint32
        L.cvb_try_init_check.argtypes = [u32] * 6 + [vp, u32, vp, u32, vp, u32]
        L.cvb_add_reconstruction_dev.argtypes = [vp] * 5 + [u32] * 5 + [vp] * 14
        L.cvb_add_reconstruction.argtypes = [vp] * 5 + [u32] * 5 + [vp] * 14
        L.cvb_try_init_dev.argtypes = [vp] * 5 + [u32] + [vp] * 4 + [u32] * 3 + [vp, u32] + [vp] * 10
        L.cvb_try_init.argtypes = [vp] * 5 + [u32] + [vp] * 4 + [u32] * 3 + [vp, u32] + [vp] * 10
        _TRY_INIT_LIB = L
    return _TRY_INIT_LIB


class Context:
    """A cvb_ctx: one CUDA stream + workspaces on one device. Not thread-safe; use one per thread."""

    def __init__(self, device=0, stream=None):
        self.lib = load_library()
        h = C.c_void_p()
        rc = self.lib.cvb_ctx_create_on_stream(int(device), C.c_void_p(stream) if stream else None, C.byref(h))
        if rc != 0:
            raise CvbError(rc, "cvb_ctx_create failed (a Hopper (sm_90) CUDA device is required; there is no CPU fallback)")
        self.handle = h
        self.device = device

    def close(self):
        if getattr(self, "handle", None):
            self.lib.cvb_ctx_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def check(self, rc):
        if rc != 0:
            raise CvbError(rc, self.lib.cvb_last_error(self.handle).decode())

    def sync(self):
        self.check(self.lib.cvb_ctx_sync(self.handle))

    def launch_count(self):
        return int(self.lib.cvb_ctx_launch_count(self.handle))

    def profile(self, enable=True):
        self.check(self.lib.cvb_ctx_profile(self.handle, 1 if enable else 0))

    def profile_report(self):
        """{kernel: dict(launches, ms, bytes)} accumulated since profile(True)."""
        buf = C.create_string_buffer(1 << 16)
        self.check(self.lib.cvb_ctx_profile_report(self.handle, buf, len(buf)))
        out = {}
        for line in buf.value.decode().splitlines():
            name, n, ms, by = line.split()
            out[name] = dict(launches=int(n), ms=float(ms), bytes=float(by))
        return out

    def timer_begin(self):
        self.check(self.lib.cvb_ctx_timer_begin(self.handle))

    def timer_end(self):
        ms = C.c_float()
        self.check(self.lib.cvb_ctx_timer_end(self.handle, C.byref(ms)))
        return ms.value


_default_ctx = {}


def default_context(device=0):
    if device not in _default_ctx:
        _default_ctx[device] = Context(device)
    return _default_ctx[device]
