"""cv_b200 -- H100-native (sm_90a) drop-in for rust-cv's AKAZE -> Hamming match -> RANSAC hot path.

Host-side mirror of the reference's interfaces for this path, over the C ABI in include/cvb200.h:

  Akaze                 <- akaze::Akaze                       (akaze/src/lib.rs:109-185, 295-366)
  Akaze.create_scale_space / find_image_keypoints / extract_descriptors, ScaleSpace
                        <- akaze's staged surface: evolutions, Akaze::find_image_keypoints, Akaze::extract_descriptors
                                                              (akaze/src/lib.rs:268-276, descriptors.rs:16-45)
  DynamicImage          <- image::DynamicImage's integer variants, from_dynamic on the device (akaze/src/image.rs:45-109)
  horizontal_filter, vertical_filter, separable_filter, gaussian_kernel, gaussian_blur, half_size
                        <- akaze::image                        (akaze/src/image.rs:154-389)
  KeyPoint dtype        <- akaze::KeyPoint                    (akaze/src/lib.rs:71-93)
  LinearKnn / hamming_knn <- space::LinearKnn + bitarray::Hamming (call sites akaze/tests/estimate_pose.rs:78-97)
  hash_knn / FrameHashIndex <- cv-sfm's similar-frame search, lsh_to_frame.knn_values (cv-sfm/src/lib.rs:597-668), exact
  matching / symmetric_matching <- cv-sfm/src/lib.rs:3097-3133, tutorial-code chapter4 main.rs:91-137
  CameraIntrinsics(K1Distortion) <- cv-pinhole/src/lib.rs:32-240
  *pose_reprojection_error, EssentialMatrix <- cv-pinhole/src/lib.rs:314-372, essential.rs:56-275
  frame_features        <- cv-sfm VSlam::kps_descriptors        (cv-sfm/src/lib.rs:2195-2235)
  init_two_view_options <- cv-sfm init_two_view against every candidate frame (cv-sfm/src/lib.rs:966-985, 1365-1432), one batched
                           consensus run (Arrsac.model_inliers_batch: many independent model_inliers calls)
  init_reconstruction, InitSettings <- cv-sfm VSlam::init_reconstruction (cv-sfm/src/lib.rs:966-1303): the two-view options and the
                           three-view choice over every pair of them, chained on the device
  generate_view_constraints, ConstraintSettings <- cv-sfm VSlam::generate_view_constraints / record_view_constraints
                           (cv-sfm/src/lib.rs:2092-2109, 2438-2516) for many views of one reconstruction snapshot in one call
  optimize_reconstruction, regenerate_reconstruction, ReconstructionSettings <- cv-sfm VSlam::optimize_reconstruction /
                           regenerate_reconstruction (cv-sfm/src/lib.rs:2343-2435): the three-view pose graph and the observation
                           filter of one reconstruction snapshot in one call
  robust_landmarks, normalize_reconstruction, export_reconstruction, ExportSettings <- cv-sfm VSlam::triangulate_landmark_robust /
                           normalize_reconstruction / export_reconstruction (cv-sfm/src/lib.rs:2241-2340, 2907-3000) of one
                           reconstruction snapshot in one call each
  register_frame, RegisterSettings <- cv-sfm VSlam::register_frame (cv-sfm/src/lib.rs:1452-1812): one new frame against one
                           reconstruction snapshot, from its descriptors to the refined pose and its landmark matches, in one call
  add_view, apply_optimization, incorporate_frame <- cv-sfm VSlamData::add_view / merge_landmarks, the remove_view / split_observation
                           edits of optimize_reconstruction, and VSlam::incorporate_frame followed by optimize_reconstruction
                           (cv-sfm/src/lib.rs:432-588, 699-721, 2067-2087): one reconstruction snapshot to the next, on the device
  incorporate_reconstruction, merge_reconstructions <- cv-sfm VSlam::incorporate_reconstruction and try_merge_reconstructions followed
                           by optimize_reconstruction (cv-sfm/src/lib.rs:1817-1887, 2116-2193): two reconstruction snapshots to one
  add_reconstruction, try_init <- cv-sfm VSlamData::add_reconstruction and VSlam::try_init (cv-sfm/src/lib.rs:377-427, 814-839): a frame
                           and its free frames to the first snapshot of a new reconstruction
  *Triangulator         <- cv-geom's six triangulators          (cv-geom/src/triangulation.rs)
  *_optimize_l1/_l2     <- cv-optimize's five pose optimizers   (cv-optimize/src/{single,three}_view_optimizer.rs)

There is no CPU fallback: every call runs CUDA kernels from cv_b200/libcvb200.so and raises
CvbError when the library or a Hopper (sm_90) GPU is missing.
"""
from ._lib import CvbError, Context, KP_DTYPE, lib_path, load_library  # noqa: F401
from .akaze import Akaze, AkazeConfig, ScaleSpace  # noqa: F401
from .image import DynamicImage  # noqa: F401
from .filter import gaussian_blur, gaussian_kernel, half_size, horizontal_filter, separable_filter, vertical_filter  # noqa: F401
from .knn import (FrameHashIndex, HammingHasher, LinearKnn, hash_knn, hamming_knn, lowe_ratio_matches, matching,  # noqa: F401
                  symmetric_matching)
from .pinhole import (CameraIntrinsics, CameraIntrinsicsK1Distortion, EssentialMatrix, average_pose_reprojection_error,  # noqa: F401
                      average_pose_reprojection_error_batch, pose_reprojection_error, pose_reprojection_error_batch)
from .geom import (Arrsac, EightPoint, LambdaTwist, NisterStewenius, Pcg64, Xoshiro256PlusPlus,  # noqa: F401
                   residuals_camera_to_camera, residuals_world_to_camera)
from .triangulation import (AngularL1Triangulator, AngularLInfinityTriangulator, LinearEigenTriangulator,  # noqa: F401
                            MeanMeanTriangulator, RelativeDltTriangulator, SineL1Triangulator)
from .optimize import (observation_losses, single_view_simple_optimize_l1, single_view_simple_optimize_l1_batch,  # noqa: F401
                       single_view_simple_optimize_l2, single_view_simple_optimize_l2_batch, three_view_adaptive_optimize_l2,
                       three_view_optimize_l2_batch, three_view_simple_optimize_l1, three_view_simple_optimize_l1_batch,
                       three_view_simple_optimize_l2, tri_landmarks_robust)
from .sfm_match import landmark_matches  # noqa: F401
from . import checkpoint  # noqa: F401  (bincode record images of the VSlamData checkpoint)
from .pair import (InitSettings, Intrinsics, IntrinsicsK1, TwoViewBuffers, init_reconstruction, init_two_view_options,  # noqa: F401
                   two_view_frames)
from .features import frame_features  # noqa: F401
from .constraints import ConstraintSettings, generate_view_constraints  # noqa: F401
from .reconstruction import ReconstructionSettings, optimize_reconstruction, regenerate_reconstruction  # noqa: F401
from .export import ExportSettings, export_reconstruction, normalize_reconstruction, robust_landmarks  # noqa: F401
from .register import RegisterSettings, register_frame  # noqa: F401
from .incorporate import add_view, apply_optimization, incorporate_frame  # noqa: F401
from .merge import incorporate_reconstruction, incorporate_reconstruction_dev, merge_reconstructions, merge_reconstructions_dev  # noqa: F401
from .try_init import add_reconstruction, add_reconstruction_dev, try_init, try_init_dev  # noqa: F401

__version__ = "0.1.0"
