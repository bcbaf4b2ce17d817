"""pylidar_slam_b200 -- H100-native ICP-odometry hot path of pyLiDAR-SLAM.

Python host code mirroring the reference's plug-in interfaces (OdometryAlgorithm, LocalMap,
RigidAlignment, Filter) over hand-written sm_90a CUDA behind a C ABI (include/plslam_b200.h).
Importing the package does not need a GPU; creating a context does (no CPU fallback).
"""
from . import _lib  # noqa: F401
from .common import (Pose, SphericalProjector, compute_neighbors, compute_normal_map, distort_frame,  # noqa: F401
                     grid_sample, voxel_hashing, voxel_normal_distribution, voxel_statistics, voxelise,
                     weighted_procrustes)
from .odometry import (LOCAL_MAP, ODOMETRY, RIGID_ALIGNMENT, GaussNewtonPointToPlaneAlignment,  # noqa: F401
                       GaussNewtonPointToPlaneConfig, GaussNewtonPointToPointAlignment, GNPointToPointConfig, ICPFrameToModel, ICPFrameToModelBatch, ICPFrameToModelConfig, KdTreeLocalMap,
                       KdTreeLocalMapConfig, LocalMap, OdometryAlgorithm, ProjectiveLocalMap,
                       ProjectiveLocalMapConfig)
from .preprocessing import (FILTER, Distortion, DistortionConfig, GridSample, GridSampleConfig, Preprocessing,  # noqa: F401
                            PreprocessingConfig, ToTensor, ToTensorConfig, Voxelization, VoxelizationConfig)

from . import dataset, integration, io  # noqa: F401
from .dataset import correct_scan, kitti_frame, kitti_read_scan  # noqa: F401
from .io import (compute_absolute_poses, compute_relative_poses, read_poses_from_disk,  # noqa: F401
                 write_poses_to_disk)
from .training import LossConfig, PointToPlaneLossConfig, _PointToPlaneLossModule  # noqa: F401

__version__ = "0.1.0"
