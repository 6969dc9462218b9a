"""rmcl_b200 -- H100-native (sm_90a) ray-casting correspondences for RMCL's MICP-L / particle-filter hot path.

The product is the C-ABI shared library rmcl_b200/lib/librmcl_b200.so (include/rmcl_b200.h); this package is the thin
host-side mirror of the reference's operator interface over it (rmcl::RCC..::find / computeCrossStatistics,
v1 correct(), ParticleUpdater::update).  There is no CPU fallback: importing works anywhere, but every compute call needs
the CUDA library and a GPU and raises otherwise.
"""
from .api import (B2Error, Map, RCCB200, RCCB200Spherical, RCCB200Pinhole, RCCB200O1Dn, RCCB200OnDn, CPCB200, SphereCorrectorB200, PinholeCorrectorB200, O1DnCloudFilter,
                  O1DnCorrectorB200, OnDnCorrectorB200, PCDSensorUpdaterB200, DistanceField, PFParams, GladiatorConfig, SurfaceConfig, KLDConfig, ClusterConfig, RecoveryConfig, SteinConfig, SearchConfig, umeyama_transform, micp_correct_once, micp_correct,
                  micp_pose_covariance, MICP_STEP_DTYPE, MICP_COVARIANCE_DTYPE, read_mesh_file, kernel_launch_count, lib_path, load_library)
from . import synth

__all__ = ["B2Error", "Map", "RCCB200", "RCCB200Spherical", "RCCB200Pinhole", "RCCB200O1Dn", "RCCB200OnDn", "CPCB200", "SphereCorrectorB200",
           "PinholeCorrectorB200", "O1DnCorrectorB200", "OnDnCorrectorB200", "PCDSensorUpdaterB200", "DistanceField", "PFParams", "GladiatorConfig", "SurfaceConfig", "KLDConfig", "ClusterConfig", "RecoveryConfig", "SteinConfig", "SearchConfig", "O1DnCloudFilter", "umeyama_transform", "micp_correct_once",
           "micp_correct", "micp_pose_covariance", "MICP_STEP_DTYPE", "MICP_COVARIANCE_DTYPE", "read_mesh_file", "kernel_launch_count", "lib_path", "load_library", "synth"]
