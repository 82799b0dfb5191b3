"""gh-icp_b200 — GH-ICP registration inner loop for the H100 (host-side Python face).

The product is `libghicp_b200.so` (hand-written sm_90a CUDA kernels behind the C ABI of
include/ghicp_b200.h).  This package is a thin ctypes binding plus a Python mirror of the reference's
`GHRegistration` interface (include/ghicp_reg.h:74-132) used by tests/ and bench.py.  It never imports
oracle/ and has no CPU fallback: without the compiled library or without a CUDA device it raises.

The directory name carries a hyphen, so import it through the repo-root shim:  `import ghicp_b200`.
"""
from .capi import (  # noqa: F401
    FT_BSC, FT_ROPS, FT_FPFH, FT_NONE, CT_NN, CT_NNR, CT_KM,
    GhicpError, IterStats, Config, lib, lib_path, build_library, device_count,
    km_solve, rigid_fit, rigid_fit_ex, comm_unique_id, voxel_downsample, detect_keypoints,
    bsc_extract, bsc_default_pattern, read_sample_pattern, Prep, PrepParams, fpfh_extract, fpfh_extract_radius, sac_ia,
    cloud_overlap, OverlapResult, cloud_icp, sor_filter, SorResult,
    SOLVER_SVD, SOLVER_WEIGHTED_SVD, SOLVER_POINT_TO_PLANE, SOLVER_YAW_4DOF,
)
from .registration import GHRegistration, Keypoints, Energyfunction  # noqa: F401
from . import synth  # noqa: F401
from . import capi  # noqa: F401
from . import pipeline  # noqa: F401
from .pipeline import (  # noqa: F401
    register_clouds, transform_cloud, coarsereg_fpfh_sac, cal_overlap, evaluate_registration, icp_reg, ptplicp_reg, gicp_reg,
)
