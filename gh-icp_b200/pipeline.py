"""Raw clouds -> transform: the steps of the reference's driver (test/ghicp_main.cpp:86-155) over the C ABI, in Python.

    Rt, info = register_clouds(target_xyz, source_xyz, resolution=0.1, neighborhood_radius=0.5,
                               curvature_non_max_radius=1.0)

Voxel down-sampling of both clouds (CFilter::voxelfilter), curvature keypoints (0.65 / 20 neighbours, :96-97), the
bounding-box magnitude of the down-sampled source (:91-93), GHRegistration on the keypoints.  Without a `features` callback
every stage runs on the GPU and the descriptors are computed there too:
  * feature_type = FT_BSC: the BSC encoder like :113-116 (capi.bsc_extract: radius = curvature_non_max_radius, 7 x 7 grids,
    dof_type 0 for the target, `dof_type` for the source; `bsc_pattern` = the sampling pairs, default = the pattern the
    reference's constructor generates);
  * feature_type = FT_FPFH: FPFHfeature::compute_fpfh_feature + keyfpfh like :120-127 (capi.Prep.fpfh: k-NN normals and
    histograms with k = `fpfh_k`, 20 in the reference, on the down-sampled cloud, gathered at the keypoints);
  * FT_NONE: coordinates only, which GHRegistration supports (src/ghicp_reg.cpp:66-68) although the reference's own main()
    rejects it.
`features(target_down, target_kp_idx, source_down, source_kp_idx) -> Keypoints` attaches descriptors computed elsewhere
instead.

GH-ICP is a local method.  initial_alignment = "fpfh_sac" first runs SAC-IA (FPFHfeature::fpfhalign, include/fpfh.hpp:117-133;
DESIGN.md §3.11) on the keypoints and their FPFH histograms — computed for this stage alone when the loop uses BSC or no
feature — and starts the loop from its transform; the returned transform is the whole one and info["sac"] describes the
coarse stage.  `sac` overrides the capi.sac_ia arguments (iterations, samples, k, min_sample_distance, threshold, seed); the
default threshold is the keypoint NMS radius squared: keypoints are at least one NMS radius apart, so within that distance the
nearest target keypoint of a moved source keypoint can only be its counterpart, and the error counts the keypoints that land
on their counterparts.  On small keypoint sets of repetitive scenes 1000 hypotheses may not be enough (DESIGN.md §3.11).

fpfh_radius = (normal_radius, feature_radius) computes the loop's and SAC-IA's histograms with the radius estimator
(capi.Prep.fpfh_radius, DESIGN.md §3.10) instead of k-NN with k = fpfh_k: a support of several voxels, as PCL users and the
reference's own coarse registration compute FPFH.  The default None keeps the k-NN estimator.

evaluate = {"thre_dis": r, "max_range": m} scores the result on the down-sampled clouds (capi.Prep.overlap on the device
pipeline, capi.cloud_overlap with `features`; DESIGN.md §3.12): info["evaluation"] for the final transform and, with
initial_alignment="fpfh_sac", info["sac"]["evaluation"] for the coarse one.  The default None leaves info as it was.
cal_overlap and evaluate_registration score any pair of clouds.

refine = {"max_iter": m, "reciprocal": b, "trimmed_thre_dis": r (optional)} refines the GH-ICP transform on the down-sampled
clouds with point-to-point ICP (capi.Prep.icp / capi.cloud_icp with `features`; DESIGN.md §3.13), started from that
transform, and returns the refined one; info["icp"] describes the refinement and keeps the GH-ICP transform as "Rt_before".
With "trimmed_thre_dis" the trimmed rejector's ratio is calOverlap at that start pose, where the reference's icp_reg measures
it on the unmoved source (it starts from the identity); with `evaluate`, info["evaluation"] scores the refined transform.
The default None leaves the result and info as they were.  icp_reg(source, target, ...) is CRegistration::icp_reg itself.
refine may also carry "metric": "plane" (default "point") and "covariance_k" (default 20): point-to-plane ICP against the
target's k-NN normals (DESIGN.md §3.14); ptplicp_reg(source, target, ...) is CRegistration::ptplicp_reg itself.
"metric": "gicp" refines with Generalized ICP over both clouds' k-NN normals (DESIGN.md §3.15), honouring "reciprocal" and
"trimmed_thre_dis" as the other metrics do: the library's own extension, the "G-ICP with trimmed property" the reference's
author was working on (PCL's GICP ignores both, src/common_reg.cpp:213-215); gicp_reg(source, target, ...) is
CRegistration::gicp_reg itself, with both options off in the loop as PCL has them.

sor = (mean_k, std_mul) removes statistical outliers (CFilter::SORFilter, capi.sor_filter, DESIGN.md §3.16) from each
down-sampled cloud between the voxel filter and the keypoints, on the device pipeline (capi.Prep(sor=...)) and with
`features` alike: isolated returns would otherwise stretch the bounding box that scales the loop's energy, and reach every
later stage.  info["sor"] = {"target": ..., "source": ...} then holds each cloud's filter result (the keys of capi.Prep.sor_info
on both branches).  The default None leaves
the result and info as they were.

coarsereg_fpfh_sac(source_xyz, target_xyz, search_radius) is CRegistration::Coarsereg_FPFHSAC (src/common_reg.cpp:393-423):
radius FPFH on every point of both clouds, then SAC-IA with correspondence randomness 15.
"""
import numpy as np

from . import capi
from .registration import Energyfunction, GHRegistration, Keypoints


def register_clouds(target_xyz, source_xyz, resolution, neighborhood_radius, curvature_non_max_radius, corr_type=capi.CT_NN,
                    feature_type=capi.FT_NONE, features=None, weight_adjustment_ratio=1.1, weight_adjustment_step=0.1,
                    dof_type=6, estimated_IoU=0.5, max_iter=0, device=0, bsc_pattern=None, fpfh_k=20, initial_alignment=None,
                    sac=None, fpfh_radius=None, evaluate=None, refine=None, sor=None, **reg_kw):
    ev_kw = _evaluate_kw(evaluate)
    if sor is not None:
        if len(sor) != 2:
            raise capi.GhicpError(-1, "sor must be a (mean_k, std_mul) pair")
        sor = capi._sor_args(sor)
    icp_kw = _refine_kw(refine)
    if initial_alignment not in (None, "fpfh_sac"):
        raise capi.GhicpError(-1, f"initial_alignment must be None or 'fpfh_sac', not {initial_alignment!r}")
    if fpfh_radius is not None:
        fpfh_radius = tuple(float(r) for r in fpfh_radius)
        if len(fpfh_radius) != 2:
            raise capi.GhicpError(-1, "fpfh_radius must be a (normal_radius, feature_radius) pair")
    sac_kw = dict(threshold=float(curvature_non_max_radius) ** 2)
    sac_kw.update(sac or {})
    T = np.ascontiguousarray(target_xyz, dtype=np.float32)
    S = np.ascontiguousarray(source_xyz, dtype=np.float32)
    if features is None:
        # device-resident pipeline: each raw cloud is uploaded once, the stages chain on the GPU, the keypoint coordinates and
        # descriptors go device-to-device into the registration context (ghicp_prep_run + ghicp_set_from_prep)
        want_bsc = feature_type == capi.FT_BSC
        radius = curvature_non_max_radius if want_bsc else 0.0
        pt = capi.Prep(T, resolution, neighborhood_radius, curvature_non_max_radius, radius, 0, pairs=bsc_pattern, device=device,
                       sor=sor)                                                                                                    # :89-115
        ps = capi.Prep(S, resolution, neighborhood_radius, curvature_non_max_radius, radius, dof_type, pairs=bsc_pattern, device=device,
                       sor=sor)                                                                                                    # :116
        try:
            for name, pr in (("target", pt), ("source", ps)):
                if pr.n_kp == 0:
                    raise capi.GhicpError(-1, f"no keypoints in the {name} cloud: check the radii")
            if feature_type == capi.FT_FPFH or initial_alignment == "fpfh_sac":          # :120-127
                for pr in (pt, ps):
                    if fpfh_radius is None:
                        pr.fpfh(fpfh_k)
                    else:
                        pr.fpfh_radius(*fpfh_radius)
            Rt0, sac_info = None, None
            if initial_alignment == "fpfh_sac":
                Rt0, sac_info = ps.sac_ia(pt, **sac_kw)
            bbx = ps.bbx_magnitude                                                       # getCloudBound, :91-93
            Ef = Energyfunction().init(ps.n_kp, pt.n_kp, bbx)
            reg = GHRegistration((ps, pt), Ef, feature_type, corr_type, curvature_non_max_radius, weight_adjustment_ratio,
                                 weight_adjustment_step, dof_type, estimated_IoU, max_iter=max_iter, device=device, **reg_kw)
            if Rt0 is not None:
                reg.set_initial_transform(Rt0)
            Rt, iterations = reg.ghicp_reg()
            info = dict(iterations=iterations, n_target_down=pt.n_down, n_source_down=ps.n_down, n_target_kp=pt.n_kp,
                        n_source_kp=ps.n_kp, bbx_magnitude=bbx, cor=len(reg.pairs()[0]),
                        stage_ms=dict(target=pt.stage_ms, source=ps.stage_ms))
            if feature_type == capi.FT_FPFH:
                info["fpfh_ms"] = dict(target=pt.fpfh_ms, source=ps.fpfh_ms)
            if sor is not None:
                info["sor"] = dict(target=pt.sor_info, source=ps.sor_info)
            if sac_info is not None:
                info["sac"] = dict(sac_info, Rt=Rt0)
            if icp_kw is not None:
                Rt = _refine(Rt, icp_kw, info, lambda G, thr: ps.overlap(pt, G, thre_dis=thr, fitness=False)["ratio"],
                             lambda G, **kw: ps.icp(pt, G, **kw))
            if ev_kw is not None:
                info["evaluation"] = ps.overlap(pt, Rt, **ev_kw)
                if sac_info is not None:
                    info["sac"]["evaluation"] = ps.overlap(pt, Rt0, **ev_kw)
            reg.close()
        finally:
            pt.close(); ps.close()
        return Rt, info
    down, kp_idx, sor_info = {}, {}, {}
    for name, P in (("T", T), ("S", S)):
        keep = capi.voxel_downsample(P, resolution, device=device)                       # :89-90
        D = np.ascontiguousarray(P[keep])
        if sor is not None:
            kept, sor_info[name] = capi.sor_filter(D, *sor, device=device)
            sor_info[name].update(n_voxel=len(D), ms=sor_info[name]["stage_ms"]["total"])   # the keys of Prep.sor_info
            D = np.ascontiguousarray(D[kept])
        kp, _, _, _ = capi.detect_keypoints(D, neighborhood_radius, 0.65, 20, curvature_non_max_radius, device=device)   # :96-100
        if len(kp) == 0:
            raise capi.GhicpError(-1, f"no keypoints in the {'target' if name == 'T' else 'source'} cloud: check the radii")
        down[name], kp_idx[name] = D, kp
    ext = down["S"].max(axis=0) - down["S"].min(axis=0)                                   # getCloudBound, :91-93
    bbx = float(np.float32(ext[0] + ext[1] + ext[2]))
    Kp = features(down["T"], kp_idx["T"], down["S"], kp_idx["S"])
    Ef = Energyfunction().init(Kp.kps_num, Kp.kpt_num, bbx)
    reg = GHRegistration(Kp, Ef, feature_type, corr_type, curvature_non_max_radius, weight_adjustment_ratio,
                         weight_adjustment_step, dof_type, estimated_IoU, max_iter=max_iter, device=device, **reg_kw)
    sac_info = None
    if initial_alignment == "fpfh_sac":
        if fpfh_radius is None:
            fs, _, _ = capi.fpfh_extract(down["S"], kp_idx["S"], fpfh_k, device=device)
            ft, _, _ = capi.fpfh_extract(down["T"], kp_idx["T"], fpfh_k, device=device)
        else:
            fs, _, _ = capi.fpfh_extract_radius(down["S"], kp_idx["S"], *fpfh_radius, device=device)
            ft, _, _ = capi.fpfh_extract_radius(down["T"], kp_idx["T"], *fpfh_radius, device=device)
        Rt0, sac_info = capi.sac_ia(down["S"][kp_idx["S"]], fs, down["T"][kp_idx["T"]], ft, device=device, **sac_kw)
        reg.set_initial_transform(Rt0)
        sac_info = dict(sac_info, Rt=Rt0)
    Rt, iterations = reg.ghicp_reg()
    info = dict(iterations=iterations, n_target_down=len(down["T"]), n_source_down=len(down["S"]), n_target_kp=len(kp_idx["T"]),
                n_source_kp=len(kp_idx["S"]), bbx_magnitude=bbx, cor=len(reg.pairs()[0]))
    if sor is not None:
        info["sor"] = dict(target=sor_info["T"], source=sor_info["S"])
    if sac_info is not None:
        info["sac"] = sac_info
    if icp_kw is not None:
        Rt = _refine(Rt, icp_kw, info,
                     lambda G, thr: capi.cloud_overlap(down["S"], down["T"], G, thre_dis=thr, fitness=False, device=device)["ratio"],
                     lambda G, **kw: capi.cloud_icp(down["S"], down["T"], G, device=device, **kw))
    if ev_kw is not None:
        info["evaluation"] = capi.cloud_overlap(down["S"], down["T"], Rt, device=device, **ev_kw)
        if sac_info is not None:
            info["sac"]["evaluation"] = capi.cloud_overlap(down["S"], down["T"], sac_info["Rt"], device=device, **ev_kw)
    reg.close()
    return Rt, info


def _evaluate_kw(evaluate):
    if evaluate is None:
        return None
    if not isinstance(evaluate, dict) or "thre_dis" not in evaluate or set(evaluate) - {"thre_dis", "max_range"}:
        raise capi.GhicpError(-1, "evaluate must be a dict {thre_dis, max_range (optional)}")
    return dict(thre_dis=float(evaluate["thre_dis"]), max_range=float(evaluate.get("max_range", float("inf"))))


def _refine_kw(refine):
    if refine is None:
        return None
    keys = {"max_iter", "reciprocal", "trimmed_thre_dis", "metric", "covariance_k"}
    if not isinstance(refine, dict) or "max_iter" not in refine or set(refine) - keys:
        raise capi.GhicpError(-1, "refine must be a dict {max_iter, reciprocal (optional), trimmed_thre_dis (optional), "
                                  "metric ('point', 'plane' or 'gicp', optional), covariance_k (optional)}")
    metric = refine.get("metric", "point")
    if metric not in capi.ICP_METRICS:
        raise capi.GhicpError(-1, f"refine: metric must be 'point', 'plane' or 'gicp', not {metric!r}")
    return dict(max_iter=int(refine["max_iter"]), reciprocal=bool(refine.get("reciprocal", False)),
                thre_dis=refine.get("trimmed_thre_dis"), metric=metric, normal_k=int(refine.get("covariance_k", 20)))


def _refine(Rt, kw, info, ratio_at, icp_from):
    """ICP from Rt (icp_from(guess, **cloud_icp options)); the trimmed ratio is calOverlap at Rt (ratio_at(Rt, thre_dis))."""
    rho = 0.0 if kw["thre_dis"] is None else float(ratio_at(Rt, float(kw["thre_dis"])))
    Rt_icp, icp_info = icp_from(Rt, max_iterations=kw["max_iter"], reciprocal=kw["reciprocal"], trim_ratio=min(rho, 1.0),
                                metric=kw["metric"], normal_k=kw["normal_k"])
    info["icp"] = dict(icp_info, Rt_before=Rt, trim_ratio=rho)
    return Rt_icp


def icp_reg(source_xyz, target_xyz, max_iter, use_reciprocal_correspondence, use_trimmed_rejector, thre_dis,
            min_overlap_for_reg=0.0, device=0):
    """CRegistration::icp_reg (src/common_reg.cpp:44-107) on the GPU: point-to-point ICP of the source onto the target from
    the identity, transformation epsilon 1e-8 and fitness epsilon 1e-5 as :86-88 set them (capi.cloud_icp, DESIGN.md §3.13).
    With use_trimmed_rejector the trimmed rejector's ratio is calOverlap(source, target, thre_dis) of the unmoved source, and
    the call returns None when that ratio is below min_overlap_for_reg (the reference returns false).  Returns (Rt 4x4, info
    with the transformed source under "moved"; info["overlap_ratio"] when trimmed)."""
    S = np.ascontiguousarray(source_xyz, dtype=np.float32).reshape(-1, 3)
    T = np.ascontiguousarray(target_xyz, dtype=np.float32).reshape(-1, 3)
    rho = 0.0
    if use_trimmed_rejector:
        rho = cal_overlap(S, T, thre_dis, device=device)
        if rho < min_overlap_for_reg:
            return None
    Rt, info = capi.cloud_icp(S, T, None, max_iterations=max_iter, reciprocal=use_reciprocal_correspondence,
                              trim_ratio=min(rho, 1.0), transformation_epsilon=1e-8, fitness_epsilon=1e-5, return_moved=True,
                              device=device)
    if use_trimmed_rejector:
        info["overlap_ratio"] = rho
    return Rt, info


def ptplicp_reg(source_xyz, target_xyz, max_iter, use_reciprocal_correspondence, use_trimmed_rejector, thre_dis, covariance_K,
                min_overlap_for_reg=0.0, device=0):
    """CRegistration::ptplicp_reg (src/common_reg.cpp:123-199) on the GPU: point-to-plane ICP of the source onto the target
    from the identity against the target's k-NN normals (k = covariance_K, 3..32), transformation epsilon 1e-8 and fitness
    epsilon 1e-5 (capi.cloud_icp with metric="plane", DESIGN.md §3.14).  The source's normals, which the reference also
    computes, take no part in PCL's estimate and are not computed.  With use_trimmed_rejector the ratio is
    calOverlap(source, target, thre_dis) of the unmoved source, and the call returns None below min_overlap_for_reg.  Returns
    (Rt 4x4, info with the transformed source under "moved"; info["overlap_ratio"] when trimmed), as icp_reg."""
    S = np.ascontiguousarray(source_xyz, dtype=np.float32).reshape(-1, 3)
    T = np.ascontiguousarray(target_xyz, dtype=np.float32).reshape(-1, 3)
    rho = 0.0
    if use_trimmed_rejector:
        rho = cal_overlap(S, T, thre_dis, device=device)
        if rho < min_overlap_for_reg:
            return None
    Rt, info = capi.cloud_icp(S, T, None, max_iterations=max_iter, reciprocal=use_reciprocal_correspondence,
                              trim_ratio=min(rho, 1.0), transformation_epsilon=1e-8, fitness_epsilon=1e-5, return_moved=True,
                              device=device, metric="plane", normal_k=covariance_K)
    if use_trimmed_rejector:
        info["overlap_ratio"] = rho
    return Rt, info


def gicp_reg(source_xyz, target_xyz, max_iter, use_reciprocal_correspondence, use_trimmed_rejector, thre_dis, covariance_K,
             min_overlap_for_reg=0.0, device=0):
    """CRegistration::gicp_reg (src/common_reg.cpp:217-284) on the GPU: Generalized ICP of the source onto the target from the
    identity with both clouds' k-NN normals as covariances (k = covariance_K, 3..32), transformation epsilon 1e-8 and rotation
    epsilon 1e-6 (capi.cloud_icp with metric="gicp", DESIGN.md §3.15).  PCL's GICP ignores the reciprocal option and the
    correspondence rejectors, so the loop runs without them whatever use_reciprocal_correspondence says; use_trimmed_rejector
    only gates the call: the ratio calOverlap(source, target, thre_dis) of the unmoved source below min_overlap_for_reg returns
    None.  Returns (Rt 4x4, info with the transformed source under "moved"; info["overlap_ratio"] when trimmed), as icp_reg."""
    S = np.ascontiguousarray(source_xyz, dtype=np.float32).reshape(-1, 3)
    T = np.ascontiguousarray(target_xyz, dtype=np.float32).reshape(-1, 3)
    rho = None
    if use_trimmed_rejector:
        rho = cal_overlap(S, T, thre_dis, device=device)
        if rho < min_overlap_for_reg:
            return None
    Rt, info = capi.cloud_icp(S, T, None, max_iterations=max_iter, reciprocal=False, trim_ratio=0.0, transformation_epsilon=1e-8,
                              return_moved=True, device=device, metric="gicp", normal_k=covariance_K, rotation_epsilon=1e-6)
    if rho is not None:
        info["overlap_ratio"] = rho
    return Rt, info


def cal_overlap(cloud1, cloud2, thre_dis, device=0):
    """CRegistration::calOverlap (src/common_reg.cpp:294-317) on the GPU: the share of cloud1 with a cloud2 point within
    thre_dis (d2 < thre_dis^2 in float32), as the reference's float (0.01 + overlap) / n.  Overlap-only mode (DESIGN.md §3.12)."""
    return capi.cloud_overlap(cloud1, cloud2, None, thre_dis=thre_dis, fitness=False, device=device)["ratio"]


def evaluate_registration(source_xyz, target_xyz, Rt, thre_dis, max_range=float("inf"), device=0):
    """Scores Rt (4x4, the source onto the target) on the two clouds: capi.cloud_overlap's dict (overlap, ratio, overlap_rmse
    within thre_dis; fitness = PCL's getFitnessScore over d2 <= max_range, a bound on squared distances)."""
    return capi.cloud_overlap(source_xyz, target_xyz, Rt, thre_dis=thre_dis, max_range=max_range, device=device)


def coarsereg_fpfh_sac(source_xyz, target_xyz, search_radius, sac=None, device=0):
    """CRegistration::Coarsereg_FPFHSAC (src/common_reg.cpp:393-423) on the GPU: normals over `search_radius` and FPFH over
    2 * search_radius on every point of both clouds (compute_fpfh_feature, :373-389; capi.fpfh_extract_radius), then SAC-IA
    with correspondence randomness 15 and PCL's other defaults: 1000 hypotheses of 3 samples, threshold 100 on squared
    distances, no minimum sample distance, seed 0 (capi.sac_ia; `sac` overrides these).  Returns (Rt 4x4 mapping the source
    onto the target, info: the sac_ia result with its fitness, plus the histograms' stage times in ms)."""
    import time
    S = np.ascontiguousarray(source_xyz, dtype=np.float32).reshape(-1, 3)
    T = np.ascontiguousarray(target_xyz, dtype=np.float32).reshape(-1, 3)
    rn, rf = float(np.float32(search_radius)), float(np.float32(2.0 * np.float32(search_radius)))
    t0 = time.perf_counter()
    fs, _, _ = capi.fpfh_extract_radius(S, None, rn, rf, device=device)
    ft, _, _ = capi.fpfh_extract_radius(T, None, rn, rf, device=device)
    t1 = time.perf_counter()
    kw = dict(iterations=1000, samples=3, k=15, min_sample_distance=0.0, threshold=100.0, seed=0)
    kw.update(sac or {})
    Rt, info = capi.sac_ia(S, fs, T, ft, device=device, **kw)
    info = dict(info, fpfh_ms=1e3 * (t1 - t0), normal_radius=rn, feature_radius=rf)
    return Rt, info


def transform_cloud(xyz, Rt):
    """pcl::transformPointCloud with the float32 matrix (test/ghicp_main.cpp:153)."""
    P = np.ascontiguousarray(xyz, dtype=np.float32)
    R, t = Rt[:3, :3].astype(np.float32), Rt[:3, 3].astype(np.float32)
    return P @ R.T + t
