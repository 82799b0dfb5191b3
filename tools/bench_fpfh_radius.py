"""Stage times of the FPFH estimator over radius neighbourhoods (ghicp_prep.cu: prep_fpfh_radius, DESIGN.md §3.10) next to
the k-NN estimator's, on synthetic scans voxel-filtered on the device-resident pipeline (ghicp_prep_run).

    python tools/bench_fpfh_radius.py [--points 1000000 5000000] [--voxel 0.05] [--radii 0.15,0.3 0.3,0.6] [--reps 3]

Per scan size and radius pair: the CUDA-event stage times of Prep.fpfh_radius at the keypoints (lists, normals, SPFH + FPFH;
best of `reps`), its work (list entries at both radii, SPFH points) and rates (list entries per second over the list stage,
SPFH pair features per second over the SPFH + FPFH stage: one pair per feature-list entry of an SPFH point, an upper bound);
the whole down-sampled cloud through fpfh_extract_radius (wall clock, host copies included); Prep.fpfh(20) (k-NN) on the same
scan.  Prints one JSON line with the card's name and power limit, read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    from bench_prep import gpu_info, scan_cloud
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, nargs="+", default=[1000000, 5000000])
    ap.add_argument("--voxel", type=float, default=0.05)
    ap.add_argument("--radii", nargs="+", default=["0.15,0.3", "0.3,0.6"])
    ap.add_argument("--nbr", type=float, default=0.5)
    ap.add_argument("--nms", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import ghicp_b200 as g
    if g.device_count() <= 0:
        raise SystemExit("bench_fpfh_radius.py: no CUDA device (the product has no CPU fallback)")
    radii = [tuple(float(x) for x in r.split(",")) for r in args.radii]
    out = {"tool": "bench_fpfh_radius", "voxel": args.voxel, "data": "synthetic scan_like_cloud", "runs": []}
    for n in args.points:
        side = (n / 1.0e6) ** 0.5 * 60.0
        P = scan_cloud(n, 1, (side, side, 6.0))
        pr = g.Prep(P, args.voxel, args.nbr, args.nms)
        try:
            D = pr.down()
            knn = min((pr.fpfh(20) for _ in range(args.reps)), key=lambda r: r["total"])
            run = dict(points=n, downsampled=pr.n_down, keypoints=pr.n_kp, knn_k20_keypoints_ms=knn, radius=[])
            for rn, rf in radii:
                best = min((pr.fpfh_radius(rn, rf) for _ in range(args.reps)), key=lambda r: r["total"])
                w = dict(pr.fpfh_work)
                t = time.perf_counter()
                g.fpfh_extract_radius(D, normal_radius=rn, feature_radius=rf)
                whole = (time.perf_counter() - t) * 1e3
                run["radius"].append(dict(normal_radius=rn, feature_radius=rf, keypoints_ms=best, work=w,
                                          list_entries_per_s=(w["normal_entries"] + w["feature_entries"]) / (best["lists"] * 1e-3),
                                          pair_features_per_s=w["feature_entries"] / (best["spfh_fpfh"] * 1e-3),
                                          whole_cloud_wall_ms=whole))
            out["runs"].append(run)
        finally:
            pr.close()
    out["gpu"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
