"""SAC-IA on the H100 (ghicp_sac.cu, DESIGN.md §3.11): stage times and hypothesis x point rate.

    python tools/bench_sac.py [--runs 3] [--iterations 1000] [--out result.json]

Workloads (synthetic scans of synth.scan_pair, voxel 0.05 m, keypoint radii 0.6 / NMS 1.2 m like tools/bench_prep.py):
  kp_1M      keypoints + FPFH of the 1 M point scan pair   (Prep.sac_ia, device to device)
  kp_5M      keypoints + FPFH of the 5 M point scan pair
  down_1M    every point of the down-sampled 1 M point scans with its FPFH (capi.sac_ia from host arrays)
The threshold is the NMS radius squared (register_clouds' default).  Times are CUDA events of the library (stage_ms) and a host
clock around the call; the median of --runs runs after one warm-up run.  Card name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ghicp_b200 as g  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"
    except Exception:
        return "unknown"


def measure(fn, runs):
    fn()   # warm-up: module load, pool growth
    rows = []
    for _ in range(runs):
        t0 = time.perf_counter()
        Rt, info = fn()
        info["wall_ms"] = (time.perf_counter() - t0) * 1e3
        rows.append((Rt, info))
    for Rt, info in rows[1:]:
        assert np.array_equal(Rt, rows[0][0]), "SAC-IA is deterministic: runs must agree"
    med = lambda key: float(np.median([r[1]["stage_ms"][key] for r in rows]))  # noqa: E731
    out = {k: med(k) for k in ("sample_knn", "estimate", "score", "pick", "total")}
    out["wall_ms"] = float(np.median([r[1]["wall_ms"] for r in rows]))
    info = rows[0][1]
    out.update(best_hypothesis=info["best_hypothesis"], inliers=info["inliers"], error=info["error"], fitness=info["fitness"])
    return out, rows[0][0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iterations", type=int, default=1000)
    ap.add_argument("--sizes", default="1000000,5000000")
    ap.add_argument("--skip-down", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if g.device_count() <= 0:
        raise SystemExit("bench_sac: no CUDA device")
    res, nbr, nms = 0.05, 0.6, 1.2
    thr = nms * nms
    result = dict(card=card(), iterations=a.iterations, threshold=thr, runs=a.runs, workloads={})
    for n in [int(v) for v in a.sizes.split(",")]:
        T, S, R_gt, _ = g.synth.scan_pair(n, seed=4)
        pt, ps = g.Prep(T, res, nbr, nms), g.Prep(S, res, nbr, nms)
        try:
            pt.fpfh(); ps.fpfh()
            name = "kp_%dM" % (n // 1000000)
            r, Rt = measure(lambda: ps.sac_ia(pt, iterations=a.iterations, threshold=thr), a.runs)
            r.update(n_source=ps.n_kp, n_target=pt.n_kp, rot_err_deg=float(np.degrees(g.synth.rot_angle(Rt[:3, :3], R_gt))))
            r["hyp_points_per_s"] = a.iterations * ps.n_kp / (r["score"] * 1e-3)
            result["workloads"][name] = r
            print(name, json.dumps(r), flush=True)
            if n == 1000000 and not a.skip_down:
                Ds, Dt = ps.down(), pt.down()
                fs, _, _ = g.fpfh_extract(Ds)
                ft, _, _ = g.fpfh_extract(Dt)
                r, Rt = measure(lambda: g.sac_ia(Ds, fs, Dt, ft, iterations=a.iterations, threshold=thr), a.runs)
                r.update(n_source=len(Ds), n_target=len(Dt), rot_err_deg=float(np.degrees(g.synth.rot_angle(Rt[:3, :3], R_gt))))
                r["hyp_points_per_s"] = a.iterations * len(Ds) / (r["score"] * 1e-3)
                result["workloads"]["down_1M"] = r
                print("down_1M", json.dumps(r), flush=True)
        finally:
            pt.close(); ps.close()
    result["card_after"] = card()
    print(json.dumps(result))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
