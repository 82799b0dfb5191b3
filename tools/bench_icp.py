"""Stage times of point-to-point ICP on the dense clouds (ghicp_icp.cu, DESIGN.md §3.13) on the synthetic scan pairs
(synth.scan_pair), down-sampled at 0.05 m on the device as tools/bench_overlap.py scores them.  --metric plane times
point-to-plane ICP (§3.14) instead, with the target normals' k = --normal-k, and adds the one-time normal estimation
(normals_ms: the first point-to-plane call's stage_ms["grid"], the target's grid being cached by then).  --metric gicp times
Generalized ICP (§3.15), whose normals_ms covers both clouds' normals.

    python tools/bench_icp.py [--points 1000000 5000000] [--reps 3] [--voxel 0.05] [--metric point|plane|gicp] [--normal-k 20]

Per scan size: the target grid build, then from the truth perturbed by 2 degrees / 0.5 m and from the truth itself, with and
without reciprocal correspondences, with and without the trimmed rejector (ratio = calOverlap at the start within 0.3 m):
ms per iteration (CUDA events, best of `reps` after a warm-up), cells and candidates per query, iterations to convergence,
final rotation / translation error against the truth.  Also one fitness-mode overlap query pass at the start pose (the
reference point of an iteration without reciprocal).  Prints one JSON line with the card's name and power limit, read in the
same run."""
import argparse
import json
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def errors(Rt, G):
    M = Rt[:3, :3].T @ G[:3, :3]
    v = 0.5 * np.array([M[2, 1] - M[1, 2], M[0, 2] - M[2, 0], M[1, 0] - M[0, 1]])
    return math.degrees(math.asin(min(1.0, float(np.linalg.norm(v))))), float(np.linalg.norm(Rt[:3, 3] - G[:3, 3]))


def main():
    from bench_prep import gpu_info
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, nargs="+", default=[1000000, 5000000])
    ap.add_argument("--voxel", type=float, default=0.05)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-iter", type=int, default=50)
    ap.add_argument("--metric", choices=["point", "plane", "gicp"], default="point")
    ap.add_argument("--normal-k", type=int, default=20)
    args = ap.parse_args()
    mkw = {} if args.metric == "point" else dict(metric=args.metric, normal_k=args.normal_k)
    import ghicp_b200 as g
    if g.device_count() <= 0:
        raise SystemExit("bench_icp.py: no CUDA device (the product has no CPU fallback)")
    out = {"tool": "bench_icp", "voxel": args.voxel, "data": "synth.scan_pair", "runs": []}
    if mkw:
        out.update(metric=args.metric, normal_k=args.normal_k)
    off = np.eye(4)
    off[:3, :3] = g.synth.rot_xyz_deg(0.6, -0.4, 2.0 * math.sqrt(1.0 - 0.13))   # 2 degrees in all
    off[:3, 3] = [0.3, -0.3, 0.25]                                               # 0.49 m
    for n in args.points:
        T, S, R, t = g.synth.scan_pair(n, seed=4)
        G = np.eye(4)
        G[:3, :3], G[:3, 3] = R, t
        pt, ps = g.Prep(T, args.voxel, 1.0, 1.5), g.Prep(S, args.voxel, 1.0, 1.5)
        run = dict(points=n, n_source_down=ps.n_down, n_target_down=pt.n_down, cases=[])
        try:
            run["grid_ms"] = ps.overlap(pt, None, thre_dis=0.3)["stage_ms"]["grid"]   # the first call on the target builds it
            if mkw:   # the first point-to-plane (GICP) call estimates the target's (both clouds') normals; the grid is cached
                run["normals_ms"] = ps.icp(pt, None, max_iterations=1, **mkw)[1]["stage_ms"]["grid"]
            for start, G0 in (("2deg_0.5m", off @ G), ("truth", G)):
                ov = [ps.overlap(pt, G0, thre_dis=0.3) for _ in range(args.reps + 1)][1:]
                rho = min(ps.overlap(pt, G0, thre_dis=0.3, fitness=False)["ratio"], 1.0)
                for recip in (False, True):
                    for trim in (0.0, rho):
                        kw = dict(max_iterations=args.max_iter, reciprocal=recip, trim_ratio=trim, **mkw)
                        ps.icp(pt, G0, **kw)   # warm-up
                        rs = [ps.icp(pt, G0, **kw) for _ in range(args.reps)]
                        Rt, best = min(rs, key=lambda r: r[1]["stage_ms"]["iterations"])
                        k = best["iterations"]
                        e0, e = errors(G0, G), errors(Rt, G)
                        run["cases"].append(dict(start=start, reciprocal=recip, trim_ratio=trim, iterations=k, state=best["state"],
                                                 ms_per_iteration=best["stage_ms"]["iterations"] / k,
                                                 ms_per_iteration_spread=[min(r[1]["stage_ms"]["iterations"] / k for r in rs),
                                                                          max(r[1]["stage_ms"]["iterations"] / k for r in rs)],
                                                 fitness_ms=best["stage_ms"]["fitness"],
                                                 cells_per_query=best["cells_visited"] / (k * ps.n_down),
                                                 candidates_per_query=best["candidates"] / (k * ps.n_down),
                                                 start_error_deg_m=e0, final_error_deg_m=e, fitness=best["fitness"]))
                run["cases"].append(dict(start=start, overlap_fitness_query_ms=min(o["stage_ms"]["queries"] for o in ov),
                                         cells_per_query=ov[0]["cells_visited"] / ps.n_down))
        finally:
            pt.close(); ps.close()
        out["runs"].append(run)
    out["gpu"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
