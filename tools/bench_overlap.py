"""Stage times of the dense-cloud overlap and fitness evaluation (ghicp_overlap.cu, DESIGN.md §3.12) on synthetic scan pairs
built as tools/bench_fpfh_radius.py builds its scans.

    python tools/bench_overlap.py [--points 1000000 5000000] [--thre 0.1] [--reps 5]

Per scan size: B is the synthetic scan, A a shuffled copy with 1 cm of noise.  For the identity, a pose 2 degrees / 0.5 m off
and the identity with 1 % of A placed 10 km away; in fitness mode (max_range = inf) and overlap-only mode; with the queries in
input order and in B-cell order (GHICP_OVERLAP_ORDER): the CUDA-event times of the grid build and of the queries (best of
`reps` after a warm-up), queries per second, and the work counters.  Prints one JSON line with the card's name and power
limit, read in the same run."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    from bench_prep import gpu_info, scan_cloud
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, nargs="+", default=[1000000, 5000000])
    ap.add_argument("--thre", type=float, default=0.1)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import ghicp_b200 as g
    if g.device_count() <= 0:
        raise SystemExit("bench_overlap.py: no CUDA device (the product has no CPU fallback)")
    out = {"tool": "bench_overlap", "thre_dis": args.thre, "data": "synthetic scan_like_cloud pair", "runs": []}
    off = np.eye(4)
    off[:3, :3] = g.synth.rot_xyz_deg(0.0, 0.0, 2.0)
    off[:3, 3] = [0.5, 0.0, 0.0]
    for n in args.points:
        side = (n / 1.0e6) ** 0.5 * 60.0
        B = scan_cloud(n, 1, (side, side, 6.0))
        rng = np.random.default_rng(2)
        A = (B[rng.permutation(n)] + rng.normal(0.0, 0.01, (n, 3))).astype(np.float32)
        F = A.copy()
        F[rng.choice(n, n // 100, replace=False)] += np.float32([10000.0, 0.0, 0.0])
        run = dict(points=n, cases=[])
        for name, X, Rt in (("identity", A, None), ("pose_2deg_0.5m", A, off), ("far_outliers_1pct", F, None)):
            for fitness in (True, False):
                for order in ("input", "cell"):
                    os.environ["GHICP_OVERLAP_ORDER"] = order
                    g.cloud_overlap(X, B, Rt, thre_dis=args.thre, fitness=fitness)   # warm-up
                    rs = [g.cloud_overlap(X, B, Rt, thre_dis=args.thre, fitness=fitness) for _ in range(args.reps)]
                    best = min(rs, key=lambda r: r["stage_ms"]["queries"])
                    ms = best["stage_ms"]
                    run["cases"].append(dict(case=name, mode="fitness" if fitness else "overlap_only", order=order,
                                             grid_ms=ms["grid"], query_ms=ms["queries"],
                                             queries_per_s=n / (ms["queries"] * 1e-3), ratio=best["ratio"],
                                             fitness=best["fitness"], cells_per_query=best["cells_visited"] / n,
                                             candidates_per_query=best["candidates"] / n,
                                             query_ms_spread=[min(r["stage_ms"]["queries"] for r in rs),
                                                              max(r["stage_ms"]["queries"] for r in rs)]))
        os.environ.pop("GHICP_OVERLAP_ORDER", None)
        out["runs"].append(run)
    out["gpu"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
