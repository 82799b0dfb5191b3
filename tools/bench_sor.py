"""Stage times of the statistical outlier removal (CFilter::SORFilter, DESIGN.md §3.16) on synthetic scans.

    python tools/bench_sor.py [--points 1000000 5000000] [--voxel 0.05] [--k 8 20 31 50 128] [--reps 5]

Per scan size (synth.scan_pair's target scan): the raw scan and its voxel-filtered cloud, for each mean_k: the CUDA-event
times of the grid, the distances, the statistics and the compaction (best of `reps` by total after a warm-up, with the spread
of the totals), points per second, candidates examined per query and exhaustive-scan fallbacks.  mean_k <= 31 runs on k_knn's
register top-k; for those k the same run also times the warp kernel that serves larger k (GHICP_SOR_FORCE_WARP=1, "warp"), the
other side of the path choice, and checks that both give the same distances.  Prints one JSON line with the card's name and
power limit, read in the same run."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, os.path.join(os.path.dirname(ROOT), "tests"))
sys.path.insert(0, ROOT)


def main():
    from bench_prep import gpu_info
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, nargs="+", default=[1000000, 5000000])
    ap.add_argument("--voxel", type=float, default=0.05)
    ap.add_argument("--k", type=int, nargs="+", default=[8, 20, 31, 50, 128])
    ap.add_argument("--std", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import ghicp_b200 as g
    if g.device_count() <= 0:
        raise SystemExit("bench_sor.py: no CUDA device (the product has no CPU fallback)")
    out = {"tool": "bench_sor", "voxel": args.voxel, "std_mul": args.std, "data": "synth.scan_pair target scan", "runs": []}
    for n in args.points:
        T, _, _, _ = g.synth.scan_pair(n, seed=6)
        raw = np.ascontiguousarray(T, np.float32)
        clouds = dict(raw=raw, voxel=np.ascontiguousarray(raw[g.voxel_downsample(raw, args.voxel)]))
        for name, P in clouds.items():
            for k in args.k:
                g.sor_filter(P, k, args.std)   # warm-up
                rs = [g.sor_filter(P, k, args.std)[1] for _ in range(args.reps)]
                best = min(rs, key=lambda r: r["stage_ms"]["total"])
                ms = best["stage_ms"]
                row = dict(points=n, cloud=name, n=len(P), mean_k=k, kept=best["n_kept"], stage_ms=ms,
                           total_ms_spread=[min(r["stage_ms"]["total"] for r in rs), max(r["stage_ms"]["total"] for r in rs)],
                           points_per_s=len(P) / (ms["total"] * 1e-3), distances_points_per_s=len(P) / (ms["distances"] * 1e-3),
                           candidates_per_query=best["candidates"] / max(best["n_finite"], 1), fallbacks=best["fallbacks"])
                if k <= 31:
                    os.environ["GHICP_SOR_FORCE_WARP"] = "1"
                    try:
                        g.sor_filter(P, k, args.std)
                        ws = [g.sor_filter(P, k, args.std, return_distances=True)[1] for _ in range(args.reps)]
                    finally:
                        os.environ.pop("GHICP_SOR_FORCE_WARP")
                    wb = min(ws, key=lambda r: r["stage_ms"]["total"])
                    same = np.array_equal(wb["distances"].view(np.uint32),
                                          g.sor_filter(P, k, args.std, return_distances=True)[1]["distances"].view(np.uint32))
                    row["warp"] = dict(stage_ms=wb["stage_ms"], candidates_per_query=wb["candidates"] / max(wb["n_finite"], 1),
                                       same_distances=bool(same))
                out["runs"].append(row)
    out["gpu"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
