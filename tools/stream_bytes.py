"""True bytes and bandwidth of one k_stream launch, from a bench.py JSON line.

bench.py's `roofline.achieved` / `roofline.frac` count 2 bytes per pair (the fp16 plane the library used to stream).  The BSC
plane is now packed (gh-icp_b200/csrc/ghicp_internal.h): per 4-row x 256-column quad block, 1024 low bytes + 128 * hb bytes of
high bits, hb = 1 / 2 / 4 for descriptors of <= 511 / <= 1023 / <= 2048 bits, rows padded to quads and columns to panels.
This script recomputes the algorithmic bytes with that layout and divides by `roofline.kernel_ms`.

    python bench.py --workload config2 | python tools/stream_bytes.py
    python tools/stream_bytes.py results.jsonl      # one report per JSON line
"""
import json
import sys


def fd_hb(bits):
    return 1 if bits <= 511 else 2 if bits <= 1023 else 4


def plane_bytes(rows, M, bits):
    return -(-M // 256) * -(-rows // 4) * (1024 + 128 * fd_hb(bits))


def report(line):
    cfg, rf = line["config"], line["roofline"]
    bits, M, nloc = int(cfg["descriptor_bits"]), int(cfg["N_tgt"]), int(rf["rows_per_gpu"])
    fd = plane_bytes(nloc, M, bits) if bits > 0 else 0
    true_bytes = fd + 16 * (nloc + M) + 12 * nloc
    ms = float(rf["kernel_ms"])
    rate = true_bytes / (ms * 1e-3) / 1e9 if ms > 0 else 0.0
    peak = float(rf["peak"])
    return {"workload": cfg["workload"], "descriptor_bits": bits, "hb": fd_hb(bits) if bits else None,
            "bytes_per_pair": fd / (float(nloc) * M) if bits else 0.0, "true_bytes_per_launch": true_bytes,
            "bench_bytes_per_launch": rf.get("algorithmic_bytes_per_launch"), "kernel_ms": ms,
            "achieved_GBps": rate, "peak_GBps": peak, "frac": rate / peak if peak > 0 else None}


def main():
    src = open(sys.argv[1]) if len(sys.argv) > 1 else sys.stdin
    for raw in src:
        raw = raw.strip()
        if raw.startswith("{"):
            line = json.loads(raw)
            if "roofline" in line and line["roofline"].get("bound") == "hbm":
                print(json.dumps(report(line)))


if __name__ == "__main__":
    main()
