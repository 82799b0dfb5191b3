"""The FP32 correspondence filters on the H100 (tests/test_filter_margins.py restates them on the CPU):
  * the approximate MUFU instructions they use (tests/harness/mufu_error.cu) against float64, inside the error figures the
    restatement budgets for;
  * near-tie scenes (a decoy the float filter ranks at or below the true nearest target) in lock step against the
    library's all-double route and the oracle, at ~3000^2 and at 48k^2 (full grid, multi-CTA column blocks);
  * a power-of-two scale sweep from 2^-40 to 2^40: identical pair lists and R, t scaled exactly, and the all-double route
    outside the filter's float window (exact_fallback bit 2)."""
import os
import subprocess

import pytest

from test_filter_margins import EX2_REL, LG2_ABS, SQRT_REL, near_tie_scene, run_near_ties, run_scale_sweep, START

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.gpu
def test_mufu_errors_inside_the_budget(tmp_path):
    exe = str(tmp_path / "mufu_error")
    r = subprocess.run(["nvcc", "-O2", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
                        os.path.join(HERE, "harness", "mufu_error.cu")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    f = r.stdout.split()
    got = {f[k]: float(f[k + 1]) for k in range(0, len(f), 2)}
    print(f"\nmeasured: sqrt.approx.ftz rel {got['sqrt_rel']:.3e} (2^{_log2(got['sqrt_rel']):.2f}), "
          f"lg2.approx.ftz abs {got['lg2_abs']:.3e} (2^{_log2(got['lg2_abs']):.2f}; / (1 + |lg2|): 2^{_log2(got['lg2_model']):.2f}), "
          f"ex2.approx.ftz rel {got['ex2_rel']:.3e} (2^{_log2(got['ex2_rel']):.2f})")
    assert got["sqrt_rel"] <= SQRT_REL
    assert got["lg2_model"] <= LG2_ABS        # |error| / (1 + |lg2 x|): the restatement's model
    assert got["ex2_rel"] <= EX2_REL
    assert got["sqrt_sub_nonzero"] == 0       # .ftz: a subnormal d2' is read as 0, as the restatement models it


def _log2(x):
    import math
    return math.log2(x) if x > 0 else float("-inf")


NEAR_TIE_CASES = [("none", "nn"), ("none", "nnr"), ("none", "km"), ("bsc", "nn"), ("bsc", "nnr"), ("bsc", "km"),
                  ("fpfh", "nn"), ("fpfh", "nnr")]


@pytest.mark.gpu
@pytest.mark.parametrize("ft,ct", NEAR_TIE_CASES)
def test_near_ties(g, orc, scratch_cwd, ft, ct):
    run_near_ties(g, orc, ft, ct, N=3000)


@pytest.mark.gpu
@pytest.mark.parametrize("ct", ["nn", "km"])
def test_near_ties_48k(g, orc, scratch_cwd, ct):
    sc = near_tie_scene(g, "none", 48000, START["none"], max_decoys=4000)
    run_near_ties(g, orc, "none", ct, N=48000, iters=1, scene=sc, with_oracle=False)   # (the CPU oracle: too slow here)


@pytest.mark.gpu
@pytest.mark.parametrize("ft,ct", [("none", "nn"), ("none", "nnr"), ("none", "km"), ("bsc", "nn"), ("bsc", "nnr"),
                                   ("bsc", "km"), ("fpfh", "nn"), ("fpfh", "nnr")])
def test_scale_sweep(g, orc, scratch_cwd, ft, ct):
    run_scale_sweep(g, orc, ft, ct, N=1000, iters=4)
