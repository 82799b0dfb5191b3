"""Every route of one registration iteration (ghicp_capi.cu: choose_route) on the emulated library, against statistics
recorded from an earlier build of the same library.  A change to the orchestration that reorders or drops a launch, moves
an event, or changes what a route reports shows up here as a changed launch count or field, without a GPU.

Case -> route(s) it exercises (iterations 0, 1, ... of the case):
  none_nn, none_nnr           stream NN / NNR in every iteration
  none_km                     stream KM, general (no feature: never settled)
  bsc_nn, bsc_nnr_dof4        stream NN / NNR (dof 4: two source variants)
  bsc_km                      stream KM, general in iterations 0-1, stream KM, settled from iteration 2
  bsc_km_fill                 GHICP_KM_FILL: stream KM, general, always with the fill pass
  bsc_km_general              GHICP_KM_GENERAL: stream KM, general in every iteration
  bsc_km_xuse8                GHICP_KM_XUSE_MAX=8: stream KM, settled from iteration 2, whose block overflows, then the
                              redo on stream KM, general (bit 1 of exact_fallback)
  exact_bsc_nn/_nnr/_km       force_exact: all-double in every iteration
  fpfh_nn                     all-double in iterations 0-1, FPFH filter NN from iteration 2
  fpfh_nnr                    FPFH filter NNR in every iteration
  fpfh_km                     all-double while the graph is dense (iterations 0-2 here), then FPFH + KM, settled
  fpfh_nn_exact               GHICP_FPFH_EXACT: all-double (matrix-free sweeps) in every iteration
  fpfh_plane_nn, _km          fpfh_matrix_free = -1 (stored FPFH plane): all-double in every iteration
  probe_bsc, probe_fpfh       ghicp_probe_rowmin after ghicp_reset: the all-double route's row stage

Per iteration the integer fields of ghicp_iter_stats, every double field but the ms_* timings (as float.hex) and SHA-256
digests of the pair lists and of the moved source keypoints are compared.  Recording (from the build to compare against):
    python tests/test_iteration_routes.py --record"""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "iteration_routes.json")
ITERS = 8

# name: (feature, correspondence, dof, environment, GHRegistration keyword arguments)
CASES = {
    "none_nn": ("none", "nn", 6, {}, {}),
    "none_nnr": ("none", "nnr", 6, {}, {}),
    "none_km": ("none", "km", 6, {}, {}),
    "bsc_nn": ("bsc", "nn", 6, {}, {}),
    "bsc_nnr_dof4": ("bsc", "nnr", 4, {}, {}),
    "bsc_km": ("bsc", "km", 6, {}, {}),
    "bsc_km_fill": ("bsc", "km", 6, {"GHICP_KM_FILL": "1"}, {}),
    "bsc_km_general": ("bsc", "km", 6, {"GHICP_KM_GENERAL": "1"}, {}),
    "bsc_km_xuse8": ("bsc", "km", 6, {"GHICP_KM_XUSE_MAX": "8"}, {}),
    "exact_bsc_nn": ("bsc", "nn", 6, {}, {"force_exact": True}),
    "exact_bsc_nnr": ("bsc", "nnr", 6, {}, {"force_exact": True}),
    "exact_bsc_km": ("bsc", "km", 6, {}, {"force_exact": True}),
    "fpfh_nn": ("fpfh", "nn", 6, {}, {}),
    "fpfh_nnr": ("fpfh", "nnr", 6, {}, {}),
    "fpfh_km": ("fpfh", "km", 6, {}, {}),
    "fpfh_nn_exact": ("fpfh", "nn", 6, {"GHICP_FPFH_EXACT": "1"}, {}),
    "fpfh_plane_nn": ("fpfh", "nn", 6, {}, {"fpfh_matrix_free": -1}),
    "fpfh_plane_km": ("fpfh", "km", 6, {}, {"fpfh_matrix_free": -1}),
    "probe_bsc": ("bsc", "nn", 6, {}, {}),
    "probe_fpfh": ("fpfh", "nn", 6, {}, {}),
}
HOOKS = ("GHICP_KM_FILL", "GHICP_KM_GENERAL", "GHICP_KM_XUSE_MAX", "GHICP_FPFH_EXACT", "GHICP_FPFH_MATRIX_FREE", "GHICP_FD_POPC",
         "GHICP_CAND_CAP_MAX")
INT_FIELDS = ("iteration", "cor", "converged", "warnings", "nnz", "km_rounds", "km_phases", "gpu_launches", "exact_fallback",
              "stream_passes", "candidates")
DOUBLE_FIELDS = ("cd_mean", "cd_std", "penalty", "rmse", "rmse_after", "fdm", "fdstd", "iou", "para1", "para2", "km_energy",
                 "ax", "ay", "az")


def _sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def _hex(xs):
    return [float(x).hex() for x in xs]


def run_case(g, name):
    """The case's per-iteration records; the caller sets the case's environment."""
    ft, ct, dof, _, kw = CASES[name]
    FT = {"none": g.FT_NONE, "bsc": g.FT_BSC, "fpfh": g.FT_FPFH}[ft]
    CT = {"nn": g.CT_NN, "nnr": g.CT_NNR, "km": g.CT_KM}[ct]
    N, M = (110, 100) if ct == "km" else (260, 230)
    sc = g.synth.gen_points(N, M, overlap=0.9, seed=11)
    if ft == "bsc":
        g.synth.add_bsc(sc, V=4 if dof == 6 else 2)
    if ft == "fpfh":
        g.synth.add_fpfh(sc)
    reg = g.registration.from_scene(sc, FT, CT, dof=dof, **kw)
    out = []
    try:
        if name.startswith("probe_"):
            for _ in range(2):
                reg.iterate()
            reg.reset()
            idx, cd, mean, std, penalty = reg.probe_rowmin()
            return [{"idx": _sha(idx), "cd": _sha(cd), "scalars": _hex((mean, std, penalty))}]
        for _ in range(ITERS):
            st = reg.iterate()
            sp, tp = reg.pairs()
            rec = {f: int(getattr(st, f)) for f in INT_FIELDS}
            rec.update({f: float(getattr(st, f)).hex() for f in DOUBLE_FIELDS})
            rec["Rt"], rec["Rt_tillnow"] = _hex(st.Rt), _hex(st.Rt_tillnow)
            rec["pairs"], rec["source"] = _sha(sp, tp), _sha(reg.source())
            out.append(rec)
    finally:
        reg.close()
    return out


@pytest.fixture()
def ge(g, emu_library_path):
    """The product package with the emulated library swapped in for this test only."""
    from conftest import swap_in_library
    real = swap_in_library(g, emu_library_path)
    try:
        yield g
    finally:
        g.capi._lib = real


@pytest.mark.parametrize("name", list(CASES))
def test_iteration_route_reproduces_recorded_statistics(ge, monkeypatch, name):
    for k in HOOKS + ("GHICP_EMU_SCHED",):
        monkeypatch.delenv(k, raising=False)
    for k, v in CASES[name][3].items():
        monkeypatch.setenv(k, v)
    with open(GOLDEN) as f:
        want = json.load(f)[name]
    got = run_case(ge, name)
    assert len(got) == len(want)
    for it, (a, b) in enumerate(zip(got, want)):
        assert a == b, (name, it, {k: (a[k], b[k]) for k in b if a.get(k) != b[k]})


if __name__ == "__main__" and sys.argv[1:] == ["--record"]:
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import tempfile

    from conftest import build_emulated_library, swap_in_library

    import ghicp_b200
    ghicp_b200.build_library()
    swap_in_library(ghicp_b200, build_emulated_library(tempfile.mkdtemp()))
    for k in HOOKS + ("GHICP_EMU_SCHED",):
        os.environ.pop(k, None)
    golden = {}
    for name, case in CASES.items():
        os.environ.update(case[3])
        golden[name] = run_case(ghicp_b200, name)
        for k in case[3]:
            del os.environ[k]
        print(name, "recorded", flush=True)
    with open(GOLDEN, "w") as f:
        json.dump(golden, f, indent=0, sort_keys=True)
        f.write("\n")
