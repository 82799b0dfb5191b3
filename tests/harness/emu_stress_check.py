"""Run by tests/test_emulated_abi.py in a fresh process (the emulator reads its stress switches once): loads the emulated
library given on the command line in place of libghicp_b200.so and checks, against the oracle,
  * the wgmma FD build (ghicp_fdtc.cu: TMA ring -> wgmma -> register epilogue) on two shapes, bit for bit;
  * a BSC + reciprocal-NN registration through the TMA streaming kernel (ghicp_stream.cu), pair lists per iteration.
Exit status 0 = everything equal, 1 = a mismatch.  Test infrastructure only."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main(lib):
    import ghicp_b200 as g
    import oracle as orc
    from conftest import swap_in_library
    swap_in_library(g, lib)
    ok = True
    for (N, M, bits, V, dof) in [(70, 150, 441, 4, 6), (33, 260, 64, 2, 4)]:
        sc = g.synth.add_bsc(g.synth.gen_points(N, M, seed=bits + N), bits=bits, V=V)
        reg = g.registration.from_scene(sc, g.FT_BSC, g.CT_NN, dof=dof)
        reg.build_fd()
        o = orc.Oracle(g.FT_BSC, g.CT_NN, dof=dof, bbx_magnitude=sc.bbx_magnitude)
        o.set_keypoints(sc.S, sc.T); o.set_bsc(sc.bsc_s, sc.bsc_t, sc.bits); o.build_fd()
        ok = ok and np.array_equal(reg.fd(), o.fd())
        reg.close()
    sc = g.synth.add_bsc(g.synth.gen_points(300, 280, overlap=0.9, seed=3))
    reg = g.registration.from_scene(sc, g.FT_BSC, g.CT_NNR, max_iter=6)
    o = orc.Oracle(g.FT_BSC, g.CT_NNR, bbx_magnitude=sc.bbx_magnitude, solve_mode=1, max_iter=6)
    o.set_keypoints(sc.S, sc.T); o.set_bsc(sc.bsc_s, sc.bsc_t, sc.bits); o.build_fd()
    for _ in range(4):
        a, b = reg.iterate(), o.iterate()
        ok = ok and a.stream_passes > 0
        ok = ok and np.array_equal(reg.pairs()[0], o.pairs()[0]) and np.array_equal(reg.pairs()[1], o.pairs()[1])
        if a.converged or b.converged:
            break
    reg.close()
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main(sys.argv[1]))
