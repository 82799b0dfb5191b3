"""Wall-clock time of the one-time FD build (ghicp_build_fd) at 50k x 50k for several descriptor lengths, three builds each in
one process (the first one carries module loading and the first growth of the allocator's pool).
    python tools/fd_time.py [bits ...]      GHICP_FD_POPC=1 selects the XOR + POPC kernel"""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ghicp_b200 as g  # noqa: E402

for bits in [int(x) for x in sys.argv[1:]] or [441, 672]:
    sc = g.synth.add_bsc(g.synth.gen_points(50000, 50000, overlap=0.6, extent=(200, 200, 40), noise=0.05, seed=2), bits=bits, V=4)
    out = []
    for rep in range(3):
        reg = g.registration.from_scene(sc, g.FT_BSC, g.CT_NN)
        t0 = time.perf_counter()
        reg.build_fd()
        out.append(round((time.perf_counter() - t0) * 1e3, 2))
        reg.close()
    print("bits", bits, "POPC" if os.environ.get("GHICP_FD_POPC") else "wgmma", "build_fd ms (3 builds in one process):", out, flush=True)
