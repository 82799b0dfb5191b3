"""The packed BSC feature-distance plane (gh-icp_b200/csrc/ghicp_internal.h: fd_at and the quad-block layout).

  * the layout's encoder helpers and fd_at round-trip every value 0 ... 2^(8+hb) - 1 for hb = 1, 2, 4, with row counts that
    are not whole quads and column counts that are not whole panels;
  * on the emulated C ABI (tests/harness: the product's kernels on the CPU), the plane that the wgmma build and the POPC
    build write, read back through ghicp_get_fd, equals the oracle's Hamming distances for descriptor lengths on both sides
    of every hb boundary.  Distances 0 and `bits` are forced into the plane, so the largest code of each hb is stored;
  * the same for the row block of each rank of a sharded run (a context holding rows [r0, r0 + nloc) only, nloc not a
    multiple of 4), with the builders and launch_get_fd driven directly on the emulated kernels."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_CODEC = r"""
#include "ghicp_internal.h"
using namespace ghicp_b200;
extern "C" int fd_hb_of(int bits) { return fd_hb(bits); }
extern "C" size_t plane_bytes(size_t rows, int M, int hb) { return fd_plane_bytes(rows, M, hb); }
// v: rows x M row-major values; plane: fd_plane_bytes zeroed bytes
extern "C" void encode(const unsigned *v, size_t rows, int M, int hb, unsigned char *plane) {
  for (size_t i = 0; i < rows; ++i)
    for (int j = 0; j < M; ++j) {
      const unsigned x = v[i * M + j];
      unsigned char *blk = plane + fd_block_offset(rows, hb, (int)i, j);
      const int u = (int)(i & 3), col = j & (FD_PANEL - 1), c = col & 7;
      blk[u * FD_PANEL + col] = (unsigned char)(x & 0xffu);
      reinterpret_cast<unsigned *>(blk + FD_LOW_BYTES)[fd_hi_word(hb, u, c) * 32 + (col >> 3)] |= fd_hi_part(hb, u, c, x);
    }
}
extern "C" void decode(const unsigned char *plane, size_t rows, int M, int hb, unsigned *v) {
  for (size_t i = 0; i < rows; ++i)
    for (int j = 0; j < M; ++j) v[i * M + j] = fd_at(plane, rows, hb, (int)i, j);
}
"""


@pytest.fixture(scope="module")
def codec(tmp_path_factory):
    d = tmp_path_factory.mktemp("fdcodec")
    src, out = os.path.join(str(d), "codec.cpp"), os.path.join(str(d), "codec.so")
    with open(src, "w") as f:
        f.write(_CODEC)
    r = subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-DGHICP_EMU_HOST",
                        "-I" + os.path.join(ROOT, "tests", "harness", "cuda_emu"), "-I" + os.path.join(ROOT, "include"),
                        "-I" + os.path.join(ROOT, "gh-icp_b200", "csrc"), "-o", out, src], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(out)
    L.plane_bytes.restype = C.c_size_t
    L.plane_bytes.argtypes = [C.c_size_t, C.c_int, C.c_int]
    L.encode.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p]
    L.decode.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p]
    return L


def test_hb_rule(codec):
    for bits, hb in ((9, 1), (441, 1), (511, 1), (512, 2), (672, 2), (1023, 2), (1024, 4), (2048, 4)):
        assert codec.fd_hb_of(bits) == hb, bits


@pytest.mark.parametrize("hb", [1, 2, 4])
@pytest.mark.parametrize("rows,M", [(37, 300), (5, 513), (64, 256)])
def test_every_code_round_trips_through_the_encoder_and_fd_at(codec, hb, rows, M):
    n = 1 << (8 + hb)
    rng = np.random.default_rng(hb * 1000 + rows)
    v = rng.permutation(np.arange(rows * M) % n).astype(np.uint32).reshape(rows, M)
    assert len(np.unique(v)) == min(n, rows * M)
    size = codec.plane_bytes(rows, M, hb)
    assert size == -(-M // 256) * -(-rows // 4) * (1024 + 128 * hb)
    plane = np.zeros(size, np.uint8)
    codec.encode(v.ctypes.data, rows, M, hb, plane.ctypes.data)
    out = np.zeros_like(v)
    codec.decode(plane.ctypes.data, rows, M, hb, out.ctypes.data)
    assert np.array_equal(out, v)


def _bsc_case(bits, V, N, M, seed):
    from ghicp_b200.synth import pack_bits
    rng = np.random.default_rng(seed)
    tb = rng.random((M, bits)) < 0.4
    sb = rng.random((V, N, bits)) < 0.4
    sb[:, 0] = ~tb[M - 1]          # FD(0, M-1) = bits: the largest code of the plane
    sb[:, N - 1] = tb[0]           # FD(N-1, 0) = 0
    sb[:, 1] = ~tb[1]
    sb[0, 1, : bits // 3] = tb[1, : bits // 3]   # FD(1, 1) = bits - bits // 3
    return pack_bits(sb), pack_bits(tb)


@pytest.mark.parametrize("popc", [False, True])
@pytest.mark.parametrize("bits", [9, 441, 511, 512, 672, 1023, 1024, 2048])
def test_emulated_get_fd_equals_the_oracle(g, orc, emu_library_path, monkeypatch, bits, popc):
    from conftest import swap_in_library
    if popc:
        monkeypatch.setenv("GHICP_FD_POPC", "1")
    N, M, dof = 37, 300, (6 if bits % 2 else 4)
    V = 4 if dof == 6 else 2
    bs, bt = _bsc_case(bits, V, N, M, bits)
    real = swap_in_library(g, emu_library_path)
    try:
        Kp = g.Keypoints().setCoordinate(np.zeros((N, 3)), np.zeros((M, 3))).setBSCfeature(bs, bt, bits)
        reg = g.GHRegistration(Kp, g.Energyfunction().init(N, M, 10.0), g.FT_BSC, g.CT_NN, dof_type=dof)
        fd = reg.fd()
    finally:
        g.capi._lib = real
    o = orc.Oracle(orc.FT_BSC, orc.CT_NN, dof=dof, bbx_magnitude=10.0, solve_mode=1)
    o.set_keypoints(np.zeros((N, 3)), np.zeros((M, 3)))
    o.set_bsc(bs, bt, bits)
    o.build_fd()
    ref = o.fd()
    assert ref[0, M - 1] == bits and ref[N - 1, 0] == 0
    assert np.array_equal(fd, ref)


_SHARD = r"""
#include "%s"
// one rank's FD plane: rows [r0, r0 + nloc) of an N x M problem; bs [V][N][B], bt [M][B]; out N x M (other rows zero)
extern "C" int shard_fd(int popc, int V, int bits, int N, int M, int r0, int nloc, const uint8_t *bs, const uint8_t *bt, double *out) {
  using namespace ghicp_b200;
  Ctx c;
  c.cfg.dof = V == 4 ? 6 : 4; c.N = N; c.M = M; c.r0 = r0; c.nloc = nloc; c.V = V; c.bits = bits;
  c.Bbytes = (bits + 7) / 8; c.W64 = (c.Bbytes + 7) / 8; c.fd_rows = (size_t)nloc;
  std::vector<uint64_t> ws((size_t)V * c.W64 * N), wt((size_t)c.W64 * M);
  c.d_bs = ws.data(); c.d_bt = wt.data();
  if (launch_pack_bsc(&c, bs, bt) != cudaSuccess) return 1;
  std::vector<uint16_t> plane((fd_plane_bytes(c.fd_rows, M, fd_hb(bits)) + 1) / 2, 0);
  c.d_fd16 = plane.data();
  if ((popc ? launch_fd_bsc(&c) : launch_fd_bsc_tc(&c)) != cudaSuccess) return 2;
  return launch_get_fd(&c, out) == cudaSuccess ? 0 : 3;
}
"""


@pytest.fixture(scope="module")
def shard_lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("fdshard")
    src, out = os.path.join(str(d), "shard.cpp"), os.path.join(str(d), "shard.so")
    with open(src, "w") as f:
        f.write(_SHARD % os.path.join(ROOT, "tests", "harness", "emu_library.cpp"))
    r = subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-DGHICP_EMU_HOST",
                        "-I" + os.path.join(ROOT, "tests", "harness", "cuda_emu"), "-I" + os.path.join(ROOT, "include"),
                        "-o", out, src, "-ldl"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(out)
    L.shard_fd.argtypes = [C.c_int] * 7 + [C.c_void_p] * 3
    return L


@pytest.mark.parametrize("popc", [False, True])
@pytest.mark.parametrize("bits", [441, 672, 2048])
def test_sharded_row_blocks_equal_the_oracle(shard_lib, orc, bits, popc):
    N, M, world = 37, 300, 3
    V = 4
    bs, bt = _bsc_case(bits, V, N, M, bits + 1)
    o = orc.Oracle(orc.FT_BSC, orc.CT_NN, dof=6, bbx_magnitude=10.0, solve_mode=1)
    o.set_keypoints(np.zeros((N, 3)), np.zeros((M, 3)))
    o.set_bsc(bs, bt, bits)
    o.build_fd()
    ref = o.fd()
    shard = -(-N // world)
    for rank in range(world):
        r0 = min(N, rank * shard)
        nloc = max(0, min(N, r0 + shard) - r0)
        out = np.full((N, M), -1.0)
        assert shard_lib.shard_fd(int(popc), V, bits, N, M, r0, nloc, np.ascontiguousarray(bs).ctypes.data,
                                  np.ascontiguousarray(bt).ctypes.data, out.ctypes.data) == 0
        assert np.array_equal(out[r0:r0 + nloc], ref[r0:r0 + nloc]), rank
        assert not out[:r0].any() and not out[r0 + nloc:].any()
