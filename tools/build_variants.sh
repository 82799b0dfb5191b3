#!/bin/bash
# A/B builds of libghicp_b200.so with other compile-time tuning knobs of the streaming kernel (ghicp_stream.cu:
# GHICP_ST_RING_KB ring bytes per warp, GHICP_ST_MINB resident CTAs per SM; the batch is the plane's 4-row quad).  Output:
# gh-icp_b200/variants/lib_<name>.so (git-ignored; select with GHICP_B200_LIB=<path> python bench.py ...).
set -e
cd "$(dirname "$0")/../gh-icp_b200/csrc"
make -j4 > /dev/null
mkdir -p ../variants
NV="/usr/local/cuda/bin/nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC -Xcompiler -O3 -ccbin /usr/bin/g++"
OTHERS="ghicp_kernels.o ghicp_fpfh.o ghicp_solvers.o ghicp_prep.o ghicp_fdtc.o ghicp_auction.o ghicp_comm.o ghicp_capi.o"
for v in "$@"; do
  name=${v%%:*}; flags=${v#*:}
  $NV $flags -c ghicp_stream.cu -o ../variants/stream_$name.o
  /usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../variants/lib_$name.so ../variants/stream_$name.o $OTHERS -lcudart -ldl
  rm -f ../variants/stream_$name.o
  echo "built variants/lib_$name.so ($flags)"
done
