#!/bin/sh
# Build librsb200.so in-tree for sm_90a (H100). Usage: sh robosat_b200/csrc/build.sh
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Xptxas -v --expt-relaxed-constexpr"
OBJS=""
for f in rsb_host rsb_conv rsb_conv_row rsb_elementwise rsb_loss rsb_train rsb_wgrad rsb_morph rsb_raster; do
  $NVCC $FLAGS -c $f.cu -o $f.o 2> $f.ptxas.log || { cat $f.ptxas.log; exit 1; }
  OBJS="$OBJS $f.o"
done
# host-side PNG codec (plain C++ over zlib)
${CXX:-g++} -O3 -std=c++17 -fPIC -I/usr/local/cuda/include -c rsb_png.cpp -o rsb_png.o
${CXX:-g++} -O3 -std=c++17 -fPIC -c rsb_inflate.cpp -o rsb_inflate.o
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o ../librsb200.so $OBJS rsb_png.o rsb_inflate.o -cudart static -lz -lpthread
echo "built $(cd .. && pwd)/librsb200.so"
