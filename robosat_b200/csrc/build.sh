#!/bin/sh
# Build librsb200.so in-tree for sm_90a (H100). Usage: sh robosat_b200/csrc/build.sh
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Xptxas -v --expt-relaxed-constexpr"
OBJS=""
for f in rsb_host rsb_conv rsb_conv_row rsb_elementwise rsb_loss rsb_train rsb_wgrad rsb_morph rsb_label rsb_raster rsb_cover rsb_dedupe rsb_merge rsb_extract rsb_compare rsb_tile rsb_bands rsb_mosaic rsb_road rsb_jpeg; do
  $NVCC $FLAGS -c $f.cu -o $f.o 2> $f.ptxas.log || { cat $f.ptxas.log; exit 1; }
  OBJS="$OBJS $f.o"
done
# host-side PNG codec (plain C++ over zlib)
${CXX:-g++} -O3 -std=c++17 -fPIC -I/usr/local/cuda/include -c rsb_png.cpp -o rsb_png.o
${CXX:-g++} -O3 -std=c++17 -fPIC -c rsb_inflate.cpp -o rsb_inflate.o
# host-side TIFF strip / tile decoder of `rs tile` and tile encoder of `rs mosaic` (plain C++ over zlib)
${CXX:-g++} -O3 -std=c++17 -fPIC -I/usr/local/cuda/include -c rsb_tiff.cpp -o rsb_tiff.o
# host-side JPEG chunk header parser of `rs tile` / `rs segment` (plain C++; the decode itself is rsb_jpeg.cu)
${CXX:-g++} -O3 -std=c++17 -fPIC -I/usr/local/cuda/include -c rsb_jpeg_parse.cpp -o rsb_jpeg_parse.o
# host-side OpenStreetMap PBF framing, inflate and parsing (plain C++ over zlib)
${CXX:-g++} -O3 -std=c++17 -fPIC -I/usr/local/cuda/include -c rsb_pbf.cpp -o rsb_pbf.o
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o ../librsb200.so $OBJS rsb_png.o rsb_inflate.o rsb_pbf.o rsb_tiff.o rsb_jpeg_parse.o -cudart static -lz -lpthread
echo "built $(cd .. && pwd)/librsb200.so"
