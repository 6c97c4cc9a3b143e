#!/bin/bash
# Build a kernel-parameter variant of libmalio_b200.so under build/variants/<name>/ (git-ignored).
#   tools/build_variant.sh t1b6 "-DMALIO_PASS_TILES=1 -DMALIO_PASS_MINB=6"
# Use it with MALIO_LIB_PATH=build/variants/<name>/libmalio_b200.so
set -e
name=$1; extra=$2
root=$(cd "$(dirname "$0")/.." && pwd)
out=$root/build/variants/$name
mkdir -p $out
cd $root/ma-lio_b200/csrc
NVCC=${NVCC:-nvcc}
NV="$NVCC -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -fmad=false -Xcompiler -fPIC -ccbin /usr/bin/g++ -I../../include -I. $extra"
for cu in *.cu; do
  f=${cu%.cu}
  $NV -Xptxas -v -c $cu -o $out/$f.o 2> $out/ptxas_$f.log &
done
/usr/bin/g++ -O3 -std=c++17 -fPIC -fopenmp -Wall -I../../include -I. -c malio_host.cpp -o $out/malio_host.o
/usr/bin/g++ -O3 -std=c++17 -fPIC -fopenmp -Wall -ffp-contract=off -I../../include -I. -c malio_dataset.cpp -o $out/malio_dataset.o
wait
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -ccbin /usr/bin/g++ -Xcompiler -fPIC $out/*.o -o $out/libmalio_b200.so -lgomp -ldl
grep -A2 "pass_kernel" $out/ptxas_malio_pass.log | grep -E "registers|spill" | head -8
echo "built $out/libmalio_b200.so"
