#!/bin/bash
# Builds libtaiga_b200.so in-tree for sm_90a (H100); the package loads it from taiga_b200/.  Then the test probe
# libtaiga_b200_probe.so (probe/, kept out of the *.cu loop below), which the tests load next to it.
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
ARCH="-gencode arch=compute_90a,code=sm_90a"
FLAGS="$ARCH -O3 -std=c++17 -lineinfo -Xcompiler -fPIC --expt-relaxed-constexpr -Xptxas -v"
mkdir -p build
# object files built for another architecture are stale even when the sources are not
if [ "$(cat build/ARCH 2>/dev/null)" != "$FLAGS" ]; then rm -f build/*.o build/probe/*.o; echo "$FLAGS" > build/ARCH; fi
pids=()
for f in *.cu; do
  o=build/${f%.cu}.o
  if [ ! -f "$o" ] || [ "$f" -nt "$o" ] || [ -n "$(find . -maxdepth 1 -name '*.cuh' -newer "$o")" ] || [ ../../include/taiga_b200.h -nt "$o" ]; then
    ( $NVCC $FLAGS -c "$f" -o "$o" > build/${f%.cu}.log 2>&1 || { cat build/${f%.cu}.log; exit 1; } ) &
    pids+=($!)
  fi
done
for p in "${pids[@]}"; do wait $p; done
$NVCC $ARCH -shared -o ../libtaiga_b200.so build/*.o -lcudart
echo "built $(realpath ../libtaiga_b200.so)"
# the test probe: C entry points over the internal kernel drivers, linked against the library above (not a copy of it)
mkdir -p build/probe
o=build/probe/tb_probe.o
if [ ! -f "$o" ] || [ probe/tb_probe.cu -nt "$o" ] || [ -n "$(find . -maxdepth 1 -name '*.cuh' -newer "$o")" ] || [ ../../include/taiga_b200.h -nt "$o" ]; then
  $NVCC $FLAGS -c probe/tb_probe.cu -o "$o" > build/probe/tb_probe.log 2>&1 || { cat build/probe/tb_probe.log; exit 1; }
fi
$NVCC $ARCH -shared -o ../libtaiga_b200_probe.so "$o" -L.. -ltaiga_b200 -lcudart -Xlinker -rpath,'$ORIGIN'
echo "built $(realpath ../libtaiga_b200_probe.so)"
