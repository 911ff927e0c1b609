#!/bin/bash
# Builds libb200grasp.so (sm_90a only) in-tree.  nvcc cross-compiles without a GPU.
set -e
cd "$(dirname "$0")/deep-rl-grasping_b200"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xcompiler -Wall -Xcompiler -fopenmp"
mkdir -p build
objs=""
pids=""
for f in csrc/*.cu; do
  o=build/$(basename "${f%.cu}").o
  stale=0
  for dep in "$f" csrc/*.cuh ../include/b200grasp.h; do          # every header is a dependency of every object
    if [ ! -f "$o" ] || [ "$dep" -nt "$o" ]; then stale=1; fi
  done
  if [ $stale = 1 ]; then
    rm -f "$o"                     # a failed compile must not leave a stale object for the link step
    $NVCC $FLAGS -c "$f" -o "$o" &
    pids="$pids $!"
  fi
  objs="$objs $o"
done
for p in $pids; do wait $p || { echo "build.sh: compilation failed" >&2; exit 1; }; done
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o libb200grasp.so $objs -ldl -lgomp
echo "built $(pwd)/libb200grasp.so"
