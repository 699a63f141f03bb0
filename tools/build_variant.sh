#!/bin/bash
# A/B build of the C-ABI library with extra -D flags:  tools/build_variant.sh <name> -DMDB_MBAR_WAIT_MODE=1
# -> magicdrive_b200/lib/variants/lib<name>.so   (select with MDB_LIB_PATH=<that file>)
# Each source gets the product's flags (magicdrive_b200/build.py): --use_fast_math except for the files in its PRECISE set.
set -e
name=$1; shift
root=$(cd "$(dirname "$0")/.." && pwd)
out=$root/magicdrive_b200/lib/variants; mkdir -p $out/$name
precise=" $(python3 -c "import runpy, sys; print(' '.join(sorted(runpy.run_path(sys.argv[1])['PRECISE'])))" \
  $root/magicdrive_b200/build.py) "
pids=()
for f in $root/magicdrive_b200/csrc/*.cu; do
  b=$(basename $f .cu)
  fm="--use_fast_math"; case "$precise" in *" $b.cu "*) fm="";; esac
  nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC $fm "$@" -c $f -o $out/$name/$b.o 2>/dev/null &
  pids+=($!)
done
for p in "${pids[@]}"; do wait $p; done
nvcc -shared -o $out/lib$name.so $out/$name/*.o -lcudart_static -lpthread -ldl -lrt 2>/dev/null
rm -rf $out/$name
echo $out/lib$name.so
