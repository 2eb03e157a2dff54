#!/usr/bin/env bash
# A/B build of the library with extra -D flags: tools/build_variant.sh <name> "<defs>"  ->  end2end-asr-pytorch_b200/csrc/build/variants/libb200asr_<name>.so
# (select it at run time with B200ASR_LIB=<path>)
set -euo pipefail
cd "$(dirname "$0")/.."
name=$1; defs=$2
SRC=end2end-asr-pytorch_b200/csrc
OBJ=$SRC/build/variants/$name
mkdir -p "$OBJ"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
pids=()
for f in "$SRC"/*.cu; do
  $NVCC -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC $defs -c "$f" -o "$OBJ/$(basename "${f%.cu}").o" &
  pids+=($!)
done
for p in "${pids[@]}"; do wait "$p"; done
$NVCC -shared -o "$SRC/build/variants/libb200asr_$name.so" "$OBJ"/*.o -gencode arch=compute_90a,code=sm_90a
echo "built $SRC/build/variants/libb200asr_$name.so"
