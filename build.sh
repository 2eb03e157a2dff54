#!/usr/bin/env bash
# Build libb200asr.so in-tree for sm_90a (H100; cross-compiles without a GPU).
set -euo pipefail
cd "$(dirname "$0")"
PKG="end2end-asr-pytorch_b200"
SRC="$PKG/csrc"
OUT="$PKG/libb200asr.so"
OBJ="$SRC/build"
mkdir -p "$OBJ"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC ${B200ASR_DEFS:-}"
pids=()
objs=()
for f in "$SRC"/*.cu; do
  o="$OBJ/$(basename "${f%.cu}").o"
  objs+=("$o")
  if [ ! -f "$o" ] || [ "$f" -nt "$o" ] || [ -n "$(find "$SRC" include -name '*.h' -newer "$o" -o -name '*.cuh' -newer "$o" | head -1)" ]; then
    $NVCC $FLAGS -c "$f" -o "$o" &
    pids+=($!)
  fi
done
for p in "${pids[@]:-}"; do [ -n "$p" ] && wait "$p"; done
$NVCC -shared -o "$OUT" "${objs[@]}" -gencode arch=compute_90a,code=sm_90a
echo "built $OUT"
