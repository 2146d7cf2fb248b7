#!/bin/bash
# Build the C-ABI library in-tree for sm_90a (cross-compiles without a GPU), in its two storage flavours:
#   lib/libb200gen.so       16-bit storage = IEEE fp16 (default)
#   lib/libb200gen_bf16.so  16-bit storage = bfloat16  (-DB200_H16_IS_BF16; B200_ACT_DTYPE=bf16 selects it)
set -euo pipefail
here="$(cd "$(dirname "$0")" && pwd)"
out="$here/../lib"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC"
SRCS="core igemm norm elementwise vq attention_small flash_attn decode repack metrics fid perceptual"
mkdir -p "$out" "$here/.obj" "$here/.obj/bf16"
pids=()
for flavour in fp16 bf16; do
  if [ "$flavour" = bf16 ]; then obj="$here/.obj/bf16"; extra="-DB200_H16_IS_BF16"; else obj="$here/.obj"; extra=""; fi
  for f in $SRCS; do
    [ -f "$here/$f.cu" ] || continue
    if [ ! -f "$obj/$f.o" ] || [ "$here/$f.cu" -nt "$obj/$f.o" ] || [ "$here/common.cuh" -nt "$obj/$f.o" ] || [ "$here/wgmma.cuh" -nt "$obj/$f.o" ] || [ "$here/../../include/b200gen.h" -nt "$obj/$f.o" ] || [ "$here/../../include/b200gen_metrics.h" -nt "$obj/$f.o" ] || [ "$here/../../include/b200gen_fid.h" -nt "$obj/$f.o" ] || [ "$here/../../include/b200gen_perceptual.h" -nt "$obj/$f.o" ]; then
      $NVCC $FLAGS $extra -c "$here/$f.cu" -o "$obj/$f.o" &
      pids+=($!)
    fi
  done
done
for p in "${pids[@]:-}"; do [ -n "$p" ] && wait "$p"; done
$NVCC -shared -o "$out/libb200gen.so" "$here"/.obj/*.o -Xcompiler -fPIC
$NVCC -shared -o "$out/libb200gen_bf16.so" "$here"/.obj/bf16/*.o -Xcompiler -fPIC
echo "built $out/libb200gen.so $out/libb200gen_bf16.so"
