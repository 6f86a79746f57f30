#!/bin/bash
# Builds libmono_emb.so (sm_90a only: H100) next to the Python package: monolith_b200/lib/libmono_emb.so
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
OUT="$HERE/../lib"
mkdir -p "$OUT" "$HERE/obj"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
ARCH="-gencode arch=compute_90a,code=sm_90a"
FLAGS="$ARCH -O3 -lineinfo -std=c++17 -fmad=false -Xcompiler -fPIC -Xptxas -v --threads 4"
pids=()
for f in table ops bwd xstep dedup layout peer ckpt tower clip capi; do
  ( $NVCC $FLAGS -c "$HERE/$f.cu" -o "$HERE/obj/$f.o" > "$HERE/obj/$f.log" 2>&1 || { cat "$HERE/obj/$f.log"; exit 1; } ) &
  pids+=($!)
done
rc=0
for p in "${pids[@]}"; do wait $p || rc=1; done
[ $rc -eq 0 ] || { echo "compile failed"; exit 1; }
$NVCC $ARCH -shared -o "$OUT/libmono_emb.so" "$HERE"/obj/{table,ops,bwd,xstep,dedup,layout,peer,ckpt,tower,clip,capi}.o -cudart static
echo "built $OUT/libmono_emb.so"
