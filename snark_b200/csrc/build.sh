#!/usr/bin/env bash
# Build libb200snark.so in-tree for sm_90a (nvcc cross-compiles without a GPU).
set -euo pipefail
cd "$(dirname "$0")"
OUT=../libb200snark.so
OBJ=../../build/obj
mkdir -p "$OBJ"
ARCH="-gencode arch=compute_90a,code=sm_90a"
FLAGS="$ARCH -O3 -std=c++17 -lineinfo -Xcompiler -fPIC --expt-relaxed-constexpr"
# objects compiled with other flags (architecture, B2S_NVCC_EXTRA) are never reused: the flags are kept in a stamp
STAMP="$OBJ/flags"
if [ "$(cat "$STAMP" 2>/dev/null)" != "$FLAGS ${B2S_NVCC_EXTRA:-}" ]; then rm -f "$OBJ"/*.o "$STAMP"; fi
pids=()
for f in api group ntt dntt msm msm_acc_g1 msm_acc_g2 r1cs lcmap gr1cs sr1cs groth16 setup setup_groth16 serialize deserialize verify verify_rlc verify_bytes zkey testops poly; do
  if [ ! -f "$OBJ/$f.o" ] || [ -n "$(find . ../../include -newer "$OBJ/$f.o" \( -name '*.cu' -o -name '*.cuh' -o -name '*.h' \) | head -1)" ]; then
    ( s=$SECONDS; nvcc $FLAGS ${B2S_NVCC_EXTRA:-} -c -o "$OBJ/$f.o" "$f.cu"; echo "$f.cu: $((SECONDS-s))s" ) &
    pids+=($!)
  fi
done
for p in "${pids[@]:-}"; do [ -n "$p" ] && wait "$p"; done
echo "$FLAGS ${B2S_NVCC_EXTRA:-}" > "$STAMP"
nvcc -shared $ARCH -o "$OUT" "$OBJ"/{api,group,ntt,dntt,msm,msm_acc_g1,msm_acc_g2,r1cs,lcmap,gr1cs,sr1cs,groth16,setup,setup_groth16,serialize,deserialize,verify,verify_rlc,verify_bytes,zkey,testops,poly}.o -lcudart_static -ldl -lrt -lpthread
echo "built $(readlink -f $OUT)"
