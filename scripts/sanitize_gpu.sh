#!/bin/bash
# compute-sanitizer over single-GPU cases, bounded by small shapes and per-case timeouts:
#   memcheck  : GEMM library cases + whole federated rounds (bf16 / fp8, SGD / Adam)
#   racecheck : shared-memory hazards of the persistent trainer, validation chain, consensus kernel
#   initcheck : reads of uninitialised device memory (symmetric heap regions, scale chunks)
# Usage (on the GPU box):  bash scripts/sanitize_gpu.sh [out_dir]
OUT=${1:-sanitize_out}
mkdir -p "$OUT"
export BFLC_NO_AUTOBUILD=1 PYTHONPATH=$PWD:$PYTHONPATH
L=$OUT/summary.log; : > "$L"
run() {  # tool, name, command...
  local tool=$1 name=$2; shift 2
  echo "=== $tool $name" >> "$L"
  timeout "${SAN_TIMEOUT:-200}" compute-sanitizer --tool "$tool" --error-exitcode 9 "$@" > "$OUT/$tool.$name.log" 2>&1
  echo "exit=$?" >> "$L"
  grep -E "RESULT|ERROR SUMMARY|RACECHECK SUMMARY|hazard|Invalid|Uninitialized" "$OUT/$tool.$name.log" | cut -c1-300 | head -8 >> "$L"
}
for c in kk_300_200_784 epi xent; do run memcheck "gemm_$c" python scripts/gemm_case.py $c; done
for c in fp8_adam bf16_sgd; do run memcheck "round_$c" python scripts/sanitize_cases.py $c; done
for c in fp8_adam bf16_sgd; do run racecheck "round_$c" python scripts/sanitize_cases.py $c; done
run initcheck round_fp8_adam python scripts/sanitize_cases.py fp8_adam
for c in conv attn attn_varlen attn_packed attn_dropout; do run memcheck "$c" python scripts/sanitize_cases.py $c; done
for c in attn attn_varlen attn_packed attn_dropout; do run racecheck "$c" python scripts/sanitize_cases.py $c; done
tail -c 4000 "$L"
