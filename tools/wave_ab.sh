#!/bin/bash
# Alternating A/B of the flagship bench between a baseline build of the library and the current one, in one session on
# one GPU.  The baseline is built beforehand (from a git checkout; the copy that runs the A/B need not be one):
#   bash tools/wave_ab.sh base [REV]     # REV (default HEAD^) -> better_fastlio2_b200/libfastlio_b200_base.so (git-ignored)
#   bash tools/wave_ab.sh [RUNS]         # RUNS (default 3) runs per build, base and new alternating
# Each run is `bench.py --steps 400 --warmup 10 --no-cpu-baseline`; one line per run gives value (scans/s), e2e (scans/s)
# and kernel_ms_per_step.  Raw JSON lines go to $OUT (default: a temporary directory).
set -e
cd "$(dirname "$0")/.."
LIB=better_fastlio2_b200
BASE=$LIB/libfastlio_b200_base.so
NEW=$LIB/libfastlio_b200.so
if [ "$1" = base ]; then
  REV=${2:-HEAD^}
  TMP=$(mktemp -d)
  git archive "$REV" better_fastlio2_b200/csrc include | tar -x -C "$TMP"
  /usr/local/cuda/bin/nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -fmad=false -Xcompiler -fPIC -shared \
    -ccbin /usr/bin/g++ -o "$BASE" "$TMP/better_fastlio2_b200/csrc/fastlio_b200.cu"
  rm -rf "$TMP"
  echo "built $BASE from $(git rev-parse --short "$REV")"
  exit 0
fi
RUNS=${1:-3}
[ -f "$BASE" ] || { echo "no $BASE: run 'bash tools/wave_ab.sh base' first" >&2; exit 1; }
[ -f "$NEW" ] || { echo "no $NEW: run build() first" >&2; exit 1; }
OUT=${OUT:-$(mktemp -d)}
mkdir -p "$OUT"
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv,noheader
for r in $(seq 1 "$RUNS"); do
  for tag in base new; do
    lib=$BASE; [ $tag = new ] && lib=$NEW
    FLB_LIB=$lib python bench.py --gpus 1 --steps 400 --warmup 10 --no-cpu-baseline > "$OUT/wave_ab_${tag}_$r.json" 2> "$OUT/wave_ab_${tag}_$r.err"
    python - "$OUT/wave_ab_${tag}_$r.json" "$tag" "$r" <<'EOF'
import json, sys
d = json.loads(open(sys.argv[1]).read().strip().splitlines()[-1])
k = " ".join(f"{n}={v:.4f}" for n, v in d["kernel_ms_per_step"].items())
print(f"{sys.argv[2]:<5} run {sys.argv[3]}: value={d['value']:.1f} e2e={d['e2e']['value']:.1f} kernel_ms_per_step: {k}")
EOF
  done
done
