#!/bin/bash
# Alternated A/B of the chain kernel launched with programmatic dependent launch (the default
# build) and without it (-DPK_CHAIN_PDL=0), same session, same GPU.  Needs both libraries:
#   build/pdl/libpink_b200.so    the library build() makes (pink_b200/libpink_b200.so)
#   build/nopdl/libpink_b200.so  nvcc <__graft_entry__.NVCC_FLAGS> -DPK_CHAIN_PDL=0 -o ... pink_b200/csrc/pk_cabi.cu
# Usage: scripts/pdl_ab.sh [output directory] [runs per arm]; leaves the PDL library in place.
# The JSON lines, logs and output dumps go to the output directory (default: a new temporary one).
OUT=${1:-$(mktemp -d)}
RUNS=${2:-3}
mkdir -p $OUT
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv,noheader | tee $OUT/gpu.txt
use() { cp build/$1/libpink_b200.so pink_b200/libpink_b200.so; }
run() {
  name=$1; shift
  env $ENVS timeout 900 python bench.py --gpus 1 "$@" > $OUT/$name.json 2> $OUT/$name.err
  python - "$OUT/$name.json" "$name" <<'PY'
import json, sys
try:
    d = json.load(open(sys.argv[1]))
    cfg = " ".join("%.3f" % c["ms_per_step"] for c in d.get("configs", []))
    print(sys.argv[2], "us/step %.2f" % (1e3 * d["ms_per_step"]), "value %.3e" % d["value"],
          "two_streams_us %.2f" % (1e3 * d["roofline"]["two_batches_in_flight_ms_per_step"]),
          "eager_us %.2f" % (1e3 * d["roofline"]["eager_ms_per_step"]), "e2e_us %.1f" % (1e3 * d["e2e"]["ms_per_step"]),
          "e2e_bitwise", d["e2e"]["bitwise_equal_to_device_path"], "status", d["nonzero_status"],
          "sm_mhz", d["clocks"].get("sm_mhz"), "configs_ms", cfg,
          "kkt", [c.get("kkt_selfcheck") for c in d.get("configs", [])], flush=True)
except Exception as e:
    print(sys.argv[2], "ERR", e)
    print(open(sys.argv[1].replace(".json", ".err")).read()[-1500:])
PY
}
for r in $(seq 1 $RUNS); do
  for b in pdl nopdl; do
    use $b
    run ${b}_k2000_r$r --steps 2000 --warmup 20 --no-cpu --dump-outputs $OUT/${b}_k2000_dump
  done
done
for r in $(seq 1 $RUNS); do
  for b in pdl nopdl; do
    use $b
    run ${b}_k20_r$r --steps 20 --warmup 5
  done
done
use pdl
python - $OUT <<'PY'
import numpy as np, sys
o = sys.argv[1]
for n in ("v", "status"):
    a, b = np.load(f"{o}/pdl_k2000_dump/{n}.npy"), np.load(f"{o}/nopdl_k2000_dump/{n}.npy")
    print(n, "bitwise equal (PDL vs no PDL):", a.shape == b.shape and a.tobytes() == b.tobytes())
PY
