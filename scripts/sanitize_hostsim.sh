#!/bin/bash
# AddressSanitizer + UBSan pass over the kernel bodies: the host build of pink_b200/csrc
# (tests/hostsim, test harness only) compiled with -fsanitize=address,undefined and driven
# by the hostsim / host-API suites.  Prints the number of sanitizer reports (expected: 0).
set -u
cd "$(dirname "$0")/.."
export LD_PRELOAD="$(g++ -print-file-name=libasan.so):$(g++ -print-file-name=libubsan.so)"
export ASAN_OPTIONS=detect_leaks=0:halt_on_error=0 UBSAN_OPTIONS=print_stacktrace=1
export PK_HOSTSIM_SANITIZE=1
LOG=${1:-/tmp/pk_sanitize.log}
python -m pytest tests/test_hostsim_dualqp.py tests/test_hostsim_coop.py tests/test_hostsim_kernel_paths.py tests/test_hostsim_parity.py tests/test_hostsim_extras.py tests/test_hostsim_degenerate_inputs.py tests/test_hostsim_converge.py tests/test_hostsim_multistart.py tests/test_hostsim_rollout.py tests/test_hostsim_instance_glue.py \
  tests/test_api_host.py tests/test_api_extras_host.py tests/test_reference_scenarios_host.py \
  tests/test_reference_task_semantics_host.py tests/test_reference_limit_barrier_semantics_host.py \
  -q -s -m "not gpu" > "$LOG" 2>&1
tail -2 "$LOG"
echo "sanitizer reports: $(grep -c 'runtime error\|ERROR: AddressSanitizer' "$LOG")"
rm -f tests/hostsim/libpk_hostsim_asan.so
