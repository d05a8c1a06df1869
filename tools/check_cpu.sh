#!/usr/bin/env bash
# Everything that can be checked without a GPU, in the order the round-end driver does it:
#   1. build(): nvcc cross-compiles libb200gp.so for sm_90a, gcc builds the C oracle (+ oracle/_ref when the reference is here)
#   2. the CPU test suite (oracle vs reference goldens, host layer over the mock C-ABI, device source compiled for the host,
#      C-ABI symbols, gloo world_size 2)
#   3. the GPU test files' host-side Python over the mock C-ABI (catches host-level errors in `-m gpu` tests before a GPU call;
#      failures that say "is not mocked" or time out are limits of the mock, not findings)
set -u
cd "$(dirname "$0")/.."
python -c "import __graft_entry__ as g; g.build()" || exit 1
python -m pytest tests/ -x -q -m "not gpu" -n "${JOBS:-8}" || exit 1
if [ "${1:-}" = "--gpu-files-on-mock" ]; then
    cd tests
    python - "$@" <<'PY'
import sys
sys.path.insert(0, ".."); sys.path.insert(0, ".")
from ctypes import c_void_p
import pytest
import hostmock
from tinygp_b200 import _cabi
ctx = _cabi.Context.__new__(_cabi.Context)
ctx.lib, ctx.handle, ctx.device = hostmock.MockLib(), c_void_p(1), -1
ctx.reset_options = lambda: None
_cabi.set_context(ctx)
files = ["test_zx_reference_tests_gpu.py", "test_zy_reference_golden_gpu.py", "test_zzx_wide_state_gpu.py",
         "test_zzy_quasisep_reference_gpu.py", "test_zzzzz_late_additions_gpu.py"]
sys.exit(pytest.main(["-m", "gpu", "-q", "--no-header", "-p", "no:cacheprovider", "--timeout", "60"] + files))
PY
fi
