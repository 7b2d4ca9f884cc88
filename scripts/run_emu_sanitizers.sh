#!/bin/bash
# The kernel sources on the host emulation under AddressSanitizer + UndefinedBehaviorSanitizer (no GPU needed):
# the emulated GPU suite and a fuzz campaign through both K1 tiers.   bash scripts/run_emu_sanitizers.sh [first_seed last_seed]
set -eu
cd "$(dirname "$0")/.."
make -C tests/host_emu SAN=1 > /dev/null
export LD_PRELOAD="$(gcc -print-file-name=libasan.so):$(gcc -print-file-name=libubsan.so)"
export ASAN_OPTIONS=detect_leaks=0:halt_on_error=1
export UGVC_LIB_PATH="$PWD/tests/host_emu/_build_san/libugvc_emu.so"
python -m pytest -q -m gpu -p no:cacheprovider tests/test_gpu_parity.py tests/test_gpu_edges.py tests/test_gpu_fuzz.py \
    tests/test_gpu_cnv.py tests/test_gpu_cli.py tests/test_gpu_multiallelics.py tests/test_gpu_x_model_apply.py \
    tests/test_gpu_x_deepvariant.py tests/test_gpu_x_bgzf.py tests/test_gpu_x_inflate_edges.py tests/test_gpu_y_tiletok.py tests/test_gpu_y_deviations.py \
    tests/test_gpu_feature_edges.py \
    tests/test_gpu_z_multiallelic_device.py \
    --deselect tests/test_gpu_edges.py::test_device_generator_text_parity \
    --deselect tests/test_gpu_parity.py::test_full_size_properties_batching_invariance 2>&1 | tee /tmp/emu_san_tests.log | tail -2
UGVC_EMU_LIB="$UGVC_LIB_PATH" python scripts/fuzz_host_emu.py "${1:-900}" "${2:-905}" 2>&1 | tee /tmp/emu_san_fuzz.log | tail -2
if grep -q "runtime error\|AddressSanitizer" /tmp/emu_san_tests.log /tmp/emu_san_fuzz.log; then echo "SANITIZER REPORTS"; exit 1; fi
echo "no sanitizer report"
