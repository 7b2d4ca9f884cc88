// tests/host_emu/emu_capi.cpp -- TEST INFRASTRUCTURE.  The product's C ABI (csrc/capi.cu) compiled for
// the host over the emulated runtime, and refusing stubs for the entry points whose kernels are not
// emulated (device synthetic generator, concordance: both are CUB pipelines).
#define UGVC_HOST_EMU 1
#include <cuda_runtime.h>

#include "../../variantcalling_b200/csrc/capi.cu"

static const char* NOT_EMULATED = "not available in the host emulation (tests/host_emu)";
extern "C" int ugvc_synth_device(ugvc_ctx* ctx, uint64_t, int64_t, int64_t, int64_t, int, uint8_t*, size_t, size_t*, void*) {
    return fail(ctx, UGVC_E_CUDA, NOT_EMULATED);
}
extern "C" int64_t ugvc_synth_header(int, char*, size_t) { return UGVC_E_CUDA; }
struct ugvc_conc;
extern "C" int ugvc_conc_create(int, ugvc_conc**) { return UGVC_E_CUDA; }
extern "C" void ugvc_conc_free(ugvc_conc*) {}
extern "C" const char* ugvc_conc_last_error(const ugvc_conc*) { return NOT_EMULATED; }
extern "C" long long ugvc_conc_launch_count(const ugvc_conc*) { return 0; }
// ugvc_conc_run writes UGVC_CONC_GROUPS x UGVC_CONC_COUNTERS (9 x 8) counters on the device; refused here
extern "C" int ugvc_conc_run(ugvc_conc*, int64_t, const double*, const uint8_t*, const uint8_t*, const uint8_t*, const int32_t*,
                             const int8_t*, int, int, int64_t*, int64_t*, double*, int64_t*) { return UGVC_E_CUDA; }
extern "C" int ugvc_conc_classify(ugvc_conc*, int64_t, const int8_t*, const int8_t*, const uint8_t*, uint8_t*, uint8_t*) { return UGVC_E_CUDA; }
extern "C" int ugvc_conc_curve(ugvc_conc*, int, double*, double*, double*, size_t) { return UGVC_E_CUDA; }
