// tests/host_emu/emu_conc.cpp -- TEST INFRASTRUCTURE.  The host emulation of the product's C ABI (emu_capi.cpp) with
// the real ugvc_conc handle (csrc/conc_handle.cu) and the concordance-frame annotation kernel and its C ABI
// (csrc/conc_annotate.cu) in place of the refusing handle stubs; the metrics entry points of the handle stay refused
// (CUB pipelines).  Built by conc_annotate.mk into a library of its own.  ca_annotate is a grid-stride loop, so one
// emulated thread runs it whole.
#define UGVC_HOST_EMU 1
#include <cuda_runtime.h>

// the handle reads the SM count with cudaDeviceGetAttribute, which the shared shim does not provide
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount = 16 };
static inline cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr, int) {
    *v = 1;
    return cudaSuccess;
}

// emu_capi.cpp's refusing handle stubs are renamed out of the way of the real handle below
#define ugvc_conc_create emu_refused_conc_create
#define ugvc_conc_free emu_refused_conc_free
#define ugvc_conc_last_error emu_refused_conc_last_error
#define ugvc_conc_launch_count emu_refused_conc_launch_count
#include "emu_capi.cpp"
#undef ugvc_conc_create
#undef ugvc_conc_free
#undef ugvc_conc_last_error
#undef ugvc_conc_launch_count

#include "../../variantcalling_b200/csrc/conc_handle.cu"
#include "../../variantcalling_b200/csrc/conc_annotate.cu"
