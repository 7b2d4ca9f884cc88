// tests/host_emu/emu_afr.cpp -- TEST INFRASTRUCTURE.  The filter_low_af_ratio_to_background kernels and their test hook
// (csrc/low_af_ratio.cu) compiled for the host, linked with the objects of the main emulation build (emu_capi.cpp keeps
// refusing the device file path).  Built by low_af_ratio.mk into a library of its own.  Every kernel is a grid-stride
// loop, so one emulated thread runs it whole.
#define UGVC_HOST_EMU 1
#include <cuda_runtime.h>

#include "../../variantcalling_b200/csrc/low_af_ratio.cu"
