// tests/host_emu/emu_hcr.cpp -- TEST INFRASTRUCTURE.  The gvcf_hcr kernels and their test hook (csrc/gvcf_hcr.cu), with
// the scan they share with filter_low_af_ratio_to_background (csrc/low_af_ratio.cu), compiled for the host and linked
// with the objects of the main emulation build (emu_capi.cpp keeps refusing the device file path).  Built by gvcf_hcr.mk
// into a library of its own.  Every kernel is a grid-stride loop, so one emulated thread runs it whole.
#define UGVC_HOST_EMU 1
#include <cuda_runtime.h>

#include "../../variantcalling_b200/csrc/low_af_ratio.cu"
#include "../../variantcalling_b200/csrc/gvcf_hcr.cu"
