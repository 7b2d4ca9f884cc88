// concordance.cuh -- the ugvc_conc handle, shared by its lifecycle (conc_handle.cu), the metrics pipeline
// (concordance.cu, CUB) and the frame annotation (conc_annotate.cu, CUB-free).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/ugvc_b200.h"

#define CONC_GROUPS UGVC_CONC_GROUPS      // 7 default groups + INDELS + H-INDELS
#define CONC_COUNTERS UGVC_CONC_COUNTERS  // tp, fp, missed (call < truth), initial_tp, n_called, n_fn, n_nan, n_inf
#define CONC_TPB 256

struct ugvc_conc {
    int device = 0;
    int sm_count = 132;  // replaced by the device's count when the handle opens
    cudaStream_t st = nullptr;
    std::string err;
    long long launches = 0;
    double* curve[CONC_GROUPS][3] = {};  // precision, recall, threshold
    int64_t curve_len[CONC_GROUPS] = {};
    // reference contigs uploaded for ugvc_conc_annotate (raw FASTA bytes, case kept), by contig id
    std::vector<uint8_t*> annot_seq;
    std::vector<int64_t> annot_len;
    // lowest failing record of the last ugvc_conc_annotate call and its UGVC_ANNOT_E_* reason (0 = none)
    int64_t annot_err_row = -1;
    int annot_err_reason = 0;
    float annot_kernel_ms = 0.f;  // CUDA-event time of the last ca_annotate launch
};

int conc_fail(ugvc_conc* h, int code, const std::string& msg);
void conc_drop_curves(ugvc_conc* h);
void conc_drop_contigs(ugvc_conc* h);

#define CCU(call)                                                                                   \
    do {                                                                                            \
        cudaError_t e_ = (call);                                                                    \
        if (e_ != cudaSuccess)                                                                      \
            return conc_fail(h, UGVC_E_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
    } while (0)
