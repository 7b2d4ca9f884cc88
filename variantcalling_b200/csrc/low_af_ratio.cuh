// low_af_ratio.cuh -- launchers of the filter_low_af_ratio_to_background kernels (low_af_ratio.cu), used by capi.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ugvc_b200.h"

// ugvc_afr_params as the kernels take it (by value)
struct AfrDev {
    double thr, thr_h, vthr_h;
    uint8_t nf[UGVC_AFR_MAX_FILTER_BYTES];
    int nf_len;
    int vt_kind, vaf_kind, bg_kind, vaf_int, bg_int;
};

// ugvc_afr_params -> AfrDev; false when a field is out of range
bool afr_params(const ugvc_afr_params* p, AfrDev* d);

// Per record of text / line_start (n + 1 entries): the decision (flags[i]: bit 0 failed, bit 1 FILTER rewritten), the
// length of the written line (len, n + 1 entries: the last one is set to 0), INFO/END (end, may be NULL); then the
// exclusive scan of len into out_ls (n + 1 entries) with agg (2 * (n / AFR_CHUNK + 2) int64 of scratch); totals[0] = the
// written bytes, totals[1] = failed records.  err: atomicMin of (record << 4 | UGVC_AFR_E_*), all ones when none.
void afr_launch_decide(const uint8_t* text, const int64_t* line_start, int64_t n, const AfrDev& P, uint8_t* flags,
                       int64_t* len, int64_t* end, int64_t* out_ls, int64_t* agg, int64_t* totals,
                       unsigned long long* err, int sm_count, cudaStream_t st);
// The scan step of afr_launch_decide alone, also used by the calibrate_bridging_snvs kernels (bridging_snvs.cu): the
// exclusive scan of len (n entries) into out_ls, totals[0] = the summed bytes, totals[1] = records with flags bit 0 set.
void afr_launch_scan(const int64_t* len, const uint8_t* flags, int64_t n, int64_t* out_ls, int64_t* agg, int64_t* totals,
                     int sm_count, cudaStream_t st);
// every line with its new FILTER column, at out + out_ls[i]
void afr_launch_copy(const uint8_t* text, const int64_t* line_start, int64_t n, const AfrDev& P, const uint8_t* flags,
                     const int64_t* out_ls, uint8_t* out, int sm_count, cudaStream_t st);
#define AFR_CHUNK 1024
#define AFR_NO_ERROR 0xFFFFFFFFFFFFFFFFull
