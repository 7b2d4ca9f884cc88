// bridging_snvs.cuh -- launchers of the calibrate_bridging_snvs kernels (bridging_snvs.cu), used by capi.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/ugvc_b200.h"

// ugvc_bsn_params as the kernels take it (by value); keys in the order AD, DP, BG_AD, BG_DP
struct BsnDev {
    int m, min_edge;
    double min_qual, min_tvaf, max_nvaf, min_ndepth;
    uint8_t qual[UGVC_BSN_MAX_QUAL_BYTES + 1];
    int qual_len;
    int kind[4], integer[4];
};

// The contig table on the device: names sorted bytewise, name k at names[name_off[k] .. name_off[k+1]), its bytes at
// seq[k] (len[k] of them)
struct BsnContigs {
    const uint8_t* names;
    const int64_t* name_off;
    const uint8_t* const* seq;
    const int64_t* len;
    int n;
};

// The device arrays behind a BsnContigs (the sequences themselves belong to the caller)
struct BsnTable {
    uint8_t* d_names = nullptr;
    int64_t* d_name_off = nullptr;
    const uint8_t** d_seq = nullptr;
    int64_t* d_len = nullptr;
    int n = 0;
    BsnContigs view() const { return BsnContigs{d_names, d_name_off, d_seq, d_len, n}; }
};

// ugvc_bsn_params -> BsnDev; false when a field is out of range
bool bsn_params(const ugvc_bsn_params* p, BsnDev* d);
// (Re)build the table of the given contigs (device sequence pointers); frees what *t held before
cudaError_t bsn_table_build(const std::vector<std::string>& names, const std::vector<const uint8_t*>& seq,
                            const std::vector<int64_t>& len, BsnTable* t);
void bsn_table_free(BsnTable* t);

// Per record of text / line_start (n + 1 entries): flags[i] (UGVC_BSN_RESCUED | UGVC_BSN_NEW_CONTIG), hmer[i] (the
// hmer_size of a walked window, else 0), the length of the written line (len) and INFO/END (end); then afr_launch_scan
// of len into out_ls with agg (2 * (n / AFR_CHUNK + 2) int64 of scratch): totals[0] = the written bytes, totals[1] =
// rescued records.  err: atomicMin of (record << 4 | UGVC_BSN_E_*), all ones when none.
void bsn_launch_decide(const uint8_t* text, const int64_t* line_start, int64_t n, const BsnDev& P, const BsnContigs& C,
                       uint8_t* flags, int32_t* hmer, int64_t* len, int64_t* end, int64_t* out_ls, int64_t* agg,
                       int64_t* totals, unsigned long long* err, int sm_count, cudaStream_t st);
// every line, a rescued one with its QUAL and FILTER columns replaced, at out + out_ls[i]
void bsn_launch_copy(const uint8_t* text, const int64_t* line_start, int64_t n, const BsnDev& P, const uint8_t* flags,
                     const int64_t* out_ls, uint8_t* out, int sm_count, cudaStream_t st);
