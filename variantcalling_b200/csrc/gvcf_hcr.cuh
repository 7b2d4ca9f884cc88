// gvcf_hcr.cuh -- the gvcf_hcr kernels (gvcf_hcr.cu) and the host halves that chain them, used by capi.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ugvc_b200.h"

// Records a reset point's thread walks before the segment it heads takes the parallel form (pointer doubling)
#define HCR_SEG_BOUND 1024

// ugvc_hcr_params as the kernels take it (by value)
struct HcrDev {
    int64_t gq_threshold;
    int gt;        // 1: select GQ >= threshold; 0: GQ absent or < threshold
    int merge;     // 1: one line per merged interval; 0: one per selected record
    int info_end;  // the header declares INFO/END
    int gq_kind;   // UGVC_HCR_GQ_*
    int gq_integer;
};

// ugvc_hcr_params -> HcrDev; false when a field is out of range
bool hcr_params(const ugvc_hcr_params* p, HcrDev* d);

// Device buffers of one piece, kept from the scan to the emit (grown on demand, never shrunk)
struct HcrBufs {
    size_t cap = 0;           // records
    int64_t* start = nullptr;  // [cap] POS - 1
    int64_t* end = nullptr;    // [cap] the interval end (RefCall deletions: start + 1)
    int64_t* pm = nullptr;     // [cap] max end of the earlier records of the contig run in the piece (-1: none)
    int32_t* rs = nullptr;     // [cap] index of the record that starts the contig run
    uint8_t* flags = nullptr;  // [cap] UGVC_HCR_* bits
    int64_t* runs = nullptr;   // [2 * cap] (record, line start) of the records that start a contig run (unordered)
    int32_t* ms_rec = nullptr; // [cap] record that starts output line r
    int64_t* run_end = nullptr;  // [cap] end of output line r
    int64_t* len = nullptr;    // [cap + 1] bytes of output line r
    int64_t* out_ls = nullptr; // [cap + 1]
    int64_t* agg = nullptr;    // [5 * (cap / AFR_CHUNK + 2)]
    int64_t* seg = nullptr;    // [3 * (cap + 2)]: long segments' heads, ends, flat offsets
    int64_t* stat = nullptr;   // [HCR_STAT_N]
    int32_t* jump = nullptr;   // jump tables of the long segments, grown on demand
    int8_t* lvl = nullptr;
    size_t cap_jump = 0, cap_lvl = 0;
    // the piece between the scan and the emit
    const uint8_t* text = nullptr;
    const int64_t* line_start = nullptr;
    int64_t n = 0;
};

enum {
    HCR_STAT_ERR = 0,      // atomicMin of (record << 4 | UGVC_HCR_E_*), all ones when none
    HCR_STAT_N_RUNS = 1,   // contig runs that start in the piece
    HCR_STAT_R0 = 2,       // first record > 0 that starts a contig run (n: none)
    HCR_STAT_FIRST_START = 3,
    HCR_STAT_LAST_START = 4,
    HCR_STAT_N_LONG = 5,   // segments longer than the bound
    HCR_STAT_MAX_SEG = 6,  // longest segment (records from a reset point to the next)
    HCR_STAT_N_LINES = 7,  // output lines
    HCR_STAT_SKIPPED = 8,
    HCR_STAT_LAST_KEPT = 9,
    HCR_STAT_LAST_END = 10,
    HCR_STAT_BYTES = 11,   // output bytes (and 12: scratch of the scan)
    HCR_STAT_N = 14
};

// What the emit hands back to the host
struct HcrEmitOut {
    int64_t n_lines, skipped, last_kept, exit_extent, bytes, longest, err;
};

void hcr_bufs_free(HcrBufs* b);
cudaError_t hcr_bufs_reserve(HcrBufs* b, size_t cap);
// decide + the per-contig prefix max of the piece's n records; leaves b->stat (except the emit's fields) on the device
void hcr_launch_scan(const uint8_t* text, const int64_t* line_start, int64_t n, const HcrDev& P, HcrBufs* b, int sm_count,
                     cudaStream_t st);
// kept flags from the entry state, selection, merge marks, the BED text at out (device) and its stats; synchronizes st.
// seg_bound: records a thread walks before a segment takes the parallel form.
cudaError_t hcr_emit(HcrBufs* b, const HcrDev& P, int continues_contig, int64_t entry_extent, int64_t seg_bound, uint8_t* out,
                     size_t out_capacity, HcrEmitOut* res, int sm_count, cudaStream_t st);
