// fileio.cuh -- launchers of the device-side record writer and BGZF encoder (fileio.cu), used by capi.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ugvc_b200.h"

struct DefTables;
cudaError_t fio_scan_i64(void* tmp, size_t& tmp_bytes, const int64_t* in, int64_t* out, int64_t n, cudaStream_t st);
cudaError_t fio_scan_u64(void* tmp, size_t& tmp_bytes, const uint64_t* in, uint64_t* out, int n, cudaStream_t st);

// What the record writer edits besides FILTER (ugvc_filter_bgzf_edits), all device pointers.  Annotation bit 0 of a
// record is the CG insertion flag (UGVC_FILE_BLACKLIST_CG), bit k + 1 blacklist k.
struct FioEdits {
    int with_model;              // 0: FILTER keeps its pieces, no TREE_SCORE, QUAL untouched
    int flags;                   // UGVC_FILE_*
    const double* phreds;        // [n][n_classes]: GT / GQ / PL of the first sample are rewritten (NULL: they are not)
    int n_classes;
    int n_bl;                    // blacklists, <= UGVC_MAX_BLACKLISTS
    const int64_t* bl_pos;       // sorted POS of each blacklist, concatenated; blacklist k at [bl_pos_off[k], bl_pos_off[k + 1])
    const int64_t* bl_pos_off;
    const uint8_t* bl_name;      // the value text of each blacklist (',' joined pieces, maybe empty) at [bl_name_off[k], ..[k + 1])
    const int32_t* bl_name_off;
    uint32_t* bl_mask;           // [n] scratch: the annotation bits of each record (splice_len -> splice_copy)
    unsigned long long* n_blacklisted;  // += records with at least one annotation bit
    int64_t* out_end;            // [n] INFO/END of each record, 0 where none (ugvc_info_end's rule); NULL: not wanted
};
void fio_launch_splice_len(const uint8_t* text, const int64_t* line_start, const ugvc_recinfo* recinfo, const uint8_t* low,
                           const double* qual, int64_t n, const FioEdits& ed, int64_t* out_len, uint8_t* score_txt,
                           int* fallback, int sm_count, cudaStream_t st);
void fio_launch_splice_copy(const uint8_t* text, const int64_t* line_start, const ugvc_recinfo* recinfo, const uint8_t* low,
                            int64_t n, const FioEdits& ed, const int64_t* out_start, const uint8_t* score_txt, uint8_t* out,
                            int* fallback, int sm_count, cudaStream_t st);
// encoder: FIO_ENC_WARP (fio_deflate_warp, the default) or FIO_ENC_THREAD (fio_deflate, one thread per block)
#define FIO_ENC_WARP 0
#define FIO_ENC_THREAD 1
cudaError_t fio_launch_deflate(const uint8_t* text, size_t n_bytes, const DefTables* tables, uint8_t* blocks, uint32_t* bsize,
                               int n_blocks, int encoder, cudaStream_t st);
void fio_launch_pack(const uint8_t* blocks, const uint32_t* bsize, uint64_t* wide, const uint64_t* boff, int n_blocks,
                     uint8_t* packed, int sm_count, cudaStream_t st);
void fio_launch_widen(const uint32_t* bsize, uint64_t* wide, int n, cudaStream_t st);
void fio_launch_first_records(const int64_t* line_start, int64_t n, const uint64_t* offsets, int m, int64_t* out, cudaStream_t st);
// test hook: the record writer's "%g" (fio_format_g) of n values, 16 bytes each as splice_len writes them
void fio_launch_test_format_g(const float* v, int64_t n, uint8_t* out, int sm_count, cudaStream_t st);
