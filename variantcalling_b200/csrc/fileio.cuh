// fileio.cuh -- launchers of the device-side record writer and BGZF encoder (fileio.cu), used by capi.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ugvc_b200.h"

struct DefTables;
cudaError_t fio_scan_i64(void* tmp, size_t& tmp_bytes, const int64_t* in, int64_t* out, int64_t n, cudaStream_t st);
cudaError_t fio_scan_u64(void* tmp, size_t& tmp_bytes, const uint64_t* in, uint64_t* out, int n, cudaStream_t st);
void fio_launch_splice_len(const uint8_t* text, const int64_t* line_start, const ugvc_recinfo* recinfo, const uint8_t* low,
                           const double* qual, int64_t n, int flags, int64_t* out_len, uint8_t* score_txt, int* fallback,
                           int sm_count, cudaStream_t st);
void fio_launch_splice_copy(const uint8_t* text, const int64_t* line_start, const ugvc_recinfo* recinfo, const uint8_t* low,
                            int64_t n, int flags, const int64_t* out_start, const uint8_t* score_txt, uint8_t* out,
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
