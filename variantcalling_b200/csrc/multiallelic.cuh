// multiallelic.cuh -- the --treat_multiallelics stages of multiallelic.cu on device pointers and a caller's stream, for the
// device file path of capi.cu (ugvc_filter_bgzf_split).  The public entries ugvc_ma_build / ugvc_ma_merge copy their host
// inputs to the handle's buffers and call the same functions.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ugvc_b200.h"

// ugvc_ma_build on device text / line starts / recinfo of one contig (the reference sequence is host memory and is
// uploaded on `st`).  Synchronises `st`; same return codes and out[8] as ugvc_ma_build.
int ma_build_on(ugvc_ma* h, const uint8_t* d_text, size_t n_bytes, const int64_t* d_line_start, const ugvc_recinfo* d_recinfo,
                int64_t n_records, const uint8_t* ref_seq, size_t ref_len, cudaStream_t st, int64_t out[8]);
// The text of the scored pass the last build wrote on the device (out[4] + out[5] bytes; 64 writable bytes follow it).
uint8_t* ma_scored_text(ugvc_ma* h);
// ugvc_ma_merge on device likelihoods: the N x width matrix stays on the device (*d_mat).  Synchronises `st`; UGVC_E_DATA
// when a 2-class model meets a two-row group.
int ma_merge_on(ugvc_ma* h, const double* d_lik, int64_t n_rows, int n_classes, int width, cudaStream_t st, double** d_mat);
// ma_score: phreds / qual / low of multiallelics.score_math over n rows of `width` likelihoods.  `phreds` may be NULL, or
// `lik` itself (each thread overwrites its row in place).
void ma_launch_score(const double* lik, int64_t n, int width, double threshold, double* phreds, double* qual, uint8_t* low,
                     int sm_count, cudaStream_t st);
int ma_device_of(const ugvc_ma* h);
