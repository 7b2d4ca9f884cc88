// tests/host_emu/emu_kernels.cpp -- TEST INFRASTRUCTURE.  The K1 (field parse), K2 (feature assembly)
// and K3 (inference) kernel bodies of variantcalling_b200/csrc/kernels.cu, compiled unchanged for the
// host through shim_include/cuda_runtime.h with one emulated thread per CTA, plus host launchers
// with the product's launch_* signatures (K3's is in kernels.cu, next to the device launcher).
// K0 (a cooperative 256-thread tile scan with inline PTX) is not emulated: lines are indexed by a
// plain loop that reproduces its outputs and error codes.
// The emulated library lets `pytest -m "not gpu"` run the parity tests against the very kernel
// source the GPU executes; it is built under tests/ only and the package never loads it.
#define UGVC_HOST_EMU 1
#define K1_TPB 1
#define K2_TPB 1
#include <cuda_runtime.h>

thread_local dim3 threadIdx, blockIdx, blockDim, gridDim;
alignas(16) uint8_t k1_smem[64 * 1024];
alignas(16) uint8_t smem3[8 * 1024 * 1024];  // K3: feature tile + the whole forest
alignas(16) uint8_t kt_smem_emu[128 * 1024];  // K1 tile kernel

#include "../../variantcalling_b200/csrc/kernels.cu"

static_assert(K1_SMEM_BYTES <= sizeof(k1_smem), "k1_smem too small");
static_assert(KT_SMEM_BYTES <= sizeof(kt_smem_emu), "kt_smem_emu too small");

static void one_thread_grid() {
    threadIdx = dim3(0, 0, 0);
    blockIdx = dim3(0, 0, 0);
    blockDim = dim3(1, 1, 1);
    gridDim = dim3(1, 1, 1);
}

void launch_k0(const uint8_t* d_text, size_t n_bytes, uint32_t*, int64_t* line_start, size_t cap_records,
               int64_t* d_n_records, unsigned long long* d_err, int, cudaStream_t) {
    // K0's contract: line_start[i] for every record, line_start[n] = n_bytes, *d_n_records = n; a batch that
    // does not end with '\n' is malformed, more lines than cap_records is REASON_TOO_MANY_ELEMS
    int64_t n = 0;
    line_start[0] = 0;
    for (size_t i = 0; i < n_bytes; ++i)
        if (d_text[i] == '\n') {
            ++n;
            if ((size_t)n <= cap_records) line_start[n] = (int64_t)i + 1;
        }
    if (n_bytes && d_text[n_bytes - 1] != '\n') atomicMin(d_err, ugvc_pack_error(n, 0xFFFF, REASON_MALFORMED_LINE));
    if ((size_t)n > cap_records) {
        atomicMin(d_err, ugvc_pack_error((long long)cap_records, 0xFFFF, REASON_TOO_MANY_ELEMS));
        n = (int64_t)cap_records;
    }
    *d_n_records = n;
}

void launch_k1(const DevPlan& plan, const DevSchedule& sched, const uint8_t* d_text, const int64_t* line_start,
               const int64_t* d_n_records, uint32_t* raw, size_t row_stride, ugvc_recinfo* recinfo,
               unsigned long long* d_err, long long* d_counts, int, cudaStream_t) {
    one_thread_grid();
    if (plan.h.n_slots) {
        gridDim = dim3(1, 1, 1);
        k1_fill(raw, row_stride, (int)plan.h.n_slots, d_n_records);
    }
    one_thread_grid();
#ifdef UGVC_K1_SPLIT
    k1_parse_info(plan, sched, d_text, line_start, d_n_records, raw, row_stride, recinfo, d_err, d_counts, nullptr, nullptr);
    one_thread_grid();
    k1_parse_frame(plan, sched, d_text, line_start, d_n_records, raw, row_stride, recinfo, d_err, d_counts, nullptr, nullptr);
#else
    k1_parse(plan, sched, d_text, line_start, d_n_records, raw, row_stride, recinfo, d_err, d_counts, nullptr, nullptr);
#endif
}

// both K1 tiers: the tile kernel emulates all 512 threads of its CTA phase by phase (KT_FOR_THREADS), then the generic
// parser takes the slow list.  UGVC_EMU_WCAP=<n> caps the records per window (several windows per tile).
void launch_k1_fast(const DevPlan& plan, const DevFast& fast, const DevSchedule& sched, const uint8_t* d_text, size_t n_bytes,
                    uint32_t* scratch, int64_t* line_start, size_t cap_records, int64_t* d_n_records, uint32_t* raw,
                    size_t row_stride, ugvc_recinfo* recinfo, uint32_t* slow_list, unsigned long long* d_err,
                    long long* d_counts, int, cudaStream_t) {
    const size_t n_tiles = (n_bytes + KT_TILE - 1) / KT_TILE;
    memset(scratch, 0, 8 + n_tiles * sizeof(unsigned long long));
    if (n_tiles == 0) {
        *d_n_records = 0;
        line_start[0] = 0;
        return;
    }
    one_thread_grid();
    uint32_t wcap = kt_window_records(plan.h.n_slots);
    if (const char* w = getenv("UGVC_EMU_WCAP")) wcap = (uint32_t)atoi(w) < wcap ? (uint32_t)atoi(w) : wcap;
    k1_tok(plan, fast, d_text, n_bytes, reinterpret_cast<unsigned long long*>(scratch) + 1, scratch, scratch + 1, n_tiles,
           line_start, cap_records, d_n_records, raw, row_stride, recinfo, slow_list, d_err, d_counts, wcap);
    one_thread_grid();
    k1_parse(plan, sched, d_text, line_start, d_n_records, raw, row_stride, recinfo, d_err, d_counts, slow_list, scratch + 1);
}

void launch_k2(const DevPlan& plan, const uint32_t* raw, size_t row_stride, const int64_t* d_n_records, float* feats,
               unsigned long long* d_err, int, cudaStream_t) {
    one_thread_grid();
    k2_features(plan, raw, row_stride, d_n_records, feats, d_err);
}

cudaError_t kernels_configure(const DevPlan&) { return cudaSuccess; }
