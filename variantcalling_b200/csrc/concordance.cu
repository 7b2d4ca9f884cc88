// concordance.cu -- precision / recall of a filtered call set against truth labels on the GPU
// (BASELINE.json configs[4]; SURVEY.md section 8 row f3).
//
// Replaces the array work of ugbio_core/concordance/concordance_utils.py:
//   calc_accuracy_metrics :11-106 / calc_recall_precision_curve :109-188  (per-group selection)
//   get_concordance_metrics :346-458                                     (tp / fp / fn counts)
//   stats_utils.precision_recall_curve :141-210 -> sklearn.metrics.precision_recall_curve
//                                                  (sort by score, cumulative counts per distinct score)
// The host mirror (variantcalling_b200/concordance.py) keeps the reference's function signatures and
// does the O(#groups) arithmetic; everything that touches N records runs here:
//   C1 conc_classify   one pass over the records: group membership, truth / call bits, and the
//                      9 x 6 counters (block-local shared-memory atomics, one global atomic per counter
//                      per block).  HBM-bound: 15 B read + 3 B written per record.
//   per group g with a curve:
//   C2 conc_flags      membership & not-false-negative flag
//      cub::DeviceSelect::Flagged          scores / truth of the group, compacted
//      cub::DeviceRadixSort::SortPairsDescending   (score fp64 key, truth byte)
//      cub::DeviceScan::InclusiveSum       cumulative true positives
//   C3 conc_boundary   last element of every run of equal scores (np.diff(score) != 0)
//      cub::DeviceSelect::Flagged          their indices
//   C4 conc_curve      precision = tps / (tps + fps), recall = tps / tps[-1] in fp64 (IEEE division, the
//                      same bits as NumPy), written in increasing-threshold order like sklearn returns them
#include <cub/cub.cuh>

#include <algorithm>

#include "concordance.cuh"

// meta bits: 0-3 default group + 1 (0 = none), 4 truth, 5 false negative, 6 call, 7 indel, 8 hmer > 0
__device__ __forceinline__ bool conc_member(unsigned meta, int g) {
    if (g < 7) return (meta & 0xFu) == (unsigned)(g + 1);
    return g == 7 ? ((meta >> 7) & 1u) : ((meta >> 8) & 1u);
}

__global__ void __launch_bounds__(CONC_TPB) conc_classify(int64_t n, const uint8_t* __restrict__ pred,
                                                           const uint8_t* __restrict__ cls,
                                                           const uint8_t* __restrict__ indel,
                                                           const int32_t* __restrict__ hmer,
                                                           const int8_t* __restrict__ group, uint16_t* __restrict__ meta,
                                                           uint8_t* __restrict__ truth8,
                                                           unsigned long long* __restrict__ counts) {
    __shared__ unsigned int s_cnt[CONC_GROUPS * CONC_COUNTERS];
    for (int i = threadIdx.x; i < CONC_GROUPS * CONC_COUNTERS; i += CONC_TPB) s_cnt[i] = 0u;
    __syncthreads();
    const int64_t stride = (int64_t)gridDim.x * CONC_TPB;
    for (int64_t i = (int64_t)blockIdx.x * CONC_TPB + threadIdx.x; i < n; i += stride) {
        const bool ind = indel[i] != 0;
        const int h = hmer[i];
        int gid;
        if (group) {
            gid = group[i];
        } else if (!ind) {
            gid = 0;
        } else if (h == 0) {
            gid = 1;
        } else if (h < 0) {
            gid = -1;
        } else {
            gid = h <= 4 ? 2 : h <= 7 ? 3 : h <= 10 ? 4 : h <= 12 ? 5 : 6;
        }
        const unsigned c = cls[i];  // 0 fp, 1 tp, 2 fn, 3 tn
        const bool truth = c == 1u || c == 2u, fnm = c == 2u, call = pred[i] != 0;
        const unsigned m = (unsigned)(gid + 1) | (truth ? 16u : 0u) | (fnm ? 32u : 0u) | (call ? 64u : 0u) |
                           (ind ? 128u : 0u) | (h > 0 ? 256u : 0u);
        meta[i] = (uint16_t)m;
        truth8[i] = truth ? 1 : 0;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int g = k == 0 ? gid : (k == 1 ? (ind ? 7 : -1) : (h > 0 ? 8 : -1));
            if (g < 0) continue;
            unsigned int* cg = s_cnt + g * CONC_COUNTERS;
            if (fnm) {
                atomicAdd(cg + 5, 1u);
            } else {
                atomicAdd(cg + 4, 1u);
                if (truth) atomicAdd(cg + 3, 1u);
                if (truth && call) atomicAdd(cg + 0, 1u);
                if (call && !truth) atomicAdd(cg + 1, 1u);
                if (!call && truth) atomicAdd(cg + 2, 1u);
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < CONC_GROUPS * CONC_COUNTERS; i += CONC_TPB)
        if (s_cnt[i]) atomicAdd(counts + i, (unsigned long long)s_cnt[i]);
}

__global__ void __launch_bounds__(CONC_TPB) conc_flags(int64_t n, const uint16_t* __restrict__ meta, int g,
                                                        uint8_t* __restrict__ flags) {
    const int64_t stride = (int64_t)gridDim.x * CONC_TPB;
    for (int64_t i = (int64_t)blockIdx.x * CONC_TPB + threadIdx.x; i < n; i += stride) {
        const unsigned m = meta[i];
        flags[i] = (conc_member(m, g) && !((m >> 5) & 1u)) ? 1 : 0;
    }
}

__global__ void __launch_bounds__(CONC_TPB) conc_boundary(int64_t n, const double* __restrict__ s,
                                                           uint8_t* __restrict__ flags) {
    const int64_t stride = (int64_t)gridDim.x * CONC_TPB;
    for (int64_t i = (int64_t)blockIdx.x * CONC_TPB + threadIdx.x; i < n; i += stride)
        flags[i] = (i == n - 1 || s[i] != s[i + 1]) ? 1 : 0;
}

__global__ void __launch_bounds__(CONC_TPB) conc_curve(int64_t d, int64_t n_sel, const int64_t* __restrict__ idx,
                                                        const double* __restrict__ s, const int64_t* __restrict__ cum,
                                                        double* __restrict__ out_p, double* __restrict__ out_r,
                                                        double* __restrict__ out_t) {
    const double total = (double)cum[n_sel - 1];
    const int64_t stride = (int64_t)gridDim.x * CONC_TPB;
    for (int64_t k = (int64_t)blockIdx.x * CONC_TPB + threadIdx.x; k < d; k += stride) {
        const int64_t at = idx[k];
        const double tps = (double)cum[at];
        const double fps = (double)(1 + at) - tps;
        const double ps = tps + fps;
        const int64_t o = d - 1 - k;
        out_p[o] = ps != 0.0 ? __ddiv_rn(tps, ps) : 0.0;
        out_r[o] = total == 0.0 ? 1.0 : __ddiv_rn(tps, total);
        out_t[o] = s[at];
    }
}

struct U8ToI64 {
    __host__ __device__ __forceinline__ int64_t operator()(const uint8_t& v) const { return (int64_t)v; }
};

namespace {
struct DevBuf {  // frees on scope exit
    std::vector<void*> ptrs;
    ~DevBuf() {
        for (void* p : ptrs) cudaFree(p);
    }
    template <class T>
    cudaError_t get(T** p, size_t count) {
        cudaError_t e = cudaMalloc(reinterpret_cast<void**>(p), (count ? count : 1) * sizeof(T));
        if (e == cudaSuccess) ptrs.push_back(*p);
        return e;
    }
};
template <class T>
cudaError_t upload(DevBuf& b, const T* src, int64_t n, bool on_device, const T** dst, cudaStream_t st) {
    if (on_device || !src) {
        *dst = src;
        return cudaSuccess;
    }
    T* d = nullptr;
    cudaError_t e = b.get(&d, (size_t)n);
    if (e != cudaSuccess) return e;
    *dst = d;
    return cudaMemcpyAsync(d, src, (size_t)n * sizeof(T), cudaMemcpyHostToDevice, st);
}
}  // namespace

extern "C" int ugvc_conc_run(ugvc_conc* h, int64_t n, const double* scores, const uint8_t* pred, const uint8_t* cls,
                             const uint8_t* indel, const int32_t* hmer_len, const int8_t* group, int inputs_on_device,
                             int want_curves, int64_t* out_counts, int64_t* out_curve_len, double* out_cutoff,
                             int64_t* out_selected) {
    if (!h) return UGVC_E_ARG;
    if (n < 0 || !out_counts) return conc_fail(h, UGVC_E_ARG, "conc_run: bad arguments");
    if (n > 0 && (!scores || !pred || !cls || !indel || !hmer_len))
        return conc_fail(h, UGVC_E_ARG, "conc_run: NULL input column");
    CCU(cudaSetDevice(h->device));
    conc_drop_curves(h);
    for (int i = 0; i < CONC_GROUPS * CONC_COUNTERS; ++i) out_counts[i] = 0;
    for (int g = 0; g < CONC_GROUPS; ++g) {
        if (out_curve_len) out_curve_len[g] = 0;
        if (out_cutoff) out_cutoff[g] = 0.0;
        if (out_selected) out_selected[2 * g] = out_selected[2 * g + 1] = 0;
    }
    if (n == 0) return UGVC_OK;
    if (n > 0x7FFFFFF0ll) return conc_fail(h, UGVC_E_ARG, "conc_run: more than 2^31 records per call are not supported");
    cudaStream_t st = h->st;
    const bool dev = inputs_on_device != 0;
    DevBuf buf;
    const double* d_scores;
    const uint8_t *d_pred, *d_cls, *d_indel;
    const int32_t* d_hmer;
    const int8_t* d_group;
    CCU(upload(buf, scores, n, dev, &d_scores, st));
    CCU(upload(buf, pred, n, dev, &d_pred, st));
    CCU(upload(buf, cls, n, dev, &d_cls, st));
    CCU(upload(buf, indel, n, dev, &d_indel, st));
    CCU(upload(buf, hmer_len, n, dev, &d_hmer, st));
    CCU(upload(buf, group, n, dev, &d_group, st));
    uint16_t* d_meta;
    uint8_t *d_truth, *d_flags;
    unsigned long long* d_counts;
    CCU(buf.get(&d_meta, (size_t)n));
    CCU(buf.get(&d_truth, (size_t)n));
    CCU(buf.get(&d_flags, (size_t)n));
    CCU(buf.get(&d_counts, (size_t)CONC_GROUPS * CONC_COUNTERS));
    CCU(cudaMemsetAsync(d_counts, 0, sizeof(unsigned long long) * CONC_GROUPS * CONC_COUNTERS, st));
    const int grid = h->sm_count * 8;
    conc_classify<<<grid, CONC_TPB, 0, st>>>(n, d_pred, d_cls, d_indel, d_hmer, d_group, d_meta, d_truth, d_counts);
    ++h->launches;
    CCU(cudaGetLastError());
    unsigned long long h_counts[CONC_GROUPS * CONC_COUNTERS];
    CCU(cudaMemcpyAsync(h_counts, d_counts, sizeof(h_counts), cudaMemcpyDeviceToHost, st));
    CCU(cudaStreamSynchronize(st));
    for (int i = 0; i < CONC_GROUPS * CONC_COUNTERS; ++i) out_counts[i] = (int64_t)h_counts[i];
    if (!want_curves) return UGVC_OK;

    // work buffers sized for the largest group
    int64_t max_sel = 0;
    for (int g = 0; g < CONC_GROUPS - 1; ++g) max_sel = std::max<int64_t>(max_sel, (int64_t)h_counts[g * CONC_COUNTERS + 4]);
    if (max_sel == 0) return UGVC_OK;
    double *d_sel_s, *d_sorted_s;
    uint8_t *d_sel_t, *d_sorted_t, *d_bflag;
    int64_t *d_cum, *d_idx, *d_num;
    CCU(buf.get(&d_sel_s, (size_t)max_sel));
    CCU(buf.get(&d_sorted_s, (size_t)max_sel + 1));
    CCU(buf.get(&d_sel_t, (size_t)max_sel));
    CCU(buf.get(&d_sorted_t, (size_t)max_sel));
    CCU(buf.get(&d_bflag, (size_t)max_sel));
    CCU(buf.get(&d_cum, (size_t)max_sel));
    CCU(buf.get(&d_idx, (size_t)max_sel));
    CCU(buf.get(&d_num, 2));
    size_t tmp_bytes = 0, need = 0;
    const int n32 = (int)n, m32 = (int)max_sel;
    cub::DeviceSelect::Flagged(nullptr, need, d_scores, d_flags, d_sel_s, d_num, n32, st);
    tmp_bytes = std::max(tmp_bytes, need);
    cub::DeviceSelect::Flagged(nullptr, need, d_truth, d_flags, d_sel_t, d_num, n32, st);
    tmp_bytes = std::max(tmp_bytes, need);
    cub::DeviceRadixSort::SortPairsDescending(nullptr, need, d_sel_s, d_sorted_s, d_sel_t, d_sorted_t, m32, 0, 64, st);
    tmp_bytes = std::max(tmp_bytes, need);
    cub::TransformInputIterator<int64_t, U8ToI64, const uint8_t*> truth_it(d_sorted_t, U8ToI64());
    cub::DeviceScan::InclusiveSum(nullptr, need, truth_it, d_cum, m32, st);
    tmp_bytes = std::max(tmp_bytes, need);
    cub::CountingInputIterator<int64_t> count_it(0);
    cub::DeviceSelect::Flagged(nullptr, need, count_it, d_bflag, d_idx, d_num, m32, st);
    tmp_bytes = std::max(tmp_bytes, need);
    uint8_t* d_tmp;
    CCU(buf.get(&d_tmp, tmp_bytes));

    for (int g = 0; g < CONC_GROUPS - 1; ++g) {  // the reference draws no curve for H-INDELS
        const int64_t expect = (int64_t)h_counts[g * CONC_COUNTERS + 4];
        if (expect == 0) continue;
        conc_flags<<<grid, CONC_TPB, 0, st>>>(n, d_meta, g, d_flags);
        ++h->launches;
        size_t tb = tmp_bytes;
        CCU(cub::DeviceSelect::Flagged(d_tmp, tb, d_scores, d_flags, d_sel_s, d_num, n32, st));
        tb = tmp_bytes;
        CCU(cub::DeviceSelect::Flagged(d_tmp, tb, d_truth, d_flags, d_sel_t, d_num + 1, n32, st));
        int64_t h_num[2];
        CCU(cudaMemcpyAsync(h_num, d_num, sizeof(h_num), cudaMemcpyDeviceToHost, st));
        CCU(cudaStreamSynchronize(st));
        if (h_num[0] != expect || h_num[1] != expect) return conc_fail(h, UGVC_E_CUDA, "conc_run: selection size mismatch");
        const int ns = (int)expect;
        tb = tmp_bytes;
        CCU(cub::DeviceRadixSort::SortPairsDescending(d_tmp, tb, d_sel_s, d_sorted_s, d_sel_t, d_sorted_t, ns, 0, 64, st));
        cub::TransformInputIterator<int64_t, U8ToI64, const uint8_t*> it(d_sorted_t, U8ToI64());
        tb = tmp_bytes;
        CCU(cub::DeviceScan::InclusiveSum(d_tmp, tb, it, d_cum, ns, st));
        conc_boundary<<<grid, CONC_TPB, 0, st>>>(expect, d_sorted_s, d_bflag);
        ++h->launches;
        tb = tmp_bytes;
        CCU(cub::DeviceSelect::Flagged(d_tmp, tb, count_it, d_bflag, d_idx, d_num, ns, st));
        int64_t d_len = 0, sel_true = 0;
        double cutoff = 0.0;
        CCU(cudaMemcpyAsync(&d_len, d_num, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        CCU(cudaMemcpyAsync(&sel_true, d_cum + (expect - 1), sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        // the 20th largest score: below it the curve is too noisy (stats_utils.py:202-207)
        CCU(cudaMemcpyAsync(&cutoff, d_sorted_s + std::min<int64_t>(expect - 1, 19), sizeof(double), cudaMemcpyDeviceToHost, st));
        CCU(cudaStreamSynchronize(st));
        for (int a = 0; a < 3; ++a) CCU(cudaMalloc(&h->curve[g][a], (size_t)d_len * sizeof(double)));
        conc_curve<<<grid, CONC_TPB, 0, st>>>(d_len, expect, d_idx, d_sorted_s, d_cum, h->curve[g][0], h->curve[g][1],
                                              h->curve[g][2]);
        ++h->launches;
        CCU(cudaGetLastError());
        h->launches += 5;  // the cub passes above
        h->curve_len[g] = d_len;
        if (out_curve_len) out_curve_len[g] = d_len;
        if (out_cutoff) out_cutoff[g] = cutoff;
        if (out_selected) {
            out_selected[2 * g] = expect;
            out_selected[2 * g + 1] = sel_true;
        }
    }
    CCU(cudaStreamSynchronize(st));
    return UGVC_OK;
}

extern "C" int ugvc_conc_curve(ugvc_conc* h, int group, double* precision, double* recall, double* thresholds,
                               size_t capacity) {
    if (!h) return UGVC_E_ARG;
    if (group < 0 || group >= CONC_GROUPS) return conc_fail(h, UGVC_E_ARG, "conc_curve: group out of range");
    const int64_t d = h->curve_len[group];
    if ((size_t)d > capacity) return conc_fail(h, UGVC_E_ARG, "conc_curve: capacity too small");
    if (d == 0) return UGVC_OK;
    CCU(cudaSetDevice(h->device));
    double* dst[3] = {precision, recall, thresholds};
    for (int a = 0; a < 3; ++a)
        if (dst[a]) CCU(cudaMemcpy(dst[a], h->curve[group][a], (size_t)d * sizeof(double), cudaMemcpyDeviceToHost));
    return UGVC_OK;
}

// ------------------------------------------------------------------------------------------
// per-record classification of a comparison frame (vcf2concordance, comparison_utils.py:153-229)
// ------------------------------------------------------------------------------------------
// Genotypes arrive as two int8 per record: allele index, -1 for None, -2 when the tuple has one element.
// classify (allele match): :153-182; classify_gt (allele + genotype match): :186-213; fix-ups :214-229.
__device__ __forceinline__ bool conc_gt_none(int a, int b) { return a == -1 && (b == -1 || b == -2); }
__global__ void __launch_bounds__(CONC_TPB) conc_classify_gt(int64_t n, const int8_t* __restrict__ gu, const int8_t* __restrict__ gt,
                                                             const uint8_t* __restrict__ base_fn, uint8_t* __restrict__ cls,
                                                             uint8_t* __restrict__ cls_gt) {
    enum { TP = 0, FP = 1, FN = 2 };
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int u0 = gu[2 * i], u1 = gu[2 * i + 1], t0 = gt[2 * i], t1 = gt[2 * i + 1];
        int c, g;
        if (conc_gt_none(u0, u1)) {
            c = g = FN;
        } else if (conc_gt_none(t0, t1)) {
            c = g = FP;
        } else {
            // sets of non-reference alleles (None is an element like any other)
            const bool u0_in = u0 != 0, u1_in = u1 != 0 && u1 != -2, t0_in = t0 != 0, t1_in = t1 != 0 && t1 != -2;
            const bool u0_hit = u0_in && ((t0_in && u0 == t0) || (t1_in && u0 == t1));
            const bool u1_hit = u1_in && ((t0_in && u1 == t0) || (t1_in && u1 == t1));
            if (u0_hit || u1_hit) c = TP;
            else if (u0_in || u1_in) c = FP;  // an allele of the call that the truth does not have
            else c = FN;
            const int nref_t = (t0 == 0) + (t1 == 0), nref_u = (u0 == 0) + (u1 == 0);
            if (nref_t < nref_u) g = FN;
            else if (nref_t > nref_u) g = FP;
            else if (u0 != t0 || u1 != t1) g = FP;  // tuples differ (order and length count)
            else g = TP;
        }
        if (g == TP && c == FP) g = FP;
        if (base_fn && base_fn[i]) {  // vcfeval's BASE says FN / FN_CA: a wrong call that was filtered is a miss
            if (c == FP) c = FN;
            if (g == FP) g = FN;
        }
        cls[i] = (uint8_t)c;
        cls_gt[i] = (uint8_t)g;
    }
}

extern "C" int ugvc_conc_classify(ugvc_conc* h, int64_t n, const int8_t* gt_ultima, const int8_t* gt_truth, const uint8_t* base_fn,
                                  uint8_t* out_classify, uint8_t* out_classify_gt) {
    if (!h || n < 0 || (n && (!gt_ultima || !gt_truth || !out_classify || !out_classify_gt))) return conc_fail(h, UGVC_E_ARG, "conc_classify: bad arguments");
    if (n == 0) return UGVC_OK;
    if (cudaSetDevice(h->device) != cudaSuccess) return conc_fail(h, UGVC_E_CUDA, "cudaSetDevice failed");
    int8_t *d_u = nullptr, *d_t = nullptr;
    uint8_t *d_b = nullptr, *d_c = nullptr, *d_g = nullptr;
    cudaError_t e = cudaMalloc(&d_u, 2 * n);
    if (e == cudaSuccess) e = cudaMalloc(&d_t, 2 * n);
    if (e == cudaSuccess && base_fn) e = cudaMalloc(&d_b, n);
    if (e == cudaSuccess) e = cudaMalloc(&d_c, n);
    if (e == cudaSuccess) e = cudaMalloc(&d_g, n);
    if (e == cudaSuccess) e = cudaMemcpy(d_u, gt_ultima, 2 * n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(d_t, gt_truth, 2 * n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && base_fn) e = cudaMemcpy(d_b, base_fn, n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        int64_t blocks = (n + CONC_TPB - 1) / CONC_TPB;
        if (blocks > h->sm_count * 16) blocks = h->sm_count * 16;
        conc_classify_gt<<<(unsigned)blocks, CONC_TPB>>>(n, d_u, d_t, d_b, d_c, d_g);
        h->launches += 1;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(out_classify, d_c, n, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(out_classify_gt, d_g, n, cudaMemcpyDeviceToHost);
    cudaFree(d_u);
    cudaFree(d_t);
    cudaFree(d_b);
    cudaFree(d_c);
    cudaFree(d_g);
    return e == cudaSuccess ? UGVC_OK : conc_fail(h, UGVC_E_CUDA, cudaGetErrorString(e));
}
