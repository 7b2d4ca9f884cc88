// bridging_snvs.cu -- calibrate_bridging_snvs on the GPU (DESIGN.md 4d).
//
// Replaces the per-record loop of ugvc/pipelines/vcfbed/calibrate_bridging_snvs.py (run, :91-130) and its
// is_homopolymer_snp (:9-66): a filtered SNV whose ALT base extends a reference homopolymer, with a high tumor VAF and a
// low normal VAF, gets FILTER PASS and a new QUAL.  Three steps, one thread per record, grid-stride and CUB-free, so that
// the host emulation runs this source:
//   bsn_decide        finds REF, ALT, QUAL, FILTER, FORMAT and sample 0 (no column or line-length limit), evaluates the
//                     candidate test, resolves CHROM in the contig table (candidates only), walks the FASTA window in
//                     place, types AD / DP / BG_AD / BG_DP of sample 0 as pysam does and evaluates the rescue; writes
//                     the decision, hmer_size, the length of the written line and INFO/END
//   afr_launch_scan   the chunked scan of low_af_ratio.cu over the lengths (and the rescued count)
//   bsn_copy          writes each line; a rescued one gets "<qual>\tPASS" in place of its QUAL and FILTER columns
// Where the reference raises, the record is recorded: atomicMin of (record << 4 | reason).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <numeric>
#include <vector>

#include "bridging_snvs.cuh"
#include "low_af_ratio.cuh"
#include "numparse.h"
#include "vcf_text.cuh"

#define BSN_TPB 256

#ifdef UGVC_HOST_EMU
#define BSN_LAUNCH(kern, grid, block, st, ...)                  \
    do {                                                        \
        threadIdx = dim3(0, 0, 0); blockIdx = dim3(0, 0, 0);     \
        blockDim = dim3(1, 1, 1); gridDim = dim3(1, 1, 1);       \
        kern(__VA_ARGS__);                                      \
    } while (0)
#else
#define BSN_LAUNCH(kern, grid, block, st, ...) kern<<<grid, block, 0, st>>>(__VA_ARGS__)
#endif

enum : uint8_t { BSN_RESCUED = UGVC_BSN_RESCUED, BSN_NEW_CONTIG = UGVC_BSN_NEW_CONTIG };
enum { K_AD = 0, K_DP = 1, K_BG_AD = 2, K_BG_DP = 3 };

bool bsn_params(const ugvc_bsn_params* p, BsnDev* d) {
    if (!p || !d || !p->qual_text || p->qual_len < 1 || p->qual_len > UGVC_BSN_MAX_QUAL_BYTES) return false;
    if (p->min_query_hmer_size < 0) return false;
    const int32_t kinds[4] = {p->ad_kind, p->dp_kind, p->bg_ad_kind, p->bg_dp_kind};
    const int32_t ints[4] = {p->ad_integer, p->dp_integer, p->bg_ad_integer, p->bg_dp_integer};
    memset(d, 0, sizeof(*d));
    for (int k = 0; k < 4; ++k) {
        if (kinds[k] < UGVC_BSN_KIND_NONE || kinds[k] > UGVC_BSN_KIND_TUPLE) return false;
        d->kind[k] = kinds[k];
        d->integer[k] = ints[k] ? 1 : 0;
    }
    d->m = p->min_query_hmer_size;
    d->min_edge = p->min_distance_from_edge;
    d->min_qual = p->min_initial_qual;
    d->min_tvaf = p->min_tumor_vaf;
    d->max_nvaf = p->max_normal_vaf;
    d->min_ndepth = p->min_normal_depth;
    memcpy(d->qual, p->qual_text, (size_t)p->qual_len);
    d->qual_len = p->qual_len;
    return true;
}

// bytewise order of two names (memcmp, then length)
__device__ __forceinline__ int bsn_cmp(const uint8_t* a, int64_t na, const uint8_t* b, int64_t nb) {
    const int64_t n = na < nb ? na : nb;
    for (int64_t k = 0; k < n; ++k)
        if (a[k] != b[k]) return a[k] < b[k] ? -1 : 1;
    return na < nb ? -1 : (na > nb ? 1 : 0);
}

// index of contig `name` in the sorted table, -1 when absent
__device__ __forceinline__ int bsn_contig(const BsnContigs& C, const uint8_t* name, int64_t nl) {
    int lo = 0, hi = C.n - 1;
    while (lo <= hi) {
        const int mid = (lo + hi) >> 1;
        const int64_t o = C.name_off[mid];
        const int c = bsn_cmp(C.names + o, C.name_off[mid + 1] - o, name, nl);
        if (c == 0) return mid;
        if (c < 0) lo = mid + 1;
        else hi = mid - 1;
    }
    return -1;
}

// sum(v[1:]) as Python computes it: 0 ok (*s), 1 TypeError (a slice of None / of a scalar, or None among the
// elements).  Integer values are exact; Float values take CPython's compensated float sum (3.12: Neumaier), which equals
// the plain left-to-right sum for one or two elements.
__device__ __forceinline__ int bsn_sum_tail(const AfrVal& v, double* s) {
    if (v.kind != 2) return 1;
    double f = 0.0, c = 0.0;
    *s = 0.0;
    if (!v.p) return 0;  // (None,)[1:] == ()
    int64_t at = 0;
    afr_piece(v.p, &at, v.n, ',');
    while (at <= v.n) {
        const int64_t b = at;
        const int64_t m = afr_piece(v.p, &at, v.n, ',');
        double x = 0.0;
        if (afr_number(v.p + b, m, v.integer, &x) != 0) return 1;
        if (v.integer) {
            f += x;
            continue;
        }
        const double t = f + x;
        if (fabs(f) >= fabs(x)) c += (f - t) + x;
        else c += (x - t) + f;
        f = t;
    }
    if (!v.integer && c != 0.0 && isfinite(c)) f += c;
    *s = f;
    return 0;
}

// a scalar number (Number=1 and a value): 0 ok (*x), 1 TypeError (None or a tuple)
__device__ __forceinline__ int bsn_scalar(const AfrVal& v, double* x) {
    if (v.kind != 1) return 1;
    return afr_number(v.p, v.n, v.integer, x) == 0 ? 0 : 1;
}

__device__ __forceinline__ void bsn_error(unsigned long long* err, int64_t i, int reason) {
    atomicMin(err, ((unsigned long long)i << 4) | (unsigned long long)reason);
}

// The rescue of a qualifying record (run, :96-103) on sample 0's typed values, in Python's order of evaluation:
// 0 = not rescued, 1 = rescued, else -(UGVC_BSN_E_* reason).  have[k]: the key is declared and the record's FORMAT and
// sample 0 carry it (else reading it raises KeyError).
__device__ __forceinline__ int bsn_rescue(const BsnDev& P, const bool* have, const AfrVal* v) {
    if (!have[K_BG_DP]) return -UGVC_BSN_E_KEY;  // normal_depth = samples[0]["BG_DP"]
    if (!have[K_AD]) return -UGVC_BSN_E_KEY;
    double s_ad, dp, s_bg, nd;
    if (bsn_sum_tail(v[K_AD], &s_ad)) return -UGVC_BSN_E_TYPE;
    if (!have[K_DP]) return -UGVC_BSN_E_KEY;
    if (bsn_scalar(v[K_DP], &dp)) return -UGVC_BSN_E_TYPE;
    if (dp == 0.0) return -UGVC_BSN_E_ZERO_DIVISION;
    const double tumor_vaf = __ddiv_rn(s_ad, dp);
    if (!have[K_BG_AD]) return -UGVC_BSN_E_KEY;
    if (bsn_sum_tail(v[K_BG_AD], &s_bg)) return -UGVC_BSN_E_TYPE;
    if (bsn_scalar(v[K_BG_DP], &nd)) return -UGVC_BSN_E_TYPE;  // max(0.01, None / tuple)
    const double normal_vaf = __ddiv_rn(s_bg, nd > 0.01 ? nd : 0.01);
    return tumor_vaf >= P.min_tvaf && normal_vaf <= P.max_nvaf && nd > P.min_ndepth;
}

__global__ void __launch_bounds__(BSN_TPB) bsn_decide(const uint8_t* __restrict__ t, const int64_t* __restrict__ ls, int64_t n,
                                                      BsnDev P, BsnContigs C, uint8_t* __restrict__ flags,
                                                      int32_t* __restrict__ hmer_out, int64_t* __restrict__ len,
                                                      int64_t* __restrict__ end_out, unsigned long long* __restrict__ err) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int64_t a = ls[i], e = ls[i + 1] - 1;  // [a, e): the line without its '\n'
        int64_t at = a;
        while (at < e && t[at] != '\t') ++at;
        const int64_t chrom_len = at - a;
        bool new_contig = i == 0;
        if (i > 0) {
            const int64_t p = ls[i - 1];
            new_contig = ls[i] - 1 - p < chrom_len + 1 || !afr_eq(t + p, chrom_len + 1, t + a, chrom_len + 1);
        }
        // columns 1 (POS) .. 9 (sample 0): [c0[k], c1[k])
        int64_t c0[10], c1[10];
        int nc = 1;
        for (++at; nc < 10 && at <= e; ++nc, ++at) {
            const int64_t b = at;
            while (at < e && t[at] != '\t') ++at;
            c0[nc] = b, c1[nc] = at;
        }
        hmer_out[i] = 0;
        if (nc < 8) {  // fewer than 8 columns: refused by the index pass before this kernel runs
            flags[i] = new_contig ? BSN_NEW_CONTIG : 0;
            len[i] = e + 1 - a;
            end_out[i] = 0;
            continue;
        }
        // INFO: the first END=
        int64_t endv = 0;
        const uint8_t* in = t + c0[7];
        const int64_t il = c1[7] - c0[7];
        if (!(il == 1 && in[0] == '.'))
            for (int64_t q = 0; q <= il;) {
                const int64_t b = q, m = afr_piece(in, &q, il, ';');
                const uint8_t* pc = in + b;
                if (m >= 4 && pc[0] == 'E' && pc[1] == 'N' && pc[2] == 'D' && pc[3] == '=') {
                    bool digits = m > 4 && m <= 14;
                    for (int64_t d = 4; d < m && digits; ++d) {
                        digits = pc[d] >= '0' && pc[d] <= '9';
                        endv = endv * 10 + (pc[d] - '0');
                    }
                    if (!digits) endv = 0;
                    break;
                }
            }
        end_out[i] = endv;
        // QUAL, typed for every record
        double qual = 0.0;
        const int qk = afr_number(t + c0[5], c1[5] - c0[5], 0, &qual);
        bool bad = qk == 2;
        // AD / DP / BG_AD / BG_DP of sample 0, typed for every record that carries them
        bool have[4] = {false, false, false, false};
        AfrVal v[4];
        int fi[4] = {-1, -1, -1, -1};
        if (nc == 10 && !(c1[8] - c0[8] == 1 && t[c0[8]] == '.')) {
            const uint8_t* fm = t + c0[8];
            const int64_t fml = c1[8] - c0[8];
            int k = 0;
            for (int64_t q = 0; q <= fml; ++k) {
                const int64_t b = q, m = afr_piece(fm, &q, fml, ':');
                if (afr_eq(fm + b, m, (const uint8_t*)"AD", 2)) fi[K_AD] = k;
                else if (afr_eq(fm + b, m, (const uint8_t*)"DP", 2)) fi[K_DP] = k;
                else if (afr_eq(fm + b, m, (const uint8_t*)"BG_AD", 5)) fi[K_BG_AD] = k;
                else if (afr_eq(fm + b, m, (const uint8_t*)"BG_DP", 5)) fi[K_BG_DP] = k;
            }
            const uint8_t* sp[4] = {nullptr, nullptr, nullptr, nullptr};
            int64_t sn[4] = {0, 0, 0, 0};
            bool spres[4] = {false, false, false, false};
            k = 0;
            for (int64_t q = c0[9]; q <= c1[9]; ++k) {
                const int64_t b = q, m = afr_piece(t, &q, c1[9], ':');
                for (int j = 0; j < 4; ++j)
                    if (k == fi[j]) sp[j] = t + b, sn[j] = m, spres[j] = true;
            }
            for (int j = 0; j < 4; ++j) {
                have[j] = P.kind[j] != UGVC_BSN_KIND_NONE && fi[j] >= 0;
                v[j] = afr_value(have[j] ? P.kind[j] : 0, P.integer[j], spres[j], sp[j], sn[j], &bad);
            }
        }
        // the candidate test (:16-22), short-circuit as there
        const int64_t ref_len = c1[3] - c0[3];
        const uint8_t* alt = t + c0[4];
        const int64_t alt_len = c1[4] - c0[4];
        int reason = 0;
        bool cand = false;
        if (ref_len == 1) {
            if (alt_len == 1 && alt[0] == '.') {
                reason = UGVC_BSN_E_TYPE;  // len(None)
            } else if (alt_len == 1) {
                const uint8_t* f = t + c0[6];
                const int64_t fl = c1[6] - c0[6];
                bool pass = false;
                if (!(fl == 1 && f[0] == '.'))
                    for (int64_t q = 0; q <= fl;) {
                        const int64_t b = q, m = afr_piece(f, &q, fl, ';');
                        pass |= afr_eq(f + b, m, (const uint8_t*)"PASS", 4);
                    }
                if (!pass) {
                    if (qk == 1) reason = UGVC_BSN_E_TYPE;  // None >= min_initial_qual
                    else cand = qual >= P.min_qual;
                }
            }
        }
        bool rescued = false;
        if (cand && !bad) {
            // the window reference.fetch(chrom, pos - m - 1, pos + m), walked in place
            int64_t pos = 0;
            for (int64_t q = c0[1]; q < c1[1] && pos < ((int64_t)1 << 40); ++q) pos = pos * 10 + (t[q] - '0');
            const int64_t s = pos - P.m - 1, stop = pos + P.m;
            const int ci = s < 0 ? -1 : bsn_contig(C, t + a, chrom_len);
            if (ci < 0) {
                reason = UGVC_BSN_E_FETCH;
            } else {
                const uint8_t* sq = C.seq[ci];
                const int64_t hi = stop < C.len[ci] ? stop : C.len[ci];
                const int64_t wl = hi > s ? hi - s : 0;  // len(reference_seq)
                const uint8_t ab = alt[0], rb = t[c0[3]];
                int64_t up = 0, down = 0;
                int before = -1, after = -1;  // -1: the walk ran out ("")
                for (int64_t j = (int64_t)P.m + 1; j < wl; ++j) {
                    if (sq[s + j] != ab) {
                        after = sq[s + j];
                        break;
                    }
                    ++down;
                }
                // seq[m - 1::-1]: from index m - 1 (clipped to the last one; for m = 0 the last one) down to 0
                const int64_t u0 = P.m == 0 ? wl - 1 : ((int64_t)P.m - 1 < wl - 1 ? (int64_t)P.m - 1 : wl - 1);
                for (int64_t j = u0; j >= 0; --j) {
                    if (sq[s + j] != ab) {
                        before = sq[s + j];
                        break;
                    }
                    ++up;
                }
                const int64_t hmer = 1 + up + down;
                const bool tandem = before >= 0 && before == after && before == rb && up == down;
                const int64_t edge = up < down ? up : down;
                hmer_out[i] = (int32_t)(hmer < 0x7FFFFFFF ? hmer : 0x7FFFFFFF);
                if (hmer >= P.m && !tandem && edge >= P.min_edge) {
                    const int r = bsn_rescue(P, have, v);
                    if (r < 0) reason = -r;
                    else rescued = r == 1;
                }
            }
        }
        if (bad) bsn_error(err, i, UGVC_BSN_E_LITERAL);
        else if (reason) bsn_error(err, i, reason);
        flags[i] = (uint8_t)((rescued ? BSN_RESCUED : 0) | (new_contig ? BSN_NEW_CONTIG : 0));
        len[i] = (e + 1 - a) + (rescued ? (P.qual_len + 5) - (c1[6] - c0[5]) : 0);
    }
}

__global__ void __launch_bounds__(BSN_TPB) bsn_copy(const uint8_t* __restrict__ t, const int64_t* __restrict__ ls, int64_t n,
                                                    BsnDev P, const uint8_t* __restrict__ flags,
                                                    const int64_t* __restrict__ out_ls, uint8_t* __restrict__ out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int64_t a = ls[i], e = ls[i + 1];
        uint8_t* o = out + out_ls[i];
        if (!(flags[i] & BSN_RESCUED)) {
            memcpy(o, t + a, (size_t)(e - a));
            continue;
        }
        // [q0, f1): the QUAL and FILTER columns (a rescued record has at least 8 columns)
        int64_t q0 = a;
        for (int tabs = 0; tabs < 5; ++q0) tabs += t[q0] == '\t';
        int64_t f1 = q0;
        while (t[f1] != '\t') ++f1;  // the end of QUAL
        ++f1;
        while (t[f1] != '\t') ++f1;  // the end of FILTER
        memcpy(o, t + a, (size_t)(q0 - a));
        o += q0 - a;
        memcpy(o, P.qual, (size_t)P.qual_len);
        o += P.qual_len;
        memcpy(o, "\tPASS", 5);
        o += 5;
        memcpy(o, t + f1, (size_t)(e - f1));
    }
}

static unsigned bsn_grid(int64_t n, int sm_count) {
    int64_t g = (n + BSN_TPB - 1) / BSN_TPB;
    if (g > (int64_t)sm_count * 16) g = (int64_t)sm_count * 16;
    return (unsigned)(g > 0 ? g : 1);
}

void bsn_launch_decide(const uint8_t* text, const int64_t* line_start, int64_t n, const BsnDev& P, const BsnContigs& C,
                       uint8_t* flags, int32_t* hmer, int64_t* len, int64_t* end, int64_t* out_ls, int64_t* agg,
                       int64_t* totals, unsigned long long* err, int sm_count, cudaStream_t st) {
    BSN_LAUNCH(bsn_decide, bsn_grid(n, sm_count), BSN_TPB, st, text, line_start, n, P, C, flags, hmer, len, end, err);
    afr_launch_scan(len, flags, n, out_ls, agg, totals, sm_count, st);
}

void bsn_launch_copy(const uint8_t* text, const int64_t* line_start, int64_t n, const BsnDev& P, const uint8_t* flags,
                     const int64_t* out_ls, uint8_t* out, int sm_count, cudaStream_t st) {
    BSN_LAUNCH(bsn_copy, bsn_grid(n, sm_count), BSN_TPB, st, text, line_start, n, P, flags, out_ls, out);
}

void bsn_table_free(BsnTable* t) {
    cudaFree(t->d_names);
    cudaFree(t->d_name_off);
    cudaFree(t->d_seq);
    cudaFree(t->d_len);
    *t = BsnTable();
}

cudaError_t bsn_table_build(const std::vector<std::string>& names, const std::vector<const uint8_t*>& seq,
                            const std::vector<int64_t>& len, BsnTable* t) {
    bsn_table_free(t);
    std::vector<size_t> order(names.size());
    std::iota(order.begin(), order.end(), (size_t)0);
    std::sort(order.begin(), order.end(), [&](size_t x, size_t y) { return names[x] < names[y]; });
    std::string blob;
    std::vector<int64_t> off(1, 0), lens;
    std::vector<const uint8_t*> ptrs;
    for (size_t k : order) {
        blob += names[k];
        off.push_back((int64_t)blob.size());
        ptrs.push_back(seq[k]);
        lens.push_back(len[k]);
    }
    cudaError_t e;
    if ((e = cudaMalloc(&t->d_names, blob.size() + 1)) != cudaSuccess) return e;
    if ((e = cudaMalloc(&t->d_name_off, off.size() * sizeof(int64_t))) != cudaSuccess) return e;
    if ((e = cudaMalloc(&t->d_seq, (ptrs.size() + 1) * sizeof(uint8_t*))) != cudaSuccess) return e;
    if ((e = cudaMalloc(&t->d_len, (lens.size() + 1) * sizeof(int64_t))) != cudaSuccess) return e;
    if (!blob.empty() && (e = cudaMemcpy(t->d_names, blob.data(), blob.size(), cudaMemcpyHostToDevice)) != cudaSuccess) return e;
    if ((e = cudaMemcpy(t->d_name_off, off.data(), off.size() * sizeof(int64_t), cudaMemcpyHostToDevice)) != cudaSuccess) return e;
    if (!ptrs.empty() && (e = cudaMemcpy(t->d_seq, ptrs.data(), ptrs.size() * sizeof(uint8_t*), cudaMemcpyHostToDevice)) != cudaSuccess)
        return e;
    if (!lens.empty() && (e = cudaMemcpy(t->d_len, lens.data(), lens.size() * sizeof(int64_t), cudaMemcpyHostToDevice)) != cudaSuccess)
        return e;
    t->n = (int)names.size();
    return cudaSuccess;
}

// ---- test hook: decide + scan + copy on caller records and contigs --------------------------------------------------------
namespace {
struct BsnBufs {  // frees on scope exit
    std::vector<void*> ptrs;
    BsnTable table;
    ~BsnBufs() {
        bsn_table_free(&table);
        for (void* p : ptrs) cudaFree(p);
    }
    template <class T>
    cudaError_t get(T** p, size_t count) {
        cudaError_t e = cudaMalloc(reinterpret_cast<void**>(p), (count ? count : 1) * sizeof(T));
        if (e == cudaSuccess) ptrs.push_back(*p);
        return e;
    }
};
}  // namespace

#define BSN_CU(call)                                 \
    do {                                             \
        if ((call) != cudaSuccess) return UGVC_E_CUDA; \
    } while (0)

extern "C" int64_t ugvc_test_bsn(const uint8_t* text, size_t n_bytes, const int64_t* line_start, int64_t n, const uint8_t* names,
                                 const int64_t* name_off, const uint8_t* seq, const int64_t* seq_off, int32_t n_contigs,
                                 const ugvc_bsn_params* params, uint8_t* out, size_t capacity, int64_t* out_line_start,
                                 uint8_t* out_rescued, int32_t* out_hmer, int64_t* out_end, int64_t* out_n_rescued,
                                 int64_t* out_err_record, int32_t* out_err_reason) {
    BsnDev P;
    if (!bsn_params(params, &P) || n < 0 || n_contigs < 0 || !line_start || !out_line_start || !out_err_record ||
        !out_err_reason || (n && (!text || !out_rescued || !out_hmer || !out_end)) ||
        (n_contigs && (!names || !name_off || !seq_off)))
        return UGVC_E_ARG;
    *out_err_record = -1;
    *out_err_reason = 0;
    if (line_start[0] != 0 || (size_t)line_start[n] != n_bytes) return UGVC_E_ARG;
    for (int64_t i = 0; i < n; ++i)
        if (line_start[i + 1] <= line_start[i] || text[line_start[i + 1] - 1] != '\n') return UGVC_E_ARG;
    BsnBufs b;
    // the contigs: one device buffer of every sequence, the table over it
    const int64_t seq_bytes = n_contigs ? seq_off[n_contigs] : 0;
    uint8_t* d_seq;
    BSN_CU(b.get(&d_seq, (size_t)seq_bytes));
    if (seq_bytes) BSN_CU(cudaMemcpy(d_seq, seq, (size_t)seq_bytes, cudaMemcpyHostToDevice));
    std::vector<std::string> cn;
    std::vector<const uint8_t*> cs;
    std::vector<int64_t> cl;
    for (int32_t k = 0; k < n_contigs; ++k) {
        cn.emplace_back((const char*)names + name_off[k], (size_t)(name_off[k + 1] - name_off[k]));
        cs.push_back(d_seq + seq_off[k]);
        cl.push_back(seq_off[k + 1] - seq_off[k]);
    }
    BSN_CU(bsn_table_build(cn, cs, cl, &b.table));
    uint8_t *d_text, *d_flags, *d_out;
    int32_t* d_hmer;
    int64_t *d_ls, *d_len, *d_end, *d_out_ls, *d_agg, *d_tot;
    unsigned long long* d_err;
    BSN_CU(b.get(&d_text, n_bytes + 16));
    BSN_CU(b.get(&d_ls, (size_t)n + 1));
    BSN_CU(b.get(&d_flags, (size_t)n));
    BSN_CU(b.get(&d_hmer, (size_t)n));
    BSN_CU(b.get(&d_len, (size_t)n + 1));
    BSN_CU(b.get(&d_end, (size_t)n));
    BSN_CU(b.get(&d_out_ls, (size_t)n + 1));
    BSN_CU(b.get(&d_agg, 2 * ((size_t)n / AFR_CHUNK + 2)));
    BSN_CU(b.get(&d_tot, 2));
    BSN_CU(b.get(&d_err, 1));
    BSN_CU(cudaMemcpy(d_text, text, n_bytes, cudaMemcpyHostToDevice));
    BSN_CU(cudaMemset(d_text + n_bytes, 0, 16));
    BSN_CU(cudaMemcpy(d_ls, line_start, ((size_t)n + 1) * sizeof(int64_t), cudaMemcpyHostToDevice));
    BSN_CU(cudaMemset(d_err, 0xFF, sizeof(unsigned long long)));
    BSN_CU(cudaMemset(d_tot, 0, 2 * sizeof(int64_t)));
    bsn_launch_decide(d_text, d_ls, n, P, b.table.view(), d_flags, d_hmer, d_len, d_end, d_out_ls, d_agg, d_tot, d_err, 132,
                      nullptr);
    BSN_CU(cudaGetLastError());
    int64_t tot[2] = {0, 0};
    unsigned long long h_err = AFR_NO_ERROR;
    BSN_CU(cudaMemcpy(tot, d_tot, sizeof(tot), cudaMemcpyDeviceToHost));
    BSN_CU(cudaMemcpy(&h_err, d_err, sizeof(h_err), cudaMemcpyDeviceToHost));
    if (h_err != AFR_NO_ERROR) {
        *out_err_record = (int64_t)(h_err >> 4);
        *out_err_reason = (int32_t)(h_err & 0xF);
        return UGVC_E_DATA;
    }
    if ((size_t)tot[0] > capacity || (tot[0] && !out)) return UGVC_E_ARG;
    BSN_CU(b.get(&d_out, (size_t)tot[0]));
    bsn_launch_copy(d_text, d_ls, n, P, d_flags, d_out_ls, d_out, 132, nullptr);
    BSN_CU(cudaGetLastError());
    if (tot[0]) BSN_CU(cudaMemcpy(out, d_out, (size_t)tot[0], cudaMemcpyDeviceToHost));
    BSN_CU(cudaMemcpy(out_line_start, d_out_ls, ((size_t)n + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost));
    if (n) {
        BSN_CU(cudaMemcpy(out_rescued, d_flags, (size_t)n, cudaMemcpyDeviceToHost));
        for (int64_t i = 0; i < n; ++i) out_rescued[i] &= BSN_RESCUED;
        BSN_CU(cudaMemcpy(out_hmer, d_hmer, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost));
        BSN_CU(cudaMemcpy(out_end, d_end, (size_t)n * sizeof(int64_t), cudaMemcpyDeviceToHost));
    }
    if (out_n_rescued) *out_n_rescued = tot[1];
    return tot[0];
}
