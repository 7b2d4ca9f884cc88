// low_af_ratio.cu -- filter_low_af_ratio_to_background on the GPU (DESIGN.md 4c).
//
// Replaces the per-record loop of ugbio_filtering/filter_low_af_ratio_to_background.py:35-65 and its process_record
// (:75-114): the AF-ratio rule over every sample of a record and the FILTER edit that pysam / htslib's bcf_add_filter
// make of it.  Three steps, one thread per record, grid-stride and CUB-free, so that the host emulation runs this source:
//   afr_decide        scans the line for FILTER, INFO, FORMAT and every sample column (no column or sample limit), types
//                     GT / VAF / BG_VAF of each sample as pysam does, evaluates the rule, and writes the decision, the
//                     length of the written line and INFO/END
//   afr_agg / afr_spine / afr_apply   the chunked three-phase scan of the lengths (and the failed count)
//   afr_copy          writes each line with its new FILTER column; every other byte is copied as read
// Where the reference raises, the record is recorded: atomicMin of (record << 4 | reason).
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "low_af_ratio.cuh"
#include "numparse.h"
#include "vcf_text.cuh"

#define AFR_TPB 256

#ifdef UGVC_HOST_EMU
#define AFR_LAUNCH(kern, grid, block, st, ...)                  \
    do {                                                        \
        threadIdx = dim3(0, 0, 0); blockIdx = dim3(0, 0, 0);     \
        blockDim = dim3(1, 1, 1); gridDim = dim3(1, 1, 1);       \
        kern(__VA_ARGS__);                                      \
    } while (0)
#else
#define AFR_LAUNCH(kern, grid, block, st, ...) kern<<<grid, block, 0, st>>>(__VA_ARGS__)
#endif

enum : uint8_t { AFR_FAILED = UGVC_AFR_FAILED, AFR_REWRITE = UGVC_AFR_REWRITTEN, AFR_NEW_CONTIG = UGVC_AFR_NEW_CONTIG };

bool afr_params(const ugvc_afr_params* p, AfrDev* d) {
    if (!p || !d || p->new_filter_len < 1 || p->new_filter_len > UGVC_AFR_MAX_FILTER_BYTES || !p->new_filter) return false;
    if (p->variant_type_kind < 0 || p->variant_type_kind > 1) return false;
    if (p->vaf_kind < 0 || p->vaf_kind > 2 || p->bg_vaf_kind < 0 || p->bg_vaf_kind > 2) return false;
    memset(d, 0, sizeof(*d));
    d->thr = p->af_ratio_threshold;
    d->thr_h = p->af_ratio_threshold_h_indels;
    d->vthr_h = p->t_vaf_threshold;
    memcpy(d->nf, p->new_filter, (size_t)p->new_filter_len);
    d->nf_len = p->new_filter_len;
    d->vt_kind = p->variant_type_kind;
    d->vaf_kind = p->vaf_kind;
    d->bg_kind = p->bg_vaf_kind;
    d->vaf_int = p->vaf_integer ? 1 : 0;
    d->bg_int = p->bg_vaf_integer ? 1 : 0;
    return true;
}

// The new FILTER column of a rewritten record (bcf_add_filter's rules, DESIGN.md 4c), written to out when it is not NULL;
// returns its length.  f / fl = the FILTER column as read.
__device__ __forceinline__ int64_t afr_filter(const uint8_t* f, int64_t fl, const AfrDev& P, bool failed, uint8_t* out) {
    const bool dot = fl == 1 && f[0] == '.';
    bool has_nf = false;
    if (!dot) {
        for (int64_t at = 0; at <= fl;) {
            const int64_t b = at, m = afr_piece(f, &at, fl, ';');
            has_nf |= afr_eq(f + b, m, P.nf, P.nf_len);
        }
    }
    int64_t o = 0;
    if (!has_nf) {  // the list as read (duplicates kept), with new_filter added
        const bool pass = fl == 4 && f[0] == 'P' && f[1] == 'A' && f[2] == 'S' && f[3] == 'S';
        if (!dot && !pass) {
            if (out) memcpy(out, f, (size_t)fl);
            o = fl;
            if (out) out[o] = ';';
            ++o;
        }
        if (out) memcpy(out + o, P.nf, (size_t)P.nf_len);
        return o + P.nf_len;
    }
    // rebuilt: the pieces other than new_filter added back in order.  Adding skips a piece already in the list, PASS
    // replaces the list, anything added to [PASS] replaces it -- so the list is the distinct pieces from `start` on.
    int64_t start = 0;
    bool list_pass = false;
    for (int64_t at = 0; at <= fl;) {
        const int64_t b = at, m = afr_piece(f, &at, fl, ';');
        if (afr_eq(f + b, m, P.nf, P.nf_len)) continue;
        bool present = false;
        for (int64_t a2 = start; a2 < b && !present;) {
            const int64_t b2 = a2, m2 = afr_piece(f, &a2, b - 1, ';');
            present = !afr_eq(f + b2, m2, P.nf, P.nf_len) && afr_eq(f + b2, m2, f + b, m);
        }
        if (present) continue;
        const bool is_pass = m == 4 && f[b] == 'P' && f[b + 1] == 'A' && f[b + 2] == 'S' && f[b + 3] == 'S';
        if (is_pass || list_pass) start = b;
        list_pass = is_pass;
    }
    int64_t kept = 0;
    for (int64_t at = start; at <= fl;) {
        const int64_t b = at, m = afr_piece(f, &at, fl, ';');
        if (afr_eq(f + b, m, P.nf, P.nf_len)) continue;
        bool dup = false;
        for (int64_t a2 = start; a2 < b && !dup;) {
            const int64_t b2 = a2, m2 = afr_piece(f, &a2, b - 1, ';');
            dup = !afr_eq(f + b2, m2, P.nf, P.nf_len) && afr_eq(f + b2, m2, f + b, m);
        }
        if (dup) continue;
        if (failed && list_pass) break;  // [PASS] + new_filter -> [new_filter]
        if (kept) {
            if (out) out[o] = ';';
            ++o;
        }
        if (out) memcpy(out + o, f + b, (size_t)m);
        o += m;
        ++kept;
    }
    if (failed) {
        if (kept) {
            if (out) out[o] = ';';
            ++o;
        }
        if (out) memcpy(out + o, P.nf, (size_t)P.nf_len);
        o += P.nf_len;
    } else if (!kept) {
        if (out) out[o] = '.';
        ++o;
    }
    return o;
}

// byte offsets of the FILTER column of line [a, e): [*f0, *f1); false when the line has fewer than 8 columns
__device__ __forceinline__ bool afr_filter_col(const uint8_t* t, int64_t a, int64_t e, int64_t* f0, int64_t* f1) {
    int col = 0;
    int64_t k = a;
    for (; k < e && col < 6; ++k) col += t[k] == '\t';
    if (col < 6) return false;
    *f0 = k;
    while (k < e && t[k] != '\t') ++k;
    *f1 = k;
    return k < e;
}

__device__ __forceinline__ void afr_error(unsigned long long* err, int64_t i, int reason) {
    atomicMin(err, ((unsigned long long)i << 4) | (unsigned long long)reason);
}

__global__ void __launch_bounds__(AFR_TPB) afr_decide(const uint8_t* __restrict__ t, const int64_t* __restrict__ ls, int64_t n,
                                                      AfrDev P, uint8_t* __restrict__ flags, int64_t* __restrict__ len,
                                                      int64_t* __restrict__ end_out, unsigned long long* __restrict__ err) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int64_t a = ls[i], e = ls[i + 1] - 1;  // [a, e): the line without its '\n'
        // CHROM against the previous line's; FILTER, INFO, FORMAT; the first sample column
        int64_t at = a;
        while (at < e && t[at] != '\t') ++at;
        bool new_contig = i == 0;
        if (i > 0) {
            const int64_t p = ls[i - 1];
            new_contig = ls[i] - 1 - p < at - a + 1 || !afr_eq(t + p, at - a + 1, t + a, at - a + 1);
        }
        int64_t c0[3] = {0, 0, 0}, c1[3] = {0, 0, 0};
        int nc = 1;
        for (++at; nc < 9 && at <= e; ++nc, ++at) {
            const int64_t b = at;
            while (at < e && t[at] != '\t') ++at;
            if (nc >= 6) c0[nc - 6] = b, c1[nc - 6] = at;
        }
        if (nc < 8) {  // fewer than 8 columns: refused by the index pass before this kernel runs
            flags[i] = new_contig ? AFR_NEW_CONTIG : 0;
            len[i] = e + 1 - a;
            if (end_out) end_out[i] = 0;
            continue;
        }
        const int64_t samples = at;  // first byte of the first sample column (> e: none)
        const uint8_t* f = t + c0[0];
        const int64_t fl = c1[0] - c0[0];
        // FILTER: RefCall
        bool refcall = false;
        if (!(fl == 1 && f[0] == '.'))
            for (int64_t q = 0; q <= fl;) {
                const int64_t b = q, m = afr_piece(f, &q, fl, ';');
                refcall |= m == 7 && afr_eq(f + b, 7, (const uint8_t*)"RefCall", 7);
            }
        // INFO: the last VARIANT_TYPE, the first END=
        bool h_indel = false;
        int64_t endv = 0;
        bool end_seen = false;
        const uint8_t* in = t + c0[1];
        const int64_t il = c1[1] - c0[1];
        if (!(il == 1 && in[0] == '.'))
            for (int64_t q = 0; q <= il;) {
                const int64_t b = q, m = afr_piece(in, &q, il, ';');
                const uint8_t* pc = in + b;
                if (m >= 12 && afr_eq(pc, 12, (const uint8_t*)"VARIANT_TYPE", 12) && (m == 12 || pc[12] == '='))
                    h_indel = P.vt_kind == 1 && m == 20 && afr_eq(pc + 13, 7, (const uint8_t*)"h-indel", 7);
                if (!end_seen && m >= 4 && pc[0] == 'E' && pc[1] == 'N' && pc[2] == 'D' && pc[3] == '=') {
                    end_seen = true;
                    bool digits = m > 4 && m <= 14;
                    for (int64_t d = 4; d < m && digits; ++d) {
                        digits = pc[d] >= '0' && pc[d] <= '9';
                        endv = endv * 10 + (pc[d] - '0');
                    }
                    if (!digits) endv = 0;
                }
            }
        if (end_out) end_out[i] = endv;
        // FORMAT: where GT / VAF / BG_VAF sit (the last of a repeated key)
        int gi = -1, vi = -1, bi = -1, n_keys = 0;
        if (nc == 9 && !(c1[2] - c0[2] == 1 && t[c0[2]] == '.')) {
            const uint8_t* fm = t + c0[2];
            const int64_t fml = c1[2] - c0[2];
            for (int64_t q = 0; q <= fml; ++n_keys) {
                const int64_t b = q, m = afr_piece(fm, &q, fml, ':');
                if (afr_eq(fm + b, m, (const uint8_t*)"GT", 2)) gi = n_keys;
                else if (afr_eq(fm + b, m, (const uint8_t*)"VAF", 3)) vi = n_keys;
                else if (afr_eq(fm + b, m, (const uint8_t*)"BG_VAF", 6)) bi = n_keys;
            }
        }
        const double thr = h_indel ? P.thr_h : P.thr;
        const double vthr = h_indel ? P.vthr_h : 1.0;
        bool failed = false, bad = false, type_error = false;
        for (int64_t s0 = samples; n_keys > 0 && s0 <= e;) {
            int64_t s1 = s0;
            while (s1 < e && t[s1] != '\t') ++s1;
            // the sub-fields of this sample
            const uint8_t *gp = nullptr, *vp = nullptr, *bp = nullptr;
            int64_t gn = 0, vn = 0, bn = 0;
            bool gpres = false, vpres = false, bpres = false;
            int k = 0;
            for (int64_t q = s0; q <= s1; ++k) {
                const int64_t b = q, m = afr_piece(t, &q, s1, ':');
                if (k == gi) gp = t + b, gn = m, gpres = true;
                if (k == vi) vp = t + b, vn = m, vpres = true;
                if (k == bi) bp = t + b, bn = m, bpres = true;
            }
            s0 = s1 + 1;
            const AfrVal vaf = afr_value(vi < 0 ? 0 : P.vaf_kind, P.vaf_int, vpres, vp, vn, &bad);
            const AfrVal bg = afr_value(bi < 0 ? 0 : P.bg_kind, P.bg_int, bpres, bp, bn, &bad);
            // GT: every allele token is "." / "" (None) or digits
            if (gi >= 0 && gpres) {
                for (int64_t j = 0; j < gn; ++j) {
                    const uint8_t c = gp[j];
                    if (c != '/' && c != '|' && c != '.' && (c < '0' || c > '9')) bad = true;
                }
                for (int64_t j = 0, b = 0; j <= gn; ++j) {
                    if (j < gn && gp[j] != '/' && gp[j] != '|') continue;
                    const int64_t m = j - b;
                    bool dots = m == 1 && gp[b] == '.';
                    for (int64_t z = b; z < j; ++z) bad |= (gp[z] == '.' && !dots);
                    b = j + 1;
                }
            }
            if (refcall || type_error || gi < 0 || vaf.kind == 0 || bg.kind == 0) continue;
            if (!gpres) continue;  // GT dropped: (None,)
            for (int64_t j = 0, b = 0; j <= gn; ++j) {
                if (j < gn && gp[j] != '/' && gp[j] != '|') continue;
                const int64_t m = j - b;
                const uint8_t* ap = gp + b;
                b = j + 1;
                if (m == 0 || (m == 1 && ap[0] == '.')) continue;  // None
                int64_t allele = 0;
                for (int64_t z = 0; z < m; ++z) allele = allele < 1000000000 ? allele * 10 + (ap[z] - '0') : allele;
                if (allele == 0) continue;
                // (allele - 1 >= len(vaf)) or (allele - 1 >= len(bg_vaf)): len() of a scalar raises TypeError
                if (vaf.kind == 1) {
                    type_error = true;
                    break;
                }
                if (allele - 1 >= vaf.len) continue;
                if (bg.kind == 1) {
                    type_error = true;
                    break;
                }
                if (allele - 1 >= bg.len) continue;
                double v = 0.0, w = 0.0;
                if (afr_elem(vaf, allele - 1, &v) || v == 0.0) {
                    failed = true;
                    continue;
                }
                if (afr_elem(bg, allele - 1, &w) || w == 0.0) {
                    failed = false;
                    break;
                }
                const double ratio = __ddiv_rn(v, w);
                if (ratio >= thr || v >= vthr) {
                    failed = false;
                    break;
                }
                failed = true;
            }
        }
        if (bad) afr_error(err, i, UGVC_AFR_E_LITERAL);
        else if (type_error) afr_error(err, i, UGVC_AFR_E_TYPE);
        // the FILTER edit
        bool has_nf = false;
        if (!(fl == 1 && f[0] == '.'))
            for (int64_t q = 0; q <= fl;) {
                const int64_t b = q, m = afr_piece(f, &q, fl, ';');
                has_nf |= afr_eq(f + b, m, P.nf, P.nf_len);
            }
        failed = failed && !refcall;
        const bool rewrite = !refcall && (has_nf || failed);
        flags[i] = (uint8_t)((failed ? AFR_FAILED : 0) | (rewrite ? AFR_REWRITE : 0) | (new_contig ? AFR_NEW_CONTIG : 0));
        len[i] = (e + 1 - a) + (rewrite ? afr_filter(f, fl, P, failed, nullptr) - fl : 0);
    }
}

// the three-phase scan over chunks of AFR_CHUNK records of {line bytes, failed}
__global__ void afr_agg(const int64_t* __restrict__ len, const uint8_t* __restrict__ flags, int64_t n, int64_t* __restrict__ agg) {
    const int64_t n_chunks = (n + AFR_CHUNK - 1) / AFR_CHUNK;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks; c += stride) {
        const int64_t e = (c + 1) * AFR_CHUNK < n ? (c + 1) * AFR_CHUNK : n;
        int64_t bytes = 0, failed = 0;
        for (int64_t i = c * AFR_CHUNK; i < e; ++i) {
            bytes += len[i];
            failed += flags[i] & AFR_FAILED;
        }
        agg[2 * c] = bytes;
        agg[2 * c + 1] = failed;
    }
}
__global__ void afr_spine(int64_t* agg, int64_t n, int64_t* totals) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    const int64_t n_chunks = (n + AFR_CHUNK - 1) / AFR_CHUNK;
    int64_t bytes = 0, failed = 0;
    for (int64_t c = 0; c < n_chunks; ++c) {
        const int64_t b = agg[2 * c], f = agg[2 * c + 1];
        agg[2 * c] = bytes;
        bytes += b;
        failed += f;
    }
    totals[0] = bytes;
    totals[1] = failed;
}
__global__ void afr_apply(const int64_t* __restrict__ len, int64_t n, const int64_t* __restrict__ agg, int64_t* __restrict__ out_ls) {
    const int64_t n_chunks = (n + AFR_CHUNK - 1) / AFR_CHUNK;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks; c += stride) {
        const int64_t e = (c + 1) * AFR_CHUNK < n ? (c + 1) * AFR_CHUNK : n;
        int64_t off = agg[2 * c];
        for (int64_t i = c * AFR_CHUNK; i < e; ++i) {
            out_ls[i] = off;
            off += len[i];
        }
        if (e == n) out_ls[n] = off;
    }
}

__global__ void __launch_bounds__(AFR_TPB) afr_copy(const uint8_t* __restrict__ t, const int64_t* __restrict__ ls, int64_t n,
                                                    AfrDev P, const uint8_t* __restrict__ flags,
                                                    const int64_t* __restrict__ out_ls, uint8_t* __restrict__ out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int64_t a = ls[i], e = ls[i + 1];
        uint8_t* o = out + out_ls[i];
        const uint8_t fg = flags[i];
        int64_t f0, f1;
        if (!(fg & AFR_REWRITE) || !afr_filter_col(t, a, e - 1, &f0, &f1)) {
            memcpy(o, t + a, (size_t)(e - a));
            continue;
        }
        memcpy(o, t + a, (size_t)(f0 - a));
        o += f0 - a;
        o += afr_filter(t + f0, f1 - f0, P, (fg & AFR_FAILED) != 0, o);
        memcpy(o, t + f1, (size_t)(e - f1));
    }
}

static unsigned afr_grid(int64_t n, int sm_count) {
    int64_t g = (n + AFR_TPB - 1) / AFR_TPB;
    if (g > (int64_t)sm_count * 16) g = (int64_t)sm_count * 16;
    return (unsigned)(g > 0 ? g : 1);
}

void afr_launch_decide(const uint8_t* text, const int64_t* line_start, int64_t n, const AfrDev& P, uint8_t* flags,
                       int64_t* len, int64_t* end, int64_t* out_ls, int64_t* agg, int64_t* totals,
                       unsigned long long* err, int sm_count, cudaStream_t st) {
    AFR_LAUNCH(afr_decide, afr_grid(n, sm_count), AFR_TPB, st, text, line_start, n, P, flags, len, end, err);
    afr_launch_scan(len, flags, n, out_ls, agg, totals, sm_count, st);
}

void afr_launch_scan(const int64_t* len, const uint8_t* flags, int64_t n, int64_t* out_ls, int64_t* agg, int64_t* totals,
                     int sm_count, cudaStream_t st) {
    const int64_t n_chunks = (n + AFR_CHUNK - 1) / AFR_CHUNK;
    AFR_LAUNCH(afr_agg, afr_grid(n_chunks, sm_count), AFR_TPB, st, len, flags, n, agg);
    AFR_LAUNCH(afr_spine, 1, 1, st, agg, n, totals);
    AFR_LAUNCH(afr_apply, afr_grid(n_chunks, sm_count), AFR_TPB, st, len, n, agg, out_ls);
}

void afr_launch_copy(const uint8_t* text, const int64_t* line_start, int64_t n, const AfrDev& P, const uint8_t* flags,
                     const int64_t* out_ls, uint8_t* out, int sm_count, cudaStream_t st) {
    AFR_LAUNCH(afr_copy, afr_grid(n, sm_count), AFR_TPB, st, text, line_start, n, P, flags, out_ls, out);
}

// ---- test hook: decide + scan + copy on caller records ------------------------------------------------------------------
namespace {
struct AfrBufs {  // frees on scope exit
    std::vector<void*> ptrs;
    ~AfrBufs() {
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

#define AFR_CU(call)                                 \
    do {                                             \
        if ((call) != cudaSuccess) return UGVC_E_CUDA; \
    } while (0)

extern "C" int64_t ugvc_test_afr(const uint8_t* text, size_t n_bytes, const int64_t* line_start, int64_t n,
                                 const ugvc_afr_params* params, uint8_t* out, size_t capacity, int64_t* out_line_start,
                                 uint8_t* out_failed, int64_t* out_end, int64_t* out_n_filtered, int64_t* out_err_record,
                                 int32_t* out_err_reason) {
    AfrDev P;
    if (!afr_params(params, &P) || n < 0 || !line_start || !out_line_start || !out_err_record || !out_err_reason ||
        (n && (!text || !out_failed || !out_end)))
        return UGVC_E_ARG;
    *out_err_record = -1;
    *out_err_reason = 0;
    if (line_start[0] != 0 || (size_t)line_start[n] != n_bytes) return UGVC_E_ARG;
    for (int64_t i = 0; i < n; ++i)
        if (line_start[i + 1] <= line_start[i] || text[line_start[i + 1] - 1] != '\n') return UGVC_E_ARG;
    AfrBufs b;
    uint8_t *d_text, *d_flags, *d_out;
    int64_t *d_ls, *d_len, *d_end, *d_out_ls, *d_agg, *d_tot;
    unsigned long long* d_err;
    AFR_CU(b.get(&d_text, n_bytes + 16));
    AFR_CU(b.get(&d_ls, (size_t)n + 1));
    AFR_CU(b.get(&d_flags, (size_t)n));
    AFR_CU(b.get(&d_len, (size_t)n + 1));
    AFR_CU(b.get(&d_end, (size_t)n));
    AFR_CU(b.get(&d_out_ls, (size_t)n + 1));
    AFR_CU(b.get(&d_agg, 2 * ((size_t)n / AFR_CHUNK + 2)));
    AFR_CU(b.get(&d_tot, 2));
    AFR_CU(b.get(&d_err, 1));
    AFR_CU(cudaMemcpy(d_text, text, n_bytes, cudaMemcpyHostToDevice));
    AFR_CU(cudaMemset(d_text + n_bytes, 0, 16));
    AFR_CU(cudaMemcpy(d_ls, line_start, ((size_t)n + 1) * sizeof(int64_t), cudaMemcpyHostToDevice));
    AFR_CU(cudaMemset(d_err, 0xFF, sizeof(unsigned long long)));
    AFR_CU(cudaMemset(d_tot, 0, 2 * sizeof(int64_t)));
    afr_launch_decide(d_text, d_ls, n, P, d_flags, d_len, d_end, d_out_ls, d_agg, d_tot, d_err, 132, nullptr);
    AFR_CU(cudaGetLastError());
    int64_t tot[2] = {0, 0};
    unsigned long long h_err = AFR_NO_ERROR;
    AFR_CU(cudaMemcpy(tot, d_tot, sizeof(tot), cudaMemcpyDeviceToHost));
    AFR_CU(cudaMemcpy(&h_err, d_err, sizeof(h_err), cudaMemcpyDeviceToHost));
    if (h_err != AFR_NO_ERROR) {
        *out_err_record = (int64_t)(h_err >> 4);
        *out_err_reason = (int32_t)(h_err & 0xF);
        return UGVC_E_DATA;
    }
    if ((size_t)tot[0] > capacity || (tot[0] && !out)) return UGVC_E_ARG;
    AFR_CU(b.get(&d_out, (size_t)tot[0]));
    afr_launch_copy(d_text, d_ls, n, P, d_flags, d_out_ls, d_out, 132, nullptr);
    AFR_CU(cudaGetLastError());
    if (tot[0]) AFR_CU(cudaMemcpy(out, d_out, (size_t)tot[0], cudaMemcpyDeviceToHost));
    AFR_CU(cudaMemcpy(out_line_start, d_out_ls, ((size_t)n + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost));
    if (n) {
        AFR_CU(cudaMemcpy(out_failed, d_flags, (size_t)n, cudaMemcpyDeviceToHost));
        for (int64_t i = 0; i < n; ++i) out_failed[i] &= AFR_FAILED;
        AFR_CU(cudaMemcpy(out_end, d_end, (size_t)n * sizeof(int64_t), cudaMemcpyDeviceToHost));
    }
    if (out_n_filtered) *out_n_filtered = tot[1];
    return tot[0];
}
