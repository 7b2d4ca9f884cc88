// gvcf_hcr.cu -- gvcf_hcr on the GPU (DESIGN.md 4e).
//
// Replaces ugvc/joint/gvcf_bed.py:gvcf_to_bed (a pysam loop over every record of a gVCF) and the bedtools merge of
// ugvc/pipelines/vcfbed/gvcf_hcr_main.py.  A record is skipped when it starts before the end of the last record of its
// contig that was not skipped, so whether a record is kept depends on every earlier record of the contig.  The kept flags
// come from reset points instead of a walk over the contig: a record that starts at or after the end of every earlier
// record of its contig (a prefix maximum) is kept whatever came before.  Between two reset points one thread walks the
// reference's rule; a segment longer than a bound is resolved by pointer doubling over next-kept pointers.  Every kernel
// is CUB-free with grid-stride loops, so that the host emulation runs this source:
//   hcr_decide                  per record: CHROM against the previous line, the interval (INFO/END, the RefCall
//                               deletion rule on sample 0's GQ / GT), the selection and what would raise
//   hcr_pm_agg / _spine / _apply  the per-contig exclusive prefix maximum of the ends (chunked three-phase scan)
//   -- the scan call ends here; the emit call takes the entry state from the previous piece --
//   hcr_reset                   reset points, the first contig run seeded with the entry extent
//   hcr_walk                    one thread per reset point walks its segment up to the bound
//   hcr_seg_end, hcr_next, hcr_jump, hcr_mark, hcr_kept   the long segments: end, next-kept pointers, jump tables,
//                               chain marking from the highest level down
//   hcr_em_agg / _spine / _apply  kept -> selected -> output lines (merge marks), skipped count, GQ errors of kept records
//   hcr_bed_len, afr_launch_scan, hcr_bed_copy   the BED lines: lengths, offsets, text
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "gvcf_hcr.cuh"
#include "low_af_ratio.cuh"
#include "numparse.h"
#include "vcf_text.cuh"

#define HCR_TPB 256

#ifdef UGVC_HOST_EMU
#define HCR_LAUNCH(kern, grid, block, st, ...)                  \
    do {                                                        \
        threadIdx = dim3(0, 0, 0); blockIdx = dim3(0, 0, 0);     \
        blockDim = dim3(1, 1, 1); gridDim = dim3(1, 1, 1);       \
        kern(__VA_ARGS__);                                      \
    } while (0)
#else
#define HCR_LAUNCH(kern, grid, block, st, ...) kern<<<grid, block, 0, st>>>(__VA_ARGS__)
#endif

enum : uint8_t {
    HCR_SEL = UGVC_HCR_SELECTED,
    HCR_GQERR = UGVC_HCR_GQ_ERROR,
    HCR_NEWC = UGVC_HCR_NEW_CONTIG,
    HCR_RESET = UGVC_HCR_RESET,
    HCR_KEPT = UGVC_HCR_KEPT,
    HCR_LINE = UGVC_HCR_LINE
};

bool hcr_params(const ugvc_hcr_params* p, HcrDev* d) {
    if (!p || !d) return false;
    if (p->gq_kind < UGVC_HCR_GQ_STRING || p->gq_kind > UGVC_HCR_GQ_TUPLE) return false;
    d->gq_threshold = p->gq_threshold;
    d->gt = p->gt ? 1 : 0;
    d->merge = p->merge ? 1 : 0;
    d->info_end = p->info_end ? 1 : 0;
    d->gq_kind = p->gq_kind;
    d->gq_integer = p->gq_integer ? 1 : 0;
    return true;
}

__device__ __forceinline__ void hcr_error(int64_t* err, int64_t i, int reason) {
    atomicMin(reinterpret_cast<unsigned long long*>(err), ((unsigned long long)i << 4) | (unsigned long long)reason);
}

__device__ __forceinline__ int64_t hcr_digits(const uint8_t* p, int64_t n) {
    int64_t v = 0;
    for (int64_t k = 0; k < n && v < ((int64_t)1 << 50); ++k) v = v * 10 + (p[k] - '0');
    return v;
}

__global__ void __launch_bounds__(HCR_TPB) hcr_decide(const uint8_t* __restrict__ t, const int64_t* __restrict__ ls, int64_t n,
                                                      HcrDev P, int64_t* __restrict__ start_out, int64_t* __restrict__ end_out,
                                                      uint8_t* __restrict__ flags, int64_t* __restrict__ runs,
                                                      int64_t* __restrict__ stat) {
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
        if (new_contig) {
            const unsigned long long k = atomicAdd(reinterpret_cast<unsigned long long*>(stat + HCR_STAT_N_RUNS), 1ull);
            runs[2 * k] = i;
            runs[2 * k + 1] = a;
        }
        // columns 1 (POS) .. 9 (sample 0): [c0[k], c1[k])
        int64_t c0[10], c1[10];
        int nc = 1;
        for (++at; nc < 10 && at <= e; ++nc, ++at) {
            const int64_t b = at;
            while (at < e && t[at] != '\t') ++at;
            c0[nc] = b, c1[nc] = at;
        }
        if (nc < 8) {  // fewer than 8 columns: refused by the index pass before this kernel runs
            start_out[i] = 0;
            end_out[i] = 1;
            flags[i] = new_contig ? HCR_NEWC : 0;
            continue;
        }
        const int64_t start = hcr_digits(t + c0[1], c1[1] - c0[1]) - 1;
        int reason = 0;
        if (!new_contig) {  // POS of the previous line, on the same contig
            int64_t q = ls[i - 1] + chrom_len + 1, pp = 0;
            while (t[q] >= '0' && t[q] <= '9' && pp < ((int64_t)1 << 50)) pp = pp * 10 + (t[q++] - '0');
            if (start + 1 < pp) reason = UGVC_HCR_E_UNSORTED;
        }
        // INFO: the first END= (1..10 digits), the index rule
        const int64_t ref_len = c1[3] - c0[3];
        int64_t stop = start + (ref_len > 1 ? ref_len : 1);
        if (P.info_end) {
            const uint8_t* in = t + c0[7];
            const int64_t il = c1[7] - c0[7];
            int64_t endv = 0;
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
            if (endv > start) stop = endv;
        }
        // FORMAT: where GQ and GT sit; sample 0's sub-fields
        int gq_at = -1, gt_at = -1;
        const uint8_t *gq_p = nullptr, *gt_p = nullptr;
        int64_t gq_n = 0, gt_n = 0;
        bool gq_sub = false, gt_sub = false;
        if (nc >= 9 && !(c1[8] - c0[8] == 1 && t[c0[8]] == '.')) {
            const uint8_t* fm = t + c0[8];
            const int64_t fml = c1[8] - c0[8];
            int k = 0;
            for (int64_t q = 0; q <= fml; ++k) {
                const int64_t b = q, m = afr_piece(fm, &q, fml, ':');
                if (gq_at < 0 && afr_eq(fm + b, m, (const uint8_t*)"GQ", 2)) gq_at = k;
                else if (gt_at < 0 && afr_eq(fm + b, m, (const uint8_t*)"GT", 2)) gt_at = k;
            }
            if (nc == 10) {
                k = 0;
                for (int64_t q = c0[9]; q <= c1[9]; ++k) {
                    const int64_t b = q, m = afr_piece(t, &q, c1[9], ':');
                    if (k == gq_at) gq_p = t + b, gq_n = m, gq_sub = true;
                    if (k == gt_at) gt_p = t + b, gt_n = m, gt_sub = true;
                }
            }
        }
        // GQ typed as pysam types it; a scalar number is the only value that compares
        const bool gq_in = gq_at >= 0;
        bool bad = false;
        bool gq_num = false;
        double gq_f = 0.0;
        int64_t gq_i = 0;
        if (gq_in && P.gq_kind != UGVC_HCR_GQ_STRING) {
            const AfrVal v = afr_value(P.gq_kind, P.gq_integer, gq_sub, gq_p, gq_n, &bad);
            if (v.kind == 1 && !bad) {
                gq_num = true;
                if (P.gq_integer) {
                    const bool neg = v.p[0] == '-';
                    const int64_t k0 = (v.p[0] == '-' || v.p[0] == '+') ? 1 : 0;
                    gq_i = hcr_digits(v.p + k0, v.n - k0);
                    if (neg) gq_i = -gq_i;
                } else {
                    afr_number(v.p, v.n, 0, &gq_f);
                }
            }
        }
        // GT: (0, 0), (None, None) or anything else; read only by the RefCall test, typed for every record
        bool g00 = false, gnn = false;
        if (gt_sub) {
            int64_t alleles = 0, zeros = 0, nones = 0;
            for (int64_t q = 0; q <= gt_n;) {
                const int64_t b = q;
                while (q < gt_n && gt_p[q] != '/' && gt_p[q] != '|') ++q;
                const int64_t m = q - b;
                ++q;
                ++alleles;
                if (m == 0 || (m == 1 && gt_p[b] == '.')) {
                    ++nones;
                    continue;
                }
                bool zero = true;
                for (int64_t d = b; d < b + m; ++d) {
                    if (gt_p[d] < '0' || gt_p[d] > '9' || m > 9) bad = true;
                    zero &= gt_p[d] == '0';
                }
                zeros += zero;
            }
            g00 = alleles == 2 && zeros == 2;
            gnn = alleles == 2 && nones == 2;
        }
        // the RefCall deletion: its interval is its first base
        bool refcall = false;
        if (ref_len > 1) {
            if (!gq_in) refcall = true;
            else if (gt_at < 0) reason = reason ? reason : UGVC_HCR_E_KEY;
            else refcall = g00 || gnn;
        }
        if (bad) reason = UGVC_HCR_E_LITERAL;
        if (reason) hcr_error(stat + HCR_STAT_ERR, i, reason);
        bool sel;
        if (P.gt) sel = gq_num && (P.gq_integer ? gq_i >= P.gq_threshold : gq_f >= (double)P.gq_threshold);
        else sel = !gq_in || (gq_num && (P.gq_integer ? gq_i < P.gq_threshold : gq_f < (double)P.gq_threshold));
        start_out[i] = start;
        end_out[i] = refcall ? start + 1 : stop;
        flags[i] = (uint8_t)((sel ? HCR_SEL : 0) | (gq_in && !gq_num ? HCR_GQERR : 0) | (new_contig ? HCR_NEWC : 0));
    }
}

// ---- per-contig exclusive prefix maximum of the ends, chunks of AFR_CHUNK records -----------------------------------------
// agg[4c] = the last record of chunk c that starts a contig run (-1: none), agg[4c + 1] = the max end after it (of the
// whole chunk when none), agg[4c + 2] = the first record > 0 of the chunk that starts a contig run (n: none)
__global__ void hcr_pm_agg(const int64_t* __restrict__ end, const uint8_t* __restrict__ flags, int64_t n, int64_t* __restrict__ agg) {
    const int64_t n_chunks = (n + AFR_CHUNK - 1) / AFR_CHUNK;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks; c += stride) {
        const int64_t e = (c + 1) * AFR_CHUNK < n ? (c + 1) * AFR_CHUNK : n;
        int64_t last = -1, mx = -1, first = n;
        for (int64_t i = c * AFR_CHUNK; i < e; ++i) {
            if (flags[i] & HCR_NEWC) {
                last = i;
                mx = -1;
                if (i > 0 && first == n) first = i;
            }
            mx = end[i] > mx ? end[i] : mx;
        }
        agg[4 * c] = last;
        agg[4 * c + 1] = mx;
        agg[4 * c + 2] = first;
    }
}
// carry-in of each chunk into agg[4c] (run start) and agg[4c + 1] (max); the summary fields of the scan
__global__ void hcr_pm_spine(int64_t* agg, const int64_t* start, int64_t n, int64_t* stat) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    const int64_t n_chunks = (n + AFR_CHUNK - 1) / AFR_CHUNK;
    int64_t run = 0, mx = -1, r0 = n;
    for (int64_t c = 0; c < n_chunks; ++c) {
        const int64_t last = agg[4 * c], m = agg[4 * c + 1], first = agg[4 * c + 2];
        agg[4 * c] = run;
        agg[4 * c + 1] = mx;
        if (last >= 0) {
            run = last;
            mx = m;
        } else {
            mx = m > mx ? m : mx;
        }
        r0 = first < r0 ? first : r0;
    }
    stat[HCR_STAT_R0] = r0;
    stat[HCR_STAT_FIRST_START] = n ? start[0] : -1;
    stat[HCR_STAT_LAST_START] = n ? start[n - 1] : -1;
}
__global__ void hcr_pm_apply(const int64_t* __restrict__ end, const uint8_t* __restrict__ flags, int64_t n,
                             const int64_t* __restrict__ agg, int64_t* __restrict__ pm, int32_t* __restrict__ rs) {
    const int64_t n_chunks = (n + AFR_CHUNK - 1) / AFR_CHUNK;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks; c += stride) {
        const int64_t e = (c + 1) * AFR_CHUNK < n ? (c + 1) * AFR_CHUNK : n;
        int64_t run = agg[4 * c], mx = agg[4 * c + 1];
        for (int64_t i = c * AFR_CHUNK; i < e; ++i) {
            if (flags[i] & HCR_NEWC) {
                run = i;
                mx = -1;
            }
            pm[i] = mx;
            rs[i] = (int32_t)run;
            mx = end[i] > mx ? end[i] : mx;
        }
    }
}

// ---- kept flags ----------------------------------------------------------------------------------------------------------
// A record is a reset point when it starts at or after every earlier end of its contig run in the piece and, in a first
// run that continues the previous piece's contig, at or after the entry extent.
__global__ void hcr_reset(const int64_t* __restrict__ start, const int64_t* __restrict__ pm, int64_t n, int64_t r0, int cont,
                          int64_t entry, uint8_t* __restrict__ flags) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        int64_t m = pm[i];
        if (cont && i < r0 && entry > m) m = entry;
        flags[i] = (uint8_t)((flags[i] & (HCR_SEL | HCR_GQERR | HCR_NEWC)) | (start[i] >= m ? HCR_RESET : 0));
    }
}

// Thread k heads record k - 1 when that is a reset point (k = 0: the piece's entry state, when record 0 is not one) and
// walks the reference's rule up to the next reset point, at most `bound` records; a longer segment's head is queued in
// seg[] for the parallel form.
__global__ void __launch_bounds__(HCR_TPB) hcr_walk(const int64_t* __restrict__ start, const int64_t* __restrict__ end,
                                                    uint8_t* flags, int64_t n, int cont, int64_t entry, int64_t bound,
                                                    int64_t* __restrict__ seg, int64_t* __restrict__ stat) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k <= n; k += stride) {
        const int64_t h = k - 1;
        int64_t extent;
        if (h < 0) {
            if (!(cont && n > 0 && !(flags[0] & HCR_RESET))) continue;
            extent = entry;
        } else {
            if (!(flags[h] & HCR_RESET)) continue;
            flags[h] |= HCR_KEPT;
            extent = end[h];
        }
        int64_t j = h + 1, walked = 0;
        while (j < n && !(flags[j] & HCR_RESET) && walked < bound) {
            if (start[j] >= extent) {
                flags[j] |= HCR_KEPT;
                extent = end[j];
            }
            ++j;
            ++walked;
        }
        if (j < n && !(flags[j] & HCR_RESET)) {
            const unsigned long long s = atomicAdd(reinterpret_cast<unsigned long long*>(stat + HCR_STAT_N_LONG), 1ull);
            seg[s] = h;
        } else {
            atomicMax(reinterpret_cast<unsigned long long*>(stat + HCR_STAT_MAX_SEG), (unsigned long long)(j - (h < 0 ? 0 : h)));
        }
    }
}

// index of the last s in [0, m) with v[s] <= x (v ascending; -1 when none)
__device__ __forceinline__ int64_t hcr_last_le(const int64_t* v, int64_t m, int64_t x) {
    int64_t lo = 0, hi = m;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (v[mid] <= x) lo = mid + 1;
        else hi = mid;
    }
    return lo - 1;
}

// tend[s] = the first reset point after head[s] (n when none): heads ascending, tend preset to n
__global__ void hcr_seg_end(const uint8_t* __restrict__ flags, int64_t n, const int64_t* __restrict__ head, int64_t m, int64_t* tend) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
        if (!(flags[j] & HCR_RESET)) continue;
        const int64_t s = hcr_last_le(head, m, j - 1);
        if (s >= 0) atomicMin(reinterpret_cast<long long*>(tend + s), (long long)j);
    }
}

// The long segments as one flat array: segment s holds its head (record head[s], or the entry state for head -1) and the
// records after it up to tend[s], at flat positions off[s] .. off[s + 1).  J0[f] = the flat position of the next kept
// record after f's (the first later record of the segment that starts at or after f's end: binary search over the sorted
// starts), T when none; lvl[f] = top + 2 for heads, 0 elsewhere.
__global__ void hcr_next(const int64_t* __restrict__ start, const int64_t* __restrict__ end, const int64_t* __restrict__ head,
                         const int64_t* __restrict__ tend, const int64_t* __restrict__ off, int64_t m, int64_t T, int64_t entry,
                         int top, int32_t* __restrict__ J0, int8_t* __restrict__ lvl) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f <= T; f += stride) {
        if (f == T) {
            J0[T] = (int32_t)T;
            lvl[T] = 0;
            continue;
        }
        const int64_t s = hcr_last_le(off, m, f);
        const int64_t i = head[s] + (f - off[s]);
        const int64_t e = i < 0 ? entry : end[i];
        int64_t lo = i + 1, hi = tend[s];
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (start[mid] >= e) hi = mid;
            else lo = mid + 1;
        }
        J0[f] = (int32_t)(lo < tend[s] ? off[s] + (lo - head[s]) : T);
        lvl[f] = (int8_t)(f == off[s] ? top + 2 : 0);
    }
}
__global__ void hcr_jump(const int32_t* __restrict__ prev, int32_t* __restrict__ next, int64_t T) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f <= T; f += stride) next[f] = prev[prev[f]];
}
// level k: every chain position marked at a higher level (lvl >= k + 2) marks the one 2^k links further
__global__ void hcr_mark(const int32_t* __restrict__ Jk, int8_t* lvl, int64_t T, int k) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < T; f += stride) {
        if (lvl[f] < k + 2) continue;
        const int32_t y = Jk[f];
        if (y != T && lvl[y] == 0) lvl[y] = (int8_t)(k + 1);
    }
}
__global__ void hcr_kept(const int64_t* __restrict__ head, const int64_t* __restrict__ off, int64_t m, int64_t T,
                         const int8_t* __restrict__ lvl, uint8_t* flags) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < T; f += stride) {
        if (!lvl[f]) continue;
        const int64_t s = hcr_last_le(off, m, f);
        const int64_t i = head[s] + (f - off[s]);
        if (i >= 0) flags[i] |= HCR_KEPT;
    }
}

// ---- selection, merge marks, skipped count --------------------------------------------------------------------------------
// Selected record i starts an output line unless merging and the previous kept record p is selected, on the same contig
// run and ends where i starts (bedtools merge -d 0: kept records never overlap, so only book-ended ones join)
__device__ __forceinline__ bool hcr_starts_line(const int64_t* start, const int64_t* end, const uint8_t* flags, const int32_t* rs,
                                                int merge, int64_t p, int64_t i) {
    return !merge || !(p >= 0 && (flags[p] & HCR_SEL) && rs[p] == rs[i] && end[p] == start[i]);
}
// agg[5c] = first kept record of chunk c (-1: none), agg[5c + 1] = last kept, agg[5c + 2] = lines started by the chunk's
// later selected records, agg[5c + 3] = skipped records
__global__ void hcr_em_agg(const int64_t* __restrict__ start, const int64_t* __restrict__ end, const uint8_t* __restrict__ flags,
                           const int32_t* __restrict__ rs, int64_t n, int merge, int64_t* __restrict__ agg) {
    const int64_t n_chunks = (n + AFR_CHUNK - 1) / AFR_CHUNK;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks; c += stride) {
        const int64_t e = (c + 1) * AFR_CHUNK < n ? (c + 1) * AFR_CHUNK : n;
        int64_t fk = -1, lk = -1, lines = 0, skipped = 0;
        for (int64_t i = c * AFR_CHUNK; i < e; ++i) {
            const uint8_t fl = flags[i];
            if (!(fl & HCR_KEPT)) {
                ++skipped;
                continue;
            }
            if (fk < 0) fk = i;
            else if (fl & HCR_SEL) lines += hcr_starts_line(start, end, flags, rs, merge, lk, i);
            lk = i;
        }
        agg[5 * c] = fk;
        agg[5 * c + 1] = lk;
        agg[5 * c + 2] = lines;
        agg[5 * c + 3] = skipped;
    }
}
// carry-in of each chunk: agg[5c + 1] = the last kept record before it, agg[5c + 2] = the lines before it, agg[5c + 4] =
// whether its first kept record starts a line; the emit's summary fields
__global__ void hcr_em_spine(const int64_t* start, const int64_t* end, const uint8_t* flags, const int32_t* rs, int64_t n,
                             int merge, int64_t* agg, int64_t* stat) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    const int64_t n_chunks = (n + AFR_CHUNK - 1) / AFR_CHUNK;
    int64_t p = -1, lines = 0, skipped = 0;
    for (int64_t c = 0; c < n_chunks; ++c) {
        const int64_t fk = agg[5 * c], lk = agg[5 * c + 1], later = agg[5 * c + 2];
        skipped += agg[5 * c + 3];
        agg[5 * c + 1] = p;
        agg[5 * c + 2] = lines;
        agg[5 * c + 4] = 0;
        if (fk < 0) continue;
        const bool first = (flags[fk] & HCR_SEL) && hcr_starts_line(start, end, flags, rs, merge, p, fk);
        agg[5 * c + 4] = first;
        lines += first + later;
        p = lk;
    }
    stat[HCR_STAT_N_LINES] = lines;
    stat[HCR_STAT_SKIPPED] = skipped;
    stat[HCR_STAT_LAST_KEPT] = p;
    stat[HCR_STAT_LAST_END] = p >= 0 ? end[p] : -1;
}
// line r's first record (ms_rec) and end (run_end, preset to 0: atomicMax over its records, whose ends increase); the GQ
// comparison of every kept record
__global__ void hcr_em_apply(const int64_t* __restrict__ start, const int64_t* __restrict__ end, uint8_t* flags,
                             const int32_t* __restrict__ rs, int64_t n, int merge, const int64_t* __restrict__ agg,
                             int32_t* __restrict__ ms_rec, int64_t* run_end, int64_t* stat) {
    const int64_t n_chunks = (n + AFR_CHUNK - 1) / AFR_CHUNK;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks; c += stride) {
        const int64_t e = (c + 1) * AFR_CHUNK < n ? (c + 1) * AFR_CHUNK : n;
        int64_t p = agg[5 * c + 1], r = agg[5 * c + 2];
        bool first = true;
        for (int64_t i = c * AFR_CHUNK; i < e; ++i) {
            const uint8_t fl = flags[i];
            if (!(fl & HCR_KEPT)) continue;
            if (fl & HCR_GQERR) hcr_error(stat + HCR_STAT_ERR, i, UGVC_HCR_E_TYPE);
            if (fl & HCR_SEL) {
                const bool line = first ? agg[5 * c + 4] != 0 : hcr_starts_line(start, end, flags, rs, merge, p, i);
                if (line) {
                    flags[i] = fl | HCR_LINE;
                    ms_rec[r++] = (int32_t)i;
                }
                atomicMax(reinterpret_cast<long long*>(run_end + r - 1), (long long)end[i]);
            }
            first = false;
            p = i;
        }
    }
}

// ---- the BED lines --------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int hcr_ndig(int64_t v) {
    int d = 1;
    for (; v >= 10; v /= 10) ++d;
    return d;
}
__device__ __forceinline__ uint8_t* hcr_put(uint8_t* o, int64_t v) {
    const int d = hcr_ndig(v);
    for (int k = d - 1; k >= 0; --k, v /= 10) o[k] = (uint8_t)('0' + v % 10);
    return o + d;
}
__device__ __forceinline__ int64_t hcr_chrom_len(const uint8_t* t, int64_t a) {
    int64_t q = a;
    while (t[q] != '\t') ++q;
    return q - a;
}
__global__ void hcr_bed_len(const uint8_t* __restrict__ t, const int64_t* __restrict__ ls, const int64_t* __restrict__ start,
                            const int32_t* __restrict__ ms_rec, const int64_t* __restrict__ run_end, int64_t R,
                            int64_t* __restrict__ len) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < R; r += stride) {
        const int64_t i = ms_rec[r];
        len[r] = hcr_chrom_len(t, ls[i]) + hcr_ndig(start[i]) + hcr_ndig(run_end[r]) + 3;
    }
}
__global__ void hcr_bed_copy(const uint8_t* __restrict__ t, const int64_t* __restrict__ ls, const int64_t* __restrict__ start,
                             const int32_t* __restrict__ ms_rec, const int64_t* __restrict__ run_end, int64_t R,
                             const int64_t* __restrict__ out_ls, uint8_t* __restrict__ out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < R; r += stride) {
        const int64_t i = ms_rec[r], a = ls[i], cl = hcr_chrom_len(t, a);
        uint8_t* o = out + out_ls[r];
        memcpy(o, t + a, (size_t)cl);
        o += cl;
        *o++ = '\t';
        o = hcr_put(o, start[i]);
        *o++ = '\t';
        o = hcr_put(o, run_end[r]);
        *o = '\n';
    }
}

// ---- host halves ----------------------------------------------------------------------------------------------------------
static unsigned hcr_grid(int64_t n, int sm_count) {
    int64_t g = (n + HCR_TPB - 1) / HCR_TPB;
    if (g > (int64_t)sm_count * 16) g = (int64_t)sm_count * 16;
    return (unsigned)(g > 0 ? g : 1);
}

void hcr_bufs_free(HcrBufs* b) {
    cudaFree(b->start);
    cudaFree(b->end);
    cudaFree(b->pm);
    cudaFree(b->rs);
    cudaFree(b->flags);
    cudaFree(b->runs);
    cudaFree(b->ms_rec);
    cudaFree(b->run_end);
    cudaFree(b->len);
    cudaFree(b->out_ls);
    cudaFree(b->agg);
    cudaFree(b->seg);
    cudaFree(b->stat);
    cudaFree(b->jump);
    cudaFree(b->lvl);
    *b = HcrBufs();
}

cudaError_t hcr_bufs_reserve(HcrBufs* b, size_t cap) {
    if (cap <= b->cap && b->stat) return cudaSuccess;
    hcr_bufs_free(b);
    cap = cap ? cap : 1;
    cudaError_t e;
    if ((e = cudaMalloc(&b->start, cap * sizeof(int64_t))) != cudaSuccess) return e;
    if ((e = cudaMalloc(&b->end, cap * sizeof(int64_t))) != cudaSuccess) return e;
    if ((e = cudaMalloc(&b->pm, cap * sizeof(int64_t))) != cudaSuccess) return e;
    if ((e = cudaMalloc(&b->rs, cap * sizeof(int32_t))) != cudaSuccess) return e;
    if ((e = cudaMalloc(&b->flags, cap)) != cudaSuccess) return e;
    if ((e = cudaMalloc(&b->runs, 2 * cap * sizeof(int64_t))) != cudaSuccess) return e;
    if ((e = cudaMalloc(&b->ms_rec, cap * sizeof(int32_t))) != cudaSuccess) return e;
    if ((e = cudaMalloc(&b->run_end, cap * sizeof(int64_t))) != cudaSuccess) return e;
    if ((e = cudaMalloc(&b->len, (cap + 1) * sizeof(int64_t))) != cudaSuccess) return e;
    if ((e = cudaMalloc(&b->out_ls, (cap + 1) * sizeof(int64_t))) != cudaSuccess) return e;
    if ((e = cudaMalloc(&b->agg, 5 * (cap / AFR_CHUNK + 2) * sizeof(int64_t))) != cudaSuccess) return e;
    if ((e = cudaMalloc(&b->seg, 3 * (cap + 2) * sizeof(int64_t))) != cudaSuccess) return e;
    if ((e = cudaMalloc(&b->stat, HCR_STAT_N * sizeof(int64_t))) != cudaSuccess) return e;
    b->cap = cap;
    return cudaSuccess;
}

void hcr_launch_scan(const uint8_t* text, const int64_t* line_start, int64_t n, const HcrDev& P, HcrBufs* b, int sm_count,
                     cudaStream_t st) {
    cudaMemsetAsync(b->stat, 0, HCR_STAT_N * sizeof(int64_t), st);
    cudaMemsetAsync(b->stat + HCR_STAT_ERR, 0xFF, sizeof(int64_t), st);
    b->text = text;
    b->line_start = line_start;
    b->n = n;
    const int64_t n_chunks = (n + AFR_CHUNK - 1) / AFR_CHUNK;
    HCR_LAUNCH(hcr_decide, hcr_grid(n, sm_count), HCR_TPB, st, text, line_start, n, P, b->start, b->end, b->flags, b->runs, b->stat);
    HCR_LAUNCH(hcr_pm_agg, hcr_grid(n_chunks, sm_count), HCR_TPB, st, b->end, b->flags, n, b->agg);
    HCR_LAUNCH(hcr_pm_spine, 1, 1, st, b->agg, b->start, n, b->stat);
    HCR_LAUNCH(hcr_pm_apply, hcr_grid(n_chunks, sm_count), HCR_TPB, st, b->end, b->flags, n, b->agg, b->pm, b->rs);
}

#define HCR_CU(call)                                 \
    do {                                             \
        cudaError_t _e = (call);                     \
        if (_e != cudaSuccess) return _e;            \
    } while (0)

// the long segments queued by hcr_walk: their ends, then pointer doubling over one flat array of all of them
static cudaError_t hcr_long_segments(HcrBufs* b, int64_t m, int64_t entry, int64_t* longest, int sm_count, cudaStream_t st) {
    const int64_t n = b->n;
    int64_t* head = b->seg;
    int64_t* tend = b->seg + (n + 2);
    int64_t* off = b->seg + 2 * (n + 2);
    std::vector<int64_t> h((size_t)m), t((size_t)m, n), o((size_t)m + 1, 0);
    HCR_CU(cudaMemcpyAsync(h.data(), head, (size_t)m * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    HCR_CU(cudaStreamSynchronize(st));
    std::sort(h.begin(), h.end());
    HCR_CU(cudaMemcpyAsync(head, h.data(), (size_t)m * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    HCR_CU(cudaMemcpyAsync(tend, t.data(), (size_t)m * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    HCR_LAUNCH(hcr_seg_end, hcr_grid(n, sm_count), HCR_TPB, st, b->flags, n, head, m, tend);
    HCR_CU(cudaMemcpyAsync(t.data(), tend, (size_t)m * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    HCR_CU(cudaStreamSynchronize(st));
    int64_t max_len = 0;
    for (int64_t s = 0; s < m; ++s) {
        const int64_t L = t[(size_t)s] - h[(size_t)s];  // the head (or the entry state) and the records after it
        o[(size_t)s + 1] = o[(size_t)s] + L;
        max_len = L > max_len ? L : max_len;
        const int64_t seg_len = t[(size_t)s] - (h[(size_t)s] < 0 ? 0 : h[(size_t)s]);
        *longest = seg_len > *longest ? seg_len : *longest;
    }
    const int64_t T = o[(size_t)m];
    int levels = 1;
    while (((int64_t)1 << levels) <= max_len) ++levels;  // 2^levels > every chain length
    const size_t need_jump = (size_t)levels * (size_t)(T + 1), need_lvl = (size_t)(T + 1);
    if (need_jump > b->cap_jump) {
        cudaFree(b->jump);
        b->jump = nullptr;
        b->cap_jump = 0;
        HCR_CU(cudaMalloc(&b->jump, need_jump * sizeof(int32_t)));
        b->cap_jump = need_jump;
    }
    if (need_lvl > b->cap_lvl) {
        cudaFree(b->lvl);
        b->lvl = nullptr;
        b->cap_lvl = 0;
        HCR_CU(cudaMalloc(&b->lvl, need_lvl));
        b->cap_lvl = need_lvl;
    }
    HCR_CU(cudaMemcpyAsync(off, o.data(), ((size_t)m + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    const unsigned g = hcr_grid(T + 1, sm_count);
    HCR_LAUNCH(hcr_next, g, HCR_TPB, st, b->start, b->end, head, tend, off, m, T, entry, levels - 1, b->jump, b->lvl);
    for (int k = 1; k < levels; ++k)
        HCR_LAUNCH(hcr_jump, g, HCR_TPB, st, b->jump + (size_t)(k - 1) * (T + 1), b->jump + (size_t)k * (T + 1), T);
    for (int k = levels - 1; k >= 0; --k) HCR_LAUNCH(hcr_mark, g, HCR_TPB, st, b->jump + (size_t)k * (T + 1), b->lvl, T, k);
    HCR_LAUNCH(hcr_kept, g, HCR_TPB, st, head, off, m, T, b->lvl, b->flags);
    HCR_CU(cudaStreamSynchronize(st));  // before h, t and o go
    return cudaSuccess;
}

cudaError_t hcr_emit(HcrBufs* b, const HcrDev& P, int continues_contig, int64_t entry_extent, int64_t seg_bound, uint8_t* out,
                     size_t out_capacity, HcrEmitOut* res, int sm_count, cudaStream_t st) {
    const int64_t n = b->n;
    const int cont = continues_contig ? 1 : 0;
    const int64_t entry = cont ? entry_extent : -1;
    const int64_t n_chunks = (n + AFR_CHUNK - 1) / AFR_CHUNK;
    int64_t h_stat[HCR_STAT_N];
    HCR_CU(cudaMemcpyAsync(h_stat, b->stat, sizeof(h_stat), cudaMemcpyDeviceToHost, st));
    HCR_CU(cudaStreamSynchronize(st));
    const int64_t r0 = h_stat[HCR_STAT_R0];
    HCR_LAUNCH(hcr_reset, hcr_grid(n, sm_count), HCR_TPB, st, b->start, b->pm, n, r0, cont, entry, b->flags);
    HCR_LAUNCH(hcr_walk, hcr_grid(n + 1, sm_count), HCR_TPB, st, b->start, b->end, b->flags, n, cont, entry,
               seg_bound > 0 ? seg_bound : (int64_t)HCR_SEG_BOUND, b->seg, b->stat);
    HCR_CU(cudaMemcpyAsync(h_stat, b->stat, sizeof(h_stat), cudaMemcpyDeviceToHost, st));
    HCR_CU(cudaStreamSynchronize(st));
    int64_t longest = h_stat[HCR_STAT_MAX_SEG];
    if (h_stat[HCR_STAT_N_LONG] > 0) HCR_CU(hcr_long_segments(b, h_stat[HCR_STAT_N_LONG], entry, &longest, sm_count, st));
    HCR_CU(cudaMemsetAsync(b->run_end, 0, (size_t)(n ? n : 1) * sizeof(int64_t), st));
    HCR_LAUNCH(hcr_em_agg, hcr_grid(n_chunks, sm_count), HCR_TPB, st, b->start, b->end, b->flags, b->rs, n, P.merge, b->agg);
    HCR_LAUNCH(hcr_em_spine, 1, 1, st, b->start, b->end, b->flags, b->rs, n, P.merge, b->agg, b->stat);
    HCR_LAUNCH(hcr_em_apply, hcr_grid(n_chunks, sm_count), HCR_TPB, st, b->start, b->end, b->flags, b->rs, n, P.merge, b->agg,
               b->ms_rec, b->run_end, b->stat);
    HCR_CU(cudaMemcpyAsync(h_stat, b->stat, sizeof(h_stat), cudaMemcpyDeviceToHost, st));
    HCR_CU(cudaStreamSynchronize(st));
    res->err = h_stat[HCR_STAT_ERR];
    res->n_lines = h_stat[HCR_STAT_N_LINES];
    res->skipped = h_stat[HCR_STAT_SKIPPED];
    res->last_kept = h_stat[HCR_STAT_LAST_KEPT];
    res->exit_extent = res->last_kept >= 0 ? h_stat[HCR_STAT_LAST_END] : entry;
    res->longest = longest;
    res->bytes = 0;
    if ((unsigned long long)res->err != AFR_NO_ERROR) return cudaSuccess;
    const int64_t R = res->n_lines;
    HCR_LAUNCH(hcr_bed_len, hcr_grid(R, sm_count), HCR_TPB, st, b->text, b->line_start, b->start, b->ms_rec, b->run_end, R, b->len);
    afr_launch_scan(b->len, b->flags, R, b->out_ls, b->agg, b->stat + HCR_STAT_BYTES, sm_count, st);
    HCR_CU(cudaMemcpyAsync(&res->bytes, b->stat + HCR_STAT_BYTES, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    HCR_CU(cudaStreamSynchronize(st));
    if (R == 0) res->bytes = 0;
    if ((size_t)res->bytes > out_capacity) return cudaErrorMemoryAllocation;
    HCR_LAUNCH(hcr_bed_copy, hcr_grid(R, sm_count), HCR_TPB, st, b->text, b->line_start, b->start, b->ms_rec, b->run_end, R,
               b->out_ls, out);
    return cudaGetLastError();
}

// ---- test hook: scan + emit on caller records -----------------------------------------------------------------------------
extern "C" int64_t ugvc_test_hcr(const uint8_t* text, size_t n_bytes, const int64_t* line_start, int64_t n, const ugvc_hcr_params* params,
                                 int continues_contig, int64_t entry_extent, int64_t seg_bound, uint8_t* out, size_t capacity,
                                 uint8_t* out_flags, int64_t out_stats[4], int64_t* out_err_record, int32_t* out_err_reason) {
    HcrDev P;
    if (!hcr_params(params, &P) || n < 0 || !line_start || !out_stats || !out_err_record || !out_err_reason ||
        (n && (!text || !out_flags)))
        return UGVC_E_ARG;
    *out_err_record = -1;
    *out_err_reason = 0;
    if (line_start[0] != 0 || (size_t)line_start[n] != n_bytes) return UGVC_E_ARG;
    for (int64_t i = 0; i < n; ++i)
        if (line_start[i + 1] <= line_start[i] || text[line_start[i + 1] - 1] != '\n') return UGVC_E_ARG;
    HcrBufs b;
    uint8_t *d_text = nullptr, *d_out = nullptr;
    int64_t* d_ls = nullptr;
    const size_t out_cap = n_bytes + 48 * (size_t)n + 16;
    int64_t rc = UGVC_E_CUDA;
    HcrEmitOut r{};
    if (hcr_bufs_reserve(&b, (size_t)n) != cudaSuccess || cudaMalloc(&d_text, n_bytes + 16) != cudaSuccess ||
        cudaMalloc(&d_ls, ((size_t)n + 1) * sizeof(int64_t)) != cudaSuccess || cudaMalloc(&d_out, out_cap) != cudaSuccess)
        goto done;
    if (cudaMemcpy(d_text, text, n_bytes, cudaMemcpyHostToDevice) != cudaSuccess || cudaMemset(d_text + n_bytes, '\n', 16) != cudaSuccess ||
        cudaMemcpy(d_ls, line_start, ((size_t)n + 1) * sizeof(int64_t), cudaMemcpyHostToDevice) != cudaSuccess)
        goto done;
    hcr_launch_scan(d_text, d_ls, n, P, &b, 132, nullptr);
    if (cudaGetLastError() != cudaSuccess) goto done;
    if (hcr_emit(&b, P, continues_contig, entry_extent, seg_bound, d_out, out_cap, &r, 132, nullptr) != cudaSuccess) goto done;
    if (cudaDeviceSynchronize() != cudaSuccess) goto done;
    if (n && cudaMemcpy(out_flags, b.flags, (size_t)n, cudaMemcpyDeviceToHost) != cudaSuccess) goto done;
    out_stats[0] = r.n_lines;
    out_stats[1] = r.skipped;
    out_stats[2] = r.exit_extent;
    out_stats[3] = r.longest;
    if ((unsigned long long)r.err != AFR_NO_ERROR) {
        *out_err_record = (int64_t)((unsigned long long)r.err >> 4);
        *out_err_reason = (int32_t)((unsigned long long)r.err & 0xF);
        rc = UGVC_E_DATA;
        goto done;
    }
    if ((size_t)r.bytes > capacity || (r.bytes && !out)) {
        rc = UGVC_E_ARG;
        goto done;
    }
    if (r.bytes && cudaMemcpy(out, d_out, (size_t)r.bytes, cudaMemcpyDeviceToHost) != cudaSuccess) goto done;
    rc = r.bytes;
done:
    hcr_bufs_free(&b);
    cudaFree(d_text);
    cudaFree(d_ls);
    cudaFree(d_out);
    return rc;
}
