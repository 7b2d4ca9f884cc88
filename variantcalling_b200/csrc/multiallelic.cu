// multiallelic.cu -- the --treat_multiallelics branch on the device (SURVEY.md section 8 row f2).
//
// The reference removes every multi-allelic record and every spanning-deletion cluster from a contig's frame,
// appends one or two biallelic rows per removed record, scores the new frame and folds the two likelihood
// triplets of a record back into one genotype-likelihood vector (filter_variants_pipeline.py:145-166;
// training_prep.py:226-287; multiallelics.py:13-62,65-177,280-308,385-465,503-559; spandel.py:11-128;
// variant_filtering_utils.py:346-408; flow_based_read.py:55-112).  Here, per contig:
//
//   ma_scan_alleles   one thread per record: allele count, deletion length max(len(REF) - len(allele)), '*' allele
//   ma_reach_*        chunked max-scan of pos + deletion length from the first deletion on: a record beyond the
//                     running reach closes the open cluster and heads the next (select_overlapping_variants)
//   ma_owner_*        chunked max-scan of the head index: every '*' record joins the cluster of the head before it
//   ma_groups_*       multi-allelic singles and flushed clusters -> the group list (singles ascending, then the
//                     cluster records ascending: the row order of the reference's frame), kept-line offsets
//   ma_plan_rows      one warp per group (lines staged in shared memory, lane 0 runs the builder): allele pairs to genotype (strongest ALT by its hom-alt PL, '*' weakest),
//                     row sizes, the allele indices the merge needs
//   ma_write_rows     one warp per group: the rows as VCF lines -- per-allele INFO / FORMAT values sub-sampled by
//                     the header's Number, GT / PL of the pair, X_IC / X_IL, X_HIL / X_HIN from the flow-space keys of
//                     the two haplotypes in the +-20 bp reference window, VARIANT_TYPE / QUAL / GQ / QD recomputed
//   ma_copy_kept      the untouched lines, compacted in input order in front of the rows
//   ma_merge          one thread per record: likelihoods of the scored pass -> N x W matrix in input record order
//   ma_score          one thread per record: phreds / qual / LOW_SCORE of the merged matrix (the device file path,
//                     ugvc_filter_bgzf_split; the host path does this step in NumPy)
//
// The rows are TEXT on purpose: the scored pass then runs the ordinary K1..K3 kernels on them, so the split rows
// get the features any record gets.  Every kernel is a grid-stride loop (shared memory only stages copies), so the host
// emulation (tests/host_emu) runs the same source with one emulated thread.  Scans are three-phase over chunks of
// 256 records (chunk aggregate, one-thread spine over the aggregates, chunk rescan): the branch touches about 1 % of
// the records and 16 bytes of state per record, far below the cost of the scored pass.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <string>

#include "../../include/ugvc_b200.h"
#include "multiallelic.cuh"

#define MA_MAX_ALLELES 32
#define MA_CHUNK 256
#define MA_RULES_MAGIC 0x4D41524Cu  // "MARL"

enum : uint8_t { MA_KEEP = 0, MA_SUB_A = 1, MA_SUB_R = 2, MA_ERR_G = 3, MA_ERR_NUM = 4, MA_SPECIAL = 5 /* + k: x_ic, x_il, x_hil, x_hin */ };
enum : uint8_t { MA_KIND_PLAIN = 0, MA_KIND_AS_IS = 1, MA_KIND_SPANNED = 3 };
enum : int {
    MA_OK = 0,
    MA_E_GT_ASSERT = 1,   // AssertionError: one of the alleles should be present in the GT
    MA_E_NUMBER_G = 2,    // RuntimeError: a per-genotype tag other than PL
    MA_E_NUMBER = 3,      // RuntimeError: Number <n> is not supported
    MA_E_NO_SPANDEL = 4,  // RuntimeError: '*' allele without the deletion record
    MA_E_NON_ACGT = 5,    // ValueError: flow key of a sequence with other characters
    MA_E_INDEX = 6,       // IndexError: a value list shorter than the alleles ask for
    MA_E_TYPE = 7,        // TypeError: arithmetic on a missing value (no PL, '.' inside PL, no X_IL on the deletion)
    MA_E_VALUE = 8,       // ValueError: not an integer
    MA_E_LIMIT = 9,       // more alleles than MA_MAX_ALLELES / a malformed line
    MA_E_TWO_CLASS = 10   // IndexError: a 2-class model has no hom-alt likelihood to spread (merge)
};

struct MaRule {
    uint8_t name[32];  // lower-cased tag
    uint8_t len;
    uint8_t action;
    uint16_t number;
};
struct MaRulesHeader {
    uint32_t magic;
    uint32_t n_info;
    uint32_t n_fmt;
    uint32_t flags;  // bit0: QD in the header's INFO, bit1: GQ in its FORMAT, bit 4 + k: special tag k is a loaded column
    uint8_t special_tag[4][32];  // spelling of X_IC / X_IL / X_HIL / X_HIN when one has to be appended
    uint8_t special_len[4];
};
struct MaRules {
    MaRulesHeader h;
    const MaRule* info;
    const MaRule* fmt;
};
struct MaGroup {
    int32_t origin;  // record index in the contig
    int32_t head;    // the deletion record spanning this one (MA_KIND_SPANNED), else -1
    uint8_t kind, n_rows, n_alleles, err;
    uint8_t pair[4];  // row 0 (a, b), row 1 (a, b)
    uint8_t i1, i2, pad0, pad1;  // first allele index spelled like the second row's alleles (merge_and_assign_pls)
    uint32_t size[2];
    int64_t row_off[2];  // byte offset of the rows inside the split text
    int32_t row0;        // index of the first row among all split rows
    int32_t pad2;
};

#ifdef UGVC_HOST_EMU
#define MA_LAUNCH(kern, grid, block, st, ...)                                          \
    do {                                                                               \
        threadIdx = dim3(0, 0, 0); blockIdx = dim3(0, 0, 0);                            \
        blockDim = dim3(1, 1, 1); gridDim = dim3(1, 1, 1);                              \
        kern(__VA_ARGS__);                                                             \
    } while (0)
#else
#define MA_LAUNCH(kern, grid, block, st, ...) kern<<<grid, block, 0, st>>>(__VA_ARGS__)
#endif
// the row kernels give a warp to every group: the lanes stage the group's line(s) in shared memory (the builder scans
// a line many times, byte by byte: from global memory every step waits for L2), lane 0 runs the builder on the copy
#ifdef UGVC_HOST_EMU
#define MA_LANES 1u
#define MA_LANE 0u
#define MA_WARP_SYNC() ((void)0)
#else
#define MA_LANES 32u
#define MA_LANE (threadIdx.x & 31u)
#define MA_WARP_SYNC() __syncwarp()
#endif
#define MA_ROW_WARPS 4u
#define MA_STAGE_BYTES 4096u   // per line; a longer line is read where it lies
#define MA_RULES_SMEM 96u
#define MA_TID ((int64_t)blockIdx.x * blockDim.x + threadIdx.x)
#define MA_NTHREADS ((int64_t)gridDim.x * blockDim.x)

// ---------------------------------------------------------------------------------------------------
// text helpers
// ---------------------------------------------------------------------------------------------------
struct MaSpan {
    uint32_t b, e;
    __device__ uint32_t len() const { return e - b; }
};
__device__ __forceinline__ uint8_t ma_lower(uint8_t c) { return (c >= 'A' && c <= 'Z') ? (uint8_t)(c + 32) : c; }
__device__ __forceinline__ uint8_t ma_upper(uint8_t c) { return (c >= 'a' && c <= 'z') ? (uint8_t)(c - 32) : c; }
__device__ inline bool ma_eq_lit(const uint8_t* t, MaSpan s, const char* lit) {
    uint32_t i = 0;
    for (; lit[i]; ++i)
        if (s.b + i >= s.e || t[s.b + i] != (uint8_t)lit[i]) return false;
    return s.b + i == s.e;
}
__device__ inline bool ma_eq_span(const uint8_t* t, MaSpan a, MaSpan b) {
    if (a.len() != b.len()) return false;
    for (uint32_t i = 0; i < a.len(); ++i)
        if (t[a.b + i] != t[b.b + i]) return false;
    return true;
}
// first position of byte c in [b, e), else e
__device__ inline uint32_t ma_find(const uint8_t* t, uint32_t b, uint32_t e, uint8_t c) {
    while (b < e && t[b] != c) ++b;
    return b;
}
// element k of a list separated by `sep` (str.split semantics: an empty text has one empty element)
__device__ inline bool ma_elem(const uint8_t* t, MaSpan s, uint8_t sep, uint32_t k, MaSpan* out) {
    uint32_t b = s.b;
    for (;;) {
        const uint32_t q = ma_find(t, b, s.e, sep);
        if (k == 0) {
            out->b = b;
            out->e = q;
            return true;
        }
        if (q >= s.e) return false;
        b = q + 1;
        --k;
    }
}
__device__ inline uint32_t ma_count(const uint8_t* t, MaSpan s, uint8_t sep) {
    uint32_t n = 1;
    for (uint32_t p = s.b; p < s.e; ++p) n += t[p] == sep;
    return n;
}
// int(text): 0 ok, MA_E_VALUE otherwise ("." / "" are handled by the callers)
__device__ inline int ma_int(const uint8_t* t, MaSpan s, long long* out) {
    uint32_t p = s.b;
    bool neg = false;
    if (p < s.e && (t[p] == '-' || t[p] == '+')) neg = t[p++] == '-';
    if (p >= s.e || s.e - p > 18u) return MA_E_VALUE;
    long long v = 0;
    for (; p < s.e; ++p) {
        const unsigned d = (unsigned)t[p] - '0';
        if (d > 9u) return MA_E_VALUE;
        v = v * 10 + d;
    }
    *out = neg ? -v : v;
    return MA_OK;
}
__device__ inline bool ma_is_missing(const uint8_t* t, MaSpan s) { return s.len() == 0 || (s.len() == 1 && t[s.b] == '.'); }

struct MaSink {
    uint8_t* out;  // nullptr: count only
    uint32_t n;
};
__device__ inline void ma_put(MaSink& s, const uint8_t* p, uint32_t len) {
    if (s.out)
        for (uint32_t i = 0; i < len; ++i) s.out[s.n + i] = p[i];
    s.n += len;
}
__device__ inline void ma_put_span(MaSink& s, const uint8_t* t, MaSpan sp) { ma_put(s, t + sp.b, sp.len()); }
__device__ inline void ma_putc(MaSink& s, uint8_t c) {
    if (s.out) s.out[s.n] = c;
    s.n += 1;
}
__device__ inline void ma_puts(MaSink& s, const char* lit) {
    for (uint32_t i = 0; lit[i]; ++i) ma_putc(s, (uint8_t)lit[i]);
}
__device__ inline void ma_put_u64(MaSink& s, unsigned long long v) {
    uint8_t buf[20];
    int n = 0;
    do {
        buf[n++] = (uint8_t)('0' + v % 10ull);
        v /= 10ull;
    } while (v);
    while (n) ma_putc(s, buf[--n]);
}
__device__ inline void ma_put_int(MaSink& s, long long v) {
    if (v < 0) {
        ma_putc(s, '-');
        ma_put_u64(s, (unsigned long long)(-(v + 1)) + 1ull);
    } else {
        ma_put_u64(s, (unsigned long long)v);
    }
}
// A finite double >= 0 as plain decimal text, truncated after 19 significant digits: the exact binary value is
// expanded digit by digit (integer part, then a 128-bit fixed-point fraction times ten), so strtod(text) is the
// double again (the truncation is far below half an ulp) -- the same double the reference's frame holds.
__device__ inline void ma_put_double(MaSink& s, double v) {
    const unsigned long long bits = (unsigned long long)__double_as_longlong(v);
    const int bexp = (int)((bits >> 52) & 0x7FFull);
    unsigned long long m = bits & ((1ull << 52) - 1ull);
    int e;  // v = m * 2^e
    if (bexp == 0) {
        e = -1074;
    } else {
        m |= 1ull << 52;
        e = bexp - 1075;
    }
    unsigned long long ip = 0, fhi = 0, flo = 0;
    if (m == 0) {
        ma_putc(s, '0');
        return;
    }
    if (e >= 0) {
        ip = e <= 10 ? (m << e) : ~0ull;  // (callers stay far below 2^63)
    } else {
        const int sh = -e;  // binary digits behind the point
        if (sh < 64) {
            ip = m >> sh;
            const unsigned long long fr = m & ((1ull << sh) - 1ull);
            fhi = fr << (64 - sh);
        } else if (sh < 128) {
            // fraction bits = m (< 2^53), its lowest bit has weight 2^-sh: m << (128 - sh) as a 128-bit number
            const int up = 128 - sh;  // 1..64
            if (up == 64) {
                fhi = m;
            } else {
                fhi = m >> (64 - up);
                flo = m << up;
            }
        } else {
            ma_putc(s, '0');  // below 2^-75: not reachable from integer qual / depth
            return;
        }
    }
    int sig = 0;
    if (ip) {
        uint8_t buf[20];
        int n = 0;
        unsigned long long x = ip;
        do {
            buf[n++] = (uint8_t)('0' + x % 10ull);
            x /= 10ull;
        } while (x);
        sig = n;
        while (n) ma_putc(s, buf[--n]);
    } else {
        ma_putc(s, '0');
    }
    if ((fhi | flo) == 0ull || sig >= 19) return;
    ma_putc(s, '.');
    while ((fhi | flo) != 0ull && sig < 19) {
        const unsigned long long carry = __umul64hi(flo, 10ull);
        flo *= 10ull;
        unsigned long long hh = __umul64hi(fhi, 10ull);
        const unsigned long long hl = fhi * 10ull;
        fhi = hl + carry;
        if (fhi < hl) ++hh;
        ma_putc(s, (uint8_t)('0' + hh));
        if (sig || hh) ++sig;
    }
}

// ---------------------------------------------------------------------------------------------------
// one record
// ---------------------------------------------------------------------------------------------------
struct MaRec {
    const uint8_t* t;  // the pointer through which this record's absolute text offsets are read (the text, or a staged copy of the line)
    MaSpan col[10];
    uint32_t n_cols;   // columns on the line
    uint32_t rest_b;   // the tab in front of column 10 (cols[10:] travel verbatim), line end when there is none
    uint32_t le;       // line end (the newline)
    MaSpan al[MA_MAX_ALLELES];
    int n_alleles;     // > MA_MAX_ALLELES: too many
    long long pos;
    bool has_fmt;      // len(cols) > 9 and FORMAT != "."
};

// the columns and alleles of the line [ls, le): le is the position of its newline
__device__ inline int ma_parse_rec(const uint8_t* t, uint32_t ls, uint32_t le, MaRec* r) {
    r->t = t;
    r->le = le;
    uint32_t b = ls, c = 0;
    r->rest_b = le;
    for (;;) {
        const uint32_t q = ma_find(t, b, le, '\t');
        if (c < 10u) {
            r->col[c].b = b;
            r->col[c].e = q;
        }
        ++c;
        if (c == 10u) r->rest_b = q;
        if (q >= le) break;
        b = q + 1;
    }
    r->n_cols = c;
    if (c < 8u) return MA_E_LIMIT;
    for (uint32_t k = c; k < 10u; ++k) r->col[k].b = r->col[k].e = le;
    if (ma_int(t, r->col[1], &r->pos) != MA_OK) return MA_E_VALUE;
    r->al[0] = r->col[3];
    r->n_alleles = 1;
    if (!ma_eq_lit(t, r->col[4], ".")) {
        uint32_t ab = r->col[4].b;
        for (;;) {
            const uint32_t q = ma_find(t, ab, r->col[4].e, ',');
            if (r->n_alleles < MA_MAX_ALLELES) {
                r->al[r->n_alleles].b = ab;
                r->al[r->n_alleles].e = q;
            }
            ++r->n_alleles;
            if (q >= r->col[4].e) break;
            ab = q + 1;
        }
    }
    r->has_fmt = c > 9u && !ma_eq_lit(t, r->col[8], ".");
    return MA_OK;
}
// _Record.info_value: the value of the first INFO entry spelled `tag` (0: no such key, 1: value in *v, empty when
// the key stands alone)
__device__ inline int ma_info_value(const uint8_t* t, const MaRec& r, const char* tag, MaSpan* v) {
    if (ma_eq_lit(t, r.col[7], ".")) return 0;
    uint32_t b = r.col[7].b;
    const uint32_t e = r.col[7].e;
    for (;;) {
        const uint32_t q = ma_find(t, b, e, ';');
        if (q > b) {
            const uint32_t eq = ma_find(t, b, q, '=');
            if (ma_eq_lit(t, MaSpan{b, eq}, tag)) {
                v->b = eq < q ? eq + 1 : q;
                v->e = q;
                return 1;
            }
        }
        if (q >= e) return 0;
        b = q + 1;
    }
}
// index of the FORMAT key spelled `tag` (-1: none)
__device__ inline int ma_fmt_index(const uint8_t* t, const MaRec& r, const char* tag) {
    if (!r.has_fmt) return -1;
    MaSpan k;
    for (uint32_t i = 0; ma_elem(t, r.col[8], ':', i, &k); ++i)
        if (ma_eq_lit(t, k, tag)) return (int)i;
    return -1;
}
// _Record.sample_value: 0 = the key is not in FORMAT (or the sample has fewer values: None), 1 = value in *v
__device__ inline int ma_sample_value(const uint8_t* t, const MaRec& r, const char* tag, MaSpan* v) {
    const int i = ma_fmt_index(t, r, tag);
    if (i < 0) return 0;
    return ma_elem(t, r.col[9], ':', (uint32_t)i, v) ? 1 : 0;
}
// PL as the reference sees it: *n elements, all integers or '.'; MA_E_TYPE when there is no PL value at all
__device__ inline int ma_pl_check(const uint8_t* t, const MaRec& r, MaSpan* pl, uint32_t* n) {
    if (!ma_sample_value(t, r, "PL", pl)) return MA_E_TYPE;
    *n = ma_count(t, *pl, ',');
    MaSpan el;
    long long v;
    for (uint32_t i = 0; i < *n; ++i) {
        ma_elem(t, *pl, ',', i, &el);
        if (!ma_is_missing(t, el) && ma_int(t, el, &v) != MA_OK) return MA_E_VALUE;
    }
    return MA_OK;
}
__device__ inline int ma_pl_at(const uint8_t* t, MaSpan pl, uint32_t n, uint32_t k, long long* v) {
    if (k >= n) return MA_E_INDEX;
    MaSpan el;
    ma_elem(t, pl, ',', k, &el);
    if (ma_is_missing(t, el)) return MA_E_TYPE;
    return ma_int(t, el, v);
}
__device__ __forceinline__ uint32_t ma_pl_idx(uint32_t a, uint32_t b) {
    const uint32_t hi = a > b ? a : b, lo = a > b ? b : a;
    return hi * (hi + 1u) / 2u + lo;
}
// `allele index in rec.gt` for the alleles a and b (GT split on / and |; '.' is None); MA_E_VALUE on a bad integer
__device__ inline int ma_gt_has(const uint8_t* t, const MaRec& r, long long a, long long b, bool* has_a, bool* has_b) {
    *has_a = *has_b = false;
    MaSpan gt;
    if (!ma_sample_value(t, r, "GT", &gt)) return MA_OK;  // (None,)
    uint32_t p = gt.b;
    for (;;) {
        uint32_t q = p;
        while (q < gt.e && t[q] != '/' && t[q] != '|') ++q;
        const MaSpan el{p, q};
        if (!ma_is_missing(t, el)) {
            long long v;
            if (ma_int(t, el, &v) != MA_OK) return MA_E_VALUE;
            *has_a |= v == a;
            *has_b |= v == b;
        }
        if (q >= gt.e) break;
        p = q + 1;
    }
    return MA_OK;
}

// ---------------------------------------------------------------------------------------------------
// flow-space comparison of two haplotypes (multiallelics.py:385-465, flow_based_concordance.py:263-339,
// flow_based_read.py:55-112)
// ---------------------------------------------------------------------------------------------------
// Python's s[a:b] on a sequence of length n
__device__ inline void ma_pyslice(int a, int b, int n, int* ob, int* oe) {
    if (a < 0) a += n;
    if (a < 0) a = 0;
    if (a > n) a = n;
    if (b < 0) b += n;
    if (b < 0) b = 0;
    if (b > n) b = n;
    if (b < a) b = a;
    *ob = a;
    *oe = b;
}
// a haplotype: window[0:rel] + allele + window[rel:][len(ref_allele):], never materialised
struct MaHap {
    const uint8_t* win;  // the window, upper-cased, characters outside ".ATCG" already 'A'
    int l_b, l_e, r_b, r_e;
    const uint8_t* al;
    int al_len;
    __device__ int len() const { return (l_e - l_b) + al_len + (r_e - r_b); }
    __device__ uint8_t at(int i) const {
        if (i < l_e - l_b) return win[l_b + i];
        i -= l_e - l_b;
        if (i < al_len) return ma_upper(al[i]);
        return win[r_b + (i - al_len)];
    }
};
__device__ inline MaHap ma_place(const uint8_t* win, int wl, int rel, int ref_allele_len, const uint8_t* al, int al_len) {
    MaHap h;
    h.win = win;
    h.al = al;
    h.al_len = al_len;
    ma_pyslice(0, rel, wl, &h.l_b, &h.l_e);
    int tb, te;
    ma_pyslice(rel, wl, wl, &tb, &te);  // window[rel:len(window)]
    int sb, se;
    ma_pyslice(ref_allele_len, te - tb, te - tb, &sb, &se);  // [len(ref_allele):] of that
    h.r_b = tb + sb;
    h.r_e = tb + se;
    return h;
}
__device__ inline bool ma_symbolic(const uint8_t* t, MaSpan a) {  // a.startswith("<") or "*" in a
    if (a.len() && t[a.b] == '<') return true;
    for (uint32_t p = a.b; p < a.e; ++p)
        if (t[p] == '*') return true;
    return false;
}
// -> hin ('.' with hil 0 when the two keys differ in anything but one flow); MA_E_NON_ACGT like the flow-key routine
__device__ inline int ma_flow_compare(const MaHap& h0, const MaHap& h1, uint8_t* hin, int* hil) {
    *hin = '.';
    *hil = 0;
    const int n0 = h0.len(), n1 = h1.len();
    for (int i = 0; i < n0; ++i) {
        const uint8_t c = h0.at(i);
        if (c != 'A' && c != 'C' && c != 'G' && c != 'T') return MA_E_NON_ACGT;
    }
    for (int i = 0; i < n1; ++i) {
        const uint8_t c = h1.at(i);
        if (c != 'A' && c != 'C' && c != 'G' && c != 'T') return MA_E_NON_ACGT;
    }
    const uint8_t order[4] = {'T', 'G', 'C', 'A'};
    int i0 = 0, i1 = 0, flow = 0, ndiff = 0, dflow = 0, dmax = 0;
    while (i0 < n0 || i1 < n1) {
        if (i0 >= n0 || i1 >= n1) return MA_OK;  // keys of different length
        const uint8_t base = order[flow & 3];
        int r0 = 0, r1 = 0;
        while (i0 + r0 < n0 && h0.at(i0 + r0) == base) ++r0;
        while (i1 + r1 < n1 && h1.at(i1 + r1) == base) ++r1;
        if (r0 != r1) {
            ++ndiff;
            dflow = flow;
            dmax = r0 > r1 ? r0 : r1;
        }
        i0 += r0;
        i1 += r1;
        ++flow;
    }
    if (ndiff == 1) {
        *hin = order[dflow & 3];
        *hil = dmax;
    }
    return MA_OK;
}
// classify_hmer_indel_relative for the alleles (pa, pb) of record r; head: the deletion record spanning it (or null)
__device__ inline int ma_classify_hmer(const uint8_t* t, const MaRec& r, int pa, int pb, const MaRec* head, const uint8_t* ref,
                                       long long ref_len, uint8_t* hin, int* hil) {
    *hin = '.';
    *hil = 0;
    long long lo = r.pos - 20 > 0 ? r.pos - 20 : 0, hi = r.pos + 20 < ref_len ? r.pos + 20 : ref_len;
    // ref[lo - 1 : hi - 1] with Python's slice rules (a negative start counts from the end)
    long long sb = lo - 1, se = hi - 1;
    if (sb < 0) sb += ref_len;
    if (sb < 0) sb = 0;
    if (sb > ref_len) sb = ref_len;
    if (se < 0) se += ref_len;
    if (se < 0) se = 0;
    if (se > ref_len) se = ref_len;
    if (se < sb) se = sb;
    uint8_t win[48];
    int wl = (int)(se - sb);
    if (wl > 48) wl = 48;  // (at most 40 by construction)
    for (int i = 0; i < wl; ++i) {
        const uint8_t c = ma_upper(ref[sb + i]);
        win[i] = (c == '.' || c == 'A' || c == 'T' || c == 'C' || c == 'G') ? c : (uint8_t)'A';
    }
    const int lo_i = pa < pb ? pa : pb, hi_i = pa < pb ? pb : pa;  // sorted(pair)
    const bool star = ma_eq_lit(t, r.al[pa], "*") || ma_eq_lit(t, r.al[pb], "*");
    MaHap haps[2];
    int nh = 0;
    const int cand[2] = {lo_i, hi_i};
    if (star) {
        if (!head) return MA_E_NO_SPANDEL;
        for (int c = 0; c < 2; ++c) {
            const MaSpan a = r.al[cand[c]];
            if (ma_eq_lit(t, a, "*") || ma_symbolic(t, a)) continue;
            if (nh < 2) haps[nh] = ma_place(win, wl, 20, (int)r.al[0].len(), t + a.b, (int)a.len());
            ++nh;
        }
        // the deletion itself: its REF and first ALT placed where the deletion starts; the second of what is kept
        int kept = 0;
        const int rel = (int)(head->pos - (r.pos - 20));
        const uint8_t* th = head->t;
        for (int c = 0; c < 2 && c < head->n_alleles; ++c) {
            const MaSpan a = head->al[c];
            if (ma_symbolic(th, a)) continue;
            if (kept == 1) {
                if (nh < 2) haps[nh] = ma_place(win, wl, rel, (int)head->al[0].len(), th + a.b, (int)a.len());
                ++nh;
            }
            ++kept;
        }
    } else {
        for (int c = 0; c < 2; ++c) {
            const MaSpan a = r.al[cand[c]];
            if (ma_symbolic(t, a)) continue;
            if (nh < 2) haps[nh] = ma_place(win, wl, 20, (int)r.al[0].len(), t + a.b, (int)a.len());
            ++nh;
        }
    }
    if (nh < 2) return MA_OK;
    return ma_flow_compare(haps[0], haps[1], hin, hil);
}

// ---------------------------------------------------------------------------------------------------
// rules
// ---------------------------------------------------------------------------------------------------
__device__ inline const MaRule* ma_rule(const MaRule* rules, uint32_t n, const uint8_t* t, MaSpan key) {
    if (key.len() > 32u || key.len() == 0u) return nullptr;
    for (uint32_t i = 0; i < n; ++i) {
        if (rules[i].len != key.len()) continue;
        bool eq = true;
        for (uint32_t c = 0; c < key.len() && eq; ++c) eq = rules[i].name[c] == ma_lower(t[key.b + c]);
        if (eq) return &rules[i];
    }
    return nullptr;
}
// is the (lower-cased) INFO key also a FORMAT key of the record?
__device__ inline bool ma_in_format(const uint8_t* t, const MaRec& r, MaSpan key) {
    if (!r.has_fmt) return false;
    MaSpan k;
    for (uint32_t i = 0; ma_elem(t, r.col[8], ':', i, &k); ++i) {
        if (k.len() != key.len()) continue;
        bool eq = true;
        for (uint32_t c = 0; c < k.len() && eq; ++c) eq = ma_lower(t[k.b + c]) == ma_lower(t[key.b + c]);
        if (eq) return true;
    }
    return false;
}
// SplitPlan.convert: the pair's values of a per-allele value list (vcftools.py:745-778)
__device__ inline int ma_convert(MaSink& s, const uint8_t* t, MaSpan v, unsigned action, int pa, int pb) {
    MaSpan el;
    switch (action) {
        case MA_SUB_A:
            if (!ma_elem(t, v, ',', (uint32_t)(pb - 1), &el)) return MA_E_INDEX;
            ma_put_span(s, t, el);
            return MA_OK;
        case MA_SUB_R:
            if (!ma_elem(t, v, ',', (uint32_t)pa, &el)) return MA_E_INDEX;
            ma_put_span(s, t, el);
            ma_putc(s, ',');
            if (!ma_elem(t, v, ',', (uint32_t)pb, &el)) return MA_E_INDEX;
            ma_put_span(s, t, el);
            return MA_OK;
        case MA_ERR_G:
            return MA_E_NUMBER_G;
        case MA_ERR_NUM:
            return MA_E_NUMBER;
        default:
            ma_put_span(s, t, v);
            return MA_OK;
    }
}

// ---------------------------------------------------------------------------------------------------
// one row: SplitPlan._rewrite / _as_is followed by _finish (cleanup_multiallelics, multiallelics.py:503-559)
// ---------------------------------------------------------------------------------------------------
// pa < 0: the record as it is (a biallelic deletion heading a cluster)
// check: also walk the conversions in the reference's order first, so that a record with several defects fails with
// the error the reference meets first (the planning pass; the writing pass only sees rows that passed)
__device__ int ma_row(MaSink& s, const MaRules& R, const MaRec& r, int pa, int pb, const MaRec* head,
                      const uint8_t* ref, long long ref_len, bool check) {
    const uint8_t* t = r.t;
    const bool as_is = pa < 0;
    int rc;
    MaSpan plv;
    // ---- the derived tags
    const MaSpan a0 = as_is ? r.al[0] : r.al[pa], a1 = as_is ? r.al[0] : r.al[pb];
    bool il_none = true;
    long long il = 0;
    int hil = 0;
    bool hil_none = false;
    uint8_t hin = '.';
    const char* x_ic = "NA";
    bool star = false;
    if (!as_is) {
        star = ma_eq_lit(t, a0, "*") || ma_eq_lit(t, a1, "*");
        if (star && !head) return MA_E_NO_SPANDEL;
        const bool indel = star || a0.len() != a1.len();
        if (!indel) {
            x_ic = "NA";
        } else if (star) {
            const uint8_t* th = head->t;
            MaSpan v, el;
            if (!ma_info_value(th, *head, "X_IL", &v)) return MA_E_TYPE;
            ma_elem(th, v, ',', 0, &el);
            // every element is converted (int_tuple), the first one is used
            MaSpan e2;
            for (uint32_t i = 0; ma_elem(th, v, ',', i, &e2); ++i) {
                long long x;
                if (!ma_is_missing(th, e2) && ma_int(th, e2, &x) != MA_OK) return MA_E_VALUE;
            }
            x_ic = "del";
            il_none = ma_is_missing(th, el);
            if (!il_none) ma_int(th, el, &il);
        } else if (a0.len() > a1.len()) {
            x_ic = "del";
            il_none = false;
            il = (long long)a0.len() - (long long)a1.len();
        } else {
            x_ic = "ins";
            il_none = false;
            il = (long long)a1.len() - (long long)a0.len();
        }
        if ((rc = ma_classify_hmer(t, r, pa, pb, head, ref, ref_len, &hin, &hil)) != MA_OK) return rc;
    } else {
        // x_il / x_hil of the record itself: the first element of each (a missing tag is a TypeError in the reference)
        MaSpan v, el;
        long long x;
        if (!ma_info_value(t, r, "X_IL", &v)) return MA_E_TYPE;
        for (uint32_t i = 0; ma_elem(t, v, ',', i, &el); ++i)
            if (!ma_is_missing(t, el) && ma_int(t, el, &x) != MA_OK) return MA_E_VALUE;
        ma_elem(t, v, ',', 0, &el);
        il_none = ma_is_missing(t, el);
        if (!il_none) ma_int(t, el, &il);
        if (!ma_info_value(t, r, "X_HIL", &v)) return MA_E_TYPE;
        for (uint32_t i = 0; ma_elem(t, v, ',', i, &el); ++i)
            if (!ma_is_missing(t, el) && ma_int(t, el, &x) != MA_OK) return MA_E_VALUE;
        ma_elem(t, v, ',', 0, &el);
        hil_none = ma_is_missing(t, el);
        if (!hil_none) {
            ma_int(t, el, &x);
            hil = (int)x;
        }
    }
    // ---- (check) the INFO values through convert(), in line order
    if (check && !as_is && !ma_eq_lit(t, r.col[7], ".")) {
        uint32_t b = r.col[7].b;
        const uint32_t e = r.col[7].e;
        for (;;) {
            const uint32_t q = ma_find(t, b, e, ';');
            const uint32_t eq = ma_find(t, b, q, '=');
            if (q > b && eq < q) {
                const MaSpan key{b, eq}, val{eq + 1, q};
                const MaRule* rule = ma_rule(R.info, R.h.n_info, t, key);
                if (rule && rule->action != MA_KEEP && rule->action < MA_SPECIAL && !ma_in_format(t, r, key)) {
                    MaSink none{nullptr, 0};
                    if ((rc = ma_convert(none, t, val, rule->action, pa, pb)) != MA_OK) return rc;
                }
            }
            if (q >= e) break;
            b = q + 1;
        }
    }
    // ---- PL of the row, QUAL, GQ
    uint32_t pln;
    if ((rc = ma_pl_check(t, r, &plv, &pln)) != MA_OK) return rc;
    long long pl3[3] = {0, 0, 0};
    long long qual = 0, gq = 0;
    if (!as_is) {
        if ((rc = ma_pl_at(t, plv, pln, ma_pl_idx((uint32_t)pa, (uint32_t)pa), &pl3[0])) != MA_OK) return rc;
        if ((rc = ma_pl_at(t, plv, pln, ma_pl_idx((uint32_t)pa, (uint32_t)pb), &pl3[1])) != MA_OK) return rc;
        if ((rc = ma_pl_at(t, plv, pln, ma_pl_idx((uint32_t)pb, (uint32_t)pb), &pl3[2])) != MA_OK) return rc;
        const long long mn = pl3[0] < pl3[1] ? (pl3[0] < pl3[2] ? pl3[0] : pl3[2]) : (pl3[1] < pl3[2] ? pl3[1] : pl3[2]);
        for (int i = 0; i < 3; ++i) pl3[i] -= mn;
        const long long m12 = pl3[1] < pl3[2] ? pl3[1] : pl3[2];
        qual = m12 - pl3[0] > 0 ? m12 - pl3[0] : 0;
        // sorted(pl)[1] - sorted(pl)[0]
        long long a = pl3[0], b = pl3[1], c = pl3[2], x;
        if (a > b) { x = a; a = b; b = x; }
        if (b > c) { x = b; b = c; c = x; }
        if (a > b) { x = a; a = b; b = x; }
        gq = b - a;
    } else {
        if (pln < 2u) return MA_E_INDEX;  // sorted(pl)[1]
        long long first = 0, s0 = 0, s1 = 0, rest_min = 0;
        for (uint32_t i = 0; i < pln; ++i) {
            long long v;
            if ((rc = ma_pl_at(t, plv, pln, i, &v)) != MA_OK) return rc;
            if (i == 0) {
                first = v;
                s0 = v;
            } else {
                if (i == 1 || v < rest_min) rest_min = v;
                if (i == 1) {
                    s1 = v;
                    if (s1 < s0) { const long long x = s0; s0 = s1; s1 = x; }
                } else if (v < s0) {
                    s1 = s0;
                    s0 = v;
                } else if (v < s1) {
                    s1 = v;
                }
            }
        }
        qual = rest_min - first > 0 ? rest_min - first : 0;
        gq = s1 - s0;
    }
    gq = gq < 0 ? 0 : (gq > 99 ? 99 : gq);
    // ---- (check) GT and the sample values through convert(), in column order
    if (check && !as_is && r.has_fmt) {
        MaSpan k, v;
        for (uint32_t i = 0; ma_elem(t, r.col[8], ':', i, &k); ++i) {
            if (ma_eq_lit(t, k, "GT")) {
                bool h0, h1;
                if ((rc = ma_gt_has(t, r, pa, pb, &h0, &h1)) != MA_OK) return rc;
                if (!h0 && !h1) return MA_E_GT_ASSERT;
            } else if (!ma_eq_lit(t, k, "PL")) {
                const MaRule* rule = ma_rule(R.fmt, R.h.n_fmt, t, k);
                if (rule && rule->action != MA_KEEP && rule->action < MA_SPECIAL) {
                    MaSink none{nullptr, 0};
                    const uint8_t dot = '.';
                    if (ma_elem(t, r.col[9], ':', i, &v)) rc = ma_convert(none, t, v, rule->action, pa, pb);
                    else rc = ma_convert(none, &dot, MaSpan{0, 1}, rule->action, pa, pb);
                    if (rc != MA_OK) return rc;
                }
            }
        }
    }
    // ---- VARIANT_TYPE after the clean-up rules
    MaSpan vt_span{0, 0};
    const bool has_vt = ma_info_value(t, r, "VARIANT_TYPE", &vt_span) != 0;
    int vt_kind = 0;  // 0: as spelled, 1: "non-h-indel", 2: "h-indel"
    if (has_vt) {
        bool snp = ma_eq_lit(t, vt_span, "snp"), nonh = ma_eq_lit(t, vt_span, "non-h-indel"), h = ma_eq_lit(t, vt_span, "h-indel");
        if (snp && !il_none && il != 0) {
            vt_kind = 1;
            nonh = true;
        }
        if (nonh && !hil_none && hil > 0) {
            vt_kind = 2;
            nonh = false;
            h = true;
        }
        if (h && (hil_none || hil == 0)) vt_kind = 1;
    }
    // ---- depth for QD: the FORMAT value whenever the key is there, else INFO
    bool dp_none = true;
    long long dp = 0;
    {
        MaSpan v;
        int have;
        if (ma_fmt_index(t, r, "DP") >= 0) have = ma_sample_value(t, r, "DP", &v);
        else have = ma_info_value(t, r, "DP", &v);
        if (have && !ma_is_missing(t, v)) {
            if (ma_int(t, v, &dp) != MA_OK) return MA_E_VALUE;
            dp_none = false;
        }
    }
    const bool qd_on = (R.h.flags & 1u) != 0u, gq_on = (R.h.flags & 2u) != 0u;

    // ---- columns 0..6
    for (int c = 0; c < 3; ++c) {
        ma_put_span(s, t, r.col[c]);
        ma_putc(s, '\t');
    }
    if (as_is) {
        ma_put_span(s, t, r.col[3]);
        ma_putc(s, '\t');
        ma_put_span(s, t, r.col[4]);
    } else {
        ma_put_span(s, t, a0);
        ma_putc(s, '\t');
        if (ma_eq_lit(t, a1, "*")) {
            // '*' cannot be told from a base by its length: one longer than REF, so that the loader's indel is True
            for (uint32_t i = 0; i <= a0.len(); ++i) ma_putc(s, '*');
        } else {
            ma_put_span(s, t, a1);
        }
    }
    ma_putc(s, '\t');
    ma_put_int(s, qual);
    ma_putc(s, '\t');
    ma_put_span(s, t, r.col[6]);
    ma_putc(s, '\t');
    // ---- INFO
    uint32_t n_info = 0;
    bool vt_done = false, qd_done = false;
    unsigned seen = 0;  // special tags met on the line
    auto put_qd = [&]() {
        if (dp_none) {
            ma_putc(s, '.');
        } else if (dp == 0) {
            ma_puts(s, qual == 0 ? "." : "inf");
        } else {
            if (dp < 0) ma_putc(s, '-');  // (-0.0 for a zero quality)
            ma_put_double(s, (double)qual / (double)(dp < 0 ? -dp : dp));
        }
    };
    auto put_special = [&](unsigned k) {
        if (k == 0) {
            ma_puts(s, x_ic);
        } else if (k == 1) {
            if (il_none) ma_putc(s, '.');
            else ma_put_int(s, il);
        } else if (k == 2) {
            ma_put_int(s, hil);
        } else {
            ma_putc(s, hin);
        }
    };
    if (!ma_eq_lit(t, r.col[7], ".")) {
        uint32_t b = r.col[7].b;
        const uint32_t e = r.col[7].e;
        for (;;) {
            const uint32_t q = ma_find(t, b, e, ';');
            if (q > b) {
                if (n_info++) ma_putc(s, ';');
                const uint32_t eq = ma_find(t, b, q, '=');
                const MaSpan key{b, eq}, val{eq < q ? eq + 1 : q, q};
                const bool sep = eq < q;
                const MaRule* rule = ma_rule(R.info, R.h.n_info, t, key);
                const unsigned action = rule ? rule->action : MA_KEEP;
                if (!vt_done && has_vt && ma_eq_lit(t, key, "VARIANT_TYPE")) {
                    vt_done = true;
                    // (the value would first go through convert(): an unsupported Number raises there)
                    if (!as_is && sep && action != MA_KEEP && action < MA_SPECIAL && !ma_in_format(t, r, key)) {
                        MaSink none{nullptr, 0};
                        if ((rc = ma_convert(none, t, val, action, pa, pb)) != MA_OK) return rc;
                    }
                    ma_puts(s, "VARIANT_TYPE=");
                    if (vt_kind == 1) ma_puts(s, "non-h-indel");
                    else if (vt_kind == 2) ma_puts(s, "h-indel");
                    else ma_put_span(s, t, vt_span);
                } else if (!qd_done && qd_on && ma_eq_lit(t, key, "QD")) {
                    qd_done = true;
                    if (!as_is && sep && action != MA_KEEP && action < MA_SPECIAL && !ma_in_format(t, r, key)) {
                        MaSink none{nullptr, 0};
                        if ((rc = ma_convert(none, t, val, action, pa, pb)) != MA_OK) return rc;
                    }
                    ma_puts(s, "QD=");
                    put_qd();
                } else if (!as_is && action >= MA_SPECIAL) {
                    ma_put_span(s, t, key);
                    ma_putc(s, '=');
                    put_special(action - MA_SPECIAL);
                    seen |= 1u << (action - MA_SPECIAL);
                } else if (sep) {
                    ma_put_span(s, t, key);
                    ma_putc(s, '=');
                    if (as_is || action == MA_KEEP || ma_in_format(t, r, key)) ma_put_span(s, t, val);
                    else if ((rc = ma_convert(s, t, val, action, pa, pb)) != MA_OK) return rc;
                } else {
                    ma_put_span(s, t, key);
                }
            }
            if (q >= e) break;
            b = q + 1;
        }
    }
    if (!as_is) {
        for (unsigned k = 0; k < 4u; ++k) {
            if (!((R.h.flags >> (4u + k)) & 1u) || ((seen >> k) & 1u)) continue;
            if (n_info++) ma_putc(s, ';');
            ma_put(s, R.h.special_tag[k], R.h.special_len[k]);
            ma_putc(s, '=');
            put_special(k);
        }
    }
    if (qd_on && !qd_done) {
        if (n_info++) ma_putc(s, ';');
        ma_puts(s, "QD=");
        put_qd();
    }
    if (n_info == 0) ma_putc(s, '.');
    ma_putc(s, '\t');
    // ---- FORMAT keys
    uint32_t n_fmt = 0;
    int gq_at = -1;
    if (r.has_fmt) {
        MaSpan k;
        for (uint32_t i = 0; ma_elem(t, r.col[8], ':', i, &k); ++i) {
            if (i) ma_putc(s, ':');
            ma_put_span(s, t, k);
            if (gq_at < 0 && ma_eq_lit(t, k, "GQ")) gq_at = (int)i;
            ++n_fmt;
        }
    }
    if (gq_on && gq_at < 0) {
        if (n_fmt) ma_putc(s, ':');
        ma_puts(s, "GQ");
    }
    ma_putc(s, '\t');
    // ---- sample values
    for (uint32_t i = 0; i < n_fmt; ++i) {
        MaSpan k, v;
        ma_elem(t, r.col[8], ':', i, &k);
        const bool have = ma_elem(t, r.col[9], ':', i, &v) && r.n_cols > 9u;
        if (i) ma_putc(s, ':');
        if (!as_is && ma_eq_lit(t, k, "GT")) {
            bool h0, h1;
            if ((rc = ma_gt_has(t, r, pa, pb, &h0, &h1)) != MA_OK) return rc;
            if (!h0 && !h1) return MA_E_GT_ASSERT;
            ma_puts(s, h0 && h1 ? "0/1" : (h0 ? "0/0" : "1/1"));
        } else if (!as_is && ma_eq_lit(t, k, "PL")) {
            ma_put_int(s, pl3[0]);
            ma_putc(s, ',');
            ma_put_int(s, pl3[1]);
            ma_putc(s, ',');
            ma_put_int(s, pl3[2]);
        } else {
            const MaRule* rule = as_is ? nullptr : ma_rule(R.fmt, R.h.n_fmt, t, k);
            const unsigned action = rule ? rule->action : MA_KEEP;
            const bool is_gq = gq_on && (int)i == gq_at;
            MaSink none{nullptr, 0};
            MaSink& dst = is_gq ? none : s;  // GQ is replaced below, after convert() had its say
            if (!have) {
                // None -> ".": one element
                if (action == MA_KEEP || action >= MA_SPECIAL) {
                    ma_putc(dst, '.');
                } else {
                    // convert(".") of a per-allele tag: "." has one element
                    const uint8_t dot = '.';
                    if ((rc = ma_convert(dst, &dot, MaSpan{0, 1}, action, pa, pb)) != MA_OK) return rc;
                }
            } else if (action == MA_KEEP || action >= MA_SPECIAL) {
                ma_put_span(dst, t, v);
            } else if ((rc = ma_convert(dst, t, v, action, pa, pb)) != MA_OK) {
                return rc;
            }
            if (is_gq) ma_put_int(s, gq);
        }
    }
    if (gq_on && gq_at < 0) {
        if (n_fmt) ma_putc(s, ':');
        ma_put_int(s, gq);
    }
    // ---- the other samples, verbatim
    if (r.rest_b < r.le) ma_put(s, t + r.rest_b, r.le - r.rest_b);
    ma_putc(s, '\n');
    return MA_OK;
}

// ---------------------------------------------------------------------------------------------------
// kernels: overlap detection
// ---------------------------------------------------------------------------------------------------
#define MA_F_BOUNDARY 1u
#define MA_F_STAR 2u
#define MA_F_MULTI 4u
#define MA_F_MEMBER 8u
#define MA_F_HAS_MEMBER 16u
#define MA_F_IN_CLUSTER 32u
#define MA_F_SINGLE 64u

__global__ void ma_scan_alleles(const uint8_t* __restrict__ t, const int64_t* __restrict__ line_start,
                                const ugvc_recinfo* __restrict__ recinfo, int64_t n, int64_t* __restrict__ key,
                                uint8_t* __restrict__ flags, unsigned long long* first_del) {
    for (int64_t i = MA_TID; i < n; i += MA_NTHREADS) {
        const uint32_t ls = (uint32_t)line_start[i], le = (uint32_t)line_start[i + 1] - 1u;
        // REF and ALT columns
        uint32_t b = ls;
        for (int c = 0; c < 3; ++c) b = ma_find(t, b, le, '\t') + 1u;
        const uint32_t ref_e = ma_find(t, b, le, '\t');
        const long long ref_len = (long long)ref_e - (long long)b;
        uint32_t ab = ref_e + 1u;
        const uint32_t alt_e = ma_find(t, ab <= le ? ab : le, le, '\t');
        long long del_len = 0;
        int n_alleles = 1;
        bool star = ref_len == 1 && t[b] == '*';
        if (ab <= le && !(alt_e - ab == 1u && t[ab] == '.')) {
            for (;;) {
                const uint32_t q = ma_find(t, ab, alt_e, ',');
                const long long al = (long long)q - (long long)ab;
                if (ref_len - al > del_len) del_len = ref_len - al;
                star |= al == 1 && t[ab] == '*';
                ++n_alleles;
                if (q >= alt_e) break;
                ab = q + 1u;
            }
        }
        key[i] = (int64_t)recinfo[i].pos + del_len;
        flags[i] = (uint8_t)((star ? MA_F_STAR : 0u) | (n_alleles > 2 ? MA_F_MULTI : 0u));
        if (del_len > 0) atomicMin(first_del, (unsigned long long)i);
    }
}
// chunk aggregate of the reach: max of pos + del_len over the records from the first deletion on
__global__ void ma_reach_agg(const int64_t* __restrict__ key, int64_t n, const unsigned long long* first_del,
                             int64_t* __restrict__ agg) {
    const int64_t n_chunks = (n + MA_CHUNK - 1) / MA_CHUNK, first = (int64_t)*first_del;
    for (int64_t c = MA_TID; c < n_chunks; c += MA_NTHREADS) {
        int64_t m = INT64_MIN;
        const int64_t e = (c + 1) * MA_CHUNK < n ? (c + 1) * MA_CHUNK : n;
        for (int64_t i = c * MA_CHUNK; i < e; ++i)
            if (i >= first && key[i] > m) m = key[i];
        agg[c] = m;
    }
}
// exclusive running maximum over the chunk aggregates (one thread: n / 256 values)
__global__ void ma_spine_max(int64_t* agg, int64_t n_chunks) {
    if (MA_TID != 0) return;
    int64_t run = INT64_MIN;
    for (int64_t c = 0; c < n_chunks; ++c) {
        const int64_t v = agg[c];
        agg[c] = run;
        if (v > run) run = v;
    }
}
// boundaries: a record from the first deletion on whose position lies beyond the reach of the records before it
__global__ void ma_reach_apply(const int64_t* __restrict__ key, const ugvc_recinfo* __restrict__ recinfo, int64_t n,
                               const unsigned long long* first_del, const int64_t* __restrict__ agg,
                               uint8_t* __restrict__ flags, int64_t* __restrict__ head_agg) {
    const int64_t n_chunks = (n + MA_CHUNK - 1) / MA_CHUNK, first = (int64_t)*first_del;
    for (int64_t c = MA_TID; c < n_chunks; c += MA_NTHREADS) {
        int64_t run = agg[c], last = -1;
        const int64_t e = (c + 1) * MA_CHUNK < n ? (c + 1) * MA_CHUNK : n;
        for (int64_t i = c * MA_CHUNK; i < e; ++i) {
            if (i < first) continue;
            if (i == first || (int64_t)recinfo[i].pos > run) {
                flags[i] |= MA_F_BOUNDARY;
                last = i;
            }
            if (key[i] > run) run = key[i];
        }
        head_agg[c] = last;
    }
}
// members: '*' records that are no boundary join the cluster of the last boundary before them
__global__ void ma_owner_apply(int64_t n, const unsigned long long* first_del, const int64_t* __restrict__ head_agg,
                               uint8_t* __restrict__ flags, int32_t* __restrict__ owner, int64_t* open_head) {
    const int64_t n_chunks = (n + MA_CHUNK - 1) / MA_CHUNK, first = (int64_t)*first_del;
    for (int64_t c = MA_TID; c < n_chunks; c += MA_NTHREADS) {
        int64_t head = head_agg[c];  // exclusive running maximum: the last boundary before the chunk
        const int64_t e = (c + 1) * MA_CHUNK < n ? (c + 1) * MA_CHUNK : n;
        for (int64_t i = c * MA_CHUNK; i < e; ++i) {
            owner[i] = -1;
            if (i < first) continue;
            const uint8_t f = flags[i];
            if (f & MA_F_BOUNDARY) {
                head = i;
            } else if (f & MA_F_STAR) {
                flags[i] = f | MA_F_MEMBER;
                owner[i] = (int32_t)head;
            }
        }
        if (e == n) *open_head = head;
    }
}
__global__ void ma_mark_heads(int64_t n, const int32_t* __restrict__ owner, uint8_t* __restrict__ head_mark) {
    for (int64_t i = MA_TID; i < n; i += MA_NTHREADS)
        if (owner[i] >= 0) head_mark[owner[i]] = 1;  // (every writer stores the same value)
}
// the role of every record + chunk counts {singles, cluster records, kept bytes, kept records}
__global__ void ma_groups_agg(int64_t n, const int64_t* __restrict__ line_start, const int32_t* __restrict__ owner,
                              const uint8_t* __restrict__ head_mark, const int64_t* open_head, uint8_t* __restrict__ flags,
                              int64_t* __restrict__ agg4) {
    const int64_t n_chunks = (n + MA_CHUNK - 1) / MA_CHUNK, open = *open_head;
    for (int64_t c = MA_TID; c < n_chunks; c += MA_NTHREADS) {
        int64_t ns = 0, nc = 0, kb = 0, kr = 0;
        const int64_t e = (c + 1) * MA_CHUNK < n ? (c + 1) * MA_CHUNK : n;
        for (int64_t i = c * MA_CHUNK; i < e; ++i) {
            uint8_t f = flags[i];
            // the cluster still open at the end of the contig is never flushed; a cluster of one record is none
            const bool in_cluster = ((f & MA_F_MEMBER) && owner[i] != open) || ((f & MA_F_BOUNDARY) && head_mark[i] && i != open);
            const bool single = (f & MA_F_MULTI) && !in_cluster;
            f |= (uint8_t)((in_cluster ? MA_F_IN_CLUSTER : 0u) | (single ? MA_F_SINGLE : 0u));
            flags[i] = f;
            ns += single;
            nc += in_cluster;
            if (!single && !in_cluster) {
                kb += line_start[i + 1] - line_start[i];
                ++kr;
            }
        }
        agg4[4 * c + 0] = ns;
        agg4[4 * c + 1] = nc;
        agg4[4 * c + 2] = kb;
        agg4[4 * c + 3] = kr;
    }
}
__global__ void ma_spine_sum4(int64_t* agg4, int64_t n_chunks, int64_t* totals) {
    if (MA_TID != 0) return;
    int64_t run[4] = {0, 0, 0, 0};
    for (int64_t c = 0; c < n_chunks; ++c)
        for (int k = 0; k < 4; ++k) {
            const int64_t v = agg4[4 * c + k];
            agg4[4 * c + k] = run[k];
            run[k] += v;
        }
    for (int k = 0; k < 4; ++k) totals[k] = run[k];
}
// group list (singles, then cluster records, both ascending), kept-line offsets, row of every kept record
__global__ void ma_groups_apply(int64_t n, const int64_t* __restrict__ line_start, const int32_t* __restrict__ owner,
                                const uint8_t* __restrict__ flags, const ugvc_recinfo* __restrict__ recinfo,
                                const int64_t* __restrict__ agg4, const int64_t* totals, MaGroup* __restrict__ groups,
                                int64_t* __restrict__ kept_off, int64_t* __restrict__ rec_row) {
    const int64_t n_chunks = (n + MA_CHUNK - 1) / MA_CHUNK, n_singles = totals[0];
    for (int64_t c = MA_TID; c < n_chunks; c += MA_NTHREADS) {
        int64_t ns = agg4[4 * c + 0], nc = agg4[4 * c + 1], kb = agg4[4 * c + 2], kr = agg4[4 * c + 3];
        const int64_t e = (c + 1) * MA_CHUNK < n ? (c + 1) * MA_CHUNK : n;
        for (int64_t i = c * MA_CHUNK; i < e; ++i) {
            const uint8_t f = flags[i];
            if (f & (MA_F_SINGLE | MA_F_IN_CLUSTER)) {
                const int64_t g = (f & MA_F_SINGLE) ? ns++ : n_singles + nc++;
                MaGroup G;
                memset(&G, 0, sizeof(G));
                G.origin = (int32_t)i;
                G.head = -1;
                if (f & MA_F_SINGLE) {
                    G.kind = MA_KIND_PLAIN;
                } else if (f & MA_F_MEMBER) {
                    G.kind = MA_KIND_SPANNED;
                    G.head = owner[i];
                } else {
                    G.kind = 0xFFu;  // a cluster head: as it is when biallelic, a plain split otherwise (decided on its alleles)
                }
                groups[g] = G;
                kept_off[i] = -1;
                rec_row[i] = -(g + 1);
            } else {
                kept_off[i] = kb;
                kb += line_start[i + 1] - line_start[i];
                rec_row[i] = kr++;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// kernels: rows
// ---------------------------------------------------------------------------------------------------
// stable order of the ALT alleles by key (argsort(kind="stable") + 1)
__device__ inline void ma_order(const long long* keyv, int n_alt, uint8_t* order) {
    for (int i = 0; i < n_alt; ++i) {
        int j = i;
        while (j > 0 && keyv[order[j - 1] - 1] > keyv[i]) {
            order[j] = order[j - 1];
            --j;
        }
        order[j] = (uint8_t)(i + 1);
    }
}
// first allele spelled like allele a (tuple.index on the strings)
__device__ inline uint8_t ma_first_like(const uint8_t* t, const MaRec& r, int a) {
    for (int i = 0; i < a; ++i)
        if (ma_eq_span(t, r.al[i], r.al[a])) return (uint8_t)i;
    return (uint8_t)a;
}
// tr / th: the pointers through which the record's and the spanning deletion's line are read (ma_stage)
__device__ int ma_plan_group(const uint8_t* tr, const uint8_t* th, const int64_t* line_start, MaGroup& G, MaRec* r, MaRec* head,
                             bool* use_head) {
    const uint8_t* t = tr;
    int rc;
    *use_head = false;
    if ((rc = ma_parse_rec(tr, (uint32_t)line_start[G.origin], (uint32_t)line_start[G.origin + 1] - 1u, r)) != MA_OK) return rc;
    if (r->n_alleles > MA_MAX_ALLELES) return MA_E_LIMIT;
    G.n_alleles = (uint8_t)r->n_alleles;
    if (G.kind == 0xFFu) G.kind = r->n_alleles == 2 ? MA_KIND_AS_IS : MA_KIND_PLAIN;
    if (G.kind == MA_KIND_AS_IS) {
        G.n_rows = 1;
        return MA_OK;
    }
    if (G.kind == MA_KIND_SPANNED) {
        if ((rc = ma_parse_rec(th, (uint32_t)line_start[G.head], (uint32_t)line_start[G.head + 1] - 1u, head)) != MA_OK) return rc;
        if (head->n_alleles > MA_MAX_ALLELES) return MA_E_LIMIT;
        *use_head = true;
    }
    MaSpan plv;
    uint32_t pln;
    if ((rc = ma_pl_check(t, *r, &plv, &pln)) != MA_OK) return rc;
    const int n = r->n_alleles, n_alt = n - 1;
    long long keyv[MA_MAX_ALLELES];
    uint8_t order[MA_MAX_ALLELES];
    if (G.kind == MA_KIND_PLAIN) {
        // split_multiallelic_variants (multiallelics.py:65-127): strongest = lowest hom-alt PL, alleles absent from GT last
        for (int i = 1; i < n; ++i) {
            long long v;
            if ((rc = ma_pl_at(t, plv, pln, ma_pl_idx((uint32_t)i, (uint32_t)i), &v)) != MA_OK) return rc;
            bool ha, hb;
            if ((rc = ma_gt_has(t, *r, i, i, &ha, &hb)) != MA_OK) return rc;
            keyv[i - 1] = v + (ha ? 0 : 1000);
        }
        ma_order(keyv, n_alt, order);
        int m = 0;
        for (int i = 0; i < n_alt; ++i)
            if (!ma_eq_lit(t, r->al[order[i]], "*")) order[m++] = order[i];
        if (m == 0) return MA_E_INDEX;
        G.pair[0] = 0;
        G.pair[1] = order[0];
        G.n_rows = 1;
        if (m > 1) {
            G.pair[2] = order[0];
            G.pair[3] = order[1];
            G.n_rows = 2;
        }
    } else {
        // split_multiallelic_variants_with_spandel (spandel.py:11-63): '*' is forced to be the weakest allele
        int star = -1;
        for (int i = 0; i < n && star < 0; ++i)
            if (ma_eq_lit(t, r->al[i], "*")) star = i;
        if (star < 0) return MA_E_VALUE;
        for (int i = 1; i < n; ++i) {
            long long v;
            if ((rc = ma_pl_at(t, plv, pln, ma_pl_idx((uint32_t)i, (uint32_t)i), &v)) != MA_OK) return rc;
            keyv[i - 1] = v + (i == star ? 100000 : 0);
        }
        ma_order(keyv, n_alt, order);
        if (n_alt < 2) return MA_E_INDEX;
        G.pair[0] = 0;
        G.pair[1] = order[0];
        G.pair[2] = order[0];
        G.pair[3] = order[1];
        G.n_rows = 2;
    }
    if (G.n_rows == 2) {
        G.i1 = ma_first_like(t, *r, G.pair[2]);
        G.i2 = ma_first_like(t, *r, G.pair[3]);
    }
    return MA_OK;
}
// the line [ls, le] (its newline included) -> buf; returns the pointer through which the line's absolute text offsets
// reach the copy (buf - ls: only ever dereferenced at offsets inside the line), or t when the line does not fit
__device__ inline const uint8_t* ma_stage(const uint8_t* t, uint32_t ls, uint32_t le, uint8_t* buf) {
    const uint32_t len = le + 1u - ls;
    if (len > MA_STAGE_BYTES) return t;
    for (uint32_t b = MA_LANE; b < len; b += MA_LANES) buf[b] = t[ls + b];
    return buf - ls;
}
struct MaRowShared {
    uint8_t line[MA_ROW_WARPS][2][MA_STAGE_BYTES];
    MaRule rules[MA_RULES_SMEM];
};
// the rule table in shared memory when it fits (every INFO / FORMAT key of a row is looked up in it)
__device__ inline MaRules ma_stage_rules(const MaRules& R, MaRule* buf) {
    MaRules out = R;
    const uint32_t n = R.h.n_info + R.h.n_fmt;
    if (n <= MA_RULES_SMEM) {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(R.info);  // (the two tables are one array: info, then fmt)
        uint32_t* dst = reinterpret_cast<uint32_t*>(buf);
        for (uint32_t i = threadIdx.x; i < n * (uint32_t)(sizeof(MaRule) / 4u); i += blockDim.x) dst[i] = src[i];
        out.info = buf;
        out.fmt = buf + R.h.n_info;
    }
    __syncthreads();
    return out;
}
__global__ void __launch_bounds__(MA_ROW_WARPS * 32) ma_plan_rows(const uint8_t* __restrict__ t, const int64_t* __restrict__ line_start,
                             MaRules Rg, const uint8_t* __restrict__ ref, int64_t ref_len, MaGroup* __restrict__ groups,
                             int64_t n_groups, unsigned long long* err, int* width_groups) {
    __shared__ __align__(16) MaRowShared sh;
    const MaRules R = ma_stage_rules(Rg, sh.rules);
    const uint32_t warp = threadIdx.x / MA_LANES;
    const int64_t n_warps = (int64_t)gridDim.x * (blockDim.x / MA_LANES);
    for (int64_t g = (int64_t)blockIdx.x * (blockDim.x / MA_LANES) + warp; g < n_groups; g += n_warps) {
        MaGroup G = groups[g];
        const uint8_t* tr = ma_stage(t, (uint32_t)line_start[G.origin], (uint32_t)line_start[G.origin + 1] - 1u, sh.line[warp][0]);
        const uint8_t* th = G.head >= 0 ? ma_stage(t, (uint32_t)line_start[G.head], (uint32_t)line_start[G.head + 1] - 1u, sh.line[warp][1]) : t;
        MA_WARP_SYNC();
        if (MA_LANE == 0u) {
            MaRec r, head;
            bool use_head;
            int rc = ma_plan_group(tr, th, line_start, G, &r, &head, &use_head);
            for (int k = 0; rc == MA_OK && k < G.n_rows; ++k) {
                MaSink s{nullptr, 0};
                if (G.kind == MA_KIND_AS_IS) rc = ma_row(s, R, r, -1, -1, nullptr, ref, ref_len, true);
                else rc = ma_row(s, R, r, G.pair[2 * k], G.pair[2 * k + 1], use_head ? &head : nullptr, ref, ref_len, true);
                G.size[k] = s.n;
            }
            if (rc != MA_OK) {
                G.err = (uint8_t)rc;
                G.n_rows = 0;
                atomicMin(err, ((unsigned long long)g << 8) | (unsigned long long)rc);
            } else if (G.n_rows == 2) {
                atomicMax(width_groups, (int)G.n_alleles * ((int)G.n_alleles + 1) / 2);
            }
            groups[g] = G;
        }
        MA_WARP_SYNC();  // the buffers are free for the warp's next group
    }
}
// row offsets in group order: three-phase scan over chunks of MA_CHUNK groups of {bytes, rows}
__global__ void ma_rowoff_agg(const MaGroup* __restrict__ groups, int64_t n_groups, int64_t* __restrict__ agg2) {
    const int64_t n_chunks = (n_groups + MA_CHUNK - 1) / MA_CHUNK;
    for (int64_t c = MA_TID; c < n_chunks; c += MA_NTHREADS) {
        int64_t bytes = 0, rows = 0;
        const int64_t e = (c + 1) * MA_CHUNK < n_groups ? (c + 1) * MA_CHUNK : n_groups;
        for (int64_t g = c * MA_CHUNK; g < e; ++g) {
            const int nr = groups[g].n_rows;
            rows += nr;
            for (int k = 0; k < nr; ++k) bytes += groups[g].size[k];
        }
        agg2[2 * c] = bytes;
        agg2[2 * c + 1] = rows;
    }
}
__global__ void ma_spine_sum2(int64_t* agg2, int64_t n_chunks, int64_t* totals) {
    if (MA_TID != 0) return;
    int64_t bytes = 0, rows = 0;
    for (int64_t c = 0; c < n_chunks; ++c) {
        const int64_t b = agg2[2 * c], r = agg2[2 * c + 1];
        agg2[2 * c] = bytes;
        agg2[2 * c + 1] = rows;
        bytes += b;
        rows += r;
    }
    totals[4] = bytes;
    totals[5] = rows;
}
__global__ void ma_rowoff_apply(MaGroup* __restrict__ groups, int64_t n_groups, const int64_t* __restrict__ agg2) {
    const int64_t n_chunks = (n_groups + MA_CHUNK - 1) / MA_CHUNK;
    for (int64_t c = MA_TID; c < n_chunks; c += MA_NTHREADS) {
        int64_t off = agg2[2 * c], row = agg2[2 * c + 1];
        const int64_t e = (c + 1) * MA_CHUNK < n_groups ? (c + 1) * MA_CHUNK : n_groups;
        for (int64_t g = c * MA_CHUNK; g < e; ++g) {
            const int nr = groups[g].n_rows;
            groups[g].row0 = (int32_t)row;
            for (int k = 0; k < nr; ++k) {
                groups[g].row_off[k] = off;
                off += groups[g].size[k];
            }
            row += nr;
        }
    }
}
__global__ void __launch_bounds__(MA_ROW_WARPS * 32) ma_write_rows(const uint8_t* __restrict__ t, const int64_t* __restrict__ line_start,
                              MaRules Rg, const uint8_t* __restrict__ ref, int64_t ref_len, const MaGroup* __restrict__ groups,
                              int64_t n_groups, uint8_t* __restrict__ out) {
    __shared__ __align__(16) MaRowShared sh;
    const MaRules R = ma_stage_rules(Rg, sh.rules);
    const uint32_t warp = threadIdx.x / MA_LANES;
    const int64_t n_warps = (int64_t)gridDim.x * (blockDim.x / MA_LANES);
    for (int64_t g = (int64_t)blockIdx.x * (blockDim.x / MA_LANES) + warp; g < n_groups; g += n_warps) {
        const MaGroup G = groups[g];
        if (G.n_rows == 0) continue;  // (warp-uniform)
        const uint8_t* tr = ma_stage(t, (uint32_t)line_start[G.origin], (uint32_t)line_start[G.origin + 1] - 1u, sh.line[warp][0]);
        const bool use_head = G.kind == MA_KIND_SPANNED;
        const uint8_t* th = use_head ? ma_stage(t, (uint32_t)line_start[G.head], (uint32_t)line_start[G.head + 1] - 1u, sh.line[warp][1]) : t;
        MA_WARP_SYNC();
        if (MA_LANE == 0u) {
            MaRec r, head;
            ma_parse_rec(tr, (uint32_t)line_start[G.origin], (uint32_t)line_start[G.origin + 1] - 1u, &r);
            if (use_head) ma_parse_rec(th, (uint32_t)line_start[G.head], (uint32_t)line_start[G.head + 1] - 1u, &head);
            for (int k = 0; k < G.n_rows; ++k) {
                MaSink s{out + G.row_off[k], 0};
                if (G.kind == MA_KIND_AS_IS) ma_row(s, R, r, -1, -1, nullptr, ref, ref_len, false);
                else ma_row(s, R, r, G.pair[2 * k], G.pair[2 * k + 1], use_head ? &head : nullptr, ref, ref_len, false);
            }
        }
        MA_WARP_SYNC();
    }
}
// the untouched lines in input order: a CTA per chunk of records, its threads on consecutive bytes of a line
__global__ void ma_copy_kept(const uint8_t* __restrict__ t, const int64_t* __restrict__ line_start,
                             const int64_t* __restrict__ kept_off, int64_t n, uint8_t* __restrict__ out) {
    const int64_t n_chunks = (n + MA_CHUNK - 1) / MA_CHUNK;
    for (int64_t c = blockIdx.x; c < n_chunks; c += gridDim.x) {
        const int64_t e = (c + 1) * MA_CHUNK < n ? (c + 1) * MA_CHUNK : n;
        int64_t i = c * MA_CHUNK;
        while (i < e) {
            if (kept_off[i] < 0) {
                ++i;
                continue;
            }
            int64_t j = i + 1;  // a run of kept lines is one contiguous piece on both sides
            while (j < e && kept_off[j] >= 0) ++j;
            const int64_t src = line_start[i], len = line_start[j] - src, dst = kept_off[i];
            for (int64_t b = threadIdx.x; b < len; b += blockDim.x) out[dst + b] = t[src + b];
            i = j;
        }
    }
}
// merge_and_assign_pls (variant_filtering_utils.py:346-408) + the fill loop of filter_variants_pipeline.py:170-172
__global__ void ma_merge(int64_t n, const int64_t* __restrict__ rec_row, const MaGroup* __restrict__ groups, int64_t n_kept,
                         const double* __restrict__ lik, int K, double* __restrict__ out, int W, unsigned long long* err) {
    for (int64_t i = MA_TID; i < n; i += MA_NTHREADS) {
        double* o = out + i * W;
        for (int k = 0; k < W; ++k) o[k] = 0.0;
        const int64_t rr = rec_row[i];
        if (rr >= 0) {
            for (int k = 0; k < K; ++k) o[k] = lik[rr * K + k];
            continue;
        }
        const int64_t g = -rr - 1;
        const MaGroup G = groups[g];
        const double* s0 = lik + (n_kept + G.row0) * K;
        if (G.n_rows == 1) {
            for (int k = 0; k < K; ++k) o[k] = s0[k];
            continue;
        }
        if (K < 3) {
            atomicMin(err, ((unsigned long long)g << 8) | (unsigned long long)MA_E_TWO_CLASS);
            continue;
        }
        const double* s1 = s0 + K;
        const uint32_t i1 = G.i1, i2 = G.i2;
        // row[where] = vals: a later assignment to the same cell wins
        o[ma_pl_idx(0, 0)] = s0[0];
        o[ma_pl_idx(0, i1)] = s0[1];
        o[ma_pl_idx(i1, i1)] = __dmul_rn(s0[2], s1[0]);
        o[ma_pl_idx(0, i2)] = 0.0;
        o[ma_pl_idx(i1, i2)] = __dmul_rn(s0[2], s1[1]);
        o[ma_pl_idx(i2, i2)] = __dmul_rn(s0[2], s1[2]);
    }
}
// -10 log10(lik + 1e-10).  The sum is the double nearest 1e-10 for lik = 0 (the literal 0.0 ma_merge writes, the 0 / 1
// probabilities of a random forest) and anything below 1e-26: its log10 lies 2^-56 from -10, which NumPy rounds to -10
// and so prints PL 100, while a log10 one ulp short of -10 would print 99.  That case is exact; any other value is CUDA's
// log10, within an ulp of NumPy's (DESIGN.md section 4).
__device__ __forceinline__ double ma_phred(double lik) {
    const double x = __dadd_rn(lik, 1e-10);
    return x == 1e-10 ? 100.0 : __dmul_rn(-10.0, log10(x));
}
// multiallelics.score_math (filter_variants_pipeline.py:174-180,192) over the merged N x W matrix, one thread per record:
// phreds of all W columns (the zero padding included, as NumPy's min over ph[1:] sees it), qual = max(30 + ph0 -
// min(ph[1:]), 0) summed in K3's order, low = qual <= threshold.  phreds may alias lik (a thread rewrites its own row).
__global__ void ma_score(const double* lik, int64_t n, int W, double threshold, double* phreds, double* __restrict__ qual,
                         uint8_t* __restrict__ low) {
    for (int64_t i = MA_TID; i < n; i += MA_NTHREADS) {
        const double* r = lik + i * W;
        double* o = phreds ? phreds + i * W : nullptr;
        double ph0 = 0.0, mn = 0.0;
        for (int k = 0; k < W; ++k) {
            const double p = ma_phred(r[k]);
            if (o) o[k] = p;
            if (k == 0) ph0 = p;
            else if (k == 1 || p < mn) mn = p;
        }
        double q = __dadd_rn(__dadd_rn(30.0, ph0), -mn);
        q = q < 0.0 ? 0.0 : q;
        qual[i] = q;
        low[i] = q <= threshold ? 1 : 0;
    }
}

// ---------------------------------------------------------------------------------------------------
// C ABI (include/ugvc_b200.h)
// ---------------------------------------------------------------------------------------------------
struct ugvc_ma {
    int device = 0;
    int sm_count = 1;
    std::string error;
    long long launches = 0;
    cudaStream_t stream = nullptr;
    // rules
    MaRules rules{};
    MaRule* d_rules = nullptr;
    bool has_rules = false;
    // per-contig state
    int64_t n = 0, n_groups = 0, n_singles = 0, n_kept = 0, n_rows = 0, kept_bytes = 0, rows_bytes = 0;
    int width_groups = 0;
    size_t cap_bytes = 0, cap_records = 0, cap_ref = 0, cap_groups = 0, cap_out = 0, cap_lik = 0, cap_mat = 0;
    uint8_t *d_text = nullptr, *d_ref = nullptr, *d_flags = nullptr, *d_head_mark = nullptr, *d_out = nullptr;
    int64_t *d_line_start = nullptr, *d_key = nullptr, *d_agg = nullptr, *d_agg4 = nullptr, *d_kept_off = nullptr, *d_rec_row = nullptr;
    int64_t* d_scalars = nullptr;  // [0..5] totals, [6] open head, [7] first deletion, [8] error word, [9] width
    int32_t* d_owner = nullptr;
    ugvc_recinfo* d_recinfo = nullptr;
    MaGroup* d_groups = nullptr;
    double *d_lik = nullptr, *d_mat = nullptr;
    unsigned long long last_err = ~0ull;
};

static int ma_fail(ugvc_ma* h, int code, const std::string& msg) {
    if (h) h->error = msg;
    return code;
}
#define MA_CU(call)                                                                                   \
    do {                                                                                              \
        cudaError_t _e = (call);                                                                      \
        if (_e != cudaSuccess) return ma_fail(h, UGVC_E_CUDA, std::string(#call) + ": " + cudaGetErrorString(_e)); \
    } while (0)

template <class T>
static cudaError_t ma_grow(T** p, size_t* cap, size_t need, size_t slack) {
    if (*p && *cap >= need) return cudaSuccess;
    if (*p) cudaFree(*p);
    *p = nullptr;
    *cap = 0;
    const cudaError_t e = cudaMalloc(p, (need + slack) * sizeof(T));
    if (e != cudaSuccess) {
        *p = nullptr;
        return e;
    }
    *cap = need + slack;
    return cudaSuccess;
}

extern "C" int ugvc_ma_create(int device, ugvc_ma** out) {
    if (!out) return UGVC_E_ARG;
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device < 0 || device >= n) return UGVC_E_CUDA;
    if (cudaSetDevice(device) != cudaSuccess) return UGVC_E_CUDA;
    ugvc_ma* h = new ugvc_ma();
    h->device = device;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess && prop.multiProcessorCount > 0) h->sm_count = prop.multiProcessorCount;
    if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess || cudaMalloc(&h->d_scalars, 16 * sizeof(int64_t)) != cudaSuccess) {
        delete h;
        return UGVC_E_CUDA;
    }
    *out = h;
    return UGVC_OK;
}
extern "C" void ugvc_ma_free(ugvc_ma* h) {
    if (!h) return;
    cudaSetDevice(h->device);
    cudaFree(h->d_rules); cudaFree(h->d_text); cudaFree(h->d_ref); cudaFree(h->d_flags); cudaFree(h->d_head_mark);
    cudaFree(h->d_out); cudaFree(h->d_line_start); cudaFree(h->d_key); cudaFree(h->d_agg); cudaFree(h->d_agg4);
    cudaFree(h->d_kept_off); cudaFree(h->d_rec_row); cudaFree(h->d_scalars); cudaFree(h->d_owner); cudaFree(h->d_recinfo);
    cudaFree(h->d_groups); cudaFree(h->d_lik); cudaFree(h->d_mat);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
}
extern "C" const char* ugvc_ma_last_error(const ugvc_ma* h) { return h ? h->error.c_str() : "no handle"; }
extern "C" long long ugvc_ma_launch_count(const ugvc_ma* h) { return h ? h->launches : 0; }

extern "C" int ugvc_ma_set_rules(ugvc_ma* h, const void* blob, size_t n_bytes) {
    if (!h || !blob) return UGVC_E_ARG;
    if (n_bytes < sizeof(MaRulesHeader)) return ma_fail(h, UGVC_E_PLAN, "rules blob too small");
    MaRulesHeader hd;
    memcpy(&hd, blob, sizeof(hd));
    if (hd.magic != MA_RULES_MAGIC) return ma_fail(h, UGVC_E_PLAN, "bad rules magic");
    const size_t n_rules = (size_t)hd.n_info + hd.n_fmt;
    if (n_rules > 65536u || n_bytes != sizeof(hd) + n_rules * sizeof(MaRule)) return ma_fail(h, UGVC_E_PLAN, "rules blob size mismatch");
    for (int k = 0; k < 4; ++k)
        if (hd.special_len[k] == 0 || hd.special_len[k] > 32) return ma_fail(h, UGVC_E_PLAN, "bad special tag");
    const MaRule* src = reinterpret_cast<const MaRule*>(static_cast<const uint8_t*>(blob) + sizeof(hd));
    for (size_t i = 0; i < n_rules; ++i)
        if (src[i].len == 0 || src[i].len > 32 || src[i].action > MA_SPECIAL + 3) return ma_fail(h, UGVC_E_PLAN, "bad rule");
    MA_CU(cudaSetDevice(h->device));
    h->has_rules = false;  // (until the new table is in place)
    cudaFree(h->d_rules);
    h->d_rules = nullptr;
    MA_CU(cudaMalloc(&h->d_rules, (n_rules ? n_rules : 1) * sizeof(MaRule)));
    if (n_rules) MA_CU(cudaMemcpy(h->d_rules, src, n_rules * sizeof(MaRule), cudaMemcpyHostToDevice));
    h->rules.h = hd;
    h->rules.info = h->d_rules;
    h->rules.fmt = h->d_rules + hd.n_info;
    h->has_rules = true;
    return UGVC_OK;
}

// the per-record scratch of a contig of n records and its reference sequence, grown on demand
static int ma_reserve(ugvc_ma* h, int64_t n, size_t ref_len) {
    {
        size_t c;
        c = h->cap_ref; MA_CU(ma_grow(&h->d_ref, &c, ref_len + 64, 0)); h->cap_ref = c;
        if ((size_t)n + 1 > h->cap_records) {
            const size_t cap = (size_t)n + 1 + (size_t)n / 8;
            const size_t chunks = (cap + MA_CHUNK - 1) / MA_CHUNK + 1;
            cudaFree(h->d_line_start); cudaFree(h->d_recinfo); cudaFree(h->d_key); cudaFree(h->d_flags); cudaFree(h->d_head_mark);
            cudaFree(h->d_owner); cudaFree(h->d_kept_off); cudaFree(h->d_rec_row); cudaFree(h->d_agg); cudaFree(h->d_agg4);
            h->d_line_start = nullptr; h->d_recinfo = nullptr; h->d_key = nullptr; h->d_flags = nullptr; h->d_head_mark = nullptr;
            h->d_owner = nullptr; h->d_kept_off = nullptr; h->d_rec_row = nullptr; h->d_agg = nullptr; h->d_agg4 = nullptr;
            h->cap_records = 0;
            MA_CU(cudaMalloc(&h->d_line_start, cap * sizeof(int64_t)));
            MA_CU(cudaMalloc(&h->d_recinfo, cap * sizeof(ugvc_recinfo)));
            MA_CU(cudaMalloc(&h->d_key, cap * sizeof(int64_t)));
            MA_CU(cudaMalloc(&h->d_flags, cap));
            MA_CU(cudaMalloc(&h->d_head_mark, cap));
            MA_CU(cudaMalloc(&h->d_owner, cap * sizeof(int32_t)));
            MA_CU(cudaMalloc(&h->d_kept_off, cap * sizeof(int64_t)));
            MA_CU(cudaMalloc(&h->d_rec_row, cap * sizeof(int64_t)));
            MA_CU(cudaMalloc(&h->d_agg, chunks * sizeof(int64_t)));
            MA_CU(cudaMalloc(&h->d_agg4, chunks * 4 * sizeof(int64_t)));
            h->cap_records = cap;
        }
    }
    return UGVC_OK;
}

int ma_build_on(ugvc_ma* h, const uint8_t* d_text, size_t n_bytes, const int64_t* d_line_start, const ugvc_recinfo* d_recinfo,
                int64_t n_records, const uint8_t* ref_seq, size_t ref_len, cudaStream_t st, int64_t out[8]) {
    if (!h || !out || (n_bytes && !d_text) || !d_line_start || (n_records && !d_recinfo) || (ref_len && !ref_seq) || n_records < 0)
        return ma_fail(h, UGVC_E_ARG, "ma_build: bad arguments");
    if (!h->has_rules) return ma_fail(h, UGVC_E_STATE, "ma_build: set the rules first");
    if (n_bytes >= (1ull << 32) - 64u) return ma_fail(h, UGVC_E_ARG, "ma_build: a contig's text must stay below 4 GiB");
    MA_CU(cudaSetDevice(h->device));
    const int64_t n = n_records, n_chunks = (n + MA_CHUNK - 1) / MA_CHUNK;
    h->n = n;
    h->n_groups = h->n_singles = h->n_kept = h->n_rows = h->kept_bytes = h->rows_bytes = 0;
    h->width_groups = 0;
    h->last_err = ~0ull;
    memset(out, 0, 8 * sizeof(int64_t));
    int rc = ma_reserve(h, n, ref_len);
    if (rc) return rc;
    if (n == 0) return UGVC_OK;
    if (ref_len) MA_CU(cudaMemcpyAsync(h->d_ref, ref_seq, ref_len, cudaMemcpyHostToDevice, st));
    MA_CU(cudaMemsetAsync(h->d_head_mark, 0, (size_t)n, st));
    int64_t init[16];
    memset(init, 0, sizeof(init));
    init[6] = -1;
    init[7] = (int64_t)n;           // first deletion: none
    init[8] = -1;                   // error word: all ones
    MA_CU(cudaMemcpyAsync(h->d_scalars, init, sizeof(init), cudaMemcpyHostToDevice, st));
    unsigned long long* d_first = reinterpret_cast<unsigned long long*>(h->d_scalars + 7);
    unsigned long long* d_err = reinterpret_cast<unsigned long long*>(h->d_scalars + 8);
    int* d_width = reinterpret_cast<int*>(h->d_scalars + 9);
    const int tpb = 256;
    const int grid_rec = (int)((n + tpb - 1) / tpb < (int64_t)h->sm_count * 8 ? (n + tpb - 1) / tpb : (int64_t)h->sm_count * 8);
    const int grid_chunk = (int)((n_chunks + 63) / 64 < (int64_t)h->sm_count * 8 ? (n_chunks + 63) / 64 : (int64_t)h->sm_count * 8);
    MA_LAUNCH(ma_scan_alleles, grid_rec, tpb, st, d_text, d_line_start, d_recinfo, n, h->d_key, h->d_flags, d_first);
    MA_LAUNCH(ma_reach_agg, grid_chunk, 64, st, h->d_key, n, d_first, h->d_agg);
    MA_LAUNCH(ma_spine_max, 1, 1, st, h->d_agg, n_chunks);
    int64_t* d_head_agg = h->d_agg4;  // (free until ma_groups_agg)
    MA_LAUNCH(ma_reach_apply, grid_chunk, 64, st, h->d_key, d_recinfo, n, d_first, h->d_agg, h->d_flags, d_head_agg);
    MA_LAUNCH(ma_spine_max, 1, 1, st, d_head_agg, n_chunks);
    MA_LAUNCH(ma_owner_apply, grid_chunk, 64, st, n, d_first, d_head_agg, h->d_flags, h->d_owner, h->d_scalars + 6);
    MA_LAUNCH(ma_mark_heads, grid_rec, tpb, st, n, h->d_owner, h->d_head_mark);
    MA_LAUNCH(ma_groups_agg, grid_chunk, 64, st, n, d_line_start, h->d_owner, h->d_head_mark, h->d_scalars + 6, h->d_flags, h->d_agg4);
    MA_LAUNCH(ma_spine_sum4, 1, 1, st, h->d_agg4, n_chunks, h->d_scalars);
    h->launches += 9;
    int64_t totals[16];
    MA_CU(cudaMemcpyAsync(totals, h->d_scalars, sizeof(totals), cudaMemcpyDeviceToHost, st));
    MA_CU(cudaStreamSynchronize(st));
    MA_CU(cudaGetLastError());
    h->n_singles = totals[0];
    h->n_groups = totals[0] + totals[1];
    h->kept_bytes = totals[2];
    h->n_kept = totals[3];
    {
        size_t c = h->cap_groups;
        MA_CU(ma_grow(&h->d_groups, &c, (size_t)h->n_groups + 1, (size_t)h->n_groups / 4));
        h->cap_groups = c;
    }
    MA_LAUNCH(ma_groups_apply, grid_chunk, 64, st, n, d_line_start, h->d_owner, h->d_flags, d_recinfo, h->d_agg4, h->d_scalars,
              h->d_groups, h->d_kept_off, h->d_rec_row);
    // a warp per group
    const int64_t grp_ctas = (h->n_groups + MA_ROW_WARPS - 1) / MA_ROW_WARPS;
    const int grid_grp = (int)(grp_ctas < (int64_t)h->sm_count * 16 ? grp_ctas : (int64_t)h->sm_count * 16);
    const int row_tpb = (int)(MA_ROW_WARPS * MA_LANES);
    const int64_t grp_chunks = (h->n_groups + MA_CHUNK - 1) / MA_CHUNK;
    const int grid_gchunk = (int)((grp_chunks + 63) / 64 > 0 ? (grp_chunks + 63) / 64 : 1);
    if (h->n_groups) {
        MA_LAUNCH(ma_plan_rows, grid_grp, row_tpb, st, d_text, d_line_start, h->rules, h->d_ref, (int64_t)ref_len, h->d_groups, h->n_groups,
                  d_err, d_width);
        MA_LAUNCH(ma_rowoff_agg, grid_gchunk, 64, st, h->d_groups, h->n_groups, h->d_agg4);
        h->launches += 2;
    }
    MA_LAUNCH(ma_spine_sum2, 1, 1, st, h->d_agg4, grp_chunks, h->d_scalars);
    if (h->n_groups) {
        MA_LAUNCH(ma_rowoff_apply, grid_gchunk, 64, st, h->d_groups, h->n_groups, h->d_agg4);
        h->launches += 1;
    }
    h->launches += 2;
    MA_CU(cudaMemcpyAsync(totals, h->d_scalars, sizeof(totals), cudaMemcpyDeviceToHost, st));
    MA_CU(cudaStreamSynchronize(st));
    MA_CU(cudaGetLastError());
    h->rows_bytes = totals[4];
    h->n_rows = totals[5];
    h->last_err = (unsigned long long)totals[8];
    memcpy(&h->width_groups, &totals[9], sizeof(int));
    out[0] = h->n_singles;
    out[1] = h->n_groups - h->n_singles;
    out[2] = h->n_kept;
    out[3] = h->n_rows;
    out[4] = h->kept_bytes;
    out[5] = h->rows_bytes;
    out[6] = h->width_groups;
    {
        size_t c = h->cap_out;
        MA_CU(ma_grow(&h->d_out, &c, (size_t)(h->kept_bytes + h->rows_bytes) + 64, (size_t)h->kept_bytes / 16));
        h->cap_out = c;
    }
    const int grid_copy = (int)(n_chunks < (int64_t)h->sm_count * 16 ? n_chunks : (int64_t)h->sm_count * 16);  // a CTA per chunk of records
    MA_LAUNCH(ma_copy_kept, grid_copy, 128, st, d_text, d_line_start, h->d_kept_off, n, h->d_out);
    if (h->n_groups) {
        MA_LAUNCH(ma_write_rows, grid_grp, row_tpb, st, d_text, d_line_start, h->rules, h->d_ref, (int64_t)ref_len, h->d_groups, h->n_groups,
                  h->d_out + h->kept_bytes);
        h->launches += 1;
    }
    h->launches += 1;
    MA_CU(cudaStreamSynchronize(st));
    MA_CU(cudaGetLastError());
    if (h->last_err != ~0ull) return ma_fail(h, UGVC_E_DATA, "a record the reference raises on (ugvc_ma_data_error)");
    return UGVC_OK;
}
uint8_t* ma_scored_text(ugvc_ma* h) { return h->d_out; }
int ma_device_of(const ugvc_ma* h) { return h->device; }

// One contig: text + the index pass's line starts / recinfo + the contig's reference sequence -> groups, split rows,
// the text of the scored pass.  out[0..7] = {n_singles, n_cluster_records, n_kept_records, n_rows, kept_bytes,
// rows_bytes, width of the widest two-row group's genotype vector, 0}.  UGVC_E_DATA: a group the reference raises
// on (ugvc_ma_data_error tells which and why).  The host inputs are copied to the handle's buffers, then ma_build_on.
extern "C" int ugvc_ma_build(ugvc_ma* h, const uint8_t* text, size_t n_bytes, const int64_t* line_start, const ugvc_recinfo* recinfo,
                             int64_t n_records, const uint8_t* ref_seq, size_t ref_len, int64_t out[8]) {
    if (!h || !out || (n_bytes && !text) || !line_start || (n_records && !recinfo) || (ref_len && !ref_seq) || n_records < 0)
        return ma_fail(h, UGVC_E_ARG, "ma_build: bad arguments");
    if (n_bytes >= (1ull << 32) - 64u) return ma_fail(h, UGVC_E_ARG, "ma_build: a contig's text must stay below 4 GiB");
    MA_CU(cudaSetDevice(h->device));
    cudaStream_t st = h->stream;
    {
        size_t c = h->cap_bytes;
        MA_CU(ma_grow(&h->d_text, &c, n_bytes + 64, n_bytes / 8));
        h->cap_bytes = c;
    }
    int rc = ma_reserve(h, n_records, ref_len);
    if (rc) return rc;
    if (n_records) {
        MA_CU(cudaMemcpyAsync(h->d_text, text, n_bytes, cudaMemcpyHostToDevice, st));
        MA_CU(cudaMemcpyAsync(h->d_line_start, line_start, ((size_t)n_records + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, st));
        MA_CU(cudaMemcpyAsync(h->d_recinfo, recinfo, (size_t)n_records * sizeof(ugvc_recinfo), cudaMemcpyHostToDevice, st));
    }
    return ma_build_on(h, h->d_text, n_bytes, h->d_line_start, h->d_recinfo, n_records, ref_seq, ref_len, st, out);
}
// detail of the last UGVC_E_DATA: group index (singles first, then cluster records), its record, the MA_E_* code
extern "C" int ugvc_ma_data_error(const ugvc_ma* h, int64_t* group, int32_t* code) {
    if (!h || h->last_err == ~0ull) return UGVC_E_STATE;
    if (group) *group = (int64_t)(h->last_err >> 8);
    if (code) *code = (int32_t)(h->last_err & 0xFFu);
    return UGVC_OK;
}
// the text of the scored pass (kept lines, then the split rows) and the group table: origin record, rows, alleles per group
extern "C" int ugvc_ma_fetch(ugvc_ma* h, uint8_t* out_text, size_t capacity, int32_t* out_origin, uint8_t* out_n_rows,
                             uint8_t* out_n_alleles, size_t capacity_groups) {
    if (!h) return UGVC_E_ARG;
    MA_CU(cudaSetDevice(h->device));
    const size_t total = (size_t)(h->kept_bytes + h->rows_bytes);
    if (out_text) {
        if (capacity < total) return ma_fail(h, UGVC_E_ARG, "ma_fetch: text capacity too small");
        if (total) MA_CU(cudaMemcpy(out_text, h->d_out, total, cudaMemcpyDeviceToHost));
    }
    if (out_origin || out_n_rows || out_n_alleles) {
        if (capacity_groups < (size_t)h->n_groups) return ma_fail(h, UGVC_E_ARG, "ma_fetch: group capacity too small");
        if (h->n_groups) {
            MaGroup* tmp = static_cast<MaGroup*>(malloc((size_t)h->n_groups * sizeof(MaGroup)));
            if (!tmp) return ma_fail(h, UGVC_E_ARG, "ma_fetch: out of memory");
            const cudaError_t e = cudaMemcpy(tmp, h->d_groups, (size_t)h->n_groups * sizeof(MaGroup), cudaMemcpyDeviceToHost);
            if (e != cudaSuccess) {
                free(tmp);
                return ma_fail(h, UGVC_E_CUDA, cudaGetErrorString(e));
            }
            for (int64_t g = 0; g < h->n_groups; ++g) {
                if (out_origin) out_origin[g] = tmp[g].origin;
                if (out_n_rows) out_n_rows[g] = tmp[g].n_rows;
                if (out_n_alleles) out_n_alleles[g] = tmp[g].n_alleles;
            }
            free(tmp);
        }
    }
    return UGVC_OK;
}
int ma_merge_on(ugvc_ma* h, const double* d_lik, int64_t n_rows, int n_classes, int width, cudaStream_t st, double** d_mat) {
    if (!h || !d_lik || !d_mat || n_classes <= 0) return ma_fail(h, UGVC_E_ARG, "ma_merge: bad arguments");
    if (n_rows != h->n_kept + h->n_rows) return ma_fail(h, UGVC_E_ARG, "ma_merge: the scored pass returned an unexpected number of rows");
    const int need = h->width_groups > n_classes ? h->width_groups : n_classes;
    if (width != need) return ma_fail(h, UGVC_E_ARG, "ma_merge: width must be max(n_classes, widest group)");
    MA_CU(cudaSetDevice(h->device));
    size_t c = h->cap_mat;
    MA_CU(ma_grow(&h->d_mat, &c, (size_t)h->n * width + 8, 0));
    h->cap_mat = c;
    *d_mat = h->d_mat;
    const int64_t minus1 = -1;
    MA_CU(cudaMemcpyAsync(h->d_scalars + 8, &minus1, sizeof(minus1), cudaMemcpyHostToDevice, st));
    const int tpb = 256;
    const int grid = (int)((h->n + tpb - 1) / tpb < (int64_t)h->sm_count * 8 ? (h->n + tpb - 1) / tpb : (int64_t)h->sm_count * 8);
    if (h->n) {
        MA_LAUNCH(ma_merge, grid, tpb, st, h->n, h->d_rec_row, h->d_groups, h->n_kept, d_lik, n_classes, h->d_mat, width,
                  reinterpret_cast<unsigned long long*>(h->d_scalars + 8));
        h->launches += 1;
    }
    int64_t errw = -1;
    MA_CU(cudaMemcpyAsync(&errw, h->d_scalars + 8, sizeof(errw), cudaMemcpyDeviceToHost, st));
    MA_CU(cudaStreamSynchronize(st));
    MA_CU(cudaGetLastError());
    h->last_err = (unsigned long long)errw;
    if (h->last_err != ~0ull) return ma_fail(h, UGVC_E_DATA, "a 2-class model cannot be merged over a split record");
    return UGVC_OK;
}
// likelihoods of the scored pass (n_kept + n_rows rows of n_classes, row-major fp64) -> out[n_records][width],
// width = max(n_classes, widest two-row group).  The host likelihoods are copied to the handle's buffer, then ma_merge_on.
extern "C" int ugvc_ma_merge(ugvc_ma* h, const double* lik, int64_t n_rows, int n_classes, double* out, int width) {
    if (!h || !lik || !out || n_classes <= 0 || n_rows < 0) return UGVC_E_ARG;
    MA_CU(cudaSetDevice(h->device));
    cudaStream_t st = h->stream;
    size_t c = h->cap_lik;
    MA_CU(ma_grow(&h->d_lik, &c, (size_t)n_rows * n_classes + 8, 0));
    h->cap_lik = c;
    MA_CU(cudaMemcpyAsync(h->d_lik, lik, (size_t)n_rows * n_classes * sizeof(double), cudaMemcpyHostToDevice, st));
    double* d_mat = nullptr;
    const int rc = ma_merge_on(h, h->d_lik, n_rows, n_classes, width, st, &d_mat);
    if (rc) return rc;
    if (h->n) MA_CU(cudaMemcpy(out, d_mat, (size_t)h->n * width * sizeof(double), cudaMemcpyDeviceToHost));
    return UGVC_OK;
}

void ma_launch_score(const double* lik, int64_t n, int width, double threshold, double* phreds, double* qual, uint8_t* low,
                     int sm_count, cudaStream_t st) {
    if (n <= 0) return;
    const int tpb = 256;
    const int grid = (int)((n + tpb - 1) / tpb < (int64_t)sm_count * 8 ? (n + tpb - 1) / tpb : (int64_t)sm_count * 8);
    MA_LAUNCH(ma_score, grid, tpb, st, lik, n, width, threshold, phreds, qual, low);
}
