// fileio.cu -- the two file-side kernels of the tool on the device: the record writer and BGZF deflate.
//
// The reference writes every record back through pysam (FILTER / INFO setters, htslib formatter, BGZF writer:
// filter_variants_pipeline.py:188-228) and the round-1 tool did the same edit on host threads
// (hostio.cpp: ugvc_splice_records) followed by zlib.  Here the edited text never exists on the host:
//   splice_len    one thread per record: length of the edited line (new FILTER column, ";TREE_SCORE=<%g>", the
//                 BLACKLST annotations -- the CG flag and a binary search of POS in each blacklist --, the optional
//                 QUAL overwrite, the recalibrated GT / GQ / PL of the first sample)
//   (exclusive scan of the lengths -> out_line_start)
//   splice_copy   one warp per record: the pieces are copied with consecutive lanes on consecutive bytes, the short
//                 rewritten ones (FILTER, BLACKLST, the first sample) by lane 0 with the routine that measured them;
//                 INFO/END is picked up on the way.  Anything the simple INFO rule does not cover (an existing
//                 TREE_SCORE= / BLACKLST= key, empty INFO pieces, a "." INFO) raises a flag and the caller falls back
//                 to the host writer
//   deflate       one thread per 56 KiB of output text -> one BGZF block (deflate.cuh), then the blocks are
//                 packed back to back
// Same text as the host writer produces (tests compare the two), so the output contract is unchanged.
#include <cuda_runtime.h>
#include <stdint.h>

#include <cub/device/device_scan.cuh>

#include "deflate.cuh"
#include "fileio.cuh"

// ---- "%g" of a float32 >= 0 (what htslib prints for INFO / QUAL floats): six significant digits, exact
// round-half-even on the binary value, trailing zeros dropped.  Values that need the exponent form return 0.  %g
// picks the form from the exponent of the value ROUNDED to six digits: 9.999995e-5 prints as 0.0001, 999999.5 as 1e+06.
__device__ int fio_format_g(float v, char* out) {
    if (v == 0.0f) {
        out[0] = '0';
        return 1;
    }
    if (!(v >= 9.9999e-5f && v < 1e6f)) return 0;  // also NaN / negative / inf
    const uint32_t bits = __float_as_uint(v);
    const int bexp = (int)((bits >> 23) & 0xFFu);
    const uint64_t m = bexp ? ((bits & 0x7FFFFFu) | 0x800000u) : (bits & 0x7FFFFFu);
    const int s = -((bexp ? bexp : 1) - 150);  // v = m * 2^-s, s in [4, 37] for the accepted range
    const uint64_t P10[11] = {1ull,         10ull,         100ull,         1000ull,         10000ull,      100000ull,
                              1000000ull,   10000000ull,   100000000ull,   1000000000ull,   10000000000ull};
    int X = (int)floorf(log10f(v));  // decimal exponent, fixed below if the estimate is off by one
    X = X < -5 ? -5 : (X > 5 ? 5 : X);
    uint64_t q = 0;
    for (int attempt = 0; attempt < 4; ++attempt) {
        const int k = 5 - X;  // 0..10
        const uint64_t N = m * P10[k];  // v 10^k = N 2^-s, below 2^58
        const uint64_t t = N >> s;      // floor(v 10^k): v lies in decade X iff it has six digits (before rounding)
        if (t < 100000ull) {
            if (X == -5) return 0;
            --X;
            continue;
        }
        if (t >= 1000000ull) {
            if (X == 5) return 0;
            ++X;
            continue;
        }
        const uint64_t r = N & ((1ull << s) - 1ull), half = 1ull << (s - 1);
        q = t + ((r > half || (r == half && (t & 1ull))) ? 1ull : 0ull);
        if (q == 1000000ull) {  // the rounding carried into a seventh digit: 10^(X+1)
            q = 100000ull;
            ++X;
        }
        break;
    }
    if (q == 0 || X < -4 || X > 5) return 0;  // exponent form (q == 0: the estimate was off by more than the loop fixes)
    char dg[6];
    for (int i = 5; i >= 0; --i) {
        dg[i] = (char)('0' + (int)(q % 10ull));
        q /= 10ull;
    }
    int nd = 6;
    while (nd > 1 && dg[nd - 1] == '0') --nd;  // trailing zeros of the significand
    int n = 0;
    if (X >= 0) {
        for (int i = 0; i <= X; ++i) out[n++] = i < 6 ? dg[i] : '0';
        if (nd > X + 1) {
            out[n++] = '.';
            for (int i = X + 1; i < nd; ++i) out[n++] = dg[i];
        }
    } else {
        out[n++] = '0';
        out[n++] = '.';
        for (int i = 0; i < -X - 1; ++i) out[n++] = '0';
        for (int i = 0; i < nd; ++i) out[n++] = dg[i];
    }
    return n;
}

__device__ __forceinline__ bool fio_is(const uint8_t* p, uint32_t n, const char* lit, uint32_t ln) {
    if (n != ln) return false;
    for (uint32_t i = 0; i < ln; ++i)
        if (p[i] != (uint8_t)lit[i]) return false;
    return true;
}

// The FILTER column of the edited record (hostio.cpp splice_one): pieces split on ';', empty ones dropped, PASS dropped
// when the record fails, LOW_SCORE appended when it fails and is not there yet, PASS when nothing is left.
// out == nullptr: only the length.
__device__ uint32_t fio_filter(const uint8_t* fp, uint32_t fl, bool low, uint8_t* out) {
    uint32_t n = 0, written = 0;
    bool has_low = false;
    if (!(fl == 1 && fp[0] == '.')) {
        uint32_t s = 0;
        for (uint32_t e = 0; e <= fl; ++e) {
            if (e == fl || fp[e] == ';') {
                const uint32_t kn = e - s;
                const bool drop = kn == 0 || (low && fio_is(fp + s, kn, "PASS", 4));
                if (!drop) {
                    if (written) {
                        if (out) out[n] = ';';
                        ++n;
                    }
                    if (out)
                        for (uint32_t i = 0; i < kn; ++i) out[n + i] = fp[s + i];
                    n += kn;
                    ++written;
                    has_low |= fio_is(fp + s, kn, "LOW_SCORE", 9);
                }
                s = e + 1;
            }
        }
    }
    if (low && !has_low) {
        if (written) {
            if (out) out[n] = ';';
            ++n;
        }
        const char* L = "LOW_SCORE";
        if (out)
            for (int i = 0; i < 9; ++i) out[n + i] = (uint8_t)L[i];
        n += 9;
        ++written;
    }
    if (!written) {
        const char* P = "PASS";
        if (out)
            for (int i = 0; i < 4; ++i) out[n + i] = (uint8_t)P[i];
        n += 4;
    }
    return n;
}

#define FIO_SCORE_KEY ";TREE_SCORE="
#define FIO_SCORE_KEY_LEN 12u

struct FioRec {  // what both kernels need of a record
    uint32_t len, q0, f0, i0, x0;
    bool ok;
};
__device__ __forceinline__ FioRec fio_rec(const int64_t* line_start, const ugvc_recinfo* recinfo, int64_t i) {
    FioRec r;
    r.len = (uint32_t)(line_start[i + 1] - line_start[i] - 1);
    const ugvc_recinfo ri = recinfo[i];
    r.q0 = ri.qual_off;
    r.f0 = ri.filter_off;
    r.i0 = ri.info_off;
    r.x0 = ri.format_off;
    // long lines carry saturated offsets: the host writer recounts the tabs, this one hands the batch back
    r.ok = r.q0 != 0xFFFFu && r.f0 != 0xFFFFu && r.i0 != 0xFFFFu && r.x0 != 0xFFFFu && r.q0 > 0 && r.q0 <= r.f0 && r.f0 <= r.i0 &&
           r.i0 <= r.x0 && r.x0 <= r.len + 1u;
    return r;
}

// ---- small writers: out == nullptr only counts, so that the length pass and the copy pass share one routine
__device__ __forceinline__ uint32_t fio_put(uint8_t* out, uint32_t n, const uint8_t* src, uint32_t len) {
    if (out)
        for (uint32_t k = 0; k < len; ++k) out[n + k] = src[k];
    return n + len;
}
__device__ __forceinline__ uint32_t fio_putc(uint8_t* out, uint32_t n, uint8_t c) {
    if (out) out[n] = c;
    return n + 1;
}
__device__ uint32_t fio_put_int(uint8_t* out, uint32_t n, int v) {  // std::to_string(int)
    char d[10];
    int k = 0;
    uint32_t u = v < 0 ? 0u - (uint32_t)v : (uint32_t)v;
    do {
        d[k++] = (char)('0' + u % 10u);
        u /= 10u;
    } while (u);
    if (v < 0) n = fio_putc(out, n, '-');
    while (k) n = fio_putc(out, n, (uint8_t)d[--k]);
    return n;
}

// ---- BLACKLST: ";BLACKLST=" and the ','-joined values of the record's annotation bits in merge order (bit 0: the CG
// insertion flag, bit k + 1: blacklist k), values that are empty skipped, nothing at all when no value is left
// (hostio.cpp splice_one; the host side of ugvc_filter_bgzf_edits already dropped the PASS / empty pieces of each value)
__device__ uint32_t fio_blacklst(uint32_t mask, int n_bl, const uint8_t* bl_name, const int32_t* bl_name_off, uint8_t* out) {
    uint32_t n = 0;
    bool any = false;
    for (int k = 0; k <= n_bl; ++k) {
        if (!((mask >> k) & 1u)) continue;
        const uint8_t* v = reinterpret_cast<const uint8_t*>("CG_NON_HMER_INDEL");
        uint32_t vl = 17;
        if (k) {
            v = bl_name + bl_name_off[k - 1];
            vl = (uint32_t)(bl_name_off[k] - bl_name_off[k - 1]);
        }
        if (!vl) continue;
        n = any ? fio_putc(out, n, ',') : fio_put(out, n, reinterpret_cast<const uint8_t*>(";BLACKLST="), 10);
        any = true;
        n = fio_put(out, n, v, vl);
    }
    return n;
}

// the annotation bits of a record: the CG flag of K1 under UGVC_FILE_BLACKLIST_CG, then a binary search of POS in each
// blacklist's sorted positions (Blacklist.apply with selection_fcn = ALL: a (chrom, pos) set; the caller uploads the
// positions of the range's contig)
__device__ uint32_t fio_bl_mask(int64_t pos, bool cg, int n_bl, const int64_t* bl_pos, const int64_t* bl_pos_off) {
    uint32_t mask = cg ? 1u : 0u;
    for (int k = 0; k < n_bl; ++k) {
        int64_t lo = bl_pos_off[k], hi = bl_pos_off[k + 1];
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (bl_pos[mid] < pos) lo = mid + 1;
            else hi = mid;
        }
        if (lo < bl_pos_off[k + 1] && bl_pos[lo] == pos) mask |= 2u << k;
    }
    return mask;
}

// ---- --recalibrate_genotype (hostio.cpp splice_one / recalibrated_sample): GQ = int(second smallest - smallest) of the
// n_classes phreds, PL = int() of the first min(n_classes, na (na + 1) / 2) of them (at least one), GT = the genotype of
// the first smallest PL (gt_from_pl_idx).  false: a phred that is not finite or whose int() would leave int32 -- the
// record is left to the host writer.
struct FioGeno {
    const double* ph;
    double gq;  // QUAL under UGVC_FILE_OVERWRITE_QUAL prints this, not int(gq)
    int n_pl, a, b;
};
__device__ bool fio_geno(const double* ph, int n_classes, uint32_t recflags, FioGeno& g) {
    if (n_classes < 2) return false;
    for (int k = 0; k < n_classes; ++k)
        if (!(fabs(ph[k]) < 2147483647.0)) return false;
    double m1 = ph[0], m2 = ph[1];
    if (m2 < m1) {
        const double t = m1;
        m1 = m2;
        m2 = t;
    }
    for (int k = 2; k < n_classes; ++k) {
        if (ph[k] < m1) {
            m2 = m1;
            m1 = ph[k];
        } else if (ph[k] < m2)
            m2 = ph[k];
    }
    g.ph = ph;
    g.gq = m2 - m1;
    if (!(g.gq < 2147483647.0)) return false;
    const int na = (int)((recflags >> 1) & 0x7Fu);
    int n_pl = (na + 1) * na / 2;
    if (n_pl > n_classes) n_pl = n_classes;
    if (n_pl < 1) n_pl = 1;
    g.n_pl = n_pl;
    int best = 0, bv = (int)ph[0];
    for (int k = 1; k < n_pl; ++k)
        if ((int)ph[k] < bv) {
            bv = (int)ph[k];
            best = k;
        }
    int count = 0, n_alleles = 0;  // gt_from_pl_idx: triangular index -> (a, b), a <= b
    while (count < best + 1) {
        count += n_alleles;
        ++n_alleles;
    }
    g.b = n_alleles - 2;
    g.a = best - (count - n_alleles) - 1;
    return true;
}

// the new value of GQ (which = 0), PL (1) or GT (2)
__device__ uint32_t fio_geno_value(uint8_t* out, uint32_t n, const FioGeno& g, int which, uint8_t sep) {
    if (which == 0) return fio_put_int(out, n, (int)g.gq);
    if (which == 1) {
        for (int k = 0; k < g.n_pl; ++k) {
            if (k) n = fio_putc(out, n, ',');
            n = fio_put_int(out, n, (int)g.ph[k]);
        }
        return n;
    }
    n = fio_put_int(out, n, g.a);
    n = fio_putc(out, n, sep);
    return fio_put_int(out, n, g.b);
}

// FORMAT and the first sample of a recalibrated record, `fmt` = the bytes after INFO's tab (len of them): the first GQ /
// PL / GT key of FORMAT gets the new value, keys FORMAT lacks are appended in that order, the sample's values are
// padded with "." to the keys (and cut to them), FORMAT "." counts as no keys; GT's separator is '|' when a GT value
// of the input holds one.  Returns the bytes of "FORMAT\tSAMPLE1"; *s1e = where the first sample ends in fmt (the
// other samples follow untouched).  Streams over the columns: no bound on the keys or the sample's length.
__device__ uint32_t fio_sample(const uint8_t* fmt, uint32_t len, const FioGeno& g, uint8_t* out, uint32_t* s1e_out) {
    uint32_t ftab = 0;
    while (ftab < len && fmt[ftab] != '\t') ++ftab;
    const uint32_t s1 = ftab < len ? ftab + 1 : len;
    uint32_t s1e = s1;
    while (s1e < len && fmt[s1e] != '\t') ++s1e;
    *s1e_out = s1e;
    const bool dot = ftab == 1 && fmt[0] == '.';
    int f_gq = -1, f_pl = -1, f_gt = -1;  // index of the first GQ / PL / GT key
    uint8_t sep = '/';
    int nkeys = 0;
    if (!dot) {  // the keys and the first sample's values side by side: value k of [vs, ve), or none left
        uint32_t ks = 0, vs = s1;
        bool vlive = true;
        for (uint32_t e = 0; e <= ftab; ++e) {
            if (e < ftab && fmt[e] != ':') continue;
            uint32_t ve = vs;
            if (vlive)
                while (ve < s1e && fmt[ve] != ':') ++ve;
            if (e - ks == 2) {
                const uint8_t c0 = fmt[ks], c1 = fmt[ks + 1];
                const int w = (c0 == 'G' && c1 == 'Q') ? 0 : (c0 == 'P' && c1 == 'L') ? 1 : (c0 == 'G' && c1 == 'T') ? 2 : -1;
                if (w == 0 && f_gq < 0) f_gq = nkeys;
                if (w == 1 && f_pl < 0) f_pl = nkeys;
                if (w == 2 && f_gt < 0) f_gt = nkeys;
                if (w == 2 && vlive)
                    for (uint32_t u = vs; u < ve; ++u)
                        if (fmt[u] == '|') sep = '|';
            }
            ++nkeys;
            if (vlive) {
                if (ve < s1e) vs = ve + 1;
                else vlive = false;
            }
            ks = e + 1;
        }
    }
    const uint8_t* K = reinterpret_cast<const uint8_t*>("GQPLGT");
    uint32_t n = dot ? 0u : fio_put(out, 0, fmt, ftab);
    int cnt = nkeys;
    for (int w = 0; w < 3; ++w)
        if ((w == 0 ? f_gq : w == 1 ? f_pl : f_gt) < 0) {
            if (cnt++) n = fio_putc(out, n, ':');
            n = fio_put(out, n, K + 2 * w, 2);
        }
    n = fio_putc(out, n, '\t');
    uint32_t vs = s1;
    bool vlive = true;
    for (int k = 0; k < nkeys; ++k) {
        uint32_t ve = vs;
        if (vlive)
            while (ve < s1e && fmt[ve] != ':') ++ve;
        if (k) n = fio_putc(out, n, ':');
        const int w = k == f_gq ? 0 : k == f_pl ? 1 : k == f_gt ? 2 : -1;
        if (w >= 0) n = fio_geno_value(out, n, g, w, sep);
        else if (vlive) n = fio_put(out, n, fmt + vs, ve - vs);
        else n = fio_putc(out, n, '.');
        if (vlive) {
            if (ve < s1e) vs = ve + 1;
            else vlive = false;
        }
    }
    cnt = nkeys;
    for (int w = 0; w < 3; ++w)
        if ((w == 0 ? f_gq : w == 1 ? f_pl : f_gt) < 0) {
            if (cnt++) n = fio_putc(out, n, ':');
            n = fio_geno_value(out, n, g, w, sep);
        }
    return n;
}

// splice_len: the length of every edited line (and what splice_copy needs of it: the formatted score, the annotation bits);
// a record the rules here do not cover raises `fallback` and the caller hands the range to the host writer
__global__ void __launch_bounds__(256) splice_len(const uint8_t* __restrict__ text, const int64_t* __restrict__ line_start,
                                                  const ugvc_recinfo* __restrict__ recinfo, const uint8_t* __restrict__ low_score,
                                                  const double* __restrict__ qual, int64_t n, const FioEdits ed,
                                                  int64_t* __restrict__ out_len, uint8_t* __restrict__ score_txt, int* fallback) {
    const bool recal = ed.phreds != nullptr;
    const bool owq = ed.with_model && (ed.flags & UGVC_FILE_OVERWRITE_QUAL);
    const bool want_num = ed.with_model && (!recal || owq);  // TREE_SCORE, or QUAL = GQ
    unsigned long long n_bl = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const FioRec r = fio_rec(line_start, recinfo, i);
        const ugvc_recinfo ri = recinfo[i];
        FioGeno g;
        bool ok = r.ok && (!recal || fio_geno(ed.phreds + (size_t)i * ed.n_classes, ed.n_classes, ri.flags, g));
        char num[16];
        int sl = 0;
        if (ok && want_num) {
            sl = fio_format_g((float)(recal ? g.gq : qual[i]), num);
            ok = sl != 0;
        }
        if (!ok) {
            atomicExch(fallback, 1);
            out_len[i] = 0;
            continue;
        }
        uint8_t* st = score_txt + (size_t)i * 16;
        st[15] = (uint8_t)sl;
        for (int c = 0; c < sl; ++c) st[c] = (uint8_t)num[c];
        const uint32_t mask = fio_bl_mask(ri.pos, (ed.flags & UGVC_FILE_BLACKLIST_CG) && (ri.flags & 1u), ed.n_bl, ed.bl_pos, ed.bl_pos_off);
        ed.bl_mask[i] = mask;
        n_bl += mask != 0u;
        const uint8_t* line = text + line_start[i];
        const bool low = ed.with_model && low_score[i] != 0;
        const uint32_t il = r.x0 - 1u - r.i0;
        uint32_t total = r.q0;                                                    // columns 1-5 with their tabs
        total += (owq ? (uint32_t)sl : r.f0 - 1u - r.q0) + 1u;                    // QUAL, tab
        total += fio_filter(line + r.f0, r.i0 - 1u - r.f0, low, nullptr) + 1u;    // FILTER, tab
        total += il;                                                              // INFO
        if (ed.with_model && !recal) total += FIO_SCORE_KEY_LEN + (uint32_t)sl;   // ;TREE_SCORE=<score>
        if (mask) total += fio_blacklst(mask, ed.n_bl, ed.bl_name, ed.bl_name_off, nullptr);  // ;BLACKLST=<annotations>
        if (r.x0 <= r.len) {                                                      // tab, FORMAT and samples
            total += 1u + (r.len - r.x0);
            if (recal) {
                uint32_t s1e = 0;
                const uint32_t sn = fio_sample(line + r.x0, r.len - r.x0, g, nullptr, &s1e);
                total = total - s1e + sn;
            }
        }
        out_len[i] = (int64_t)total + 1;  // newline
    }
    if (n_bl) atomicAdd(ed.n_blacklisted, n_bl);
}

__device__ __forceinline__ void fio_copy(uint8_t* dst, const uint8_t* src, uint32_t n, unsigned lane) {
    for (uint32_t k = lane; k < n; k += 32u) dst[k] = src[k];
}

__global__ void __launch_bounds__(256) splice_copy(const uint8_t* __restrict__ text, const int64_t* __restrict__ line_start,
                                                   const ugvc_recinfo* __restrict__ recinfo, const uint8_t* __restrict__ low_score,
                                                   int64_t n, const FioEdits ed, const int64_t* __restrict__ out_start,
                                                   const uint8_t* __restrict__ score_txt, uint8_t* __restrict__ out, int* fallback) {
    const unsigned FULL = 0xffffffffu;
    const unsigned lane = threadIdx.x & 31u;
    const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const bool recal = ed.phreds != nullptr;
    const bool owq = ed.with_model && (ed.flags & UGVC_FILE_OVERWRITE_QUAL);
    for (int64_t i = warp0; i < n; i += n_warps) {
        const FioRec r = fio_rec(line_start, recinfo, i);
        if (!r.ok) continue;
        const uint8_t* line = text + line_start[i];
        const uint8_t* st = score_txt + (size_t)i * 16;
        const uint32_t sl = st[15];
        uint8_t* o = out + out_start[i];
        fio_copy(o, line, r.q0, lane);
        o += r.q0;
        if (owq) {
            fio_copy(o, st, sl, lane);
            o += sl;
        } else {
            fio_copy(o, line + r.q0, r.f0 - 1u - r.q0, lane);
            o += r.f0 - 1u - r.q0;
        }
        // FILTER: short, written by one lane with the same routine that measured it
        uint32_t fn = 0;
        if (lane == 0) {
            o[0] = '\t';
            fn = fio_filter(line + r.f0, r.i0 - 1u - r.f0, ed.with_model && low_score[i] != 0, o + 1);
            o[1 + fn] = '\t';
        }
        fn = __shfl_sync(FULL, fn, 0);
        o += fn + 2u;
        // INFO: copied as it is when it is "plain" (hostio.cpp: no empty piece, not ".", neither key already there).
        // Under out_end each lane also notes the first piece it sees that starts with "END=" (ugvc_info_end: the first
        // such piece of the column decides)
        const uint8_t* ip = line + r.i0;
        const uint32_t il = r.x0 - 1u - r.i0;
        bool odd = il == 0 || (il == 1 && ip[0] == '.') || ip[0] == ';' || ip[il - 1] == ';';
        uint32_t endk = 0xFFFFFFFFu;
        for (uint32_t k = lane; k < il; k += 32u) {
            const uint8_t c = ip[k];
            o[k] = c;
            if (c == ';' && k + 1 < il && ip[k + 1] == ';') odd = true;
            if (c == 'T' && k + 11 <= il) {
                const char* key = "TREE_SCORE=";
                bool eq = true;
                for (int z = 1; z < 11 && eq; ++z) eq = ip[k + z] == (uint8_t)key[z];
                odd |= eq;
            }
            if (c == 'B' && k + 9 <= il) {
                const char* key = "BLACKLST=";
                bool eq = true;
                for (int z = 1; z < 9 && eq; ++z) eq = ip[k + z] == (uint8_t)key[z];
                odd |= eq;
            }
            if (c == 'E' && endk == 0xFFFFFFFFu && k + 4 <= il && (k == 0 || ip[k - 1] == ';') && ip[k + 1] == 'N' &&
                ip[k + 2] == 'D' && ip[k + 3] == '=')
                endk = k;
        }
        if (__any_sync(FULL, odd)) {
            if (lane == 0) atomicExch(fallback, 1);
        }
        if (ed.out_end) {
            endk = __reduce_min_sync(FULL, endk);
            if (lane == 0) {
                // ugvc_info_end: a piece "END=" + 1..10 digits gives the value, any other END= piece gives none
                int64_t v = 0;
                if (endk != 0xFFFFFFFFu) {
                    uint32_t q = endk + 4u;
                    while (q < il && ip[q] != ';') ++q;
                    const uint32_t pl = q - endk;
                    bool digits = pl > 4u && pl <= 14u;
                    for (uint32_t d = endk + 4u; d < q && digits; ++d) {
                        digits = ip[d] >= '0' && ip[d] <= '9';
                        v = v * 10 + (ip[d] - '0');
                    }
                    if (!digits) v = 0;
                }
                ed.out_end[i] = v;
            }
        }
        o += il;
        if (ed.with_model && !recal) {
            if (lane < FIO_SCORE_KEY_LEN) o[lane] = (uint8_t)FIO_SCORE_KEY[lane];
            o += FIO_SCORE_KEY_LEN;
            fio_copy(o, st, sl, lane);
            o += sl;
        }
        const uint32_t mask = ed.bl_mask[i];
        if (mask) {
            uint32_t bn = 0;
            if (lane == 0) bn = fio_blacklst(mask, ed.n_bl, ed.bl_name, ed.bl_name_off, o);
            o += __shfl_sync(FULL, bn, 0);
        }
        if (r.x0 <= r.len) {
            if (lane == 0) o[0] = '\t';
            ++o;
            uint32_t from = 0;  // FORMAT and the samples from here on are copied as they are
            if (recal) {
                uint32_t sn = 0, s1e = 0;
                if (lane == 0) {
                    FioGeno g;
                    fio_geno(ed.phreds + (size_t)i * ed.n_classes, ed.n_classes, recinfo[i].flags, g);  // true: splice_len
                    sn = fio_sample(line + r.x0, r.len - r.x0, g, o, &s1e);
                }
                o += __shfl_sync(FULL, sn, 0);
                from = __shfl_sync(FULL, s1e, 0);
            }
            fio_copy(o, line + r.x0 + from, r.len - r.x0 - from, lane);
            o += r.len - r.x0 - from;
        }
        if (lane == 0) o[0] = '\n';
    }
}

// ---- deflate: one thread per block of DEF_CHUNK output-text bytes
#define FIO_DEF_TPB 32
__global__ void __launch_bounds__(FIO_DEF_TPB) fio_deflate(const uint8_t* __restrict__ text, size_t n_bytes,
                                                           const DefTables* __restrict__ T, uint8_t* __restrict__ blocks,
                                                           uint32_t* __restrict__ bsize, int n_blocks) {
    extern __shared__ __align__(16) uint16_t fio_heads[];  // [FIO_DEF_TPB][1 << DEF_HASH_BITS]
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n_blocks) return;
    const size_t off = (size_t)b * DEF_CHUNK;
    const uint32_t n = (uint32_t)(n_bytes - off < DEF_CHUNK ? n_bytes - off : DEF_CHUNK);
    bsize[b] = def_block(text + off, n, blocks + (size_t)b * DEF_BLOCK_STRIDE, fio_heads + ((size_t)threadIdx.x << DEF_HASH_BITS), *T);
}

// ---- deflate, one warp per block (the default).  A thread per block is bound by its own dependent chain (about
// 2000 clocks a token: 0.7 s for a 5 M-record file); here the 32 lanes take 32 consecutive positions at a time:
//   every lane hashes its four bytes and reads the candidate BEFORE any lane of the window inserts (so a match
//   starts at least one window back; of lanes with equal hashes the lowest inserts), verifies and extends it on its own;
//   the token starts are then picked greedily from the left with one shuffle per token (uniform loop);
//   the token bits (def_token, <= 31 each) go to their bit offsets (warp scan) in a 32-word ring in shared memory
//   with atomicOr, and the words that became complete are stored to the block coalesced;
//   the CRC32 is computed as 32 slices combined pairwise (crc(A||B) = crc(A) x^(8|B|) + crc(B)).
// hostio.cpp: ugvc_test_deflate_block_lanes is the same algorithm with the lanes as a loop (CPU tests).
#define FIO_DEFW_WARPS 16
#define FIO_DEFW_SMEM (FIO_DEFW_WARPS * ((2u << DEF_HASH_BITS) + 128u))
__global__ void __launch_bounds__(FIO_DEFW_WARPS * 32) fio_deflate_warp(const uint8_t* __restrict__ text, size_t n_bytes,
                                                                        const DefTables* __restrict__ Tp,
                                                                        uint8_t* __restrict__ blocks,
                                                                        uint32_t* __restrict__ bsize, int n_blocks) {
    extern __shared__ __align__(16) uint32_t fio_sm[];
    const unsigned FULL = 0xffffffffu;
    const int wib = threadIdx.x >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    const int b = blockIdx.x * FIO_DEFW_WARPS + wib;
    if (b >= n_blocks) return;  // warps are independent: no CTA-wide barrier below
    uint16_t* head = reinterpret_cast<uint16_t*>(fio_sm) + ((size_t)wib << DEF_HASH_BITS);
    uint32_t* ring = fio_sm + ((FIO_DEFW_WARPS << DEF_HASH_BITS) >> 1) + wib * 32;
    const DefTables& T = *Tp;
    const size_t off0 = (size_t)b * DEF_CHUNK;
    const uint32_t n = (uint32_t)(n_bytes - off0 < DEF_CHUNK ? n_bytes - off0 : DEF_CHUNK);
    const uint8_t* in = text + off0;
    uint8_t* out = blocks + (size_t)b * DEF_BLOCK_STRIDE;
    uint32_t* outw = reinterpret_cast<uint32_t*>(out + 16);  // the bit stream starts with the two BSIZE bytes
    if (lane == 0) {  // 1f 8b 08 04 | mtime 0 | xfl 0, os ff | xlen 6 | 'B' 'C' 2 0
        reinterpret_cast<uint64_t*>(out)[0] = 0x0000000004088b1full;
        reinterpret_cast<uint64_t*>(out)[1] = 0x000243420006ff00ull;
    }
    // ---- CRC32: a slice per lane, then five pairwise combines
    uint32_t crc;
    {
        const uint32_t L = (((n + 31u) >> 5) + 3u) & ~3u;
        const uint32_t s0 = lane * L;
        uint32_t cov = s0 < n ? (n - s0 < L ? n - s0 : L) : 0u;
        crc = def_crc_slice(T, in + (cov ? s0 : 0u), cov);
#pragma unroll 1
        for (uint32_t s = 1; s < 32; s <<= 1) {
            const uint32_t pc = __shfl_down_sync(FULL, crc, s), pl = __shfl_down_sync(FULL, cov, s);
            if ((lane & (2u * s - 1u)) == 0u) {
                if (pl) crc = def_crc_combine(T, crc, pc, pl);
                cov += pl;
            }
        }
    }
    // ---- LZ77 + fixed Huffman codes
    for (uint32_t i = lane; i < ((1u << DEF_HASH_BITS) >> 1); i += 32) reinterpret_cast<uint32_t*>(head)[i] = 0xFFFFFFFFu;
    ring[lane] = lane == 0 ? (3u << 16) : 0u;  // BFINAL = 1, BTYPE = 01 after the 16 BSIZE bits
    __syncwarp();
    uint32_t bp = 19, flushed = 0, carry = 0;
#pragma unroll 1
    for (uint32_t p0 = 0; p0 < n; p0 += 32) {
        const uint32_t pos = p0 + lane;
        const bool can = pos + DEF_MIN_MATCH <= n;
        const uint32_t w = can ? def_ld4(in + pos) : 0u;
        const uint32_t h = DEFW_HASH(w);
        const uint32_t cand = can ? head[h] : 0xFFFFu;
        __syncwarp();
        if (can) head[h] = (uint16_t)pos;
        __syncwarp();
        // lanes with equal hashes stored to one address, and CUDA does not say which of those stores lands: the lowest
        // position is made to win (the lanes still above it store again until none is).  On the H100 it already has
        // after the first store, so the loop only costs the check (the output is byte-identical to the unchecked store)
        bool above = can && head[h] > pos;
        while (__any_sync(FULL, above)) {
            __syncwarp();
            if (above) head[h] = (uint16_t)pos;
            __syncwarp();
            above = above && head[h] > pos;
        }
        if (carry >= 32) {  // the whole window lies inside the last match
            carry -= 32;
            continue;
        }
        uint32_t len = 0, dist = 0;
        if (cand != 0xFFFFu && pos - cand <= 32768u && def_ld4(in + cand) == w) {
            const uint32_t maxlen = n - pos < DEF_MAX_MATCH ? n - pos : DEF_MAX_MATCH;
            len = def_extend(in, cand, pos, maxlen);
            dist = pos - cand;
        }
        // token starts: follow "next" from the first position the last window left uncovered
        const uint32_t nxt = lane + (len ? len : 1u);
        const uint32_t lim = n - p0 < 32u ? n - p0 : 32u;
        uint32_t mask = 0, cur = carry;
        while (cur < lim) {
            mask |= 1u << cur;
            cur = __shfl_sync(FULL, nxt, (int)cur);
        }
        carry = cur >= 32u ? cur - 32u : 0u;
        uint32_t nb = 0, bits = 0;
        if ((mask >> lane) & 1u) bits = def_token(T, can ? (w & 0xFFu) : (uint32_t)in[pos], len, dist, nb);
        uint32_t incl = nb;
#pragma unroll
        for (int s = 1; s < 32; s <<= 1) {
            const uint32_t t = __shfl_up_sync(FULL, incl, s);
            if ((int)lane >= s) incl += t;
        }
        const uint32_t total = __shfl_sync(FULL, incl, 31);
        if (nb) {
            const uint32_t o = bp + incl - nb, wi = o >> 5, sh = o & 31u;
            atomicOr(&ring[wi & 31u], bits << sh);
            if (sh + nb > 32u) atomicOr(&ring[(wi + 1u) & 31u], bits >> (32u - sh));
        }
        bp += total;
        __syncwarp();
        const uint32_t full = bp >> 5;
        if (lane < full - flushed) {  // at most ten words a window
            const uint32_t wi = flushed + lane;
            outw[wi] = ring[wi & 31u];
            ring[wi & 31u] = 0u;
        }
        flushed = full;
        __syncwarp();
    }
    bp += 7;  // end of block: seven zero bits
    {
        const uint32_t endw = (bp + 31u) >> 5;
        if (flushed + lane < endw) outw[flushed + lane] = ring[(flushed + lane) & 31u];
    }
    __syncwarp();
    uint32_t payload = ((bp + 7u) >> 3) - 2u;
    if (payload >= n + 5u) {  // did not shrink: one stored block
        if (lane == 0) {
            uint8_t* p = out + 18;
            p[0] = 1;
            p[1] = (uint8_t)n;
            p[2] = (uint8_t)(n >> 8);
            p[3] = (uint8_t)~n;
            p[4] = (uint8_t)(~n >> 8);
        }
        for (uint32_t k = lane; k < n; k += 32) out[23 + k] = in[k];
        payload = n + 5u;
    }
    __syncwarp();
    if (lane == 0) {
        uint8_t* ft = out + 18 + payload;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            ft[k] = (uint8_t)(crc >> (8 * k));
            ft[4 + k] = (uint8_t)(n >> (8 * k));
        }
        const uint32_t bs = 18u + payload + 8u;
        out[16] = (uint8_t)(bs - 1u);
        out[17] = (uint8_t)((bs - 1u) >> 8);
        bsize[b] = bs;
    }
}

__global__ void __launch_bounds__(256) fio_pack(const uint8_t* __restrict__ blocks, const uint32_t* __restrict__ bsize,
                                                const uint64_t* __restrict__ boff, int n_blocks, uint8_t* __restrict__ packed) {
    for (int b = blockIdx.x; b < n_blocks; b += gridDim.x) {
        const uint8_t* src = blocks + (size_t)b * DEF_BLOCK_STRIDE;
        uint8_t* dst = packed + boff[b];
        const uint32_t n = bsize[b];
        // blocks start 64 KiB apart (16-byte aligned); the packed position is arbitrary: words where both agree
        for (uint32_t k = threadIdx.x; k < n; k += blockDim.x) dst[k] = src[k];
    }
}

// first record starting at or after each text offset (lower bound on line_start[0, n])
__global__ void fio_first_records(const int64_t* __restrict__ line_start, int64_t n, const uint64_t* __restrict__ offsets, int m,
                                  int64_t* __restrict__ out) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= m) return;
    const int64_t want = (int64_t)offsets[k];
    int64_t lo = 0, hi = n;  // answer in [0, n]
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (line_start[mid] < want) lo = mid + 1;
        else hi = mid;
    }
    out[k] = lo;
}
void fio_launch_first_records(const int64_t* line_start, int64_t n, const uint64_t* offsets, int m, int64_t* out, cudaStream_t st) {
    if (m <= 0) return;
    fio_first_records<<<(m + 63) / 64, 64, 0, st>>>(line_start, n, offsets, m, out);
}

__global__ void fio_widen(const uint32_t* __restrict__ bsize, uint64_t* __restrict__ wide, int n) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) wide[i] = bsize[i];
}

// ---- launchers (capi.cu owns the buffers)
cudaError_t fio_scan_i64(void* tmp, size_t& tmp_bytes, const int64_t* in, int64_t* out, int64_t n, cudaStream_t st) {
    return cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, in, out, (int)n, st);
}
cudaError_t fio_scan_u64(void* tmp, size_t& tmp_bytes, const uint64_t* in, uint64_t* out, int n, cudaStream_t st) {
    return cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, in, out, n, st);
}
void fio_launch_splice_len(const uint8_t* text, const int64_t* line_start, const ugvc_recinfo* recinfo, const uint8_t* low,
                           const double* qual, int64_t n, const FioEdits& ed, int64_t* out_len, uint8_t* score_txt,
                           int* fallback, int sm_count, cudaStream_t st) {
    if (n <= 0) return;
    int64_t blocks = (n + 255) / 256;
    if (blocks > (int64_t)sm_count * 16) blocks = (int64_t)sm_count * 16;
    splice_len<<<(unsigned)blocks, 256, 0, st>>>(text, line_start, recinfo, low, qual, n, ed, out_len, score_txt, fallback);
}
void fio_launch_splice_copy(const uint8_t* text, const int64_t* line_start, const ugvc_recinfo* recinfo, const uint8_t* low,
                            int64_t n, const FioEdits& ed, const int64_t* out_start, const uint8_t* score_txt, uint8_t* out,
                            int* fallback, int sm_count, cudaStream_t st) {
    if (n <= 0) return;
    int64_t blocks = (n + 7) / 8;
    if (blocks > (int64_t)sm_count * 32) blocks = (int64_t)sm_count * 32;
    splice_copy<<<(unsigned)blocks, 256, 0, st>>>(text, line_start, recinfo, low, n, ed, out_start, score_txt, out, fallback);
}
cudaError_t fio_launch_deflate(const uint8_t* text, size_t n_bytes, const DefTables* tables, uint8_t* blocks, uint32_t* bsize,
                               int n_blocks, int encoder, cudaStream_t st) {
    if (n_blocks <= 0) return cudaSuccess;
    cudaError_t e;
    // the attribute is set per call: it belongs to the current device, and lanes are driven from several host threads
    if (encoder == FIO_ENC_WARP) {
        if ((e = cudaFuncSetAttribute(fio_deflate_warp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FIO_DEFW_SMEM)) != cudaSuccess)
            return e;
        fio_deflate_warp<<<(n_blocks + FIO_DEFW_WARPS - 1) / FIO_DEFW_WARPS, FIO_DEFW_WARPS * 32, FIO_DEFW_SMEM, st>>>(
            text, n_bytes, tables, blocks, bsize, n_blocks);
        return cudaGetLastError();
    }
    const size_t smem = (size_t)FIO_DEF_TPB * sizeof(uint16_t) << DEF_HASH_BITS;
    if ((e = cudaFuncSetAttribute(fio_deflate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess) return e;
    fio_deflate<<<(n_blocks + FIO_DEF_TPB - 1) / FIO_DEF_TPB, FIO_DEF_TPB, smem, st>>>(text, n_bytes, tables, blocks, bsize, n_blocks);
    return cudaGetLastError();
}
void fio_launch_pack(const uint8_t* blocks, const uint32_t* bsize, uint64_t* wide, const uint64_t* boff, int n_blocks,
                     uint8_t* packed, int sm_count, cudaStream_t st) {
    if (n_blocks <= 0) return;
    (void)wide;
    fio_pack<<<n_blocks < sm_count * 8 ? n_blocks : sm_count * 8, 256, 0, st>>>(blocks, bsize, boff, n_blocks, packed);
}
void fio_launch_widen(const uint32_t* bsize, uint64_t* wide, int n, cudaStream_t st) {
    if (n <= 0) return;
    fio_widen<<<(n + 255) / 256, 256, 0, st>>>(bsize, wide, n);
}

// test hook (ugvc_test_format_g): fio_format_g of every value into the 16-byte slot layout of splice_len (text in
// bytes 0..14, zero padded; length in byte 15, 0 = left to the host writer)
__global__ void __launch_bounds__(256) fio_test_format_g(const float* __restrict__ v, int64_t n, uint8_t* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        char num[16];
        const int sl = fio_format_g(v[i], num);
        uint8_t* st = out + (size_t)i * 16;
        for (int c = 0; c < 15; ++c) st[c] = c < sl ? (uint8_t)num[c] : 0;
        st[15] = (uint8_t)sl;
    }
}
void fio_launch_test_format_g(const float* v, int64_t n, uint8_t* out, int sm_count, cudaStream_t st) {
    if (n <= 0) return;
    int64_t blocks = (n + 255) / 256;
    if (blocks > (int64_t)sm_count * 16) blocks = (int64_t)sm_count * 16;
    fio_test_format_g<<<(unsigned)blocks, 256, 0, st>>>(v, n, out);
}
