// conc_annotate.cu -- annotation of a concordance frame on the GPU (SURVEY.md section 8 row f3, DESIGN.md 4b).
//
// Replaces the per-record passes of comparison_utils.annotate_concordance (ugbio_comparison/comparison_utils.py:
// 321-380), which runs, in this order, over every row of the frame:
//   classify_indel      variant_annotation.py:259-286   indel_classify (None / ins / del), indel_length
//   is_hmer_indel       :289-334 + dna_sequence_utils.hmer_length :43-62   hmer_indel_length, hmer_indel_nuc
//   get_motif_around    :404-458 (size 5)                left_motif, right_motif
//   get_gc_content      :461-490 (window 10)             gc_content
//   annotate_cycle_skip :616-744 + flow_based_read.generate_key_from_sequence :55-112 (gt_field=None)
//                                                        cycleskip_status
// ca_annotate is one thread per record (grid-stride, so the host emulation runs it with one thread): every row reads
// a few bytes of its alleles and a window of at most ~2 x motif + hmer run bytes of the contig, then walks the two
// flow keys of a SNP in lockstep without storing them.  Contig bytes keep the FASTA's case; every read goes through
// Python str slice rules (ca_slice), which is what the reference's sequence objects follow.
//
// Where the reference raises, the row is recorded instead: the 64-bit key (stage << 48 | row << 4 | reason) of the
// lowest (stage, row) wins an atomicMin, stage being the pass of the list above that raises first.  Stage 0
// (ValueError for a row without alleles) is checked by the host before the launch.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "concordance.cuh"

#define CA_TPB 256
#define CA_NO_ERROR 0xFFFFFFFFFFFFFFFFull

enum : int8_t { CA_CLS_NONE = 0, CA_CLS_INS = 1, CA_CLS_DEL = 2 };
enum : int8_t { CA_CS_NA = 0, CA_CS_SKIP = 1, CA_CS_POSSIBLE = 2, CA_CS_NON_SKIP = 3 };
enum : int { CA_STAGE_HMER = 1, CA_STAGE_MOTIF = 2, CA_STAGE_GC = 3 };

#ifdef UGVC_HOST_EMU
#define CA_LAUNCH(kern, grid, block, st, ...)                   \
    do {                                                        \
        threadIdx = dim3(0, 0, 0); blockIdx = dim3(0, 0, 0);     \
        blockDim = dim3(1, 1, 1); gridDim = dim3(1, 1, 1);       \
        kern(__VA_ARGS__);                                      \
    } while (0)
#else
#define CA_LAUNCH(kern, grid, block, st, ...) kern<<<grid, block, 0, st>>>(__VA_ARGS__)
#endif

struct CaContig {
    const uint8_t* seq;  // NULL: the contig is not in the FASTA
    int64_t len;
};

__device__ __forceinline__ uint8_t ca_upper(uint8_t c) { return (c >= 'a' && c <= 'z') ? (uint8_t)(c - 32) : c; }

// s[a:b] of a str of length n: a negative bound counts from the end, bounds clip to [0, n], start >= stop is empty
__device__ __forceinline__ void ca_slice(int64_t n, int64_t a, int64_t b, int64_t* s, int64_t* e) {
    if (a < 0) {
        a += n;
        if (a < 0) a = 0;
    } else if (a > n) {
        a = n;
    }
    if (b < 0) {
        b += n;
        if (b < 0) b = 0;
    } else if (b > n) {
        b = n;
    }
    *s = a;
    *e = b > a ? b : a;
}

// s[i:i+1].upper() as a byte, -1 for the empty string (past the end)
__device__ __forceinline__ int ca_base(const CaContig& c, int64_t i) {
    int64_t s, e;
    ca_slice(c.len, i, i + 1, &s, &e);
    return e > s ? (int)ca_upper(c.seq[s]) : -1;
}

// dna_sequence_utils.hmer_length: run of upper-case-equal bases from `start` (whose base is not empty), ending at the
// contig end
__device__ __forceinline__ int64_t ca_hmer_run(const CaContig& c, int64_t start) {
    const int b0 = ca_base(c, start);
    int64_t i = start + 1;
    while (ca_base(c, i) == b0) ++i;
    return i - start;
}

// chrom[a:b].upper() into `size` bytes, zero-padded
__device__ __forceinline__ void ca_motif(const CaContig& c, int64_t a, int64_t b, int size, uint8_t* out,
                                         uint8_t* out_len) {
    int64_t s, e;
    ca_slice(c.len, a, b, &s, &e);
    *out_len = (uint8_t)(e - s);
    for (int64_t k = s; k < e; ++k) out[k - s] = ca_upper(c.seq[k]);
    for (int64_t k = e - s; k < size; ++k) out[k] = 0;
}

// one sequence left + mid + right of the cycle-skip test, bases upper-cased
struct CaSeq {
    const uint8_t *l, *m, *r;
    int64_t nl, nm, nr;
    __device__ __forceinline__ int64_t size() const { return nl + nm + nr; }
    __device__ __forceinline__ uint8_t at(int64_t i) const {
        if (i < nl) return l[i];
        i -= nl;
        if (i < nm) return ca_upper(m[i]);
        return r[i - nm];
    }
    __device__ __forceinline__ bool acgt() const {
        for (int64_t i = 0, n = size(); i < n; ++i) {
            const uint8_t c = at(i);
            if (c != 'A' && c != 'C' && c != 'G' && c != 'T') return false;
        }
        return true;
    }
};

// generate_key_from_sequence, one flow at a time: the run of the flow's base from the current position; the key ends
// after the flow whose run reaches the end of the sequence, or after len(flow_order) * len(seq) flows
struct CaKeyWalk {
    int64_t pos = 0, flow = 0, max_flows = 0;
    bool done = false;
    __device__ __forceinline__ bool next(const CaSeq& s, const uint8_t* fo, int fo_len, int64_t* h) {
        if (done || flow >= max_flows) {
            done = true;
            return false;
        }
        const uint8_t b = fo[flow % fo_len];
        const int64_t n = s.size();
        int64_t k = pos;
        while (k < n && s.at(k) == b) ++k;
        *h = k - pos;
        pos = k;
        ++flow;
        if (k == n) done = true;
        return true;
    }
};

__device__ __forceinline__ int8_t ca_cycle_skip(const CaSeq& ref, const CaSeq& alt, const uint8_t* fo, int fo_len) {
    if (!ref.acgt() || !alt.acgt()) return CA_CS_NA;
    CaKeyWalk wr, wa;
    wr.max_flows = (int64_t)fo_len * ref.size();
    wa.max_flows = (int64_t)fo_len * alt.size();
    bool possible = false;
    for (;;) {
        int64_t hr = 0, ha = 0;
        const bool vr = wr.next(ref, fo, fo_len, &hr), va = wa.next(alt, fo, fo_len, &ha);
        if (vr != va) return CA_CS_SKIP;  // keys of different lengths
        if (!vr) break;
        if (hr != ha && (hr == 0 || ha == 0)) possible = true;
    }
    return possible ? CA_CS_POSSIBLE : CA_CS_NON_SKIP;
}

__device__ __forceinline__ void ca_error(unsigned long long* err, int stage, int64_t row, int reason) {
    atomicMin(err, ((unsigned long long)stage << 48) | ((unsigned long long)row << 4) | (unsigned long long)reason);
}

__device__ __forceinline__ bool ca_equal(const uint8_t* a, int64_t na, const uint8_t* b, int64_t nb) {
    if (na != nb) return false;
    for (int64_t k = 0; k < na; ++k)
        if (a[k] != b[k]) return false;
    return true;
}

// a non-empty run of one byte (len(set(s)) == 1)
__device__ __forceinline__ bool ca_one_letter(const uint8_t* s, int64_t n) {
    if (n <= 0) return false;
    for (int64_t k = 1; k < n; ++k)
        if (s[k] != s[0]) return false;
    return true;
}

__global__ void __launch_bounds__(CA_TPB) ca_annotate(
    int64_t n, const CaContig* __restrict__ contigs, const int32_t* __restrict__ contig, const int64_t* __restrict__ pos,
    const uint8_t* __restrict__ indel, const uint8_t* __restrict__ ref, const int64_t* __restrict__ ref_off,
    const uint8_t* __restrict__ al, const int64_t* __restrict__ al_off, const int64_t* __restrict__ rec_al,
    const uint8_t* __restrict__ flow_order, int fo_len, int motif, int gc_window, int8_t* __restrict__ out_class,
    int32_t* __restrict__ out_indel_len, int32_t* __restrict__ out_hmer_len, uint8_t* __restrict__ out_hmer_nuc,
    uint8_t* __restrict__ out_left, uint8_t* __restrict__ out_right, uint8_t* __restrict__ out_left_len,
    uint8_t* __restrict__ out_right_len, double* __restrict__ out_gc, int8_t* __restrict__ out_cs,
    unsigned long long* __restrict__ err) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int cid = contig[i];
        const CaContig c = cid >= 0 ? contigs[cid] : CaContig{nullptr, 0};
        const bool missing = c.seq == nullptr;
        const int64_t p = pos[i];
        const bool is_indel = indel[i] != 0;
        const uint8_t* r = ref + ref_off[i];
        const int64_t nr = ref_off[i + 1] - ref_off[i];
        const int64_t a0 = rec_al[i], a1 = rec_al[i + 1];

        // classify_indel
        int64_t max_len = 0, indel_len = 0;
        for (int64_t a = a0; a < a1; ++a) {
            const int64_t na = al_off[a + 1] - al_off[a];
            max_len = na > max_len ? na : max_len;
            const int64_t d = na > nr ? na - nr : nr - na;
            indel_len = d > indel_len ? d : indel_len;
        }
        const int8_t cls = !is_indel ? CA_CLS_NONE : (nr < max_len ? CA_CLS_INS : CA_CLS_DEL);
        out_class[i] = cls;
        out_indel_len[i] = (int32_t)indel_len;

        // is_hmer_indel
        int64_t hmer = 0;
        uint8_t nuc = 0;
        if (cls == CA_CLS_INS) {
            int64_t first = -1;
            for (int64_t a = a0; a < a1 && first < 0; ++a)
                if (!ca_equal(al + al_off[a], al_off[a + 1] - al_off[a], r, nr)) first = a;
            if (first < 0) {
                ca_error(err, CA_STAGE_HMER, i, UGVC_ANNOT_E_INDEX);
            } else {
                const uint8_t* s = al + al_off[first] + 1;
                const int64_t ns = al_off[first + 1] - al_off[first] - 1;
                if (ca_one_letter(s, ns)) {
                    if (missing) {
                        ca_error(err, CA_STAGE_HMER, i, UGVC_ANNOT_E_KEY);
                    } else if (ca_base(c, p) == (int)s[0]) {
                        hmer = ca_hmer_run(c, p);
                        nuc = s[0];
                    }
                }
            }
        } else if (cls == CA_CLS_DEL && ca_one_letter(r + 1, nr - 1)) {
            if (missing) {
                ca_error(err, CA_STAGE_HMER, i, UGVC_ANNOT_E_KEY);
            } else if (ca_base(c, p + nr - 1) == (int)r[1]) {
                hmer = (nr - 1) + ca_hmer_run(c, p + nr - 1);
                nuc = r[1];
            }
        }
        out_hmer_len[i] = (int32_t)hmer;
        out_hmer_nuc[i] = nuc;

        // get_motif_around
        uint8_t* left = out_left + i * motif;
        uint8_t* right = out_right + i * motif;
        out_left_len[i] = out_right_len[i] = 0;
        if (missing) {
            ca_error(err, CA_STAGE_MOTIF, i, UGVC_ANNOT_E_KEY);
            for (int k = 0; k < motif; ++k) left[k] = right[k] = 0;
            continue;
        }
        if (is_indel && hmer > 0) {
            ca_motif(c, p - motif, p, motif, left, out_left_len + i);
            ca_motif(c, p + hmer, p + hmer + motif, motif, right, out_right_len + i);
        } else if (is_indel) {
            ca_motif(c, p - motif, p, motif, left, out_left_len + i);
            ca_motif(c, p + nr - 1, p + nr - 1 + motif, motif, right, out_right_len + i);
        } else {
            ca_motif(c, p - motif - 1, p - 1, motif, left, out_left_len + i);
            ca_motif(c, p, p + motif, motif, right, out_right_len + i);
        }

        // get_gc_content: everything but A and T counts
        {
            const int64_t beg = p - gc_window / 2;
            int64_t s, e;
            ca_slice(c.len, beg, beg + gc_window, &s, &e);
            if (e == s) {
                ca_error(err, CA_STAGE_GC, i, UGVC_ANNOT_E_ZERO_DIVISION);
                out_gc[i] = 0.0;
            } else {
                int64_t gc = 0;
                for (int64_t k = s; k < e; ++k) {
                    const uint8_t b = ca_upper(c.seq[k]);
                    gc += (b != 'A' && b != 'T');
                }
                out_gc[i] = __ddiv_rn((double)gc, (double)(e - s));
            }
        }

        // annotate_cycle_skip (gt_field=None): SNP-like rows of at most two alleles; alt = alleles[1]
        if (fo_len >= 0) {
            int8_t cs = CA_CS_NA;
            if (!is_indel && a1 - a0 == 2) {
                const CaSeq sr{left, r, right, out_left_len[i], nr, out_right_len[i]};
                const CaSeq sa{left, al + al_off[a0 + 1], right, out_left_len[i], al_off[a0 + 2] - al_off[a0 + 1],
                               out_right_len[i]};
                cs = ca_cycle_skip(sr, sa, flow_order, fo_len);
            }
            out_cs[i] = cs;
        }
    }
}

extern "C" int ugvc_conc_annot_add_contig(ugvc_conc* h, const uint8_t* seq, int64_t len, int32_t* out_id) {
    if (!h) return UGVC_E_ARG;
    if (len < 0 || (len > 0 && !seq) || !out_id) return conc_fail(h, UGVC_E_ARG, "conc_annot_add_contig: bad arguments");
    if (h->annot_seq.size() >= 0x7FFFFFFFu) return conc_fail(h, UGVC_E_ARG, "conc_annot_add_contig: too many contigs");
    CCU(cudaSetDevice(h->device));
    uint8_t* d = nullptr;
    CCU(cudaMalloc(&d, (size_t)(len ? len : 1)));
    h->annot_seq.push_back(d);
    h->annot_len.push_back(len);
    if (len) CCU(cudaMemcpy(d, seq, (size_t)len, cudaMemcpyHostToDevice));
    *out_id = (int32_t)(h->annot_seq.size() - 1);
    return UGVC_OK;
}

extern "C" int ugvc_conc_annot_clear(ugvc_conc* h) {
    if (!h) return UGVC_E_ARG;
    CCU(cudaSetDevice(h->device));
    conc_drop_contigs(h);
    return UGVC_OK;
}

extern "C" double ugvc_conc_annot_kernel_ms(const ugvc_conc* h) { return h ? (double)h->annot_kernel_ms : 0.0; }

extern "C" int ugvc_conc_annot_error(const ugvc_conc* h, int64_t* row, int* reason) {
    if (!h || !row || !reason) return UGVC_E_ARG;
    *row = h->annot_err_row;
    *reason = h->annot_err_reason;
    return UGVC_OK;
}

namespace {
struct CaBufs {  // frees on scope exit
    std::vector<void*> ptrs;
    ~CaBufs() {
        for (void* p : ptrs) cudaFree(p);
    }
    template <class T>
    cudaError_t get(T** p, size_t count) {
        cudaError_t e = cudaMalloc(reinterpret_cast<void**>(p), (count ? count : 1) * sizeof(T));
        if (e == cudaSuccess) ptrs.push_back(*p);
        return e;
    }
    template <class T>
    cudaError_t put(T** p, const T* src, size_t count, cudaStream_t st) {
        cudaError_t e = get(p, count);
        if (e == cudaSuccess && count) e = cudaMemcpyAsync(*p, src, count * sizeof(T), cudaMemcpyHostToDevice, st);
        return e;
    }
};
}  // namespace

extern "C" int ugvc_conc_annotate(ugvc_conc* h, int64_t n, const int32_t* contig, const int64_t* pos,
                                  const uint8_t* indel, const uint8_t* ref_bytes, const int64_t* ref_off,
                                  const uint8_t* allele_bytes, const int64_t* allele_off, const int64_t* rec_allele_off,
                                  const char* flow_order, int motif_size, int gc_window, int8_t* out_class,
                                  int32_t* out_indel_len, int32_t* out_hmer_len, uint8_t* out_hmer_nuc,
                                  uint8_t* out_left, uint8_t* out_right, uint8_t* out_left_len, uint8_t* out_right_len,
                                  double* out_gc, int8_t* out_cycleskip) {
    if (!h) return UGVC_E_ARG;
    h->annot_err_row = -1;
    h->annot_err_reason = 0;
    if (n < 0 || motif_size < 0 || motif_size > 255 || gc_window < 0)
        return conc_fail(h, UGVC_E_ARG, "conc_annotate: bad sizes");
    if (n == 0) return UGVC_OK;
    if (n >= (1ll << 44)) return conc_fail(h, UGVC_E_ARG, "conc_annotate: too many records");
    if (!contig || !pos || !indel || !ref_off || !allele_off || !rec_allele_off || !out_class || !out_indel_len ||
        !out_hmer_len || !out_hmer_nuc || !out_left || !out_right || !out_left_len || !out_right_len || !out_gc ||
        (flow_order && !out_cycleskip))
        return conc_fail(h, UGVC_E_ARG, "conc_annotate: NULL array");
    const int64_t n_al = rec_allele_off[n];
    const int64_t ref_bytes_n = ref_off[n], al_bytes_n = allele_off[n_al];
    if (rec_allele_off[0] != 0 || ref_off[0] != 0 || allele_off[0] != 0 || n_al < 0 || ref_bytes_n < 0 ||
        al_bytes_n < 0 || (ref_bytes_n && !ref_bytes) || (al_bytes_n && !allele_bytes))
        return conc_fail(h, UGVC_E_ARG, "conc_annotate: bad offsets");
    const int n_contigs = (int)h->annot_seq.size();
    for (int64_t i = 0; i < n; ++i) {
        if (contig[i] >= n_contigs) return conc_fail(h, UGVC_E_ARG, "conc_annotate: contig id out of range");
        if (rec_allele_off[i + 1] <= rec_allele_off[i] || ref_off[i + 1] < ref_off[i])
            return conc_fail(h, UGVC_E_ARG, "conc_annotate: every record needs alleles (offsets must increase)");
    }
    for (int64_t a = 0; a < n_al; ++a)
        if (allele_off[a + 1] < allele_off[a]) return conc_fail(h, UGVC_E_ARG, "conc_annotate: bad allele offsets");
    const int fo_len = flow_order ? (int)strlen(flow_order) : -1;
    CCU(cudaSetDevice(h->device));
    cudaStream_t st = h->st;
    CaBufs b;
    std::vector<CaContig> hc(n_contigs > 0 ? n_contigs : 1);
    for (int k = 0; k < n_contigs; ++k) hc[k] = CaContig{h->annot_seq[k], h->annot_len[k]};
    CaContig* d_contigs;
    int32_t* d_contig;
    int64_t *d_pos, *d_ref_off, *d_al_off, *d_rec_al;
    uint8_t *d_indel, *d_ref, *d_al, *d_fo;
    CCU(b.put(&d_contigs, hc.data(), hc.size(), st));
    CCU(b.put(&d_contig, contig, (size_t)n, st));
    CCU(b.put(&d_pos, pos, (size_t)n, st));
    CCU(b.put(&d_indel, indel, (size_t)n, st));
    CCU(b.put(&d_ref, ref_bytes, (size_t)ref_bytes_n, st));
    CCU(b.put(&d_ref_off, ref_off, (size_t)n + 1, st));
    CCU(b.put(&d_al, allele_bytes, (size_t)al_bytes_n, st));
    CCU(b.put(&d_al_off, allele_off, (size_t)n_al + 1, st));
    CCU(b.put(&d_rec_al, rec_allele_off, (size_t)n + 1, st));
    CCU(b.put(&d_fo, reinterpret_cast<const uint8_t*>(flow_order), (size_t)(fo_len > 0 ? fo_len : 0), st));
    int8_t *d_class, *d_cs;
    int32_t *d_indel_len, *d_hmer_len;
    uint8_t *d_nuc, *d_left, *d_right, *d_left_len, *d_right_len;
    double* d_gc;
    unsigned long long* d_err;
    CCU(b.get(&d_class, (size_t)n));
    CCU(b.get(&d_cs, fo_len >= 0 ? (size_t)n : 1));
    CCU(b.get(&d_indel_len, (size_t)n));
    CCU(b.get(&d_hmer_len, (size_t)n));
    CCU(b.get(&d_nuc, (size_t)n));
    CCU(b.get(&d_left, (size_t)n * motif_size));
    CCU(b.get(&d_right, (size_t)n * motif_size));
    CCU(b.get(&d_left_len, (size_t)n));
    CCU(b.get(&d_right_len, (size_t)n));
    CCU(b.get(&d_gc, (size_t)n));
    CCU(b.get(&d_err, 1));
    CCU(cudaMemsetAsync(d_err, 0xFF, sizeof(unsigned long long), st));
    int64_t blocks = (n + CA_TPB - 1) / CA_TPB;
    if (blocks > (int64_t)h->sm_count * 32) blocks = (int64_t)h->sm_count * 32;
    cudaEvent_t ev[2] = {nullptr, nullptr};
    CCU(cudaEventCreate(&ev[0]));
    if (cudaEventCreate(&ev[1]) != cudaSuccess) {
        cudaEventDestroy(ev[0]);
        return conc_fail(h, UGVC_E_CUDA, "conc_annotate: cudaEventCreate failed");
    }
    cudaEventRecord(ev[0], st);
    CA_LAUNCH(ca_annotate, (unsigned)blocks, CA_TPB, st, n, d_contigs, d_contig, d_pos, d_indel, d_ref, d_ref_off, d_al,
              d_al_off, d_rec_al, d_fo, fo_len, motif_size, gc_window, d_class, d_indel_len, d_hmer_len, d_nuc, d_left,
              d_right, d_left_len, d_right_len, d_gc, d_cs, d_err);
    cudaEventRecord(ev[1], st);
    ++h->launches;
    const cudaError_t launch_err = cudaGetLastError();
    if (launch_err == cudaSuccess && cudaEventSynchronize(ev[1]) == cudaSuccess)
        cudaEventElapsedTime(&h->annot_kernel_ms, ev[0], ev[1]);
    cudaEventDestroy(ev[0]);
    cudaEventDestroy(ev[1]);
    CCU(launch_err);
    unsigned long long h_err = CA_NO_ERROR;
    CCU(cudaMemcpyAsync(&h_err, d_err, sizeof(h_err), cudaMemcpyDeviceToHost, st));
    CCU(cudaMemcpyAsync(out_class, d_class, (size_t)n, cudaMemcpyDeviceToHost, st));
    CCU(cudaMemcpyAsync(out_indel_len, d_indel_len, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    CCU(cudaMemcpyAsync(out_hmer_len, d_hmer_len, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    CCU(cudaMemcpyAsync(out_hmer_nuc, d_nuc, (size_t)n, cudaMemcpyDeviceToHost, st));
    CCU(cudaMemcpyAsync(out_left, d_left, (size_t)n * motif_size, cudaMemcpyDeviceToHost, st));
    CCU(cudaMemcpyAsync(out_right, d_right, (size_t)n * motif_size, cudaMemcpyDeviceToHost, st));
    CCU(cudaMemcpyAsync(out_left_len, d_left_len, (size_t)n, cudaMemcpyDeviceToHost, st));
    CCU(cudaMemcpyAsync(out_right_len, d_right_len, (size_t)n, cudaMemcpyDeviceToHost, st));
    CCU(cudaMemcpyAsync(out_gc, d_gc, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
    if (fo_len >= 0) CCU(cudaMemcpyAsync(out_cycleskip, d_cs, (size_t)n, cudaMemcpyDeviceToHost, st));
    CCU(cudaStreamSynchronize(st));
    if (h_err != CA_NO_ERROR) {
        h->annot_err_row = (int64_t)((h_err >> 4) & ((1ull << 44) - 1));
        h->annot_err_reason = (int)(h_err & 0xF);
        return conc_fail(h, UGVC_E_DATA, "conc_annotate: the reference raises at record " +
                                             std::to_string(h->annot_err_row) + " (reason " +
                                             std::to_string(h->annot_err_reason) + ")");
    }
    return UGVC_OK;
}
