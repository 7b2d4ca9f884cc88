// kernels.cu -- the hot path of filter_variants_pipeline as sm_90a (H100) CUDA kernels.
//
//   K0  line index      : one pass over the VCF text (decoupled look-back) -> line_start[], n_records
//   K1  field parse     : one thread per record walks the 8 fixed columns, the INFO key=value
//                         list and the FORMAT/sample pair and decodes the tags the plan needs
//                         with htslib's typing rules (int32 / float32 / dictionary-encoded
//                         strings) straight into the columnar batch raw[slot][record]; keys are
//                         visited in the learned order so the lanes of a warp decode the same
//                         type together, keys off that order take a generic hash-lookup path
//                         (replaces vcftools.py:63-89 + :196-214 of the reference)
//   K2  feature assembly: raw slots -> fp32 feature matrix feats[feature][record] with the
//                         fitted transformer's missing/absent policies (transformers.py:221-344)
//   K3  inference       : feature tile + forest staged in shared memory, tree-ensemble /
//                         logistic evaluation in the training library's own arithmetic order,
//                         fp64 phred/qual math and the FILTER decision fused in
//                         (variant_filtering_utils.py:123-124, filter_variants_pipeline.py:170-195)
//
// No tensor cores: there is no dense contraction on this path.  K0/K2 are HBM-side kernels,
// K1 is bound by instruction fetch and per-warp latency, K3 by shared-memory wavefronts
// (DESIGN.md sections 3 and 6 carry the measurements).
#include "kernels.cuh"

#include <math.h>
#include <stdlib.h>

#include <array>
#include <iterator>
#include <utility>

#include "numparse.h"

// UGVC_HOST_EMU: tests/host_emu compiles the K1-K3 kernel bodies of this file with g++ (one emulated
// thread per CTA, TPB = 1) to run the parity tests without a GPU; the product build never defines it.
#ifndef K1_TPB
#define K1_TPB 128
#endif
#ifndef K1_MIN_CTAS
#define K1_MIN_CTAS 8  // resident CTAs per SM the register allocation targets (profiled: see DESIGN.md)
#endif
#ifndef K2_TPB
#define K2_TPB 256
#endif

#ifndef UGVC_HOST_EMU  // K0 (cooperative tile scan, inline PTX): the emulation indexes lines on the host
// ------------------------------------------------------------------------------------------
// small helpers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned nl_bits4(unsigned w) {
    unsigned m = __vcmpeq4(w, 0x0A0A0A0Au);
    return ((m >> 7) & 1u) | ((m >> 14) & 2u) | ((m >> 21) & 4u) | ((m >> 28) & 8u);
}
__device__ __forceinline__ uint4 ld_stream16(const uint4* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

// ------------------------------------------------------------------------------------------
// K0: line index (single pass)
// ------------------------------------------------------------------------------------------
// One read of the text.  Tiles of 64 KiB are claimed in order from an atomic ticket; each thread
// turns its 256 contiguous bytes into four 64-bit newline masks, the block scans the pop-counts, the
// tile's running record count comes from a decoupled look-back over the tile-state words
// (bit 63: inclusive prefix published, bit 62: aggregate published), and the line starts are
// written straight from the masks -- no second pass over the text.
#define K0_TPB 256
#define K0_SEGS 4
#define K0_TILE_BYTES (K0_TPB * 64 * K0_SEGS)
#define K0_FLAG_AGG (1ull << 62)
#define K0_FLAG_INC (1ull << 63)
#define K0_VAL_MASK ((1ull << 62) - 1ull)

__device__ __forceinline__ unsigned long long nl_mask64(const uint8_t* __restrict__ text, size_t off, size_t n_bytes) {
    unsigned long long m = 0;
    if (off + 64 <= n_bytes) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const uint4 v = ld_stream16(reinterpret_cast<const uint4*>(text + off) + q);
            const unsigned long long part = (unsigned long long)(nl_bits4(v.x) | (nl_bits4(v.y) << 4) |
                                                                 (nl_bits4(v.z) << 8) | (nl_bits4(v.w) << 12));
            m |= part << (16 * q);
        }
    } else {
        for (size_t q = off; q < n_bytes && q < off + 64; ++q)
            if (text[q] == '\n') m |= 1ull << (q - off);
    }
    return m;
}

__global__ void __launch_bounds__(K0_TPB) k0_index(const uint8_t* __restrict__ text, size_t n_bytes,
                                                   unsigned long long* __restrict__ tile_state,
                                                   unsigned int* __restrict__ ticket, size_t n_tiles,
                                                   int64_t* __restrict__ line_start, size_t cap_records,
                                                   int64_t* __restrict__ n_records, unsigned long long* err) {
    __shared__ unsigned s_warp[K0_TPB / 32];
    __shared__ unsigned long long s_excl;
    __shared__ unsigned s_tile;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (;;) {
        if (threadIdx.x == 0) s_tile = atomicAdd(ticket, 1u);
        __syncthreads();
        const size_t tile = s_tile;
        if (tile >= n_tiles) break;
        // each thread owns K0_SEGS * 64 contiguous bytes
        const size_t off = tile * K0_TILE_BYTES + (size_t)threadIdx.x * (64 * K0_SEGS);
        unsigned long long mask[K0_SEGS];
        unsigned cnt = 0;
#pragma unroll
        for (int g = 0; g < K0_SEGS; ++g) {
            mask[g] = off + 64 * g < n_bytes ? nl_mask64(text, off + 64 * g, n_bytes) : 0ull;
            cnt += __popcll(mask[g]);
        }
        unsigned incl = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned v = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += v;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        unsigned warp_base = 0, total = 0;
#pragma unroll
        for (int w = 0; w < K0_TPB / 32; ++w) {
            const unsigned v = s_warp[w];
            if (w < warp) warp_base += v;
            total += v;
        }
        if (threadIdx.x == 0) {
            // publish the aggregate, then look back for the exclusive prefix
            unsigned long long excl = 0;
            if (tile == 0) {
                atomicExch(&tile_state[0], K0_FLAG_INC | (unsigned long long)total);
            } else {
                atomicExch(&tile_state[tile], K0_FLAG_AGG | (unsigned long long)total);
                size_t p = tile;
                while (p > 0) {
                    --p;
                    unsigned long long st;
                    do {
                        st = atomicAdd(&tile_state[p], 0ull);
                    } while ((st & (K0_FLAG_AGG | K0_FLAG_INC)) == 0);
                    excl += st & K0_VAL_MASK;
                    if (st & K0_FLAG_INC) break;
                }
                atomicExch(&tile_state[tile], K0_FLAG_INC | (excl + total));
            }
            s_excl = excl;
            if (tile == n_tiles - 1) {
                long long all = (long long)(excl + total);
                if (n_bytes > 0 && text[n_bytes - 1] != '\n')  // contract: the batch ends with '\n'
                    atomicMin(err, ugvc_pack_error(all, 0xFFFF, REASON_MALFORMED_LINE));
                if ((size_t)all > cap_records) {
                    atomicMin(err, ugvc_pack_error((long long)cap_records, 0xFFFF, REASON_TOO_MANY_ELEMS));
                    all = (long long)cap_records;
                }
                *n_records = all;
                line_start[0] = 0;
            }
        }
        __syncthreads();
        size_t idx = (size_t)s_excl + warp_base + (incl - cnt);
#pragma unroll
        for (int g = 0; g < K0_SEGS; ++g) {
            unsigned long long m = mask[g];
            while (m) {
                const int b = __ffsll((long long)m) - 1;
                m &= m - 1;
                if (idx + 1 <= cap_records) line_start[idx + 1] = (int64_t)(off + 64 * g + b + 1);
                ++idx;
            }
        }
        __syncthreads();  // s_tile / s_excl are rewritten by the next round
    }
}

__global__ void k0_empty(int64_t* __restrict__ line_start, int64_t* __restrict__ n_records) {
    *n_records = 0;
    line_start[0] = 0;
}

void launch_k0(const uint8_t* d_text, size_t n_bytes, uint32_t* scratch, int64_t* line_start,
               size_t cap_records, int64_t* d_n_records, unsigned long long* d_err, int sm_count,
               cudaStream_t st) {
    // scratch: [0] ticket (padded to 8 bytes), then one 64-bit state word per tile
    const size_t n_tiles = (n_bytes + K0_TILE_BYTES - 1) / K0_TILE_BYTES;
    if (n_tiles == 0) {
        k0_empty<<<1, 1, 0, st>>>(line_start, d_n_records);
        return;
    }
    cudaMemsetAsync(scratch, 0, 8 + n_tiles * sizeof(unsigned long long), st);
    size_t blocks = n_tiles < (size_t)sm_count * 8 ? n_tiles : (size_t)sm_count * 8;
    k0_index<<<(unsigned)blocks, K0_TPB, 0, st>>>(d_text, n_bytes,
                                                  reinterpret_cast<unsigned long long*>(scratch) + 1,
                                                  reinterpret_cast<unsigned int*>(scratch), n_tiles, line_start,
                                                  cap_records, d_n_records, d_err);
}

#endif  // !UGVC_HOST_EMU

// ------------------------------------------------------------------------------------------
// K1: field parse
// ------------------------------------------------------------------------------------------
// One thread per record.  The record's bytes are consumed through a 64-bit register window
// (aligned 8-byte loads through L1; delimiter search is SWAR over the window with
// __vcmpeq4), keys and short string values are gathered into three 64-bit registers and
// matched word-wise against the plan tables in shared memory, numbers go through
// numparse.h.  The scanning primitives are real (non-inlined) functions taking and returning
// the cursor by value: the kernel body stays small enough for the instruction cache while
// the 32 lanes of a warp sit in different fields of different records.
#define K1_MAX_STRINGS 96
#define K1_MAX_DICTS 64
// fixed layout of the shared-memory plan tables, then the slot tile
#define K1_OFF_TAGS 0
#define K1_OFF_STRINGS (K1_OFF_TAGS + UGVC_MAX_TAGS * 40)
#define K1_OFF_SLOTS (K1_OFF_STRINGS + K1_MAX_STRINGS * 32)
#define K1_OFF_DICTS (K1_OFF_SLOTS + 256 * 4)
#define K1_OFF_HTAB (K1_OFF_DICTS + K1_MAX_DICTS * 4)
#define K1_OFF_SCHED (K1_OFF_HTAB + 256)
#define K1_SMEM_BYTES (K1_OFF_SCHED + UGVC_MAX_SCHED * 32)

extern __shared__ __align__(16) uint8_t k1_smem[];
__device__ __forceinline__ const PlanTag* s_tags() { return reinterpret_cast<const PlanTag*>(k1_smem + K1_OFF_TAGS); }
__device__ __forceinline__ const PlanString* s_strings() { return reinterpret_cast<const PlanString*>(k1_smem + K1_OFF_STRINGS); }
__device__ __forceinline__ const PlanSlot* s_slots() { return reinterpret_cast<const PlanSlot*>(k1_smem + K1_OFF_SLOTS); }
__device__ __forceinline__ const PlanDict* s_dicts() { return reinterpret_cast<const PlanDict*>(k1_smem + K1_OFF_DICTS); }
__device__ __forceinline__ const uint8_t* s_htab() { return k1_smem + K1_OFF_HTAB; }
__device__ __forceinline__ const SchedEntry* s_sched() { return reinterpret_cast<const SchedEntry*>(k1_smem + K1_OFF_SCHED); }

// Look-ahead cursor: two consecutive aligned 8-byte words of the line (the second one is always
// already loaded, so the next load is issued a word ahead of its use) and a byte offset into
// the first.  peek8() is the next 8 bytes of the stream whatever the alignment.
struct Cur {
    const unsigned long long* wp;  // word after hi
    unsigned long long lo, hi;
    int sh;                        // bytes of lo already consumed (0..7)
    __device__ __forceinline__ void init(const uint8_t* p) {
        sh = (int)(reinterpret_cast<uintptr_t>(p) & 7u);
        wp = reinterpret_cast<const unsigned long long*>(p - sh);
        lo = __ldg(wp++);
        hi = __ldg(wp++);
    }
    __device__ __forceinline__ unsigned peek() const { return (unsigned)(lo >> (8 * sh)) & 0xFFu; }
    __device__ __forceinline__ unsigned long long peek8() const {
        return sh ? ((lo >> (8 * sh)) | (hi << (64 - 8 * sh))) : lo;
    }
    __device__ __forceinline__ void adv() {
        if (++sh == 8) {
            sh = 0;
            lo = hi;
            hi = __ldg(wp++);
        }
    }
    __device__ __forceinline__ void advance(int k) {  // 0 <= k <= 8
        sh += k;
        if (sh >= 8) {
            sh -= 8;
            lo = hi;
            hi = __ldg(wp++);
        }
    }
    __device__ __forceinline__ const uint8_t* ptr() const { return reinterpret_cast<const uint8_t*>(wp - 2) + sh; }
};

struct Key {
    unsigned long long k0, k1, k2, k3;  // the first 32 bytes, little-endian, zero padded
    int len;                             // the true length (may exceed 32: then nothing matches)
};
struct KeyCur {
    Cur c;
    Key k;
};
struct NumCur {
    Cur c;
    double v;
    int st;
};

#define B4(ch) ((unsigned)(ch) * 0x01010101u)

// Bit 7 set in the FIRST byte of w that equals tab, newline or one of the two pattern bytes
// (bytes above the first match may carry false positives -- only the lowest set bit is used).
// Classic has-zero-byte SWAR on 64-bit words: sm_90 has no byte-compare instruction
// (__vcmpeq4 is emulated with five instructions).
__device__ __forceinline__ unsigned long long has_zero(unsigned long long x) {
    return (x - 0x0101010101010101ull) & ~x & 0x8080808080808080ull;
}
__device__ __forceinline__ unsigned long long delim_mask(unsigned long long w, unsigned a4, unsigned b4) {
    const unsigned long long a8 = ((unsigned long long)a4 << 32) | a4, b8 = ((unsigned long long)b4 << 32) | b4;
    // tab (0x09) and newline (0x0A) are the only bytes of a VCF line in 0x08..0x0B
    return has_zero((w & 0xFCFCFCFCFCFCFCFCull) ^ 0x0808080808080808ull) | has_zero(w ^ a8) | has_zero(w ^ b8);
}

// advance to the first byte that is tab, newline or a pattern byte (8 bytes of look-ahead per step)
__device__ __noinline__ Cur skip_until(Cur c, unsigned a4, unsigned b4) {
    for (;;) {
        const unsigned long long m = delim_mask(c.peek8(), a4, b4);
        if (m) {
            c.advance((__ffsll((long long)m) - 1) >> 3);
            return c;
        }
        c.advance(8);
    }
}

__device__ __forceinline__ void key_append(Key& key, unsigned long long bytes, int k) {
    const int pos = key.len;
    key.len = pos + k;
    if (k == 0 || pos >= 32) return;
    const int sh = (pos & 7) * 8;
    const unsigned long long lo = bytes << sh;
    const unsigned long long hi = sh ? (bytes >> (64 - sh)) : 0ull;
    const int word = pos >> 3;
    if (word == 0) {
        key.k0 |= lo;
        key.k1 |= hi;
    } else if (word == 1) {
        key.k1 |= lo;
        key.k2 |= hi;
    } else if (word == 2) {
        key.k2 |= lo;
        key.k3 |= hi;
    } else {
        key.k3 |= lo;
    }
}

// gather the bytes up to (not including) the first tab / newline / pattern byte
__device__ __noinline__ KeyCur take_until(Cur c, unsigned a4, unsigned b4) {
    KeyCur r;
    r.k.k0 = r.k.k1 = r.k.k2 = r.k.k3 = 0ull;
    r.k.len = 0;
    for (;;) {
        const unsigned long long x = c.peek8();
        const unsigned long long m = delim_mask(x, a4, b4);
        if (m) {
            const int k = (__ffsll((long long)m) - 1) >> 3;  // 0..7
            key_append(r.k, x & ((1ull << (8 * k)) - 1ull), k);
            c.advance(k);
            r.c = c;
            return r;
        }
        key_append(r.k, x, 8);
        c.advance(8);
    }
}

__device__ __noinline__ NumCur parse_num_cur(Cur c) {
    NumCur r;
    r.st = ugvc_parse_num(c, r.v);
    r.c = c;
    return r;
}

struct IntCur {
    Cur c;
    int v;
    int st;
};
// "[+-]digits" or "." -> int (int32 range, else NUM_BAD); anything else in the token is NUM_BAD
__device__ __noinline__ IntCur parse_int_cur(Cur c) {
    IntCur r;
    unsigned ch = c.peek();
    bool neg = false;
    if (ch == '-' || ch == '+') {
        neg = ch == '-';
        c.adv();
        ch = c.peek();
    }
    unsigned m = 0;
    int nd = 0;
    bool ovf = false;
    while (ugvc_is_digit(ch)) {
        const unsigned d = ch - '0';
        ovf |= m > 214748364u || (m == 214748364u && d > 7u);
        m = m * 10u + d;
        ++nd;
        c.adv();
        ch = c.peek();
    }
    r.st = NUM_OK;
    if (nd == 0) {
        if (ch == '.' && !neg) {
            c.adv();
            r.st = NUM_MISSING;
        } else
            r.st = NUM_BAD;
    } else if (ovf) {
        r.st = NUM_BAD;  // outside int32: htslib rejects the value
    }
    r.v = neg ? -(int)m : (int)m;
    r.c = c;
    return r;
}

__device__ __forceinline__ unsigned base_code(unsigned c) {
    // {A:1, T:2, G:3, C:4}  (transformers.py:72-77)
    return c == 'A' ? 1u : c == 'T' ? 2u : c == 'G' ? 3u : c == 'C' ? 4u : 0u;
}
__device__ __forceinline__ unsigned motif_code(unsigned c) { return c == 'N' ? 5u : base_code(c); }

__device__ __noinline__ int find_tag(Key key) {
    if (key.len <= 0 || key.len > UGVC_NAME_MAX) return -1;
    unsigned idx = ugvc_key_hash(key.k0, key.k1, key.k2, key.k3, key.len);
    for (int probe = 0; probe < 256; ++probe) {
        const unsigned t = s_htab()[idx];
        if (t == 0xFFu) return -1;
        const unsigned long long* tw = reinterpret_cast<const unsigned long long*>(&s_tags()[t]);
        if (tw[0] == key.k0 && tw[1] == key.k1 && tw[2] == key.k2 && tw[3] == key.k3 && (int)(tw[4] & 0xFFu) == key.len)
            return (int)t;
        idx = (idx + 1) & 255u;
    }
    return -1;
}

// Slot stores go straight to the columnar batch raw[slot][record] (rows were pre-filled with
// RAW_ABSENT by k1_fill).  A warp's lanes hit different rows at different times, so these are
// 4-byte partial-sector writes that L2 merges (8 neighbouring records share a sector); keeping
// the tile out of shared memory is what lets ~2x more warps stay resident, and this kernel is
// bound by latency per warp, not by store bandwidth.
struct RawOut {
    uint32_t* col;      // &raw[0][record]
    size_t stride;      // elements between slot rows
};
__device__ __forceinline__ void store_slot(const RawOut& o, int slot, uint32_t bits) { o.col[(size_t)slot * o.stride] = bits; }
__device__ __forceinline__ void store_slot_f(const RawOut& o, int slot, float v) { store_slot(o, slot, __float_as_uint(v)); }

#define CH3(a, b, c) ((unsigned long long)(a) | ((unsigned long long)(b) << 8) | ((unsigned long long)(c) << 16))

__device__ __forceinline__ uint32_t reduce_string(const PlanSlot sl, const Key& k) {
    switch (sl.reducer) {
        case RED_BASE:
            return __float_as_uint(k.len == 1 ? (float)base_code((unsigned)k.k0 & 0xFFu) : 0.0f);
        case RED_INSDEL:
            if (k.len == 3 && k.k0 == CH3('i', 'n', 's')) return __float_as_uint(-1.0f);
            if (k.len == 3 && k.k0 == CH3('d', 'e', 'l')) return __float_as_uint(1.0f);
            if (k.len == 2 && k.k0 == CH3('N', 'A', 0)) return __float_as_uint(0.0f);
            return RAW_ERR;
        case RED_DICT: {
            const PlanDict d = s_dicts()[sl.dict];
            for (int i = 0; i < d.n_strings; ++i) {
                const unsigned long long* sw = reinterpret_cast<const unsigned long long*>(&s_strings()[d.first_string + i]);
                if (sw[0] == k.k0 && sw[1] == k.k1 && sw[2] == k.k2 && (int)(sw[3] & 0xFFu) == k.len)
                    return __float_as_uint((float)i);
            }
            return RAW_ERR;
        }
        default:
            return RAW_ERR;
    }
}

// tuple of region names -> code of the (sorted) subset; transformers.py:108-123.  Rarely used
// (CNV flavour): kept out of line so the hot decoders stay small.
__device__ __noinline__ Cur parse_region(RawOut o, int slot, unsigned type, bool scalar, Cur c, unsigned vend) {
    const unsigned v4 = B4(vend), c4 = B4(',');
    if (type != KIND_STR) {
        store_slot(o, slot, RAW_ERR);
        return c;
    }
    const PlanDict d = s_dicts()[s_slots()[slot].dict];
    unsigned mask = 0;
    bool bad = d.n_strings != 3;
    for (;;) {
        const KeyCur r = take_until(c, scalar ? v4 : c4, v4);
        c = r.c;
        int hit = -1;
        for (int i = 0; i < 3 && !bad; ++i) {
            const unsigned long long* sw = reinterpret_cast<const unsigned long long*>(&s_strings()[d.first_string + i]);
            if (sw[0] == r.k.k0 && sw[1] == r.k.k1 && sw[2] == r.k.k2 && (int)(sw[3] & 0xFFu) == r.k.len) hit = i;
        }
        bad |= hit < 0 || (mask & (1u << hit));  // unknown or repeated name: KeyError in the reference
        if (hit >= 0) mask |= 1u << hit;
        if (c.peek() == ',' && !scalar) {
            c.adv();
            continue;
        }
        break;
    }
    // subsets of the sorted names enumerated by size, then lexicographically, from 1
    const float code = (float)((0x87645321u >> (4 * (mask & 7u))) & 0xFu);
    store_slot(o, slot, bad ? RAW_ERR : __float_as_uint(code));
    return c;
}

// Decode one tag value starting at the cursor.  vend ends a value in this column (';' in INFO,
// ':' in the sample column).  The plan lays a tag's slots out as elements 0..n_elem-1 followed
// by at most one whole-value slot, so element e lands in slot first_slot + e.  Returns the
// cursor somewhere inside / at the end of the value; the caller skips to vend.
__device__ __noinline__ Cur parse_value(RawOut o, int t, unsigned kind, Cur c, unsigned vend) {
    const PlanTag tg = s_tags()[t];
    const unsigned whole = tg.whole_red;
    const int s0 = tg.first_slot;
    const int n_elem = (int)tg.n_slots - (whole != 0xFFu ? 1 : 0);
    const unsigned type = kind & KIND_TYPE_MASK;
    const bool scalar = (kind & KIND_SCALAR) != 0;
    const unsigned v4 = B4(vend), c4 = B4(',');
    if (type == KIND_FLAG) {
        for (int s = s0; s < s0 + (int)tg.n_slots; ++s) store_slot(o, s, RAW_MISSING);
        return c;
    }
    if (whole == RED_MOTIF_L || whole == RED_MOTIF_R) {
        // list(x): characters of a str, elements of a tuple (only single-character elements can
        // match a base) -- transformers.py:36-60
        if (type != KIND_STR) {
            store_slot(o, tg.whole_slot, RAW_ERR);
            return c;
        }
        double num = 0.0, scale = 1.0;
        const bool left = whole == RED_MOTIF_L;
        unsigned ch = c.peek();
        int elen = 0;
        unsigned first = 0;
        for (;;) {
            const bool end = (ch == vend || ch == '\t' || ch == '\n');
            unsigned code = 0;
            bool emit = false;
            if (scalar) {
                if (!end) {
                    code = motif_code(ch);
                    emit = true;
                }
            } else if (end || ch == ',') {
                code = elen == 1 ? motif_code(first) : 0u;
                emit = true;
                elen = 0;
            } else {
                if (elen == 0) first = ch;
                ++elen;
            }
            if (emit) {
                if (left) {
                    num += scale * (double)code;
                    scale *= 10.0;
                } else
                    num = num * 10.0 + (double)code;
            }
            if (end) break;
            c.adv();
            ch = c.peek();
        }
        store_slot_f(o, tg.whole_slot, (float)num);
        return c;
    }
    if (whole == RED_REGION) return parse_region(o, tg.whole_slot, type, scalar, c, vend);
    if (whole == RED_GT_HOM) {
        const KeyCur r = take_until(c, v4, v4);
        const bool hom = r.k.len == 3 && (r.k.k0 == CH3('1', '/', '1') || r.k.k0 == CH3('1', '|', '1'));
        store_slot_f(o, tg.whole_slot, hom ? 1.0f : 0.0f);
        return r.c;
    }
    if (whole == RED_STRNUM) {
        // pd.to_numeric ignores spaces around the number (the tile kernel hands such values over to this parser)
        while (c.peek() == ' ') c.adv();
        NumCur r = parse_num_cur(c);
        while (r.st == NUM_OK && r.c.peek() == ' ') r.c.adv();
        const unsigned ch = r.c.peek();
        const bool ok = r.st == NUM_OK && (ch == vend || ch == '\t' || ch == '\n') && !isnan(r.v);
        store_slot(o, tg.whole_slot, ok ? __float_as_uint((float)r.v) : RAW_ERR);
        return r.c;
    }
    const bool count_all = whole == RED_LEN;
    int e = 0;
    for (;;) {
        if (type == KIND_INT) {
            // Integer tags (htslib int32): digits only, no binary64 round trip
            IntCur r = parse_int_cur(c);
            c = r.c;
            const unsigned ch = c.peek();
            if (ch != ',' && ch != vend && ch != '\t' && ch != '\n') {
                r.st = NUM_BAD;
                c = skip_until(c, c4, v4);
            }
            if (e < n_elem) {
                uint32_t bits;
                if (s_slots()[s0 + e].reducer != RED_NUM) bits = RAW_ERR;
                else if (r.st != NUM_OK) bits = r.st == NUM_MISSING ? RAW_MISSING : RAW_ERR;
                else bits = __float_as_uint((float)r.v);
                store_slot(o, s0 + e, bits);
            }
        } else if (type == KIND_FLOAT) {
            NumCur r = parse_num_cur(c);
            c = r.c;
            const unsigned ch = c.peek();
            if (ch != ',' && ch != vend && ch != '\t' && ch != '\n') {  // trailing garbage in the token
                r.st = NUM_BAD;
                c = skip_until(c, c4, v4);
            }
            if (e < n_elem) {
                uint32_t bits;
                if (s_slots()[s0 + e].reducer != RED_NUM) bits = RAW_ERR;
                else if (r.st != NUM_OK) bits = r.st == NUM_MISSING ? RAW_MISSING : RAW_ERR;
                else {
                    const float f = (float)r.v;  // float32(strtod(text))
                    bits = isnan(f) ? RAW_MISSING : __float_as_uint(f);
                }
                store_slot(o, s0 + e, bits);
            }
        } else if (e < n_elem) {
            const KeyCur r = take_until(c, scalar ? v4 : c4, v4);
            c = r.c;
            store_slot(o, s0 + e, reduce_string(s_slots()[s0 + e], r.k));
        } else {
            c = skip_until(c, scalar ? v4 : c4, v4);
        }
        ++e;
        if (c.peek() == ',' && !(scalar && type == KIND_STR) && (e < n_elem || count_all)) {
            c.adv();
            continue;
        }
        break;
    }
    for (int m = e; m < n_elem; ++m) store_slot(o, s0 + m, RAW_MISSING);  // vector shorter than needed
    if (count_all) store_slot_f(o, tg.whole_slot, (float)e);
    return c;
}

__device__ __forceinline__ bool key_is_cg(const Key& k) {
    // an allele equal to GGC or CCG (blacklist.py:85-101: tuple membership)
    return k.len == 3 && (k.k0 == CH3('G', 'G', 'C') || k.k0 == CH3('C', 'C', 'G'));
}

__device__ __forceinline__ void set_tag_missing(const RawOut& o, int t) {
    const PlanTag tg = s_tags()[t];
    for (int s = tg.first_slot; s < tg.first_slot + tg.n_slots; ++s) store_slot(o, s, RAW_MISSING);
}

// number of leading ASCII digits in the 8 look-ahead bytes (0..8)
__device__ __forceinline__ int leading_digits(unsigned long long x) {
    const unsigned long long hi = 0xF0F0F0F0F0F0F0F0ull, three = 0x3030303030303030ull;
    // a byte is a digit iff its high nibble is 3 and stays 3 after adding 6
    const unsigned long long nd = ((x & hi) ^ three) | (((x + 0x0606060606060606ull) & hi) ^ three);
    return nd ? ((__ffsll((long long)nd) - 1) >> 3) : 8;
}
__device__ __forceinline__ bool is_term(unsigned ch, unsigned vend) {
    return ch == ',' || ch == vend || ch == '\t' || ch == '\n';
}

// Decode the value of a scheduled key (every lane that gets here holds the same key, so the
// class switch is warp-uniform) and leave the cursor on the byte that ends the field.
// meta = the entry's last 8 bytes: len | cls<<8 | slot0<<16 | n_elem<<24 | dict<<32 | flags<<40 | tag<<48
__device__ __noinline__ Cur decode_sched(RawOut o, unsigned long long meta, Cur c, unsigned vend) {
    const unsigned cls = (unsigned)(meta >> 8) & 0xFFu;
    const int slot0 = (int)((meta >> 16) & 0xFFu), n_elem = (int)((meta >> 24) & 0xFFu);
    const unsigned flags = (unsigned)(meta >> 40) & 0xFFu;
    const unsigned v4 = B4(vend), c4 = B4(',');
    if (cls == CLS_INT || cls == CLS_FLOAT) {
        const bool count_all = (flags & SCHED_COUNT_ALL) != 0;
        int e = 0;
        for (;;) {
            uint32_t bits;
            // fast paths on the 8-byte look-ahead: a short unsigned integer, or digits '.' digits,
            // ending inside the window; anything else goes through the full parsers
            const unsigned long long x = c.peek8();
            const int k1 = leading_digits(x);
            bool fast = false;
            if (cls == CLS_INT) {
                if (k1 >= 1 && k1 <= 7 && is_term((unsigned)(x >> (8 * k1)) & 0xFFu, vend)) {
                    unsigned v = 0;
                    for (int i = 0; i < k1; ++i) v = v * 10u + ((unsigned)(x >> (8 * i)) & 0xFu);
                    bits = __float_as_uint((float)v);
                    c.advance(k1);
                    fast = true;
                }
                if (!fast) {
                    const IntCur r = parse_int_cur(c);  // htslib int32 -> fp32 feature
                    c = r.c;
                    bits = r.st == NUM_OK ? __float_as_uint((float)r.v) : (r.st == NUM_MISSING ? RAW_MISSING : RAW_ERR);
                }
            } else {
#ifdef UGVC_K1_NEGFAST
                // experiment (round 2): "-d.ddd" decoded on the look-ahead too (the rank-sum tags are negative half of the time)
                if ((x & 0xFFull) == '-') {
                    const unsigned long long xs = (x >> 8) | (0xFFull << 56);
                    const int n1 = leading_digits(xs);
                    if (n1 >= 1 && n1 <= 4 && ((unsigned)(xs >> (8 * n1)) & 0xFFu) == '.') {
                        const unsigned long long ys = xs >> (8 * (n1 + 1));
                        const int n2 = leading_digits(ys | (0xFFull << (8 * (7 - n1))));
                        if (n2 >= 1 && n1 + 1 + n2 <= 6 && is_term((unsigned)(ys >> (8 * n2)) & 0xFFu, vend)) {
                            unsigned m = 0;
                            for (int i = 0; i < n1; ++i) m = m * 10u + ((unsigned)(xs >> (8 * i)) & 0xFu);
                            for (int i = 0; i < n2; ++i) m = m * 10u + ((unsigned)(ys >> (8 * i)) & 0xFu);
                            bits = __float_as_uint((float)(-((double)m / ugvc_ten(n2))));
                            c.advance(1 + n1 + 1 + n2);
                            fast = true;
                        }
                    }
                } else
#endif
                if (k1 >= 1 && k1 <= 5 && ((unsigned)(x >> (8 * k1)) & 0xFFu) == '.') {
                    const unsigned long long y = x >> (8 * (k1 + 1));
                    const int k2 = leading_digits(y | (0xFFull << (8 * (7 - k1))));  // bytes past the window: non-digits
                    if (k2 >= 1 && k1 + 1 + k2 <= 7 && is_term((unsigned)(y >> (8 * k2)) & 0xFFu, vend)) {
                        unsigned m = 0;
                        for (int i = 0; i < k1; ++i) m = m * 10u + ((unsigned)(x >> (8 * i)) & 0xFu);
                        for (int i = 0; i < k2; ++i) m = m * 10u + ((unsigned)(y >> (8 * i)) & 0xFu);
                        // Clinger: m < 2^24 and 10^k2 are exact doubles, one correctly rounded division
                        const float f = (float)((double)m / ugvc_ten(k2));
                        bits = __float_as_uint(f);
                        c.advance(k1 + 1 + k2);
                        fast = true;
                    }
                }
                if (!fast) {
                    const NumCur r = parse_num_cur(c);  // float32(strtod(text))
                    c = r.c;
                    const float f = (float)r.v;
                    bits = r.st == NUM_OK ? (isnan(f) ? RAW_MISSING : __float_as_uint(f))
                                          : (r.st == NUM_MISSING ? RAW_MISSING : RAW_ERR);
                }
            }
            const unsigned ch = c.peek();
            if (ch != ',' && ch != vend && ch != '\t' && ch != '\n') {  // trailing garbage in the token
                bits = RAW_ERR;
                c = skip_until(c, c4, v4);
            }
            if (e < n_elem) store_slot(o, slot0 + e, bits);
            ++e;
            if (c.peek() == ',' && (e < n_elem || count_all)) {
                c.adv();
                continue;
            }
            break;
        }
        for (int m = e; m < n_elem; ++m) store_slot(o, slot0 + m, RAW_MISSING);  // vector shorter than needed
        if (count_all) store_slot_f(o, slot0 + n_elem, (float)e);
    } else if (cls == CLS_DICT1) {
        // category strings of up to 7 bytes are compared against the look-ahead directly
        const PlanDict d = s_dicts()[(meta >> 32) & 0xFFu];
        const unsigned long long x = c.peek8();
        int found = -1;
        bool all_short = true;
        for (int i = 0; i < d.n_strings; ++i) {
            const PlanString* ps = &s_strings()[d.first_string + i];
            const int L = ps->len;
            all_short &= L <= 7;
            if (L <= 7) {
                const unsigned long long w0 = *reinterpret_cast<const unsigned long long*>(ps);
                const unsigned nxt = (unsigned)(x >> (8 * L)) & 0xFFu;
                if ((x & ((1ull << (8 * L)) - 1ull)) == w0 && (nxt == vend || nxt == '\t' || nxt == '\n')) found = i;
            }
        }
        if (found >= 0) {
            store_slot_f(o, slot0, (float)found);
            c.advance(s_strings()[d.first_string + found].len);
        } else if (all_short) {
            store_slot(o, slot0, RAW_ERR);  // unknown category
        } else {
            const KeyCur r = take_until(c, v4, v4);
            c = r.c;
            PlanSlot sl;
            sl.reducer = RED_DICT;
            sl.dict = (uint8_t)((meta >> 32) & 0xFFu);
            store_slot(o, slot0, reduce_string(sl, r.k));
        }
    } else if (cls == CLS_GENERIC) {
        const int tag = (int)(short)(meta >> 48);
        const unsigned kind = vend == ':' ? s_tags()[tag].fmt_kind : s_tags()[tag].info_kind;
        c = parse_value(o, tag, kind, c, vend);
    }
    const unsigned ch = c.peek();
    if (ch != vend && ch != '\t' && ch != '\n') c = skip_until(c, v4, v4);
    return c;
}

#define K1_PART 0
#define K1_KERNEL_NAME k1_parse
#include "k1_parse_body.inc"
#undef K1_PART
#undef K1_KERNEL_NAME
#ifdef UGVC_K1_SPLIT
#define K1_PART 1
#define K1_KERNEL_NAME k1_parse_info
#include "k1_parse_body.inc"
#undef K1_PART
#undef K1_KERNEL_NAME
#define K1_PART 2
#define K1_KERNEL_NAME k1_parse_frame
#include "k1_parse_body.inc"
#undef K1_PART
#undef K1_KERNEL_NAME
#endif

#include "k1_tok.inc"

size_t k1_smem_bytes(const DevPlan&) { return (size_t)K1_SMEM_BYTES; }

// every slot of every record starts ABSENT (the reference's defaultdict(lambda: None)):
// coalesced 16-byte stores over the first n_records columns of each slot row
__global__ void __launch_bounds__(256) k1_fill(uint32_t* __restrict__ raw, size_t row_stride, int n_slots,
                                               const int64_t* __restrict__ n_records_p) {
    const long long n_rec = *n_records_p;
    const long long quads = (n_rec + 3) >> 2;  // rows are 16-byte aligned and padded (cap is a multiple of 128)
    const uint4 v = make_uint4(RAW_ABSENT, RAW_ABSENT, RAW_ABSENT, RAW_ABSENT);
    for (int s = blockIdx.y; s < n_slots; s += gridDim.y) {
        uint4* row = reinterpret_cast<uint4*>(raw + (size_t)s * row_stride);
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < quads; i += (long long)gridDim.x * blockDim.x)
            row[i] = v;
    }
}

#ifndef UGVC_HOST_EMU
void launch_k1(const DevPlan& plan, const DevSchedule& sched, const uint8_t* d_text, const int64_t* line_start,
               const int64_t* d_n_records,
               uint32_t* raw, size_t row_stride, ugvc_recinfo* recinfo, unsigned long long* d_err,
               long long* d_counts, int sm_count, cudaStream_t st) {
    const size_t smem = k1_smem_bytes(plan);
    // persistent grid: exactly the CTAs that can be resident (registers and shared memory decide)
    static int occ = 0;
    if (occ == 0) {
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k1_parse, K1_TPB, smem) != cudaSuccess || occ < 1) occ = 1;
    }
    int per_sm = occ;
    static const int tune = getenv("UGVC_K1_CTAS_PER_SM") ? atoi(getenv("UGVC_K1_CTAS_PER_SM")) : 0;  // profiling knob
    if (tune > 0 && tune < per_sm) per_sm = tune;
    if (plan.h.n_slots) {
        const dim3 fgrid((unsigned)(sm_count * 2), (unsigned)(plan.h.n_slots < 16 ? plan.h.n_slots : 16));
        k1_fill<<<fgrid, 256, 0, st>>>(raw, row_stride, (int)plan.h.n_slots, d_n_records);
    }
#ifdef UGVC_K1_SPLIT
    static int occ_i = 0, occ_f = 0;
    if (occ_i == 0) {
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_i, k1_parse_info, K1_TPB, smem) != cudaSuccess || occ_i < 1) occ_i = 1;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_f, k1_parse_frame, K1_TPB, smem) != cudaSuccess || occ_f < 1) occ_f = 1;
    }
    k1_parse_info<<<sm_count * occ_i, K1_TPB, smem, st>>>(plan, sched, d_text, line_start, d_n_records, raw, row_stride, recinfo,
                                                          d_err, d_counts, nullptr, nullptr);
    k1_parse_frame<<<sm_count * occ_f, K1_TPB, smem, st>>>(plan, sched, d_text, line_start, d_n_records, raw, row_stride, recinfo,
                                                           d_err, d_counts, nullptr, nullptr);
    (void)per_sm;
#else
    k1_parse<<<sm_count * per_sm, K1_TPB, smem, st>>>(plan, sched, d_text, line_start, d_n_records, raw, row_stride, recinfo,
                                                      d_err, d_counts, nullptr, nullptr);
#endif
}

// K1, both tiers: the tile kernel (line index + parse of the usual records, k1_tok.inc) and the generic parser over
// the records it put on the slow list.  scratch: [0] tile ticket, [1] slow-record count, then one
// 64-bit look-back state word per tile.
__global__ void k1_tile_empty(int64_t* __restrict__ line_start, int64_t* __restrict__ n_records) {
    *n_records = 0;
    line_start[0] = 0;
}
void launch_k1_fast(const DevPlan& plan, const DevFast& fast, const DevSchedule& sched, const uint8_t* d_text, size_t n_bytes,
                    uint32_t* scratch, int64_t* line_start, size_t cap_records, int64_t* d_n_records, uint32_t* raw,
                    size_t row_stride, ugvc_recinfo* recinfo, uint32_t* slow_list, unsigned long long* d_err,
                    long long* d_counts, int sm_count, cudaStream_t st) {
    const size_t n_tiles = (n_bytes + KT_TILE - 1) / KT_TILE;
    cudaMemsetAsync(scratch, 0, 8 + n_tiles * sizeof(unsigned long long), st);
    if (n_tiles == 0) {
        k1_tile_empty<<<1, 1, 0, st>>>(line_start, d_n_records);
        return;
    }
    const size_t blocks = n_tiles < (size_t)sm_count * 2 ? n_tiles : (size_t)sm_count * 2;  // two resident CTAs per SM
    const uint32_t wcap = kt_window_records(plan.h.n_slots);  // >= 24 for any plan (at most 255 slots)
    k1_tok<<<(unsigned)blocks, KT_TPB, KT_SMEM_BYTES, st>>>(plan, fast, d_text, n_bytes,
                                                            reinterpret_cast<unsigned long long*>(scratch) + 1, scratch, scratch + 1,
                                                            n_tiles, line_start, cap_records, d_n_records, raw, row_stride, recinfo,
                                                            slow_list, d_err, d_counts, wcap);
    // the slow tier: usually an empty list (the CTAs leave at once)
    k1_parse<<<sm_count * 2, K1_TPB, k1_smem_bytes(plan), st>>>(plan, sched, d_text, line_start, d_n_records, raw, row_stride,
                                                                recinfo, d_err, d_counts, slow_list, scratch + 1);
}

#endif  // !UGVC_HOST_EMU

// ------------------------------------------------------------------------------------------
// K2: feature assembly
// ------------------------------------------------------------------------------------------
// Four consecutive records per thread: every slot row and every feature row is touched with
// 16-byte loads / stores (rows are 512-byte aligned), policies applied lane-wise.
__device__ __forceinline__ float k2_apply(uint32_t bits, const PlanFeature& pf, long long rec, int f,
                                          unsigned long long* err) {
    float v = __uint_as_float(bits);
    if ((bits & 0x7F800000u) == 0x7F800000u) {  // the three sentinels are NaNs; the infinities share the exponent
        const bool ab = bits == RAW_ABSENT, mi = bits == RAW_MISSING;
        v = ab && pf.absent_pol == POL_VALUE ? pf.absent_val : v;
        v = mi && pf.missing_pol == POL_VALUE ? pf.missing_val : v;
        // +-inf (an overflowing literal, or "inf" itself): SimpleImputer's / the model's input check raises
        // "Input X contains infinity" in the reference whatever the column's pipeline is
        const bool bad_value = (ab && pf.absent_pol == POL_ERROR) || (!ab && !mi && (bits == RAW_ERR || (bits & 0x7FFFFFFFu) == 0x7F800000u));
        if (bad_value) atomicMin(err, ugvc_pack_error(rec, f, REASON_BAD_VALUE));
        else if (mi && pf.missing_pol == POL_ERROR) atomicMin(err, ugvc_pack_error(rec, f, REASON_NULL_FEATURE));
    }
    return v;
}

__device__ __forceinline__ void k2_combine_one(const PlanCombine cb, uint32_t bbits, float& a, long long rec, bool live,
                                               unsigned long long* err) {
    const bool b_null = bbits == RAW_ABSENT || bbits == RAW_MISSING;
    if (bbits == RAW_ERR && live) atomicMin(err, ugvc_pack_error(rec, cb.feature, REASON_BAD_VALUE));
    const float bv = __uint_as_float(bbits);
    const float r = isnan(a) ? (b_null ? a : bv) : (b_null ? a : fmaxf(a, bv));
    if (isnan(r) && live) atomicMin(err, ugvc_pack_error(rec, cb.feature, REASON_NULL_FEATURE));
    // an infinite operand wins the max: the model's input check raises "Input X contains infinity"
    if (isinf(r) && live) atomicMin(err, ugvc_pack_error(rec, cb.feature, REASON_BAD_VALUE));
    a = r;
}

__global__ void __launch_bounds__(K2_TPB) k2_features(const __grid_constant__ DevPlan plan,
                                                      const uint32_t* __restrict__ raw, size_t row_stride,
                                                      const int64_t* __restrict__ n_records_p,
                                                      float* __restrict__ feats, unsigned long long* err) {
    __shared__ PlanFeature s_feat[UGVC_MAX_FEATURES];
    const int F = plan.h.n_features;
    for (int i = threadIdx.x; i < F; i += K2_TPB) s_feat[i] = plan.feats[i];
    __syncthreads();
    const long long n_rec = *n_records_p;
    const long long n_quads = (n_rec + 3) >> 2;
    for (long long q = (long long)blockIdx.x * K2_TPB + threadIdx.x; q < n_quads; q += (long long)gridDim.x * K2_TPB) {
        const long long rec = q << 2;
        // records past n_rec inside the last quad: rows are padded to a multiple of 128, the values
        // there are the ABSENT fill and are never reported (only rec < n_rec can raise)
        const int live = (int)(n_rec - rec < 4 ? n_rec - rec : 4);
#pragma unroll 2
        for (int f = 0; f < F; ++f) {
            const PlanFeature pf = s_feat[f];
            const uint4 b = __ldg(reinterpret_cast<const uint4*>(raw + (size_t)pf.slot * row_stride + rec));
            float4 v;
            v.x = k2_apply(b.x, pf, rec, f, err);
            v.y = live > 1 ? k2_apply(b.y, pf, rec + 1, f, err) : 0.f;
            v.z = live > 2 ? k2_apply(b.z, pf, rec + 2, f, err) : 0.f;
            v.w = live > 3 ? k2_apply(b.w, pf, rec + 3, f, err) : 0.f;
            *reinterpret_cast<float4*>(feats + (size_t)f * row_stride + rec) = v;
        }
        for (unsigned c = 0; c < plan.h.n_combines; ++c) {
            // feature = max(feature, slot_b), nulls skipped (DataFrame.max(axis=1), transformers.py:200-201)
            const PlanCombine cb = plan.combines[c];
            const uint4 b = __ldg(reinterpret_cast<const uint4*>(raw + (size_t)cb.slot_b * row_stride + rec));
            float4* dst = reinterpret_cast<float4*>(feats + (size_t)cb.feature * row_stride + rec);
            float4 a = *dst;
            const uint32_t bb[4] = {b.x, b.y, b.z, b.w};
            float* av = &a.x;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                k2_combine_one(cb, bb[i], av[i], rec + i, i < live, err);
            }
            *dst = a;
        }
        for (unsigned c = 0; c < plan.h.n_checks; ++c) {
            const PlanCheck ck = plan.checks[c];
            const uint4 b = __ldg(reinterpret_cast<const uint4*>(raw + (size_t)ck.slot * row_stride + rec));
            const uint32_t bits[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                if (i >= live || bits[i] == RAW_ABSENT || bits[i] == RAW_MISSING) continue;  // handled by the feature policies
                const float v = __uint_as_float(bits[i]);
                const bool ok = ck.kind == 0 ? (v <= ck.bound) : (v >= ck.bound);
                if (!ok) atomicMin(err, ugvc_pack_error(rec + i, 0xFFFF, ck.kind == 0 ? REASON_TOO_MANY_ELEMS : REASON_BAD_VALUE));
            }
        }
    }
}

#ifndef UGVC_HOST_EMU
void launch_k2(const DevPlan& plan, const uint32_t* raw, size_t row_stride, const int64_t* d_n_records, float* feats,
               unsigned long long* d_err, int sm_count, cudaStream_t st) {
    k2_features<<<sm_count * 8, K2_TPB, 0, st>>>(plan, raw, row_stride, d_n_records, feats, d_err);
}
#endif  // !UGVC_HOST_EMU

// ------------------------------------------------------------------------------------------
// K3: inference + score math + FILTER decision
// ------------------------------------------------------------------------------------------
// One thread per record, one persistent CTA per SM.  Shared memory holds the feature tile
// [F][K3_TPB] (column f of a record tile is one coalesced row of the column-major matrix) and
// the forest in device form (8-byte nodes; leaves are absorbing: threshold = quiet NaN carrying
// the leaf row, right child = itself).  Trees are walked eight at a time with a fixed number of
// steps (the depth of the deepest leaf), branch-free, so eight independent load chains per
// thread hide the shared-memory latency; leaf values are then added in tree order in the
// arithmetic of the library that trained the model (fp64 for sklearn, fp32 for xgboost).
#ifndef K3_CHAINS
#define K3_CHAINS 8
#endif

__device__ __forceinline__ double expit64(double x) { return 1.0 / (1.0 + exp(-x)); }
// expf rounded once from the fp64 exponential.  The optimiser shrinks (float)exp((double)x) back to expf(x) (a
// library-call simplification that is only valid for a correctly rounded expf: seen on the GPU as 1-ulp differences
// in a sixth of the probabilities); the rounding therefore goes through the conversion intrinsic.
__device__ __forceinline__ float k3_expf_cr(float x) {
#ifdef __CUDA_ARCH__
    return __double2float_rn(exp((double)x));  // an intrinsic, not an fptrunc: the call is not shrunk
#else
    return (float)exp((double)x);
#endif
}

template <int CMP, int TPB>
__device__ __forceinline__ void walk8(const uint2* __restrict__ s_nodes, const uint32_t* __restrict__ s_roots,
                                      unsigned chunk_first_node, unsigned tr, unsigned tr_end, int depth,
                                      const float* __restrict__ x, int leaf[K3_CHAINS]) {
    unsigned n[K3_CHAINS];
    uint2 nd[K3_CHAINS];
#pragma unroll
    for (int j = 0; j < K3_CHAINS; ++j) {
        const unsigned t = tr + j < tr_end ? tr + j : tr;  // pad with a repeat (result ignored)
        n[j] = s_roots[t] - chunk_first_node;
    }
    for (int d = 0; d <= depth; ++d) {
#pragma unroll
        for (int j = 0; j < K3_CHAINS; ++j) nd[j] = s_nodes[n[j]];
#pragma unroll
        for (int j = 0; j < K3_CHAINS; ++j) {
            const float xv = x[(nd[j].y & 0xFFu) * TPB];
            const float thr = __uint_as_float(nd[j].x);
            const bool left = (CMP == CMP_LE) ? (xv <= thr) : (xv < thr);  // false on a leaf (NaN)
            n[j] = left ? n[j] + 1 : (nd[j].y >> 8) - chunk_first_node;
        }
    }
#pragma unroll
    for (int j = 0; j < K3_CHAINS; ++j) leaf[j] = (int)(nd[j].x & 0x3FFFFFu);
}

// K3_WALK_CAT: one node's decision (xgboost's GetNextNode / common::Decision, plan.h NODE_*).  NaN takes the default
// child; a categorical node sends a category in its set right and everything else left (not in the set, past the
// bitset, x < 0 or x >= 2^24); a numeric node goes left when x < threshold.  `word` is the threshold bits or the
// node's UGVC_CAT_REF; s_cat the category bitset words in shared memory.
__device__ __forceinline__ bool k3_cat_left(float xv, uint32_t word, uint32_t flags, const uint32_t* __restrict__ s_cat) {
    const bool cat = (flags & NODE_CATEGORICAL) != 0;
    const bool valid = xv >= 0.0f && xv < 16777216.0f;  // false for NaN too
    const unsigned c = valid ? (unsigned)xv : 0u;         // truncation, as xgboost's AsCat
    const bool in_bits = cat && valid && c < UGVC_CAT_WORDS(word) * 32u;
    const bool in_set = in_bits && ((s_cat[UGVC_CAT_FIRST(word) + (c >> 5)] >> (c & 31u)) & 1u) != 0u;
    const bool by_value = cat ? !in_set : xv < __uint_as_float(word);
    return isnan(xv) ? (flags & NODE_DEFAULT_LEFT) != 0 : by_value;
}

// walk8 for K3_WALK_CAT plans (xgboost, so x < threshold): y = feature | flags << 8 | right << 10
template <int TPB>
__device__ __forceinline__ void walk8c(const uint2* __restrict__ s_nodes, const uint32_t* __restrict__ s_roots,
                                       const uint32_t* __restrict__ s_cat, unsigned chunk_first_node, unsigned tr,
                                       unsigned tr_end, int depth, const float* __restrict__ x, int leaf[K3_CHAINS]) {
    unsigned n[K3_CHAINS];
    uint2 nd[K3_CHAINS];
#pragma unroll
    for (int j = 0; j < K3_CHAINS; ++j) {
        const unsigned t = tr + j < tr_end ? tr + j : tr;  // pad with a repeat (result ignored)
        n[j] = s_roots[t] - chunk_first_node;
    }
    for (int d = 0; d <= depth; ++d) {
#pragma unroll
        for (int j = 0; j < K3_CHAINS; ++j) nd[j] = s_nodes[n[j]];
#pragma unroll
        for (int j = 0; j < K3_CHAINS; ++j) {
            const float xv = x[(nd[j].y & 0xFFu) * TPB];
            const bool left = k3_cat_left(xv, nd[j].x, (nd[j].y >> 8) & 3u, s_cat);  // false on a leaf (NaN, no flags)
            n[j] = left ? n[j] + 1 : (nd[j].y >> 10) - chunk_first_node;
        }
    }
#pragma unroll
    for (int j = 0; j < K3_CHAINS; ++j) leaf[j] = (int)(nd[j].x & 0x3FFFFFu);
}

#ifndef UGVC_HOST_EMU
// test hook: the xgboost-flavoured fp32 sigmoid exactly as k3_finish evaluates it, on an array of margins
__global__ void k3_test_sigmoid(const float* __restrict__ m, int n, float* __restrict__ p1, float* __restrict__ e_out) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float e = k3_expf_cr(-m[i]);
        e_out[i] = e;
        p1[i] = 1.0f / (1.0f + e);
    }
}
void launch_test_sigmoid(const float* d_m, int n, float* d_p1, float* d_e, cudaStream_t st) {
    k3_test_sigmoid<<<(n + 255) / 256, 256, 0, st>>>(d_m, n, d_p1, d_e);
}
#endif

// Link function, fp64 phred / qual arithmetic and the FILTER decision of one record (shared by the two K3
// kernels): z / zf are the accumulated raw scores (fp64 for sklearn, fp32 for xgboost), x the record's
// column of the shared-memory feature tile (stride TPB).  Returns quals <= threshold.
template <int TPB>
__device__ __forceinline__ bool k3_finish(const DevPlan& plan, const float* __restrict__ x, double z[UGVC_MAX_CLASSES],
                                          float zf[UGVC_MAX_CLASSES], long long rec, double threshold,
                                          uint8_t* __restrict__ low_score, float* __restrict__ probs,
                                          double* __restrict__ qual_out, double* __restrict__ phred_out, int phred_mode) {
    const int F = plan.h.n_features, K = plan.h.n_classes, O = plan.h.n_outputs;
    const unsigned n_trees = plan.h.n_trees;
    double p[UGVC_MAX_CLASSES] = {0.0, 0.0, 0.0, 0.0};
    switch (plan.h.model_kind) {
        case MODEL_LOGISTIC: {
            // sklearn LogisticRegression: fp64 decision, expit / softmax
#pragma unroll
            for (int o = 0; o < UGVC_MAX_CLASSES; ++o) {
                if (o < O) {
                    double acc = 0.0;
                    const double* w = plan.coef + (size_t)o * F;
                    for (int f = 0; f < F; ++f) acc = fma((double)x[f * TPB], __ldg(&w[f]), acc);
                    z[o] = acc + plan.intercept[o];
                }
            }
        }
        // fall through: same link as the fp64 boosting model
        case MODEL_GB_SKLEARN: {
            if (O == 1) {
                p[1] = expit64(z[0]);
                p[0] = 1.0 - p[1];
            } else if (plan.h.model_kind == MODEL_LOGISTIC) {
                double mx = z[0];
#pragma unroll
                for (int o = 1; o < UGVC_MAX_CLASSES; ++o)
                    if (o < O) mx = fmax(mx, z[o]);
                double s = 0.0;
#pragma unroll
                for (int o = 0; o < UGVC_MAX_CLASSES; ++o)
                    if (o < O) {
                        p[o] = exp(z[o] - mx);
                        s += p[o];
                    }
#pragma unroll
                for (int o = 0; o < UGVC_MAX_CLASSES; ++o)
                    if (o < O) p[o] /= s;
            } else {
                // sklearn multiclass boosting: exp(raw - logsumexp(raw))
                double mx = z[0];
#pragma unroll
                for (int o = 1; o < UGVC_MAX_CLASSES; ++o)
                    if (o < O) mx = fmax(mx, z[o]);
                double s = 0.0;
#pragma unroll
                for (int o = 0; o < UGVC_MAX_CLASSES; ++o)
                    if (o < O) s += exp(z[o] - mx);
                const double lse = mx + log(s);
#pragma unroll
                for (int o = 0; o < UGVC_MAX_CLASSES; ++o)
                    if (o < O) p[o] = exp(z[o] - lse);
            }
            break;
        }
        case MODEL_RF_SKLEARN: {
#pragma unroll
            for (int k = 0; k < UGVC_MAX_CLASSES; ++k)
                if (k < K) p[k] = z[k] / (double)n_trees;
            break;
        }
        case MODEL_XGB: {
            // xgboost CPU predictor: fp32 margins, fp32 sigmoid / softmax
            if (O == 1) {
                const float p1 = 1.0f / (1.0f + k3_expf_cr(-zf[0]));
                p[1] = (double)p1;
                p[0] = (double)(1.0f - p1);
            } else {
                float mx = zf[0];
#pragma unroll
                for (int o = 1; o < UGVC_MAX_CLASSES; ++o)
                    if (o < O) mx = fmaxf(mx, zf[o]);
                double s = 0.0;
                float e[UGVC_MAX_CLASSES] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int o = 0; o < UGVC_MAX_CLASSES; ++o)
                    if (o < O) {
                        e[o] = k3_expf_cr(zf[o] - mx);
                        s += (double)e[o];
                    }
#pragma unroll
                for (int o = 0; o < UGVC_MAX_CLASSES; ++o)
                    if (o < O) p[o] = (double)(e[o] / (float)s);
            }
            break;
        }
        default:
            break;
    }
    // phred = -10 log10(lik + 1e-10); qual = clip(30 + ph[0] - min(ph[1:]), 0, inf)   (fp64)
    double ph[UGVC_MAX_CLASSES];
#pragma unroll
    for (int k = 0; k < UGVC_MAX_CLASSES; ++k) ph[k] = k < K ? -10.0 * log10(p[k] + 1e-10) : 0.0;
    const double ph0 = ph[0];
    double mn = ph[1];
#pragma unroll
    for (int k = 2; k < UGVC_MAX_CLASSES; ++k)
        if (k < K) mn = fmin(mn, ph[k]);
    if (phred_out) {  // --recalibrate_genotype: PL / GQ come from the per-class phreds;
                      // mode 2 (--treat_multiallelics): the fp64 likelihoods, merged on the host
#pragma unroll
        for (int k = 0; k < UGVC_MAX_CLASSES; ++k)
            if (k < K) phred_out[(size_t)rec * K + k] = phred_mode == 2 ? p[k] : ph[k];
    }
    double q = __dadd_rn(__dadd_rn(30.0, ph0), -mn);
    q = q < 0.0 ? 0.0 : q;
    const bool low = q <= threshold;
    low_score[rec] = low ? 1 : 0;
    qual_out[rec] = q;
    if (K == 2) {
        *reinterpret_cast<float2*>(&probs[(size_t)rec * 2]) = make_float2((float)p[0], (float)p[1]);
    } else {
#pragma unroll
        for (int k = 0; k < UGVC_MAX_CLASSES; ++k)
            if (k < K) probs[(size_t)rec * K + k] = (float)p[k];
    }
    return low;
}

// WALK: K3_WALK_* (one kernel per walk, chosen at plan load from plan.walk; the plain walk unless one is named)
template <int TPB, int WALK = K3_WALK_PLAIN>
__global__ void __launch_bounds__(TPB, 1)
k3_infer(const __grid_constant__ DevPlan plan, const float* __restrict__ feats, size_t row_stride,
         const int64_t* __restrict__ n_records_p, double threshold, uint8_t* __restrict__ low_score,
         float* __restrict__ probs, double* __restrict__ qual_out, double* __restrict__ phred_out, long long* counts,
         unsigned chunk_nodes_cap, int phred_mode) {
    extern __shared__ __align__(16) uint8_t smem3[];
    const int F = plan.h.n_features, K = plan.h.n_classes, O = plan.h.n_outputs;
    const unsigned n_trees = plan.h.n_trees;
    const bool forest = plan.h.model_kind != MODEL_LOGISTIC;
    float* tile = reinterpret_cast<float*>(smem3);  // [F][TPB]
    uint2* s_nodes = reinterpret_cast<uint2*>(smem3 + (size_t)F * TPB * sizeof(float));
    uint32_t* s_roots = reinterpret_cast<uint32_t*>(s_nodes + chunk_nodes_cap);  // [n_trees + 1]
    uint32_t* s_cat = s_roots + n_trees + 2;                                      // [n_cat_words], always resident
    const bool resident = forest && plan.h.n_nodes <= chunk_nodes_cap;  // whole forest fits: stage once
    if (forest) {
        for (unsigned i = threadIdx.x; i <= n_trees; i += TPB) s_roots[i] = plan.tree_root[i];
        if (WALK == K3_WALK_CAT) {
            const uint32_t* cat = reinterpret_cast<const uint32_t*>(plan.dev_nodes + plan.h.n_nodes);
            for (unsigned i = threadIdx.x; i < plan.n_cat_words; i += TPB) s_cat[i] = cat[i];
        }
        if (resident)
            for (unsigned i = threadIdx.x; i < plan.h.n_nodes; i += TPB) s_nodes[i] = plan.dev_nodes[i];
    }
    const int depth = (int)plan.max_depth;
    const long long n_rec = *n_records_p;
    const long long n_tiles = (n_rec + TPB - 1) / TPB;
    unsigned n_low = 0, n_seen = 0;
    for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const long long rec = t * TPB + threadIdx.x;
        const bool active = rec < n_rec;
        __syncthreads();
        {
            const float* src = feats + rec;
#pragma unroll 8
            for (int f = 0; f < F; ++f) tile[f * TPB + threadIdx.x] = active ? __ldg(src + (size_t)f * row_stride) : 0.f;
        }
        __syncthreads();
        const float* x = tile + threadIdx.x;
        double z[UGVC_MAX_CLASSES];   // fp64 accumulators (sklearn) ...
        float zf[UGVC_MAX_CLASSES];   // ... fp32 accumulators (xgboost)
#pragma unroll
        for (int o = 0; o < UGVC_MAX_CLASSES; ++o) {
            z[o] = plan.h.model_kind == MODEL_RF_SKLEARN ? 0.0 : plan.h.init[o];
            zf[o] = (float)plan.h.init[o];
        }
        if (forest) {
            // tree chunks: [c0, c1) are whole trees whose nodes fit the shared-memory buffer
            unsigned c0 = 0;
            while (c0 < n_trees) {
                unsigned c1 = n_trees;
                unsigned first_node = 0;
                if (!resident) {
                    first_node = s_roots[c0];
                    c1 = c0;
                    while (c1 < n_trees && s_roots[c1 + 1] - first_node <= chunk_nodes_cap) ++c1;
                    if (c1 == c0) c1 = c0 + 1;  // cannot happen: load_plan checks every tree fits
                    __syncthreads();
                    const unsigned cnt = s_roots[c1] - first_node;
                    for (unsigned i = threadIdx.x; i < cnt; i += TPB) s_nodes[i] = plan.dev_nodes[first_node + i];
                    __syncthreads();
                }
                for (unsigned tr = c0; tr < c1; tr += K3_CHAINS) {
                    int leaf[K3_CHAINS];
                    if (WALK == K3_WALK_CAT) walk8c<TPB>(s_nodes, s_roots, s_cat, first_node, tr, c1, depth, x, leaf);
                    else if (plan.h.cmp_mode == CMP_LE) walk8<CMP_LE, TPB>(s_nodes, s_roots, first_node, tr, c1, depth, x, leaf);
                    else walk8<CMP_LT, TPB>(s_nodes, s_roots, first_node, tr, c1, depth, x, leaf);
                    if (plan.h.model_kind == MODEL_GB_SKLEARN && O == 1) {
                        // raw += learning_rate * leaf (pre-scaled on the host), fp64, tree order
#pragma unroll
                        for (int j = 0; j < K3_CHAINS; ++j)
                            if (tr + j < c1) z[0] = __dadd_rn(z[0], __ldg(&plan.leaves[leaf[j]]));
                    } else if (plan.h.model_kind == MODEL_RF_SKLEARN) {
                        // sum of per-leaf class fractions, fp64, tree order
#pragma unroll
                        for (int j = 0; j < K3_CHAINS; ++j)
                            if (tr + j < c1) {
                                const double* lv = plan.leaves + (size_t)leaf[j] * plan.h.leaf_width;
#pragma unroll
                                for (int k = 0; k < UGVC_MAX_CLASSES; ++k)
                                    if (k < K) z[k] = __dadd_rn(z[k], __ldg(&lv[k]));
                            }
                    } else {
#pragma unroll
                        for (int j = 0; j < K3_CHAINS; ++j)
                            if (tr + j < c1) {
                                const int o = plan.tree_out[tr + j];
                                const double add = __ldg(&plan.leaves[leaf[j]]);
                                const float addf = (float)add;
#pragma unroll
                                for (int k = 0; k < UGVC_MAX_CLASSES; ++k) {
                                    z[k] = o == k ? __dadd_rn(z[k], add) : z[k];
                                    zf[k] = o == k ? __fadd_rn(zf[k], addf) : zf[k];
                                }
                            }
                    }
                }
                c0 = c1;
            }
        }
        if (!active) continue;
        const bool low = k3_finish<TPB>(plan, x, z, zf, rec, threshold, low_score, probs, qual_out, phred_out, phred_mode);
        n_low += low ? 1u : 0u;
        n_seen += 1u;
    }
    // pass / fail counters: warp shuffle reduction, one atomic per warp
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        n_low += __shfl_xor_sync(0xffffffffu, n_low, s);
        n_seen += __shfl_xor_sync(0xffffffffu, n_seen, s);
    }
    if ((threadIdx.x & 31) == 0 && n_seen) {
        atomicAdd((unsigned long long*)&counts[0], (unsigned long long)n_seen);
        atomicAdd((unsigned long long*)&counts[1], (unsigned long long)n_low);
        atomicAdd((unsigned long long*)&counts[2], (unsigned long long)(n_seen - n_low));
    }
}

#define K3_SMEM_BUDGET (224u * 1024u)

// ------------------------------------------------------------------------------------------
// K2 + K3 fused, heap forest
// ------------------------------------------------------------------------------------------
// K3 was bound by shared-memory wavefronts: 8-byte preorder nodes gathered by 32 lanes cost 4-5 wavefronts per
// level.  Here every tree is a complete binary tree in breadth-first order, thresholds / features / leaf rows
// in separate arrays: the 2^d nodes of level d are 2^d consecutive 4-byte words (d <= 5: distinct banks, equal
// addresses broadcast), so a level costs three conflict-free wavefronts (feature byte, threshold, x).  The
// feature tile is assembled straight from K1's raw slots with the fitted transformer's missing / absent
// policies (what k2_features did in a pass of its own), or copied from a dense matrix (ugvc_predict_features).

// NCH trees at once from the heap form in shared memory: node = (threshold bits, byte offset of the feature's row in
// the thread's tile column).  All indices are kept as byte offsets so that a level costs six instructions per chain:
// node load, address add, x load, compare, select, shift-add.
template <int CMP, int NCH>
__device__ __forceinline__ void walkh(const uint8_t* __restrict__ s_node, const uint16_t* __restrict__ s_leaf, unsigned H,
                                      int depth, unsigned tr, unsigned tr_end, const uint8_t* __restrict__ xcol,
                                      int leaf[NCH]) {
    unsigned a8[NCH];
    int go_l[NCH];  // what turns 2 * a8 into the left child's offset (the right one is 8 more)
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
        const unsigned t = tr + j < tr_end ? tr + j : tr;  // pad with a repeat (result ignored)
        const unsigned tb8 = t * H * 8u;
        a8[j] = tb8 + 8u;  // the root: node 1 of the tree
        go_l[j] = -(int)tb8;
    }
    for (int d = 0; d < depth; ++d) {
        uint2 nd[NCH];
#pragma unroll
        for (int j = 0; j < NCH; ++j) nd[j] = *reinterpret_cast<const uint2*>(s_node + a8[j]);
#pragma unroll
        for (int j = 0; j < NCH; ++j) {
            const float xv = *reinterpret_cast<const float*>(xcol + nd[j].y);
            const float th = __uint_as_float(nd[j].x);
            const bool left = (CMP == CMP_LE) ? (xv <= th) : (xv < th);
            const unsigned l8 = 2u * a8[j] + (unsigned)go_l[j];  // off the critical path: ready before the compare
            a8[j] = left ? l8 : l8 + 8u;
        }
    }
#pragma unroll
    for (int j = 0; j < NCH; ++j) leaf[j] = (int)s_leaf[(a8[j] >> 3) - H];
}

// walkh for K3_WALK_CAT plans: node = (threshold bits or UGVC_CAT_REF, byte offset of the feature | NODE_* flags << 30)
template <int NCH>
__device__ __forceinline__ void walkhc(const uint8_t* __restrict__ s_node, const uint16_t* __restrict__ s_leaf,
                                       const uint32_t* __restrict__ s_cat, unsigned H, int depth, unsigned tr,
                                       unsigned tr_end, const uint8_t* __restrict__ xcol, int leaf[NCH]) {
    unsigned a8[NCH];
    int go_l[NCH];
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
        const unsigned t = tr + j < tr_end ? tr + j : tr;  // pad with a repeat (result ignored)
        const unsigned tb8 = t * H * 8u;
        a8[j] = tb8 + 8u;
        go_l[j] = -(int)tb8;
    }
    for (int d = 0; d < depth; ++d) {
        uint2 nd[NCH];
#pragma unroll
        for (int j = 0; j < NCH; ++j) nd[j] = *reinterpret_cast<const uint2*>(s_node + a8[j]);
#pragma unroll
        for (int j = 0; j < NCH; ++j) {
            const float xv = *reinterpret_cast<const float*>(xcol + (nd[j].y & 0x3FFFFFFFu));
            const bool left = k3_cat_left(xv, nd[j].x, nd[j].y >> 30, s_cat);
            const unsigned l8 = 2u * a8[j] + (unsigned)go_l[j];
            a8[j] = left ? l8 : l8 + 8u;
        }
    }
#pragma unroll
    for (int j = 0; j < NCH; ++j) leaf[j] = (int)s_leaf[(a8[j] >> 3) - H];
}

// The leaf rows of trees [tr, min(tr + NCH, c1)) into the accumulators, in tree order (the sums both k3_heap forms
// share).  Binary sklearn boosting keeps the leaf values of a group pending (fetched from global memory, L1) while the
// next group is walked, and adds them before it: k3_add_pending adds what is left after the last group.
template <int NCH>
__device__ __forceinline__ void k3_add_pending(double z[UGVC_MAX_CLASSES], const double pend[NCH], unsigned n_pend) {
#pragma unroll
    for (int j = 0; j < NCH; ++j)
        if ((unsigned)j < n_pend) z[0] = __dadd_rn(z[0], pend[j]);
}
template <int NCH>
__device__ __forceinline__ void k3_add_leaves(const DevPlan& plan, unsigned tr, unsigned c1, const int leaf[NCH],
                                              double z[UGVC_MAX_CLASSES], float zf[UGVC_MAX_CLASSES], double pend[NCH],
                                              unsigned& n_pend) {
    const int K = plan.h.n_classes, O = plan.h.n_outputs;
    if (plan.h.model_kind == MODEL_GB_SKLEARN && O == 1) {
        // raw += learning_rate * leaf (pre-scaled on the host), fp64, tree order
        k3_add_pending<NCH>(z, pend, n_pend);
        n_pend = c1 - tr < (unsigned)NCH ? c1 - tr : (unsigned)NCH;
#pragma unroll
        for (int j = 0; j < NCH; ++j) pend[j] = __ldg(&plan.leaves[leaf[j]]);
    } else if (plan.h.model_kind == MODEL_RF_SKLEARN) {
#pragma unroll
        for (int j = 0; j < NCH; ++j)
            if (tr + j < c1) {
                const double* lv = plan.leaves + (size_t)leaf[j] * plan.h.leaf_width;
#pragma unroll
                for (int k = 0; k < UGVC_MAX_CLASSES; ++k)
                    if (k < K) z[k] = __dadd_rn(z[k], __ldg(&lv[k]));
            }
    } else {
#pragma unroll
        for (int j = 0; j < NCH; ++j)
            if (tr + j < c1) {
                const int o = plan.tree_out[tr + j];
                const double add = __ldg(&plan.leaves[leaf[j]]);
                const float addf = (float)add;
#pragma unroll
                for (int k = 0; k < UGVC_MAX_CLASSES; ++k) {
                    z[k] = o == k ? __dadd_rn(z[k], add) : z[k];
                    zf[k] = o == k ? __fadd_rn(zf[k], addf) : zf[k];
                }
            }
    }
}

// NBUF = 2: the raw rows of the NEXT record tile are fetched by 1-D bulk copies (cp.async.bulk, one per feature row,
// completion on an mbarrier) while the current tile is walked, so no warp ever waits on HBM; every thread then turns
// its own column of the landed slot words into feature values in place (K2's policies) -- a thread only ever reads
// its own column, so the tile needs no barrier between assembly and walk.
// WALK: K3_WALK_* (one kernel per walk, chosen at plan load from plan.walk; the plain walk unless one is named)
template <int TPB, int NBUF, int NCH, int GROUPS, int WALK = K3_WALK_PLAIN>
__global__ void __launch_bounds__(TPB, 1)
k3_heap(const __grid_constant__ DevPlan plan, const uint32_t* __restrict__ raw, const float* __restrict__ feats,
        size_t row_stride, const int64_t* __restrict__ n_records_p, double threshold, uint8_t* __restrict__ low_score,
        float* __restrict__ probs, double* __restrict__ qual_out, double* __restrict__ phred_out, long long* counts,
        unsigned chunk_trees, int phred_mode, unsigned long long* err, unsigned*) {
    extern __shared__ __align__(16) uint8_t smem3[];
    const int F = plan.h.n_features;
    const unsigned n_trees = plan.h.n_trees;
    const bool forest = plan.h.model_kind != MODEL_LOGISTIC;
    const int depth = (int)plan.heap_depth;
    const unsigned H = 1u << depth;
    // GROUPS = 2: the CTA is two independent halves (own tile, own mbarrier, named barrier): while one half waits for
    // its next tile the other one walks -- the forest in shared memory is paid for once
    constexpr int GS = TPB / GROUPS;                        // threads = records of one group's tile
    const int gid = GROUPS == 1 ? 0 : (int)threadIdx.x / GS, gtid = GROUPS == 1 ? (int)threadIdx.x : (int)threadIdx.x % GS;
    float* tile0 = reinterpret_cast<float*>(smem3) + (size_t)gid * NBUF * F * GS;  // this group's [NBUF][F][GS]
    uint2* s_node = reinterpret_cast<uint2*>(reinterpret_cast<float*>(smem3) + (size_t)GROUPS * NBUF * F * GS);  // [chunk_trees][H]
    PlanFeature* s_pf = reinterpret_cast<PlanFeature*>(s_node + (forest ? (size_t)chunk_trees * H : 0));  // [F]
    uint16_t* s_leaf = reinterpret_cast<uint16_t*>(s_pf + F);                                              // [chunk_trees][H]
    uint32_t* s_cat = reinterpret_cast<uint32_t*>(s_leaf + (size_t)chunk_trees * H);                        // [n_cat_words]
    const bool resident = forest && n_trees <= chunk_trees;  // whole forest fits: stage once
    for (int i = threadIdx.x; i < F; i += TPB) s_pf[i] = plan.feats[i];
    if (WALK == K3_WALK_CAT) {
        const uint32_t* cat = reinterpret_cast<const uint32_t*>(plan.dev_nodes + plan.h.n_nodes);
        for (unsigned i = threadIdx.x; i < plan.n_cat_words; i += TPB) s_cat[i] = cat[i];
    }
    // K3_WALK_CAT: the node flags follow the features in heap_feat
    const uint8_t* heap_flags = plan.heap_feat + (size_t)n_trees * H;
    if (resident) {
        const unsigned cnt = n_trees * H;
        for (unsigned i = threadIdx.x; i < cnt; i += TPB) {
            const unsigned fl = WALK == K3_WALK_CAT ? (unsigned)heap_flags[i] << 30 : 0u;
            s_node[i] = make_uint2(__float_as_uint(plan.heap_thr[i]), (unsigned)plan.heap_feat[i] * (unsigned)(GS * sizeof(float)) | fl);
            s_leaf[i] = plan.heap_leaf[i];
        }
    }
    const long long n_rec = *n_records_p;
    const long long n_tiles = (n_rec + GS - 1) / GS;
    const long long tile_first = (long long)blockIdx.x * GROUPS + gid, tile_step = (long long)gridDim.x * GROUPS;
    unsigned n_low = 0, n_seen = 0;
#ifndef UGVC_HOST_EMU
    __shared__ __align__(8) unsigned long long k3_mbar_all[4];
    unsigned long long* k3_mbar = k3_mbar_all + 2 * gid;
    if (threadIdx.x == 0) {
        for (int b = 0; b < 2 * GROUPS; ++b) {
            const uint32_t mb = (uint32_t)__cvta_generic_to_shared(&k3_mbar_all[b]);
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mb));
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    // rows [t * TPB, ...) of every feature's slot -> tile buffer b (thread 0)
    auto fetch = [&](long long t, int b) {
        const size_t rec0 = (size_t)t * GS;
        const size_t rows = row_stride - rec0 < (size_t)GS ? row_stride - rec0 : (size_t)GS;  // rows are padded to 128 records
        const uint32_t row_bytes = (uint32_t)rows * 4u;
        const uint32_t mb = (uint32_t)__cvta_generic_to_shared(&k3_mbar[b]);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mb), "r"(row_bytes * (uint32_t)F) : "memory");
        for (int f = 0; f < F; ++f) {
            const void* src = raw ? static_cast<const void*>(raw + (size_t)s_pf[f].slot * row_stride + rec0)
                                  : static_cast<const void*>(feats + (size_t)f * row_stride + rec0);
            const uint32_t dst = (uint32_t)__cvta_generic_to_shared(tile0 + ((size_t)b * F + f) * GS);
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(dst), "l"(src), "r"(row_bytes), "r"(mb)
                         : "memory");
        }
    };
    uint32_t phase0 = 0u, phase1 = 0u;
    if (gtid == 0 && tile_first < n_tiles) fetch(tile_first, 0);
#endif
    int buf = 0;
    auto group_sync = [&]() {
#ifndef UGVC_HOST_EMU
        if (GROUPS == 1) __syncthreads();
        else asm volatile("bar.sync %0, %1;" ::"r"(gid + 1), "r"(GS) : "memory");
#endif
    };
    for (long long t = tile_first; t < n_tiles; t += tile_step) {
        const long long rec = t * GS + gtid;
        const bool active = rec < n_rec;
        float* tile = tile0 + (size_t)buf * F * GS;
#ifndef UGVC_HOST_EMU
        {
            const uint32_t mb = (uint32_t)__cvta_generic_to_shared(&k3_mbar[buf]);
            uint32_t ok = 0;
            while (!ok)
                asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                             : "=r"(ok)
                             : "r"(mb), "r"(buf ? phase1 : phase0)
                             : "memory");
            if (buf) phase1 ^= 1u;
            else phase0 ^= 1u;
            // the other buffer was released by the barrier that ended the previous tile: fetch the next tile into it
            if (NBUF == 2 && gtid == 0 && t + tile_step < n_tiles) fetch(t + tile_step, buf ^ 1);
        }
#endif
        if (raw) {
            // K2: slot -> feature with the missing / absent policies (transformers.py:221-344)
            const uint32_t* src = raw + rec;
#pragma unroll 4
            for (int f = 0; f < F; ++f) {
                const PlanFeature pf = s_pf[f];
#ifdef UGVC_HOST_EMU
                const uint32_t bits = active ? src[(size_t)pf.slot * row_stride] : 0u;
#else
                const uint32_t bits = __float_as_uint(tile[f * GS + gtid]);
#endif
                tile[f * GS + gtid] = active ? k2_apply(bits, pf, rec, f, err) : 0.f;
            }
            for (unsigned c = 0; c < plan.h.n_combines; ++c) {  // feature = max(feature, slot_b), nulls skipped
                const PlanCombine cb = plan.combines[c];
                if (active) k2_combine_one(cb, __ldg(src + (size_t)cb.slot_b * row_stride), tile[cb.feature * GS + gtid], rec, true, err);
            }
            for (unsigned c = 0; c < plan.h.n_checks; ++c) {
                const PlanCheck ck = plan.checks[c];
                if (!active) continue;
                const uint32_t bits = __ldg(src + (size_t)ck.slot * row_stride);
                if (bits == RAW_ABSENT || bits == RAW_MISSING) continue;  // handled by the feature policies
                const float v = __uint_as_float(bits);
                const bool ok = ck.kind == 0 ? (v <= ck.bound) : (v >= ck.bound);
                if (!ok) atomicMin(err, ugvc_pack_error(rec, 0xFFFF, ck.kind == 0 ? REASON_TOO_MANY_ELEMS : REASON_BAD_VALUE));
            }
        } else {
#ifdef UGVC_HOST_EMU
            const float* src = feats + rec;
            for (int f = 0; f < F; ++f) tile[f * GS + gtid] = active ? src[(size_t)f * row_stride] : 0.f;
#else
            if (!active)
                for (int f = 0; f < F; ++f) tile[f * GS + gtid] = 0.f;
#endif
        }
        const float* x = tile + gtid;
        double z[UGVC_MAX_CLASSES];   // fp64 accumulators (sklearn) ...
        float zf[UGVC_MAX_CLASSES];   // ... fp32 accumulators (xgboost)
#pragma unroll
        for (int o = 0; o < UGVC_MAX_CLASSES; ++o) {
            z[o] = plan.h.model_kind == MODEL_RF_SKLEARN ? 0.0 : plan.h.init[o];
            zf[o] = (float)plan.h.init[o];
        }
        if (forest) {
            unsigned c0 = 0;
            while (c0 < n_trees) {
                unsigned c1 = n_trees;
                if (!resident) {  // tree chunks [c0, c1) staged in turn
                    c1 = c0 + chunk_trees < n_trees ? c0 + chunk_trees : n_trees;
                    __syncthreads();
                    const unsigned cnt = (c1 - c0) * H;
                    const size_t off = (size_t)c0 * H;
                    for (unsigned i = threadIdx.x; i < cnt; i += TPB) {
                        const unsigned fl = WALK == K3_WALK_CAT ? (unsigned)heap_flags[off + i] << 30 : 0u;
                        s_node[i] = make_uint2(__float_as_uint(plan.heap_thr[off + i]),
                                               (unsigned)plan.heap_feat[off + i] * (unsigned)(GS * sizeof(float)) | fl);
                        s_leaf[i] = plan.heap_leaf[off + i];
                    }
                    __syncthreads();
                }
                // the leaf values of a group are fetched (global, L1) while the next group is walked and added after
                // it, still in tree order
                double pend[NCH];
                unsigned n_pend = 0;
                for (unsigned tr = c0; tr < c1; tr += NCH) {
                    int leaf[NCH];
                    const unsigned lt = resident ? tr : tr - c0, lt_end = resident ? c1 : c1 - c0;
                    const uint8_t* xcol = reinterpret_cast<const uint8_t*>(x);
                    if (WALK == K3_WALK_CAT) walkhc<NCH>(reinterpret_cast<const uint8_t*>(s_node), s_leaf, s_cat, H, depth, lt, lt_end, xcol, leaf);
                    else if (plan.h.cmp_mode == CMP_LE) walkh<CMP_LE, NCH>(reinterpret_cast<const uint8_t*>(s_node), s_leaf, H, depth, lt, lt_end, xcol, leaf);
                    else walkh<CMP_LT, NCH>(reinterpret_cast<const uint8_t*>(s_node), s_leaf, H, depth, lt, lt_end, xcol, leaf);
                    k3_add_leaves<NCH>(plan, tr, c1, leaf, z, zf, pend, n_pend);
                }
                k3_add_pending<NCH>(z, pend, n_pend);
                c0 = c1;
            }
        }
        if (active) {
            const bool low = k3_finish<GS>(plan, x, z, zf, rec, threshold, low_score, probs, qual_out, phred_out, phred_mode);
            n_low += low ? 1u : 0u;
            n_seen += 1u;
        }
        group_sync();  // every thread of the group is done with this tile buffer
#ifndef UGVC_HOST_EMU
        if (NBUF == 1 && gtid == 0 && t + tile_step < n_tiles) fetch(t + tile_step, 0);
#endif
        buf ^= (NBUF == 2) ? 1 : 0;
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        n_low += __shfl_xor_sync(0xffffffffu, n_low, s);
        n_seen += __shfl_xor_sync(0xffffffffu, n_seen, s);
    }
    if ((threadIdx.x & 31) == 0 && n_seen) {
        atomicAdd((unsigned long long*)&counts[0], (unsigned long long)n_seen);
        atomicAdd((unsigned long long*)&counts[1], (unsigned long long)n_low);
        atomicAdd((unsigned long long*)&counts[2], (unsigned long long)(n_seen - n_low));
    }
}

// k3_heap with two threads per record (resident forests only).  Thread A of a record walks trees [0, TA), thread B
// walks [TA, T) and leaves its leaf rows in s_hand; A then adds them after its own, so the record's sums are the same
// roundings in the same tree order as k3_heap's (z = init + l0 + ... + l(T-1)).  For the same feature tile the CTA
// runs twice the warps and twice the walk chains.  The CTA is GROUPS independent groups (own tile, own mbarrier, named
// barrier), each of RS = TPB / GROUPS / 2 records: threads [0, RS) of a group are the A threads, [RS, 2 RS) the B
// threads, so every warp reads 32 distinct tile columns.  A group claims its tiles from the launch's ticket (zeroed
// by launch_k3), so the groups that finish first take the last tiles; the first warp of a group claims, then spreads
// the tile's row copies over its lanes.  NBUF = 2: the group's next tile is claimed and in flight while it walks the
// current one.  In the host emulation (one thread, RS = 1) that thread plays B, then A, through the same code.
__host__ __device__ inline unsigned k3s_trees_a(unsigned n_trees, unsigned nch) {  // TA: half the trees, whole groups of chains
    const unsigned a = ((n_trees + 1) / 2 + nch - 1) / nch * nch;
    return a < n_trees ? a : n_trees;
}
template <int TPB, int NBUF, int NCH, int GROUPS, int WALK = K3_WALK_PLAIN>
__global__ void __launch_bounds__(TPB, 1)
k3_heap_split(const __grid_constant__ DevPlan plan, const uint32_t* __restrict__ raw, const float* __restrict__ feats,
              size_t row_stride, const int64_t* __restrict__ n_records_p, double threshold, uint8_t* __restrict__ low_score,
              float* __restrict__ probs, double* __restrict__ qual_out, double* __restrict__ phred_out, long long* counts,
              unsigned, int phred_mode, unsigned long long* err, unsigned* __restrict__ ticket) {
    // NBUF = 2 (one group of 192 records, 384 threads, the next tile in flight during the walk) measured 1.35 ms per
    // bench launch against 0.96 ms for five single-buffered groups of 64 (profiles/h100_k3_budget.json): the warps
    // the second buffer costs outweigh the fetch it hides.  The buffer index is kept so that it can be timed again.
    static_assert(NBUF == 1 || NBUF == 2, "one or two tile buffers per group");
    extern __shared__ __align__(16) uint8_t smem3[];
    const int F = plan.h.n_features;
    const unsigned n_trees = plan.h.n_trees, ta = k3s_trees_a(n_trees, NCH), tb = n_trees - ta;
    const int depth = (int)plan.heap_depth;
    const unsigned H = 1u << depth;
    constexpr int GS = TPB / GROUPS;  // threads of one group
    constexpr int RS = GS / 2;        // records of one group's tile
    const int gid = GROUPS == 1 ? 0 : (int)threadIdx.x / GS, gtid = GROUPS == 1 ? (int)threadIdx.x : (int)threadIdx.x % GS;
    const int r = gtid % RS;
    float* tile0 = reinterpret_cast<float*>(smem3) + (size_t)gid * NBUF * F * RS;                               // [NBUF][F][RS]
    uint2* s_node = reinterpret_cast<uint2*>(reinterpret_cast<float*>(smem3) + (size_t)GROUPS * NBUF * F * RS);  // [T][H]
    PlanFeature* s_pf = reinterpret_cast<PlanFeature*>(s_node + (size_t)n_trees * H);                      // [F]
    uint16_t* s_leaf = reinterpret_cast<uint16_t*>(s_pf + F);                                              // [T][H]
    uint16_t* s_hand0 = s_leaf + (size_t)n_trees * H;                                                      // [GROUPS][tb][RS]
    uint32_t* s_cat = reinterpret_cast<uint32_t*>(s_hand0 + (size_t)GROUPS * tb * RS);                     // [n_cat_words]
    uint16_t* s_hand = s_hand0 + (size_t)gid * tb * RS;
    for (int i = threadIdx.x; i < F; i += blockDim.x) s_pf[i] = plan.feats[i];
    if (WALK == K3_WALK_CAT) {
        const uint32_t* cat = reinterpret_cast<const uint32_t*>(plan.dev_nodes + plan.h.n_nodes);
        for (unsigned i = threadIdx.x; i < plan.n_cat_words; i += blockDim.x) s_cat[i] = cat[i];
    }
    const uint8_t* heap_flags = plan.heap_feat + (size_t)n_trees * H;  // K3_WALK_CAT: the node flags follow the features
    // (stride blockDim.x: TPB threads on the device, one in the host emulation)
    for (unsigned i = threadIdx.x; i < n_trees * H; i += blockDim.x) {
        const unsigned fl = WALK == K3_WALK_CAT ? (unsigned)heap_flags[i] << 30 : 0u;
        s_node[i] = make_uint2(__float_as_uint(plan.heap_thr[i]), (unsigned)plan.heap_feat[i] * (unsigned)(RS * sizeof(float)) | fl);
        s_leaf[i] = plan.heap_leaf[i];
    }
    const long long n_rec = *n_records_p;
    const long long n_tiles = (n_rec + RS - 1) / RS;
    const int fa = (F + 1) / 2;  // K2: A assembles features [0, fa), B [fa, F)
    unsigned n_low = 0, n_seen = 0;
#ifdef UGVC_HOST_EMU
    constexpr int ROLES = 2;  // the one thread is B, then A
#else
    constexpr int ROLES = 1;
    __shared__ __align__(8) unsigned long long k3_mbar_all[GROUPS * NBUF];
    __shared__ unsigned s_tile_all[GROUPS * NBUF];  // the tile claimed into each buffer
    unsigned long long* k3_mbar = k3_mbar_all + gid * NBUF;
    unsigned* s_tile = s_tile_all + gid * NBUF;
    if (threadIdx.x == 0) {
        for (int b = 0; b < GROUPS * NBUF; ++b)
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"((uint32_t)__cvta_generic_to_shared(&k3_mbar_all[b])));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    // the group's first warp: claim the next tile for buffer b, then its rows [t * RS, ...) of every feature's slot ->
    // buffer b.  Past the last tile only the arrival completes the buffer's phase, and the group reads that it is done.
    auto claim_fetch = [&](int b) {
        const int lane = gtid;
        const uint32_t mb = (uint32_t)__cvta_generic_to_shared(&k3_mbar[b]);
        if (lane == 0) s_tile[b] = atomicAdd(ticket, 1u);
        __syncwarp();
        const long long t = s_tile[b];
        if (t >= n_tiles) {
            if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(mb) : "memory");
            return;
        }
        float* tile = tile0 + (size_t)b * F * RS;
        const size_t rec0 = (size_t)t * RS;
        const size_t rows = row_stride - rec0 < (size_t)RS ? row_stride - rec0 : (size_t)RS;  // rows are padded to 128 records
        const uint32_t row_bytes = (uint32_t)rows * 4u;
        if (lane == 0)
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mb), "r"(row_bytes * (uint32_t)F) : "memory");
        __syncwarp();
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        for (int f = lane; f < F; f += 32) {
            const void* src = raw ? static_cast<const void*>(raw + (size_t)s_pf[f].slot * row_stride + rec0)
                                  : static_cast<const void*>(feats + (size_t)f * row_stride + rec0);
            const uint32_t dst = (uint32_t)__cvta_generic_to_shared(tile + (size_t)f * RS);
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(dst), "l"(src), "r"(row_bytes), "r"(mb)
                         : "memory");
        }
    };
    uint32_t phases = 0u;  // bit b: the parity buffer b waits for next
    if (gtid < 32)
        for (int b = 0; b < NBUF; ++b) claim_fetch(b);
#endif
    auto group_sync = [&]() {
#ifndef UGVC_HOST_EMU
        if (GROUPS == 1) __syncthreads();
        else asm volatile("bar.sync %0, %1;" ::"r"(gid + 1), "r"(GS) : "memory");
#endif
    };
    for (int buf = 0;; buf = NBUF == 2 ? buf ^ 1 : 0) {
#ifdef UGVC_HOST_EMU
        const long long t = atomicAdd(ticket, 1u);
#else
        {
            const uint32_t mb = (uint32_t)__cvta_generic_to_shared(&k3_mbar[buf]);
            uint32_t ok = 0;
            while (!ok)
                asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                             : "=r"(ok)
                             : "r"(mb), "r"((phases >> buf) & 1u)
                             : "memory");
            phases ^= 1u << buf;
        }
        const long long t = s_tile[buf];
#endif
        if (t >= n_tiles) break;
        float* tile = tile0 + (size_t)buf * F * RS;
        const long long rec = t * RS + r;
        const bool active = rec < n_rec;
        // K2 (transformers.py:221-344): each thread of the pair assembles its half of the record's features; a combine
        // runs in the thread that assembled its feature, after it
        for (int role = 0; role < ROLES; ++role) {
            const int half = ROLES == 2 ? 1 - role : gtid / RS;
            const int f0 = half ? fa : 0, f1 = half ? F : fa;
            if (raw) {
                const uint32_t* src = raw + rec;
#pragma unroll 2
                for (int f = f0; f < f1; ++f) {
                    const PlanFeature pf = s_pf[f];
#ifdef UGVC_HOST_EMU
                    const uint32_t bits = active ? src[(size_t)pf.slot * row_stride] : 0u;
#else
                    const uint32_t bits = __float_as_uint(tile[f * RS + r]);
#endif
                    tile[f * RS + r] = active ? k2_apply(bits, pf, rec, f, err) : 0.f;
                }
                for (unsigned c = 0; c < plan.h.n_combines; ++c) {  // feature = max(feature, slot_b), nulls skipped
                    const PlanCombine cb = plan.combines[c];
                    if (active && (int)cb.feature >= f0 && (int)cb.feature < f1)
                        k2_combine_one(cb, __ldg(src + (size_t)cb.slot_b * row_stride), tile[cb.feature * RS + r], rec, true, err);
                }
                for (unsigned c = 0; c < plan.h.n_checks && half == 0; ++c) {
                    const PlanCheck ck = plan.checks[c];
                    if (!active) continue;
                    const uint32_t bits = __ldg(src + (size_t)ck.slot * row_stride);
                    if (bits == RAW_ABSENT || bits == RAW_MISSING) continue;  // handled by the feature policies
                    const float v = __uint_as_float(bits);
                    const bool ok = ck.kind == 0 ? (v <= ck.bound) : (v >= ck.bound);
                    if (!ok) atomicMin(err, ugvc_pack_error(rec, 0xFFFF, ck.kind == 0 ? REASON_TOO_MANY_ELEMS : REASON_BAD_VALUE));
                }
            } else {
#ifdef UGVC_HOST_EMU
                const float* src = feats + rec;
                for (int f = f0; f < f1; ++f) tile[f * RS + r] = active ? src[(size_t)f * row_stride] : 0.f;
#else
                if (!active)
                    for (int f = f0; f < f1; ++f) tile[f * RS + r] = 0.f;
#endif
            }
        }
        group_sync();  // the pair's features are in the tile
        const uint8_t* xcol = reinterpret_cast<const uint8_t*>(tile + r);
        const uint8_t* nodes = reinterpret_cast<const uint8_t*>(s_node);
        double z[UGVC_MAX_CLASSES];   // fp64 accumulators (sklearn) ...
        float zf[UGVC_MAX_CLASSES];   // ... fp32 accumulators (xgboost), A's only
        double pend[NCH];
        unsigned n_pend = 0;
        for (int role = 0; role < ROLES; ++role) {
            const int half = ROLES == 2 ? 1 - role : gtid / RS;
            if (half == 0) {
#pragma unroll
                for (int o = 0; o < UGVC_MAX_CLASSES; ++o) {
                    z[o] = plan.h.model_kind == MODEL_RF_SKLEARN ? 0.0 : plan.h.init[o];
                    zf[o] = (float)plan.h.init[o];
                }
            }
            const unsigned t0 = half ? ta : 0, t1 = half ? n_trees : ta;
            for (unsigned tr = t0; tr < t1; tr += NCH) {
                int leaf[NCH];
                if (WALK == K3_WALK_CAT) walkhc<NCH>(nodes, s_leaf, s_cat, H, depth, tr, t1, xcol, leaf);
                else if (plan.h.cmp_mode == CMP_LE) walkh<CMP_LE, NCH>(nodes, s_leaf, H, depth, tr, t1, xcol, leaf);
                else walkh<CMP_LT, NCH>(nodes, s_leaf, H, depth, tr, t1, xcol, leaf);
                if (half) {  // B: hand the leaf rows over, one row of s_hand per tree
#pragma unroll
                    for (int j = 0; j < NCH; ++j)
                        if (tr + j < t1) s_hand[(size_t)(tr - ta + j) * RS + r] = (uint16_t)leaf[j];
                } else {
                    k3_add_leaves<NCH>(plan, tr, t1, leaf, z, zf, pend, n_pend);
                }
            }
        }
        group_sync();  // B's leaf rows are in s_hand, and the walks are done with the tile
#ifndef UGVC_HOST_EMU
        // k3_finish reads the tile only for a linear model: this buffer takes a new tile while A finishes this one.  B
        // writes s_hand again only after the next tile's first barrier, which A reaches after reading it.
        if (gtid < 32) claim_fetch(buf);
#endif
        if (ROLES == 2 || gtid < RS) {
            // A: B's trees, in tree order after its own
            for (unsigned tr = ta; tr < n_trees; tr += NCH) {
                int leaf[NCH];
#pragma unroll
                for (int j = 0; j < NCH; ++j) leaf[j] = tr + j < n_trees ? (int)s_hand[(size_t)(tr - ta + j) * RS + r] : 0;
                k3_add_leaves<NCH>(plan, tr, n_trees, leaf, z, zf, pend, n_pend);
            }
            k3_add_pending<NCH>(z, pend, n_pend);
            if (active) {
                const bool low = k3_finish<RS>(plan, reinterpret_cast<const float*>(xcol), z, zf, rec, threshold, low_score,
                                               probs, qual_out, phred_out, phred_mode);
                n_low += low ? 1u : 0u;
                n_seen += 1u;
            }
        }
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        n_low += __shfl_xor_sync(0xffffffffu, n_low, s);
        n_seen += __shfl_xor_sync(0xffffffffu, n_seen, s);
    }
    if ((threadIdx.x & 31) == 0 && n_seen) {
        atomicAdd((unsigned long long*)&counts[0], (unsigned long long)n_seen);
        atomicAdd((unsigned long long*)&counts[1], (unsigned long long)n_low);
        atomicAdd((unsigned long long*)&counts[2], (unsigned long long)(n_seen - n_low));
    }
}

// ------------------------------------------------------------------------------------------
// The K3 launch of a plan: kernel, shape, staging, grid and walk (k3_choose, once per plan)
// ------------------------------------------------------------------------------------------
// k3_heap's instantiations {tpb, nbuf, nch, groups, split}, records per tile tpb / groups / split.  Entry 9
// (k3_heap_split: five groups of 64 records, two threads per record, 20 warps) comes first for a resident forest of
// K3S_MIN_TREES trees or more, at most K3S_MAX_DEPTH deep, that it holds and entry 0 does not; five groups keep four other tiles walking while one
// waits for its rows.  Then entries 0-7 are tried in order (UGVC_K3_SHAPE picks one of 0-7 or 9): two half-CTAs with
// one tile each first (most warps for the shared memory), then double-buffered single groups.  Where there are few
// threads per SM (the tiles are large), sixteen trees per thread in flight make up for it.  Entry 8 is entry 1 walking
// twelve trees at once (UGVC_K3_NCH448=12).
struct K3hShape {
    int tpb, nbuf, nch, groups, split = 1;
};
static constexpr K3hShape K3H_SHAPES[] = {{512, 1, 8, 2},  {448, 1, 8, 2}, {384, 1, 16, 2}, {256, 2, 16, 1}, {192, 2, 16, 1},
                                          {128, 2, 16, 1}, {256, 1, 8, 1}, {128, 1, 8, 1},  {448, 1, 12, 2}, {640, 1, 8, 5, 2}};
static constexpr int K3S_SHAPE = 9;
// k3_heap_split needs trees to share: with fewer, each thread of a pair walks at most four groups of chains and the
// two extra barriers and the hand-over of every tile weigh more (UGVC_K3_SHAPE=9 runs it on any forest it holds)
static constexpr unsigned K3S_MIN_TREES = 64;
static constexpr unsigned K3S_MAX_DEPTH = 6;
// k3_infer's instantiations: records per CTA, 384 when the feature tile and the whole forest still fit, else 256
static constexpr int K3I_TPB[] = {384, 256};

// shared-memory plan of k3_heap: records per CTA, tile buffers, trees per staged chunk
static size_t k3h_tree_bytes(const DevPlan& plan) { return (size_t)(1u << plan.heap_depth) * 10u; }  // 8-byte nodes + leaf rows
static size_t k3_cat_bytes(const DevPlan& plan) { return (size_t)plan.n_cat_words * sizeof(uint32_t); }  // resident
static size_t k3h_tile_bytes(const DevPlan& plan, K3hShape c) {  // all tile buffers of the CTA + the policy table + bitsets
    return (size_t)c.nbuf * plan.h.n_features * c.tpb * sizeof(float) + (size_t)plan.h.n_features * sizeof(PlanFeature) + 64 +
           k3_cat_bytes(plan);
}
// k3_heap_split's shared memory: the groups' tiles, the policy table, bitsets, the whole forest and the hand-over rows
static size_t k3s_bytes(const DevPlan& plan, K3hShape c) {
    const size_t rs = (size_t)c.tpb / c.groups / 2, tb = plan.h.n_trees - k3s_trees_a(plan.h.n_trees, (unsigned)c.nch);
    return (size_t)c.groups * c.nbuf * plan.h.n_features * rs * sizeof(float) + (size_t)plan.h.n_features * sizeof(PlanFeature) + 64 +
           k3_cat_bytes(plan) + (size_t)plan.h.n_trees * k3h_tree_bytes(plan) + (size_t)c.groups * tb * rs * sizeof(uint16_t);
}
// the K3H_SHAPES entry of a model with a heap form, -1 if none holds it
static int k3h_shape(const DevPlan& plan) {
    static const int force = getenv("UGVC_K3_SHAPE") ? atoi(getenv("UGVC_K3_SHAPE")) : -1;  // profiling knob: 0-7 or 9
    static const int nch448 = getenv("UGVC_K3_NCH448") ? atoi(getenv("UGVC_K3_NCH448")) : 8;  // profiling knob
    const bool forest = plan.h.model_kind != MODEL_LOGISTIC;
    const size_t all = forest ? (size_t)plan.h.n_trees * k3h_tree_bytes(plan) : 0;
    // k3_heap_split where the tile leaves the one-thread form short of its widest shape (16 warps), for forests of the
    // depth it was timed at (the bench's, 6) or shallower; deeper ones keep k3_heap until a measurement says otherwise
    const bool split_pays = force < 0 && plan.h.n_trees >= K3S_MIN_TREES && plan.heap_depth <= K3S_MAX_DEPTH &&
                            k3h_tile_bytes(plan, K3H_SHAPES[0]) + all > K3_SMEM_BUDGET;
    if (forest && (force == K3S_SHAPE || split_pays) && k3s_bytes(plan, K3H_SHAPES[K3S_SHAPE]) <= K3_SMEM_BUDGET)
        return K3S_SHAPE;
    for (int i = 0; i < 8; ++i) {
        if (force >= 0 && i != force) continue;
        if (k3h_tile_bytes(plan, K3H_SHAPES[i]) + all <= K3_SMEM_BUDGET) return i == 1 && nch448 == 12 ? 8 : i;
    }
    for (int i = 3; i < 8; ++i)  // the forest is staged in chunks (single group: the chunks need whole-CTA barriers)
        if (k3h_tile_bytes(plan, K3H_SHAPES[i]) + 16 * k3h_tree_bytes(plan) <= K3_SMEM_BUDGET) return i;
    return -1;
}
static unsigned k3h_chunk_trees(const DevPlan& plan, K3hShape sh) {
    if (plan.h.model_kind == MODEL_LOGISTIC) return 0;
    const size_t room = K3_SMEM_BUDGET - k3h_tile_bytes(plan, sh);
    size_t n = room / k3h_tree_bytes(plan);
    if (n > plan.h.n_trees) n = plan.h.n_trees;
    if (n < plan.h.n_trees) n &= ~(size_t)15;  // whole groups of chains
    return (unsigned)n;
}
// k3_heap's launch for a model with a heap form; shape -1 (and nothing else set) when no shape holds the model
static K3Config k3_heap_config(const DevPlan& plan, int sm_count) {
    K3Config c{};
    c.kernel = K3_KERNEL_HEAP;
    c.shape = k3h_shape(plan);
    if (c.shape < 0) return c;
    const K3hShape sh = K3H_SHAPES[c.shape];
    c.tpb = sh.tpb;
    c.nbuf = sh.nbuf;
    c.groups = sh.groups;
    c.nch = sh.nch;
    c.split = sh.split;
    c.chunk = sh.split == 2 ? plan.h.n_trees : k3h_chunk_trees(plan, sh);
    c.resident = plan.h.model_kind == MODEL_LOGISTIC || c.chunk >= plan.h.n_trees;
    c.smem = sh.split == 2 ? k3s_bytes(plan, sh) : k3h_tile_bytes(plan, sh) + (size_t)c.chunk * k3h_tree_bytes(plan);
    int per_sm = (int)((227u * 1024u) / (c.smem + 1024));
    per_sm = per_sm < 1 ? 1 : (per_sm > 4 ? 4 : per_sm);
    if (sh.split == 2) per_sm = 1;  // __launch_bounds__(tpb, 1) registers: a second CTA would not be resident
    if (per_sm * sh.tpb > 1536) per_sm = 1536 / sh.tpb;
    c.grid = sm_count * per_sm;
    c.walk = (int)plan.walk;
    return c;
}

static size_t k3_forest_bytes(const DevPlan& plan) {
    if (plan.h.model_kind == MODEL_LOGISTIC || plan.h.model_kind == MODEL_NONE) return 0;
    return (size_t)plan.h.n_nodes * sizeof(uint2);
}
static size_t k3_roots_bytes(const DevPlan& plan) { return ((size_t)plan.h.n_trees + 2) * sizeof(uint32_t); }
// the K3I_TPB entry of a model
static int k3i_shape(const DevPlan& plan) {
    const size_t forest = k3_forest_bytes(plan);
    if (forest == 0) return 1;
    const size_t need384 = (size_t)plan.h.n_features * K3I_TPB[0] * sizeof(float) + forest + k3_roots_bytes(plan) + k3_cat_bytes(plan);
    static const int force = getenv("UGVC_K3_TPB") ? atoi(getenv("UGVC_K3_TPB")) : 0;  // profiling knob: 256, or 384 where it fits
    return force != 256 && need384 <= K3_SMEM_BUDGET ? 0 : 1;
}
static int k3_tpb(const DevPlan& plan) { return K3I_TPB[k3i_shape(plan)]; }
// nodes the shared-memory forest buffer holds (0 for linear models)
static unsigned k3_chunk_nodes(const DevPlan& plan) {
    if (k3_forest_bytes(plan) == 0) return 0;
    const size_t tile = (size_t)plan.h.n_features * k3_tpb(plan) * sizeof(float);
    const size_t roots = k3_roots_bytes(plan) + k3_cat_bytes(plan);  // the tree roots and the bitsets stay resident
    if (tile + roots + 4096 > K3_SMEM_BUDGET) return 0;
    const size_t room = (K3_SMEM_BUDGET - tile - roots) / sizeof(uint2);
    return (unsigned)(room < plan.h.n_nodes ? room : plan.h.n_nodes);
}
static size_t k3_smem_bytes(const DevPlan& plan) {
    size_t b = (size_t)plan.h.n_features * k3_tpb(plan) * sizeof(float);
    const unsigned cap = k3_chunk_nodes(plan);
    if (cap) b += (size_t)cap * sizeof(uint2) + k3_roots_bytes(plan) + k3_cat_bytes(plan);
    return b;
}
static bool k3_plan_fits(const DevPlan& plan) {
    if (k3_forest_bytes(plan) == 0) return (size_t)plan.h.n_features * 256 * sizeof(float) <= K3_SMEM_BUDGET;
    return k3_chunk_nodes(plan) > 0;
}
// most features k3_infer holds for this model: a 256-record tile, plus for a forest the tree roots, the category
// bitsets and 4 KiB of nodes
static unsigned k3_infer_max_features(const DevPlan& plan) {
    const size_t fixed = k3_forest_bytes(plan) ? k3_roots_bytes(plan) + k3_cat_bytes(plan) + 4096 : 0;
    return fixed >= K3_SMEM_BUDGET ? 0u : (unsigned)((K3_SMEM_BUDGET - fixed) / (256 * sizeof(float)));
}
static K3Config k3_infer_config(const DevPlan& plan, int sm_count) {
    K3Config c{};
    c.kernel = K3_KERNEL_INFER;
    c.shape = k3i_shape(plan);
    c.tpb = K3I_TPB[c.shape];
    c.nbuf = c.groups = c.split = 1;
    c.nch = K3_CHAINS;
    c.chunk = k3_chunk_nodes(plan);
    c.resident = k3_forest_bytes(plan) == 0 || c.chunk >= plan.h.n_nodes;
    c.smem = k3_smem_bytes(plan);
    int per_sm = (int)((K3_SMEM_BUDGET) / (c.smem + 1024));
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 4) per_sm = 4;
    c.grid = sm_count * per_sm;
    c.walk = (int)plan.walk;
    return c;
}

bool k3_choose(const DevPlan& plan, const uint32_t* tree_root, int sm_count, K3Config* out, std::string* why) {
    // UGVC_K3_LEGACY=1 (profiling): K2 + k3_infer even where k3_heap would run
    static const bool legacy = getenv("UGVC_K3_LEGACY") && *getenv("UGVC_K3_LEGACY") != '0';
    // k3_heap (K2 fused into its tile load) when the model has a heap form: it holds every plan the compiler makes (up
    // to 250 features)
    if (!legacy && (plan.h.model_kind == MODEL_LOGISTIC || plan.heap_depth != 0)) {
        const K3Config c = k3_heap_config(plan, sm_count);
        if (c.shape >= 0) {
            *out = c;
            return true;
        }
    }
    // else K2 + k3_infer, which holds fewer features
    if (!k3_plan_fits(plan)) {
        *why = std::string("plan needs more shared memory than one sm_90 CTA has: k3_infer (") +
               (legacy ? "selected by UGVC_K3_LEGACY" : "forests deeper than 8 or with 65536 leaf rows or more") +
               ") holds at most " + std::to_string(k3_infer_max_features(plan)) + " features for this model, it has " +
               std::to_string(plan.h.n_features);
        return false;
    }
    if (plan.h.model_kind != MODEL_LOGISTIC) {
        const unsigned cap = k3_chunk_nodes(plan);
        for (uint32_t t = 0; t < plan.h.n_trees; ++t)
            if (tree_root[t + 1] - tree_root[t] > cap) {
                *why = "a single tree does not fit k3_infer's shared-memory forest buffer";
                return false;
            }
    }
    *out = k3_infer_config(plan, sm_count);
    return true;
}

#ifndef UGVC_HOST_EMU
// the instantiations of one walk, in table order
template <size_t S, int WALK>
static constexpr auto k3h_kernel() {
    constexpr K3hShape sh = K3H_SHAPES[S];
    if constexpr (sh.split == 2) return &k3_heap_split<sh.tpb, sh.nbuf, sh.nch, sh.groups, WALK>;
    else return &k3_heap<sh.tpb, sh.nbuf, sh.nch, sh.groups, WALK>;
}
template <int WALK, size_t... S>
static auto k3h_kernels(std::index_sequence<S...>) {
    return std::array{k3h_kernel<S, WALK>()...};
}
template <int WALK, size_t... S>
static auto k3i_kernels(std::index_sequence<S...>) {
    return std::array{&k3_infer<K3I_TPB[S], WALK>...};
}
// [walk][K3Config::shape]
static const auto K3H_KERNELS = std::array{k3h_kernels<K3_WALK_PLAIN>(std::make_index_sequence<std::size(K3H_SHAPES)>()),
                                           k3h_kernels<K3_WALK_CAT>(std::make_index_sequence<std::size(K3H_SHAPES)>())};
static const auto K3I_KERNELS = std::array{k3i_kernels<K3_WALK_PLAIN>(std::make_index_sequence<std::size(K3I_TPB)>()),
                                           k3i_kernels<K3_WALK_CAT>(std::make_index_sequence<std::size(K3I_TPB)>())};

void launch_k3(const DevPlan& plan, const K3Config& c, const uint32_t* raw, const float* feats, size_t row_stride,
               const int64_t* d_n_records, double threshold, uint8_t* low_score, float* probs, double* qual,
               double* phreds, int phred_mode, long long* d_counts, unsigned long long* d_err, unsigned* ticket,
               cudaStream_t st) {
    if (c.kernel == K3_KERNEL_HEAP) {
        if (c.split == 2) cudaMemsetAsync(ticket, 0, sizeof(unsigned), st);
        const auto k = K3H_KERNELS[c.walk][c.shape];
        k<<<c.grid, c.tpb, c.smem, st>>>(plan, raw, feats, row_stride, d_n_records, threshold, low_score, probs, qual, phreds,
                                         d_counts, c.chunk, phred_mode, d_err, ticket);
    } else {
        const auto k = K3I_KERNELS[c.walk][c.shape];
        k<<<c.grid, c.tpb, c.smem, st>>>(plan, feats, row_stride, d_n_records, threshold, low_score, probs, qual, phreds,
                                         d_counts, c.chunk, phred_mode);
    }
}

cudaError_t kernels_configure(const DevPlan& plan) {
    cudaError_t e = cudaFuncSetAttribute(k1_parse, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)k1_smem_bytes(plan));
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(k1_tok, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)KT_SMEM_BYTES);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(k1_tok, cudaFuncAttributePreferredSharedMemoryCarveout, 100);  // two CTAs per SM need all of it
    if (e != cudaSuccess) return e;
#ifdef UGVC_K1_SPLIT
    e = cudaFuncSetAttribute(k1_parse_info, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k1_smem_bytes(plan));
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(k1_parse_frame, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k1_smem_bytes(plan));
    if (e != cudaSuccess) return e;
#endif
    for (const auto& walk : K3H_KERNELS)  // a few static bytes (the mbarrier words) come on top of the dynamic part
        for (const auto k : walk)
            if ((e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024)) != cudaSuccess) return e;
    for (const auto& walk : K3I_KERNELS)
        for (const auto k : walk)
            if ((e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024)) != cudaSuccess) return e;
    return cudaSuccess;
}
#else
// host emulation (tests/host_emu): the chosen kernel and walk with one thread per CTA and the product's chunk, so a
// forest larger than it runs the chunk loop here too.  smem3 is the emulation's shared memory.
void launch_k3(const DevPlan& plan, const K3Config& c, const uint32_t* raw, const float* feats, size_t row_stride,
               const int64_t* d_n_records, double threshold, uint8_t* low_score, float* probs, double* qual,
               double* phreds, int phred_mode, long long* d_counts, unsigned long long* d_err, unsigned* ticket,
               cudaStream_t) {
    threadIdx = blockIdx = dim3(0, 0, 0);
    blockDim = gridDim = dim3(1, 1, 1);
    if (c.smem > sizeof(smem3)) {  // c.smem is sized for the product's tile, wider than the emulated one
        fprintf(stderr, "host_emu: K3 does not fit the emulated shared memory\n");
        abort();
    }
    const bool cat = c.walk == K3_WALK_CAT;
    if (c.kernel == K3_KERNEL_HEAP && c.split == 2) {  // one thread: RS = 1 record per tile, walked as B then A
        *ticket = 0;
        (cat ? k3_heap_split<2, 1, 8, 1, K3_WALK_CAT> : k3_heap_split<2, 1, 8, 1, K3_WALK_PLAIN>)(
            plan, raw, feats, row_stride, d_n_records, threshold, low_score, probs, qual, phreds, d_counts, c.chunk,
            phred_mode, d_err, ticket);
    }
    else if (c.kernel == K3_KERNEL_HEAP)
        (cat ? k3_heap<1, 1, 8, 1, K3_WALK_CAT> : k3_heap<1, 1, 8, 1, K3_WALK_PLAIN>)(
            plan, raw, feats, row_stride, d_n_records, threshold, low_score, probs, qual, phreds, d_counts, c.chunk,
            phred_mode, d_err, ticket);
    else
        (cat ? k3_infer<1, K3_WALK_CAT> : k3_infer<1, K3_WALK_PLAIN>)(
            plan, feats, row_stride, d_n_records, threshold, low_score, probs, qual, phreds, d_counts, c.chunk, phred_mode);
}
#endif  // !UGVC_HOST_EMU
