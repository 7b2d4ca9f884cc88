// inflate.cuh -- BGZF (RFC 1951 DEFLATE inside RFC 1952 gzip members) inflate on the device.
//
// SURVEY.md section 8 row f1: the reference reads its input through htslib's BGZF reader
// (filter_variants_pipeline.py:106,115); moving the decode to the GPU lets the host ship the
// *compressed* bytes over PCIe (4-5x fewer for VCF text), the link that bounds the end-to-end rate.
//
// Every BGZF block is self-contained (<= 64 KiB in, <= 64 KiB out, no history crosses blocks), so blocks are
// decoded independently.  Two decoders share the Huffman code builder and the symbol decoder below:
//  - inf_block_warp (the default, `bgzf_inflate_warps`): one warp per block.  The bit stream is decoded
//    warp-uniformly on tables in shared memory (10-bit literal-length and 8-bit distance look-up tables), the byte
//    moves of matches and stored blocks are spread over the lanes.
//  - inf_block (`bgzf_inflate_blocks`, UGVC_INFLATE_THREADS=1, and the host emulation): one thread per block with
//    9-bit / 7-bit tables in local memory, long matches moved as aligned 8-byte words.
// Codes longer than a table fall back to a canonical bit-by-bit walk.  Both decoders accept exactly what zlib's
// inflate accepts for a raw stream that ends inside the payload, and then check the block the way htslib's reader
// does: the output length must equal ISIZE and its CRC32 (def_crc_slice, deflate.cuh) the gzip footer's.
#pragma once
#include <stdint.h>

#include "deflate.cuh"

#ifndef __CUDACC__
#ifndef __host__
#define __host__
#define __device__
#endif
#endif

enum : int {
    INF_OK = 0,
    INF_BAD_BLOCK_TYPE = 1,
    INF_BAD_STORED_LEN = 2,
    INF_BAD_CODE_LENGTHS = 3,
    INF_BAD_SYMBOL = 4,
    INF_BAD_DISTANCE = 5,
    INF_OUTPUT_OVERRUN = 6,
    INF_INPUT_OVERRUN = 7,
    INF_SIZE_MISMATCH = 8,
    INF_BAD_CRC = 9,
};

// the CRC32 of the gzip footer, which follows the DEFLATE payload in[0, n_in)
__host__ __device__ inline uint32_t inf_footer_crc(const uint8_t* in, uint32_t n_in) {
    const uint8_t* f = in + n_in;
    return (uint32_t)f[0] | ((uint32_t)f[1] << 8) | ((uint32_t)f[2] << 16) | ((uint32_t)f[3] << 24);
}

#define INF_LIT_BITS 9
#define INF_DIST_BITS 7
#define INF_MAX_BITS 15

struct InfBits {
    const uint8_t* in;
    uint32_t n_in, pos;  // pos: next input byte to load
    uint64_t buf;
    int cnt;
    // Top the buffer up to >= 57 bits.  Whole aligned 32-bit words are loaded once `in + pos` is 4-byte
    // aligned (the caller guarantees 8 readable bytes after the input, so the last word may reach past n_in:
    // those bytes are never consumed by a valid stream and an invalid one is caught by the final position check).
    __host__ __device__ inline void refill() {
        while (cnt <= 56) {
            if (cnt <= 32 && ((reinterpret_cast<uintptr_t>(in) + pos) & 3u) == 0 && pos + 4 <= n_in + 4) {
                const uint64_t w = *reinterpret_cast<const uint32_t*>(in + pos);
                buf |= w << cnt;
                pos += 4;
                cnt += 32;
            } else {
                const uint64_t b = pos < n_in ? in[pos] : 0u;  // past the end zeros are shifted in
                ++pos;
                buf |= b << cnt;
                cnt += 8;
            }
        }
    }
    __host__ __device__ inline uint32_t peek(int n) const { return (uint32_t)(buf & ((1ull << n) - 1ull)); }
    __host__ __device__ inline void drop(int n) {
        buf >>= n;
        cnt -= n;
    }
    __host__ __device__ inline uint32_t take(int n) {
        const uint32_t v = peek(n);
        drop(n);
        return v;
    }
};

// Canonical Huffman code of `n` symbols with lengths len[0..n): count[], first-symbol offsets and the
// sorted symbol list for the slow path, plus a `bits`-wide look-up table: entry = (symbol << 4) | length,
// 0 for prefixes of longer codes.  Returns false for a set of lengths zlib's inflate_table refuses: an
// over-subscribed one, or an incomplete one -- except that a literal-length or distance code may consist of a
// single code of length 1, and a distance code may have no codes at all (a literal-only block).  The code-length
// code (`code_lengths`) must be complete.
struct InfCode {
    uint16_t count[INF_MAX_BITS + 1];
    uint16_t symbol[288];
};

__host__ __device__ inline uint32_t inf_reverse(uint32_t code, int len) {
    uint32_t r = 0;
    for (int i = 0; i < len; ++i) {
        r = (r << 1) | (code & 1u);
        code >>= 1;
    }
    return r;
}

__host__ __device__ inline bool inf_build(InfCode& c, const uint8_t* len, int n, uint16_t* lut, int bits,
                                          bool code_lengths = false) {
    for (int i = 0; i <= INF_MAX_BITS; ++i) c.count[i] = 0;
    for (int i = 0; i < n; ++i) c.count[len[i]]++;
    for (int i = 0; i < (1 << bits); ++i) lut[i] = 0;
    if (c.count[0] == n) return !code_lengths;  // no codes at all: legal for the distance code of a literal-only block
    int left = 1;
    for (int l = 1; l <= INF_MAX_BITS; ++l) {
        left <<= 1;
        left -= c.count[l];
        if (left < 0) return false;  // over-subscribed
    }
    if (left > 0 && (code_lengths || c.count[0] != n - 1 || c.count[1] != 1)) return false;  // incomplete
    uint16_t offs[INF_MAX_BITS + 2];
    offs[1] = 0;
    for (int l = 1; l < INF_MAX_BITS; ++l) offs[l + 1] = offs[l] + c.count[l];
    for (int s = 0; s < n; ++s)
        if (len[s]) c.symbol[offs[len[s]]++] = (uint16_t)s;
    // look-up table: canonical codes are assigned in symbol order within a length
    uint32_t code = 0;
    int idx = 0;
    for (int l = 1; l <= bits; ++l) {
        for (int k = 0; k < c.count[l]; ++k) {
            const uint32_t r = inf_reverse(code, l);
            const uint16_t e = (uint16_t)((c.symbol[idx] << 4) | l);
            for (uint32_t fill = r; fill < (1u << bits); fill += (1u << l)) lut[fill] = e;
            ++code;
            ++idx;
        }
        code <<= 1;
    }
    return true;
}

// decode one symbol: table first, canonical walk for codes longer than the table width
__host__ __device__ inline int inf_decode(InfBits& b, const InfCode& c, const uint16_t* lut, int bits) {
    const uint16_t e = lut[b.peek(bits)];
    if (e) {
        b.drop(e & 15);
        return e >> 4;
    }
    int code = 0, first = 0, index = 0;
    uint64_t window = b.buf;
    for (int l = 1; l <= INF_MAX_BITS; ++l) {
        code |= (int)(window & 1u);
        window >>= 1;
        const int cnt = c.count[l];
        if (code - cnt < first) {
            b.drop(l);
            return c.symbol[index + (code - first)];
        }
        index += cnt;
        first += cnt;
        first <<= 1;
        code <<= 1;
    }
    return -1;
}

// Inflate one raw DEFLATE stream of n_in bytes into exactly n_out bytes whose CRC32 is the one in the gzip footer at
// in + n_in.  Returns INF_*.
__host__ __device__ inline int inf_block(const uint8_t* in, uint32_t n_in, uint8_t* out, uint32_t n_out, const DefTables& T) {
    const uint16_t LEN_BASE[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
    const uint8_t LEN_EXTRA[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
    const uint16_t DIST_BASE[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
    const uint8_t DIST_EXTRA[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
    const uint8_t CL_ORDER[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    InfBits b;
    b.in = in;
    b.n_in = n_in;
    b.pos = 0;
    b.buf = 0;
    b.cnt = 0;
    uint32_t op = 0;
    InfCode lit, dist;
    uint16_t lit_lut[1 << INF_LIT_BITS], dist_lut[1 << INF_DIST_BITS];
    uint8_t lens[320];
    for (;;) {
        b.refill();
        const uint32_t last = b.take(1);
        const uint32_t type = b.take(2);
        if (type == 0) {  // stored
            b.drop(b.cnt & 7);
            b.refill();
            const uint32_t len = b.take(16), nlen = b.take(16);
            if ((len ^ 0xFFFFu) != nlen) return INF_BAD_STORED_LEN;
            if (op + len > n_out) return INF_OUTPUT_OVERRUN;
            // the bit buffer holds whole bytes now: give them back and copy from the input directly
            uint32_t p = b.pos - (uint32_t)(b.cnt >> 3);
            if (p + len > n_in) return INF_INPUT_OVERRUN;
            for (uint32_t i = 0; i < len; ++i) out[op++] = in[p++];
            b.pos = p;
            b.buf = 0;
            b.cnt = 0;
        } else if (type == 1 || type == 2) {
            if (type == 1) {  // fixed code
                for (int i = 0; i < 144; ++i) lens[i] = 8;
                for (int i = 144; i < 256; ++i) lens[i] = 9;
                for (int i = 256; i < 280; ++i) lens[i] = 7;
                for (int i = 280; i < 288; ++i) lens[i] = 8;
                inf_build(lit, lens, 288, lit_lut, INF_LIT_BITS);
                for (int i = 0; i < 32; ++i) lens[i] = 5;  // complete: distance codes 30 and 31 decode and are refused
                inf_build(dist, lens, 32, dist_lut, INF_DIST_BITS);
            } else {  // dynamic code
                const int hlit = (int)b.take(5) + 257, hdist = (int)b.take(5) + 1, hclen = (int)b.take(4) + 4;
                if (hlit > 286 || hdist > 30) return INF_BAD_CODE_LENGTHS;
                uint8_t cl[19];
                for (int i = 0; i < 19; ++i) cl[i] = 0;
                b.refill();
                for (int i = 0; i < hclen; ++i) {
                    if (b.cnt < 3) b.refill();
                    cl[CL_ORDER[i]] = (uint8_t)b.take(3);
                }
                InfCode clc;
                uint16_t cl_lut[1 << 7];
                if (!inf_build(clc, cl, 19, cl_lut, 7, true)) return INF_BAD_CODE_LENGTHS;
                int i = 0;
                while (i < hlit + hdist) {
                    b.refill();
                    const int sym = inf_decode(b, clc, cl_lut, 7);
                    if (sym < 0) return INF_BAD_SYMBOL;
                    if (sym < 16) {
                        lens[i++] = (uint8_t)sym;
                    } else {
                        int rep, val = 0;
                        if (sym == 16) {
                            if (i == 0) return INF_BAD_CODE_LENGTHS;
                            val = lens[i - 1];
                            rep = 3 + (int)b.take(2);
                        } else if (sym == 17) {
                            rep = 3 + (int)b.take(3);
                        } else {
                            rep = 11 + (int)b.take(7);
                        }
                        if (i + rep > hlit + hdist) return INF_BAD_CODE_LENGTHS;
                        while (rep--) lens[i++] = (uint8_t)val;
                    }
                }
                if (lens[256] == 0) return INF_BAD_CODE_LENGTHS;  // no end-of-block code
                if (!inf_build(lit, lens, hlit, lit_lut, INF_LIT_BITS)) return INF_BAD_CODE_LENGTHS;
                if (!inf_build(dist, lens + hlit, hdist, dist_lut, INF_DIST_BITS)) return INF_BAD_CODE_LENGTHS;
            }
            for (;;) {
                b.refill();  // >= 57 bits: enough for a literal-length code (15) + extra (5) + distance code (15) + extra (13)
                int sym = inf_decode(b, lit, lit_lut, INF_LIT_BITS);
                if (sym < 0) return INF_BAD_SYMBOL;
                if (sym < 256) {
                    if (op >= n_out) return INF_OUTPUT_OVERRUN;
                    out[op++] = (uint8_t)sym;
                    continue;
                }
                if (sym == 256) break;
                sym -= 257;
                if (sym >= 29) return INF_BAD_SYMBOL;
                const uint32_t len = LEN_BASE[sym] + b.take(LEN_EXTRA[sym]);
                const int ds = inf_decode(b, dist, dist_lut, INF_DIST_BITS);
                if (ds < 0 || ds >= 30) return INF_BAD_DISTANCE;
                const uint32_t d = DIST_BASE[ds] + b.take(DIST_EXTRA[ds]);
                if (d > op) return INF_BAD_DISTANCE;
                if (op + len > n_out) return INF_OUTPUT_OVERRUN;
                // The source bytes were written by this thread a moment ago and come back from L2.  A long match far
                // enough behind is moved as aligned 8-byte words (source words realigned with a funnel shift): one load
                // and one store per eight bytes instead of sixteen byte transactions; everything else byte by byte,
                // eight loads in flight where source and destination cannot overlap within a group.
                uint32_t i = 0;
                if (d >= 16 && len >= 16) {
                    while ((reinterpret_cast<uintptr_t>(out + op + i) & 7u) != 0) {  // destination up to an 8-byte boundary
                        out[op + i] = out[op + i - d];
                        ++i;
                    }
                    const uint8_t* src = out + op + i - d;
                    const unsigned sm = (unsigned)(reinterpret_cast<uintptr_t>(src) & 7u);
                    const uint64_t* sw = reinterpret_cast<const uint64_t*>(src - sm);
                    uint64_t* dw = reinterpret_cast<uint64_t*>(out + op + i);
                    if (sm == 0) {
                        for (; i + 8 <= len; i += 8) *dw++ = *sw++;
                    } else {
                        uint64_t lo = *sw++;
                        for (; i + 8 <= len; i += 8) {
                            const uint64_t hi = *sw++;  // at most 15 bytes past the source position: still behind `op` (d >= 16)
                            *dw++ = (lo >> (8 * sm)) | (hi << (64 - 8 * sm));
                            lo = hi;
                        }
                    }
                } else if (d >= 8) {
                    for (; i + 8 <= len; i += 8) {
                        const uint8_t* sp = out + op - d + i;
                        const uint8_t b0 = sp[0], b1 = sp[1], b2 = sp[2], b3 = sp[3], b4 = sp[4], b5 = sp[5], b6 = sp[6], b7 = sp[7];
                        uint8_t* dp = out + op + i;
                        dp[0] = b0, dp[1] = b1, dp[2] = b2, dp[3] = b3, dp[4] = b4, dp[5] = b5, dp[6] = b6, dp[7] = b7;
                    }
                }
                for (; i < len; ++i) out[op + i] = out[op + i - d];
                op += len;
            }
        } else {
            return INF_BAD_BLOCK_TYPE;
        }
        if (last) break;
    }
    if (b.pos - (uint32_t)(b.cnt >> 3) > n_in) return INF_INPUT_OVERRUN;
    if (op != n_out) return INF_SIZE_MISMATCH;
    return def_crc_slice(T, out, n_out) == inf_footer_crc(in, n_in) ? INF_OK : INF_BAD_CRC;
}

#if defined(__CUDACC__) && !defined(UGVC_HOST_EMU)
// ---------------------------------------------------------------------------------------------------
// One WARP per BGZF block.  The thread-per-block decoder above diverges 32 ways inside a warp and keeps its
// tables in local memory.  Here the serial part -- bit buffer, table
// look-up, symbol decode -- runs warp-uniformly (every lane holds the same state, the tables are in shared
// memory, the input word is a broadcast load), so nothing diverges, and the byte moves of the matches are spread
// over the lanes (lane k copies byte k; an overlapping match repeats with period d).  Literals are stored by
// one lane.  The output window lives in global memory: a match reads bytes the warp wrote a moment ago, so the
// source loads bypass L1 (ld.volatile) and are ordered behind the stores by __syncwarp().
#define INFW_LIT_BITS 10
#define INFW_DIST_BITS 8
struct InfWarpTables {
    uint16_t lit_lut[1 << INFW_LIT_BITS];
    uint16_t dist_lut[1 << INFW_DIST_BITS];
    InfCode lit, dist;
    uint8_t lens[320];
    uint8_t cl[32];
};

// the symbol -> base / extra-bit tables: warp-uniform indices, so the constant cache serves them
__constant__ uint16_t INFW_LEN_BASE[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t INFW_LEN_EXTRA[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t INFW_DIST_BASE[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t INFW_DIST_EXTRA[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t INFW_CL_ORDER[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

__device__ __forceinline__ int inf_block_warp(const uint8_t* __restrict__ in, uint32_t n_in, uint8_t* out, uint32_t n_out,
                                              InfWarpTables& T, const DefTables& D) {
    const unsigned lane = threadIdx.x & 31u;
    const volatile uint8_t* vout = out;
    InfBits b;
    b.in = in;
    b.n_in = n_in;
    b.pos = 0;
    b.buf = 0;
    b.cnt = 0;
    uint32_t op = 0;
    for (;;) {
        b.refill();
        const uint32_t last = b.take(1);
        const uint32_t type = b.take(2);
        if (type == 0) {  // stored: the lanes share the copy
            b.drop(b.cnt & 7);
            b.refill();
            const uint32_t len = b.take(16), nlen = b.take(16);
            if ((len ^ 0xFFFFu) != nlen) return INF_BAD_STORED_LEN;
            if (op + len > n_out) return INF_OUTPUT_OVERRUN;
            const uint32_t p = b.pos - (uint32_t)(b.cnt >> 3);
            if (p + len > n_in) return INF_INPUT_OVERRUN;
            for (uint32_t i = lane; i < len; i += 32u) out[op + i] = in[p + i];
            op += len;
            b.pos = p + len;
            b.buf = 0;
            b.cnt = 0;
        } else if (type == 1 || type == 2) {
            int err = INF_OK;
            if (type == 1) {  // fixed code
                if (lane == 0) {
                    for (int i = 0; i < 144; ++i) T.lens[i] = 8;
                    for (int i = 144; i < 256; ++i) T.lens[i] = 9;
                    for (int i = 256; i < 280; ++i) T.lens[i] = 7;
                    for (int i = 280; i < 288; ++i) T.lens[i] = 8;
                    inf_build(T.lit, T.lens, 288, T.lit_lut, INFW_LIT_BITS);
                    for (int i = 0; i < 32; ++i) T.lens[i] = 5;  // complete: distance codes 30 and 31 decode and are refused
                    inf_build(T.dist, T.lens, 32, T.dist_lut, INFW_DIST_BITS);
                }
            } else {  // dynamic code: the header is decoded by every lane (uniform), the tables are built by lane 0
                const int hlit = (int)b.take(5) + 257, hdist = (int)b.take(5) + 1, hclen = (int)b.take(4) + 4;
                if (hlit > 286 || hdist > 30) return INF_BAD_CODE_LENGTHS;
                b.refill();
                uint32_t cl3[19];
                for (int i = 0; i < 19; ++i) cl3[i] = 0;
                for (int i = 0; i < hclen; ++i) {
                    if (b.cnt < 3) b.refill();
                    cl3[i] = b.take(3);
                }
                if (lane == 0) {
                    uint8_t cl[19];
                    for (int i = 0; i < 19; ++i) cl[i] = 0;
                    for (int i = 0; i < hclen; ++i) cl[INFW_CL_ORDER[i]] = (uint8_t)cl3[i];
                    // the code-length code shares the distance tables' storage until they are built
                    if (!inf_build(T.dist, cl, 19, T.dist_lut, 7, true)) err = INF_BAD_CODE_LENGTHS;
                }
                __syncwarp();
                err = __shfl_sync(0xffffffffu, err, 0);
                if (err) return err;
                int i = 0;
                while (i < hlit + hdist) {
                    b.refill();
                    const int sym = inf_decode(b, T.dist, T.dist_lut, 7);
                    if (sym < 0) return INF_BAD_SYMBOL;
                    if (sym < 16) {
                        if (lane == 0) T.lens[i] = (uint8_t)sym;
                        ++i;
                    } else {
                        int rep, val = 0;
                        if (sym == 16) {
                            if (i == 0) return INF_BAD_CODE_LENGTHS;
                            __syncwarp();
                            val = T.lens[i - 1];
                            rep = 3 + (int)b.take(2);
                        } else if (sym == 17) {
                            rep = 3 + (int)b.take(3);
                        } else {
                            rep = 11 + (int)b.take(7);
                        }
                        if (i + rep > hlit + hdist) return INF_BAD_CODE_LENGTHS;
                        if (lane == 0)
                            for (int r = 0; r < rep; ++r) T.lens[i + r] = (uint8_t)val;
                        i += rep;
                    }
                }
                __syncwarp();
                if (lane == 0) {
                    if (T.lens[256] == 0) err = INF_BAD_CODE_LENGTHS;  // no end-of-block code
                    else if (!inf_build(T.lit, T.lens, hlit, T.lit_lut, INFW_LIT_BITS)) err = INF_BAD_CODE_LENGTHS;
                    else if (!inf_build(T.dist, T.lens + hlit, hdist, T.dist_lut, INFW_DIST_BITS)) err = INF_BAD_CODE_LENGTHS;
                }
            }
            __syncwarp();
            err = __shfl_sync(0xffffffffu, err, 0);
            if (err) return err;
            for (;;) {
                b.refill();  // >= 57 bits: a literal-length code (15) + extra (5) + distance code (15) + extra (13)
                int sym = inf_decode(b, T.lit, T.lit_lut, INFW_LIT_BITS);
                if (sym < 0) return INF_BAD_SYMBOL;
                if (sym < 256) {
                    if (op >= n_out) return INF_OUTPUT_OVERRUN;
                    if (lane == 0) out[op] = (uint8_t)sym;
                    ++op;
                    continue;
                }
                if (sym == 256) break;
                sym -= 257;
                if (sym >= 29) return INF_BAD_SYMBOL;
                const uint32_t len = INFW_LEN_BASE[sym] + b.take(INFW_LEN_EXTRA[sym]);
                const int ds = inf_decode(b, T.dist, T.dist_lut, INFW_DIST_BITS);
                if (ds < 0 || ds >= 30) return INF_BAD_DISTANCE;
                const uint32_t d = INFW_DIST_BASE[ds] + b.take(INFW_DIST_EXTRA[ds]);
                if (d > op) return INF_BAD_DISTANCE;
                if (op + len > n_out) return INF_OUTPUT_OVERRUN;
                __syncwarp();  // the bytes this match reads are in memory
                if (d >= len) {
                    for (uint32_t k = lane; k < len; k += 32u) out[op + k] = vout[op - d + k];
                } else {  // overlapping: the match repeats its first d bytes
                    for (uint32_t k = lane; k < len; k += 32u) out[op + k] = vout[op - d + k % d];
                }
                op += len;
            }
        } else {
            return INF_BAD_BLOCK_TYPE;
        }
        if (last) break;
    }
    if (b.pos - (uint32_t)(b.cnt >> 3) > n_in) return INF_INPUT_OVERRUN;
    if (op != n_out) return INF_SIZE_MISMATCH;
    // CRC32: every lane one contiguous slice, the slices' CRCs combined pairwise up the warp
    __syncwarp();  // every lane's stores are visible
    const uint32_t per = (n_out + 31u) / 32u, lo = lane * per < n_out ? lane * per : n_out;
    uint32_t len = n_out - lo < per ? n_out - lo : per;
    uint32_t crc = def_crc_slice(D, out + lo, len);
    for (unsigned s = 1; s < 32u; s <<= 1) {
        const uint32_t crc_b = __shfl_down_sync(0xffffffffu, crc, s), len_b = __shfl_down_sync(0xffffffffu, len, s);
        if ((lane & (2u * s - 1u)) == 0) {
            crc = def_crc_combine(D, crc, crc_b, len_b);
            len += len_b;
        }
    }
    crc = __shfl_sync(0xffffffffu, crc, 0);
    return crc == inf_footer_crc(in, n_in) ? INF_OK : INF_BAD_CRC;
}
#endif
