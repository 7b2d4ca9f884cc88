// hostio.cpp -- host side of the container formats around the hot path.
//
// The reference reads and writes bgzip'ed VCF through htslib (pysam.VariantFile at
// filter_variants_pipeline.py:106,115) and re-serialises every record in Python
// (filter_variants_pipeline.py:188-228).  Here: multi-threaded BGZF inflate/deflate over
// zlib, and a record splicer that rewrites FILTER / QUAL / INFO in the original line bytes
// following the same rules.  Plain C++17 + pthreads, no CUDA.
#include <stdio.h>
#include <string.h>
#include <zlib.h>

#include <atomic>
#include <algorithm>
#include <string>
#include <thread>
#include <vector>

#include "../../include/ugvc_b200.h"
#include "numparse.h"
#include "deflate.cuh"

namespace {

struct Block {
    uint64_t coff;   // file offset of the block
    uint32_t csize;  // whole block size
    uint32_t isize;  // uncompressed size
    uint64_t uoff;   // uncompressed offset of the block start
};

bool read_all(FILE* f, uint64_t off, void* dst, size_t n) {
    if (fseeko(f, (off_t)off, SEEK_SET) != 0) return false;
    return fread(dst, 1, n, f) == n;
}

// Parse one BGZF block header at p (>= 18 bytes available); returns total block size or 0.
uint32_t bgzf_block_size(const uint8_t* p, size_t avail) {
    if (avail < 18 || p[0] != 0x1f || p[1] != 0x8b || p[2] != 8 || !(p[3] & 4)) return 0;
    const uint32_t xlen = p[10] | (p[11] << 8);
    if (avail < 12 + xlen) return 0;
    const uint8_t* x = p + 12;
    const uint8_t* xe = x + xlen;
    while (x + 4 <= xe) {
        const uint32_t slen = x[2] | (x[3] << 8);
        if (x[0] == 'B' && x[1] == 'C' && slen == 2 && x + 6 <= xe) return (uint32_t)(x[4] | (x[5] << 8)) + 1;
        x += 4 + slen;
    }
    return 0;
}

int scan_blocks(FILE* f, uint64_t file_size, uint64_t begin, uint64_t end, std::vector<Block>& blocks) {
    uint64_t off = begin, uoff = 0;
    uint8_t hdr[18 + 256];
    while (off < end && off < file_size) {
        const size_t want = (size_t)std::min<uint64_t>(sizeof(hdr), file_size - off);
        if (!read_all(f, off, hdr, want)) return UGVC_E_IO;
        const uint32_t bs = bgzf_block_size(hdr, want);
        if (bs < 26 || off + bs > file_size) return UGVC_E_IO;
        uint8_t tail[4];
        if (!read_all(f, off + bs - 4, tail, 4)) return UGVC_E_IO;
        const uint32_t isize = tail[0] | (tail[1] << 8) | (tail[2] << 16) | ((uint32_t)tail[3] << 24);
        blocks.push_back({off, bs, isize, uoff});
        uoff += isize;
        off += bs;
    }
    return UGVC_OK;
}

bool inflate_block(const uint8_t* src, uint32_t csize, uint8_t* dst, uint32_t isize) {
    const uint32_t xlen = src[10] | (src[11] << 8);
    const uint32_t hdr = 12 + xlen;
    if (csize < hdr + 8) return false;
    z_stream zs;
    memset(&zs, 0, sizeof(zs));
    if (inflateInit2(&zs, -15) != Z_OK) return false;
    zs.next_in = const_cast<Bytef*>(src + hdr);
    zs.avail_in = csize - hdr - 8;
    zs.next_out = dst;
    zs.avail_out = isize;
    const int rc = inflate(&zs, Z_FINISH);
    bool ok = (rc == Z_STREAM_END) && zs.total_out == isize;
    inflateEnd(&zs);
    if (ok) {  // the gzip footer's CRC32, as htslib checks it: a corrupted block is refused, not parsed
        const uint8_t* ft = src + csize - 8;
        const uint32_t want = (uint32_t)ft[0] | ((uint32_t)ft[1] << 8) | ((uint32_t)ft[2] << 16) | ((uint32_t)ft[3] << 24);
        ok = (uint32_t)crc32(crc32(0L, Z_NULL, 0), dst, isize) == want;
    }
    return ok;
}

int clamp_threads(int n) {
    if (n <= 0) n = (int)std::thread::hardware_concurrency();
    if (n < 1) n = 1;
    if (n > 128) n = 128;
    return n;
}

const uint8_t BGZF_EOF[28] = {0x1f, 0x8b, 0x08, 0x04, 0, 0, 0, 0, 0, 0xff, 0x06, 0, 0x42, 0x43,
                              0x02, 0,    0x1b, 0,    0x03, 0, 0, 0, 0, 0, 0, 0,    0,    0};
constexpr size_t BGZF_BLOCK_DATA = 0xff00;

}  // namespace

extern "C" int64_t ugvc_bgzf_uncompressed_size(const char* path) {
    FILE* f = fopen(path, "rb");
    if (!f) return UGVC_E_IO;
    fseeko(f, 0, SEEK_END);
    const uint64_t fs = (uint64_t)ftello(f);
    std::vector<Block> blocks;
    const int rc = scan_blocks(f, fs, 0, fs, blocks);
    fclose(f);
    if (rc) return rc;
    return blocks.empty() ? 0 : (int64_t)(blocks.back().uoff + blocks.back().isize);
}

// The compressed byte range [c_begin, c_end) of the blocks that hold the virtual-offset range, the bytes of the first
// block before it and its uncompressed length: what ugvc_filter_bgzf wants to know about a contig of an indexed file.
extern "C" int ugvc_bgzf_range_info(const char* path, uint64_t voff_begin, uint64_t voff_end, uint64_t* c_begin, uint64_t* c_end,
                                    uint32_t* skip_head, uint64_t* take_bytes) {
    FILE* f = fopen(path, "rb");
    if (!f) return UGVC_E_IO;
    fseeko(f, 0, SEEK_END);
    const uint64_t fs = (uint64_t)ftello(f);
    const uint64_t cb = voff_begin >> 16, ub = voff_begin & 0xffff;
    const bool to_eof = (voff_end == 0 || voff_end == ~0ull);
    const uint64_t ce = to_eof ? fs : (voff_end >> 16), ue = to_eof ? 0 : (voff_end & 0xffff);
    std::vector<Block> blocks;
    const int rc = scan_blocks(f, fs, cb, ue ? ce + 1 : ce, blocks);
    fclose(f);
    if (rc) return rc;
    while (!blocks.empty() && blocks.back().isize == 0) blocks.pop_back();  // the EOF block carries nothing
    if (blocks.empty()) {
        *c_begin = *c_end = cb;
        *skip_head = 0;
        *take_bytes = 0;
        return UGVC_OK;
    }
    const uint64_t total_u = blocks.back().uoff + blocks.back().isize;
    uint64_t last_cut = 0;
    if (ue && blocks.back().coff == ce) {
        if (ue > blocks.back().isize) return UGVC_E_IO;
        last_cut = blocks.back().isize - ue;
    }
    if (ub > blocks.front().isize || ub + last_cut > total_u) return UGVC_E_IO;
    *c_begin = blocks.front().coff;
    *c_end = blocks.back().coff + blocks.back().csize;
    *skip_head = (uint32_t)ub;
    *take_bytes = total_u - ub - last_cut;
    return UGVC_OK;
}

extern "C" int ugvc_bgzf_inflate_file(const char* path, uint64_t voff_begin, uint64_t voff_end, uint8_t* out,
                                      size_t capacity, size_t* out_bytes, int n_threads) {
    FILE* f = fopen(path, "rb");
    if (!f) return UGVC_E_IO;
    fseeko(f, 0, SEEK_END);
    const uint64_t fs = (uint64_t)ftello(f);
    const uint64_t cb = voff_begin >> 16, ub = voff_begin & 0xffff;
    const bool to_eof = (voff_end == 0 || voff_end == ~0ull);
    const uint64_t ce = to_eof ? fs : (voff_end >> 16), ue = to_eof ? 0 : (voff_end & 0xffff);
    std::vector<Block> blocks;
    // blocks in [cb, ce) plus the block at ce when it is only partly wanted
    int rc = scan_blocks(f, fs, cb, ue ? ce + 1 : ce, blocks);
    if (rc) {
        fclose(f);
        return rc;
    }
    if (blocks.empty()) {
        fclose(f);
        if (out_bytes) *out_bytes = 0;
        return UGVC_OK;
    }
    const uint64_t total_u = blocks.back().uoff + blocks.back().isize;
    uint64_t last_cut = 0;  // bytes to drop from the tail of the last block
    if (ue && blocks.back().coff == ce) {
        if (ue > blocks.back().isize) {
            fclose(f);
            return UGVC_E_IO;
        }
        last_cut = blocks.back().isize - ue;
    }
    if (ub > blocks.front().isize || ub + last_cut > total_u) {
        fclose(f);
        return UGVC_E_IO;
    }
    const uint64_t produced = total_u - ub - last_cut;
    if (out_bytes) *out_bytes = (size_t)produced;
    if (produced > capacity) {
        fclose(f);
        return UGVC_E_ARG;
    }
    // read the compressed range once
    const uint64_t c0 = blocks.front().coff, c1 = blocks.back().coff + blocks.back().csize;
    std::vector<uint8_t> comp((size_t)(c1 - c0));
    const bool ok_read = read_all(f, c0, comp.data(), comp.size());
    fclose(f);
    if (!ok_read) return UGVC_E_IO;
    n_threads = clamp_threads(n_threads);
    std::atomic<size_t> next{0};
    std::atomic<int> failed{0};
    auto work = [&]() {
        std::vector<uint8_t> tmp;
        for (;;) {
            const size_t i = next.fetch_add(1);
            if (i >= blocks.size() || failed.load()) break;
            const Block& b = blocks[i];
            if (b.isize == 0) continue;
            const uint8_t* src = comp.data() + (b.coff - c0);
            const bool first = (i == 0 && ub > 0), last = (i + 1 == blocks.size() && last_cut > 0);
            if (!first && !last) {
                if (!inflate_block(src, b.csize, out + (b.uoff - ub), b.isize)) failed = 1;
            } else {
                tmp.resize(b.isize);
                if (!inflate_block(src, b.csize, tmp.data(), b.isize)) {
                    failed = 1;
                    continue;
                }
                const uint64_t s = first ? ub : 0, e = b.isize - (last ? last_cut : 0);
                if (e > s) memcpy(out + (b.uoff + s - ub), tmp.data() + s, (size_t)(e - s));
            }
        }
    };
    std::vector<std::thread> th;
    for (int t = 1; t < n_threads; ++t) th.emplace_back(work);
    work();
    for (auto& t : th) t.join();
    return failed.load() ? UGVC_E_IO : UGVC_OK;
}

extern "C" int ugvc_bgzf_deflate_to_file(const char* path, const char* mode, const uint8_t* data, size_t n_bytes,
                                         int level, int write_eof, int n_threads, uint64_t* out_compressed_bytes,
                                         uint32_t* out_block_csize, size_t block_capacity, size_t* out_n_blocks) {
    const size_t n_blocks = (n_bytes + BGZF_BLOCK_DATA - 1) / BGZF_BLOCK_DATA;
    if (out_n_blocks) *out_n_blocks = n_blocks;
    if (out_block_csize && block_capacity < n_blocks) return UGVC_E_ARG;
    std::vector<std::vector<uint8_t>> outb(n_blocks);
    n_threads = clamp_threads(n_threads);
    std::atomic<size_t> next{0};
    std::atomic<int> failed{0};
    if (level < 0 || level > 9) level = 6;
    auto work = [&]() {
        z_stream zs;
        memset(&zs, 0, sizeof(zs));
        if (deflateInit2(&zs, level, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY) != Z_OK) {
            failed = 1;
            return;
        }
        for (;;) {
            const size_t i = next.fetch_add(1);
            if (i >= n_blocks) break;
            const size_t off = i * BGZF_BLOCK_DATA;
            const size_t len = std::min(BGZF_BLOCK_DATA, n_bytes - off);
            std::vector<uint8_t>& o = outb[i];
            o.resize(18 + deflateBound(&zs, (uLong)len) + 8);
            deflateReset(&zs);
            zs.next_in = const_cast<Bytef*>(data + off);
            zs.avail_in = (uInt)len;
            zs.next_out = o.data() + 18;
            zs.avail_out = (uInt)(o.size() - 18 - 8);
            if (deflate(&zs, Z_FINISH) != Z_STREAM_END || 18 + zs.total_out + 8 > 65536) {
                // incompressible: store
                deflateEnd(&zs);
                z_stream z0;
                memset(&z0, 0, sizeof(z0));
                deflateInit2(&z0, 0, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY);
                z0.next_in = const_cast<Bytef*>(data + off);
                z0.avail_in = (uInt)len;
                z0.next_out = o.data() + 18;
                z0.avail_out = (uInt)(o.size() - 18 - 8);
                const int rc0 = deflate(&z0, Z_FINISH);
                zs.total_out = z0.total_out;
                deflateEnd(&z0);
                deflateInit2(&zs, level, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY);
                if (rc0 != Z_STREAM_END || 18 + zs.total_out + 8 > 65536) {
                    failed = 1;
                    break;
                }
            }
            const uint32_t clen = (uint32_t)zs.total_out;
            const uint32_t bsize = 18 + clen + 8;
            static const uint8_t H[12] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0};
            memcpy(o.data(), H, 12);
            o[12] = 'B';
            o[13] = 'C';
            o[14] = 2;
            o[15] = 0;
            o[16] = (uint8_t)((bsize - 1) & 0xff);
            o[17] = (uint8_t)((bsize - 1) >> 8);
            const uint32_t crc = (uint32_t)crc32(crc32(0L, Z_NULL, 0), data + off, (uInt)len);
            uint8_t* t = o.data() + 18 + clen;
            t[0] = crc & 0xff; t[1] = (crc >> 8) & 0xff; t[2] = (crc >> 16) & 0xff; t[3] = (crc >> 24) & 0xff;
            t[4] = len & 0xff; t[5] = (len >> 8) & 0xff; t[6] = (len >> 16) & 0xff; t[7] = (len >> 24) & 0xff;
            o.resize(bsize);
        }
        deflateEnd(&zs);
    };
    std::vector<std::thread> th;
    for (int t = 1; t < n_threads; ++t) th.emplace_back(work);
    work();
    for (auto& t : th) t.join();
    if (failed.load()) return UGVC_E_IO;
    FILE* f = fopen(path, (mode && mode[0] == 'a') ? "ab" : "wb");
    if (!f) return UGVC_E_IO;
    uint64_t total = 0;
    for (size_t i = 0; i < n_blocks; ++i) {
        if (fwrite(outb[i].data(), 1, outb[i].size(), f) != outb[i].size()) {
            fclose(f);
            return UGVC_E_IO;
        }
        if (out_block_csize) out_block_csize[i] = (uint32_t)outb[i].size();
        total += outb[i].size();
    }
    if (write_eof) {
        if (fwrite(BGZF_EOF, 1, 28, f) != 28) {
            fclose(f);
            return UGVC_E_IO;
        }
        total += 28;
    }
    if (fclose(f) != 0) return UGVC_E_IO;
    if (out_compressed_bytes) *out_compressed_bytes = total;
    return UGVC_OK;
}

// ------------------------------------------------------------------------------------------
// record splicer: filter_variants_pipeline.py:188-228 on the original line bytes
// ------------------------------------------------------------------------------------------
namespace {

struct Piece {
    const uint8_t* p;
    size_t n;
};

inline bool piece_is(const Piece& a, const char* s) {
    const size_t n = strlen(s);
    return a.n == n && memcmp(a.p, s, n) == 0;
}

// htslib prints INFO/QUAL floats (float32) with %g semantics
int format_g(double q, char* buf, size_t cap) { return snprintf(buf, cap, "%g", (double)(float)q); }

// triangular PL index -> (a, b) with a <= b  (multiallelics.py:257-277)
void gt_from_pl_idx(int idx, int& a, int& b) {
    int count = 0, n_alleles = 0;
    while (count < idx + 1) {
        count += n_alleles;
        ++n_alleles;
    }
    b = n_alleles - 2;
    a = idx - (count - n_alleles) - 1;
}

// rewrite GT / GQ / PL of the first sample (filter_variants_pipeline.py:203-215)
void recalibrated_sample(const uint8_t* fmt, size_t len, const double* ph, int n_pl, double gq, std::string& out) {
    // fmt = "FORMAT\tSAMPLE1[\tSAMPLE2...]"
    size_t ftab = 0;
    while (ftab < len && fmt[ftab] != '\t') ++ftab;
    std::vector<std::string> keys, vals;
    {
        size_t s = 0;
        for (size_t e = 0; e <= ftab; ++e)
            if (e == ftab || fmt[e] == ':') {
                keys.emplace_back(reinterpret_cast<const char*>(fmt + s), e - s);
                s = e + 1;
            }
    }
    size_t s1 = ftab < len ? ftab + 1 : len, s1e = s1;
    while (s1e < len && fmt[s1e] != '\t') ++s1e;
    {
        size_t s = s1;
        for (size_t e = s1; e <= s1e; ++e)
            if (e == s1e || fmt[e] == ':') {
                vals.emplace_back(reinterpret_cast<const char*>(fmt + s), e - s);
                s = e + 1;
            }
    }
    if (keys.size() == 1 && keys[0] == ".") keys.clear();
    vals.resize(keys.size(), ".");
    char sep = '/';
    std::vector<int> pl(n_pl);
    int best = 0;
    for (int k = 0; k < n_pl; ++k) {
        pl[k] = (int)ph[k];  // int(): truncation
        if (pl[k] < pl[best]) best = k;
    }
    int a = 0, b = 0;
    gt_from_pl_idx(best, a, b);
    auto set = [&](const char* key, const std::string& v) {
        for (size_t i = 0; i < keys.size(); ++i)
            if (keys[i] == key) {
                vals[i] = v;
                return;
            }
        keys.emplace_back(key);
        vals.push_back(v);
    };
    for (size_t i = 0; i < keys.size(); ++i)
        if (keys[i] == "GT" && vals[i].find('|') != std::string::npos) sep = '|';
    set("GQ", std::to_string((int)gq));
    std::string pls;
    for (int k = 0; k < n_pl; ++k) {
        if (k) pls.push_back(',');
        pls += std::to_string(pl[k]);
    }
    set("PL", pls);
    set("GT", std::to_string(a) + sep + std::to_string(b));
    for (size_t i = 0; i < keys.size(); ++i) {
        if (i) out.push_back(':');
        out += keys[i];
    }
    out.push_back('\t');
    for (size_t i = 0; i < vals.size(); ++i) {
        if (i) out.push_back(':');
        out += vals[i];
    }
    if (s1e < len) out.append(reinterpret_cast<const char*>(fmt + s1e), len - s1e);  // other samples untouched
}

void splice_one(const uint8_t* line, size_t len, const ugvc_recinfo& ri, bool with_model, bool low, double qual,
                bool overwrite_qual, const char* bl, size_t bl_len, const double* ph, int n_classes,
                std::string& out) {
    size_t off[4] = {ri.qual_off, ri.filter_off, ri.info_off, ri.format_off};
    if (ri.qual_off == 0xFFFF || ri.filter_off == 0xFFFF || ri.info_off == 0xFFFF || ri.format_off == 0xFFFF) {
        // long line: recount the tabs
        size_t tabs = 0, k = 0;
        for (size_t i = 0; i < len && k < 4; ++i)
            if (line[i] == '\t') {
                ++tabs;
                if (tabs >= 5) off[k++] = i + 1;
            }
        while (k < 4) off[k++] = len + 1;
    }
    const size_t q0 = off[0], f0 = off[1], i0 = off[2], x0 = off[3];  // x0: one past the tab after INFO
    if (!(q0 <= f0 && f0 <= i0 && i0 <= x0 && x0 <= len + 1) || q0 == 0) {
        out.append(reinterpret_cast<const char*>(line), len);  // malformed: pass through
        out.push_back('\n');
        return;
    }
    char num[48];
    // --recalibrate_genotype: gq = second smallest - smallest phred
    const bool recal = with_model && ph != nullptr;
    double gq = 0.0;
    int n_pl = 0;
    if (recal) {
        double m1 = ph[0], m2 = ph[1];
        if (m2 < m1) std::swap(m1, m2);
        for (int k = 2; k < n_classes; ++k) {
            if (ph[k] < m1) {
                m2 = m1;
                m1 = ph[k];
            } else if (ph[k] < m2)
                m2 = ph[k];
        }
        gq = m2 - m1;
        const int na = (int)((ri.flags >> 1) & 0x7Fu);
        n_pl = (na + 1) * na / 2;
        if (n_pl > n_classes) n_pl = n_classes;
        if (n_pl < 1) n_pl = 1;
    }
    // columns 1-5 incl. trailing tab
    out.append(reinterpret_cast<const char*>(line), q0);
    // QUAL
    if (with_model && overwrite_qual) out.append(num, (size_t)format_g(recal ? gq : qual, num, sizeof(num)));
    else out.append(reinterpret_cast<const char*>(line + q0), f0 - 1 - q0);
    out.push_back('\t');
    // FILTER
    {
        const uint8_t* fp = line + f0;
        const size_t fl = i0 - 1 - f0;
        size_t written = 0;
        bool has_low = false;
        if (!(fl == 1 && fp[0] == '.')) {
            size_t s = 0;
            for (size_t e = 0; e <= fl; ++e) {
                if (e == fl || fp[e] == ';') {
                    Piece k{fp + s, e - s};
                    const bool drop = k.n == 0 || (with_model && low && piece_is(k, "PASS"));
                    if (!drop) {
                        if (written) out.push_back(';');
                        out.append(reinterpret_cast<const char*>(k.p), k.n);
                        ++written;
                        has_low |= piece_is(k, "LOW_SCORE");
                    }
                    s = e + 1;
                }
            }
        }
        if (with_model && low && !has_low) {
            if (written) out.push_back(';');
            out.append("LOW_SCORE");
            ++written;
        }
        if (!written) out.append("PASS");
    }
    out.push_back('\t');
    // INFO
    {
        const uint8_t* ip = line + i0;
        const size_t il = x0 - 1 - i0;
        size_t written = 0;
        bool done_score = !with_model || recal, done_bl = (bl_len == 0);
        std::string score;
        if (with_model && !recal) {
            score = "TREE_SCORE=";
            score.append(num, (size_t)format_g(qual, num, sizeof(num)));
        }
        std::string blv;
        if (bl_len) {
            // ';'-joined blacklist annotations, PASS entries dropped (filter_variants_pipeline.py:217-224)
            size_t s = 0;
            for (size_t e = 0; e <= bl_len; ++e)
                if (e == bl_len || bl[e] == ';') {
                    if (e > s && !(e - s == 4 && memcmp(bl + s, "PASS", 4) == 0)) {
                        blv += blv.empty() ? "BLACKLST=" : ",";
                        blv.append(bl + s, e - s);
                    }
                    s = e + 1;
                }
            if (blv.empty()) done_bl = true;
        }
        // common case: no empty pieces and neither key already present -> the INFO bytes go out in one piece
        const bool plain = il > 0 && !(il == 1 && ip[0] == '.') && ip[0] != ';' && ip[il - 1] != ';' &&
                           !memmem(ip, il, ";;", 2) && (done_score || !memmem(ip, il, "TREE_SCORE=", 11)) &&
                           (done_bl || !memmem(ip, il, "BLACKLST=", 9));
        if (plain) {
            out.append(reinterpret_cast<const char*>(ip), il);
            written = 1;
        } else if (!(il == 1 && ip[0] == '.')) {
            size_t s = 0;
            for (size_t e = 0; e <= il; ++e) {
                if (e == il || ip[e] == ';') {
                    Piece k{ip + s, e - s};
                    if (k.n) {
                        if (written) out.push_back(';');
                        if (!done_score && k.n >= 11 && memcmp(k.p, "TREE_SCORE=", 11) == 0) {
                            out += score;
                            done_score = true;
                        } else if (!done_bl && k.n >= 9 && memcmp(k.p, "BLACKLST=", 9) == 0) {
                            out += blv;
                            done_bl = true;
                        } else
                            out.append(reinterpret_cast<const char*>(k.p), k.n);
                        ++written;
                    }
                    s = e + 1;
                }
            }
        }
        if (!done_score) {
            if (written) out.push_back(';');
            out += score;
            ++written;
        }
        if (!done_bl) {
            if (written) out.push_back(';');
            out += blv;
            ++written;
        }
        if (!written) out.push_back('.');
    }
    // FORMAT + samples (with the tab before them): untouched unless genotypes are recalibrated
    if (x0 <= len) {
        out.push_back('\t');
        if (recal) recalibrated_sample(line + x0, len - x0, ph, n_pl, gq, out);
        else out.append(reinterpret_cast<const char*>(line + x0), len - x0);
    }
    out.push_back('\n');
}

}  // namespace

extern "C" int64_t ugvc_splice_records(const uint8_t* text, const int64_t* line_start, const ugvc_recinfo* recinfo,
                                       const uint8_t* low_score, const double* qual, int64_t n_records,
                                       int overwrite_qual, int with_model, const int32_t* blacklist_code,
                                       const char* blacklist_table, const int64_t* blacklist_table_off,
                                       const double* phreds, int n_classes, uint8_t* out, size_t capacity,
                                       int64_t* out_line_start, int n_threads) {
    if (!text || !line_start || !recinfo || n_records < 0) return UGVC_E_ARG;
    if (with_model && (!low_score || !qual)) return UGVC_E_ARG;
    n_threads = clamp_threads(n_threads);
    if ((int64_t)n_threads > n_records / 4096 + 1) n_threads = (int)(n_records / 4096 + 1);
    std::vector<std::string> parts(n_threads);
    std::vector<std::vector<int64_t>> lens(n_threads);
    auto work = [&](int t) {
        const int64_t lo = n_records * t / n_threads, hi = n_records * (t + 1) / n_threads;
        std::string& o = parts[t];
        o.reserve((size_t)((line_start[hi] - line_start[lo]) + (hi - lo) * 40));
        if (out_line_start) lens[t].reserve((size_t)(hi - lo));
        for (int64_t i = lo; i < hi; ++i) {
            const size_t before = o.size();
            const uint8_t* line = text + line_start[i];
            const size_t len = (size_t)(line_start[i + 1] - line_start[i] - 1);
            const char* bl = nullptr;
            size_t bl_len = 0;
            if (blacklist_code && blacklist_table && blacklist_table_off) {
                const int32_t code = blacklist_code[i];
                bl = blacklist_table + blacklist_table_off[code];
                bl_len = (size_t)(blacklist_table_off[code + 1] - blacklist_table_off[code]);
            }
            splice_one(line, len, recinfo[i], with_model != 0, with_model && low_score[i] != 0,
                       with_model ? qual[i] : 0.0, overwrite_qual != 0, bl, bl_len,
                       phreds ? phreds + (size_t)i * n_classes : nullptr, n_classes, o);
            if (out_line_start) lens[t].push_back((int64_t)(o.size() - before));
        }
    };
    std::vector<std::thread> th;
    for (int t = 1; t < n_threads; ++t) th.emplace_back(work, t);
    work(0);
    for (auto& t : th) t.join();
    size_t total = 0;
    std::vector<size_t> part_off(n_threads);
    for (int t = 0; t < n_threads; ++t) {
        part_off[t] = total;
        total += parts[t].size();
    }
    if (total > capacity) return UGVC_E_ARG;
    // gather: every thread copies its own part (first touch of `out` is spread over the threads too)
    auto gather = [&](int t) {
        memcpy(out + part_off[t], parts[t].data(), parts[t].size());
        if (out_line_start) {
            int64_t rec = n_records * t / n_threads;
            int64_t o2 = (int64_t)part_off[t];
            for (int64_t l : lens[t]) {
                out_line_start[rec++] = o2;
                o2 += l;
            }
        }
        std::string().swap(parts[t]);
    };
    th.clear();
    for (int t = 1; t < n_threads; ++t) th.emplace_back(gather, t);
    gather(0);
    for (auto& t : th) t.join();
    if (out_line_start) out_line_start[n_records] = (int64_t)total;
    return (int64_t)total;
}

// Occurrences of `byte` in data[0, n): the record count of a contig's text (newlines), threaded.
extern "C" int64_t ugvc_count_byte(const uint8_t* data, size_t n, int byte, int n_threads) {
    if (!data && n) return UGVC_E_ARG;
    n_threads = clamp_threads(n_threads);
    if ((size_t)n_threads > n / (1u << 20) + 1) n_threads = (int)(n / (1u << 20) + 1);
    std::vector<int64_t> part(n_threads, 0);
    auto work = [&](int t) {
        const size_t lo = n * (size_t)t / n_threads, hi = n * (size_t)(t + 1) / n_threads;
        const uint8_t* p = data + lo;
        const uint8_t* end = data + hi;
        int64_t c = 0;
        while (p < end) {
            p = static_cast<const uint8_t*>(memchr(p, byte, (size_t)(end - p)));
            if (!p) break;
            ++c;
            ++p;
        }
        part[t] = c;
    };
    std::vector<std::thread> th;
    for (int t = 1; t < n_threads; ++t) th.emplace_back(work, t);
    work(0);
    for (auto& t : th) t.join();
    int64_t total = 0;
    for (int64_t c : part) total += c;
    return total;
}

// INFO/END of every record (0 where the INFO column has no END=<digits> field): what htslib's tabix takes for the end of
// a record's interval when the value lies beyond POS (gVCF blocks, symbolic alleles; bcftools index -t of the reference,
// filter_variants_pipeline.py:231).  The first END field of a line counts; the column bounds come from recinfo.  Threaded.
extern "C" int64_t ugvc_info_end(const uint8_t* text, const int64_t* line_start, const ugvc_recinfo* recinfo, int64_t n,
                                 int64_t* out_end, int n_threads) {
    if (n < 0 || (n && (!text || !line_start || !recinfo || !out_end))) return UGVC_E_ARG;
    n_threads = clamp_threads(n_threads);
    if ((int64_t)n_threads > n / 65536 + 1) n_threads = (int)(n / 65536 + 1);
    std::vector<int64_t> part(n_threads, 0);
    auto work = [&](int t) {
        const int64_t lo = n * (int64_t)t / n_threads, hi = n * (int64_t)(t + 1) / n_threads;
        int64_t found = 0;
        for (int64_t i = lo; i < hi; ++i) {
            out_end[i] = 0;
            const uint8_t* p = text + line_start[i] + recinfo[i].info_off;
            // format_off: one past the tab behind INFO, or line length + 1 when the line ends with the INFO column
            const uint8_t* end = text + line_start[i] + recinfo[i].format_off - 1;
            if (recinfo[i].format_off <= recinfo[i].info_off || end > text + line_start[i + 1]) continue;
            while (p < end) {
                const uint8_t* q = static_cast<const uint8_t*>(memchr(p, ';', (size_t)(end - p)));
                if (!q) q = end;
                if (q - p > 4 && p[0] == 'E' && p[1] == 'N' && p[2] == 'D' && p[3] == '=' && q - p <= 14) {
                    int64_t v = 0;
                    bool digits = true;
                    for (const uint8_t* d = p + 4; d < q; ++d) {
                        digits = digits && *d >= '0' && *d <= '9';
                        v = v * 10 + (*d - '0');
                    }
                    if (digits) {
                        out_end[i] = v;
                        ++found;
                    }
                    break;  // the first END field of the line
                }
                if (q - p >= 4 && p[0] == 'E' && p[1] == 'N' && p[2] == 'D' && p[3] == '=') break;  // END= without a usable value
                p = q + 1;
            }
        }
        part[t] = found;
    };
    std::vector<std::thread> th;
    for (int t = 1; t < n_threads; ++t) th.emplace_back(work, t);
    work(0);
    for (auto& t : th) t.join();
    int64_t total = 0;
    for (int64_t c : part) total += c;
    return total;
}

// The K1 numeric-literal parser compiled for the host (same header as the device code), so
// the CPU tests can check it against strtod on millions of literals.
extern "C" int ugvc_test_parse_float(const char* text, float* out_f32, double* out_f64, int* out_consumed) {
    UgvcPtrSrc s{reinterpret_cast<const uint8_t*>(text)};
    double v = 0.0;
    const int st = ugvc_parse_num(s, v);
    if (out_f64) *out_f64 = v;
    if (out_f32) *out_f32 = (float)v;
    if (out_consumed) *out_consumed = (int)(s.p - reinterpret_cast<const uint8_t*>(text));
    return st;
}

// The device BGZF encoder (deflate.cuh) compiled for the host -- the same source the GPU runs -- so that the CPU
// tests can inflate its blocks with zlib.  `in` needs 4 readable bytes after n; out: DEF_BLOCK_STRIDE bytes.
extern "C" int64_t ugvc_test_deflate_block(const uint8_t* in, uint32_t n, uint8_t* out) {
    if (!in || !out || n > DEF_CHUNK) return UGVC_E_ARG;
    static DefTables* tables = [] {
        DefTables* t = new DefTables();
        def_build_tables(*t);
        return t;
    }();
    std::vector<uint16_t> head(1u << DEF_HASH_BITS);
    alignas(16) static thread_local uint8_t buf[DEF_BLOCK_STRIDE];
    const uint32_t sz = def_block(in, n, buf, head.data(), *tables);
    memcpy(out, buf, sz);
    return (int64_t)sz;
}

// Host model of fio_deflate_warp (fileio.cu): the same windows of 32 positions, the same candidate rule (the hash
// table is read by all 32 positions before any of them is inserted), the same token selection, bit layout and
// slice-wise CRC -- with the lanes as a loop.  Test hook: the CPU suite inflates its output with zlib.
extern "C" int64_t ugvc_test_deflate_block_lanes(const uint8_t* in_, uint32_t n, uint8_t* out) {
    if (!in_ || !out || n > DEF_CHUNK) return UGVC_E_ARG;
    static DefTables* T = [] {
        DefTables* t = new DefTables();
        def_build_tables(*t);
        return t;
    }();
    std::vector<uint8_t> inbuf((size_t)n + 64, 0);  // the encoder reads whole words past the end
    memcpy(inbuf.data() + 16, in_, n);
    const uint8_t* in = inbuf.data() + 16;
    std::vector<uint16_t> head(1u << DEF_HASH_BITS, 0xFFFFu);
    std::vector<uint32_t> words((DEF_BLOCK_STRIDE >> 2), 0u);  // the bit stream from byte 16 of the block
    const uint8_t hdr[16] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0};
    memcpy(out, hdr, 16);
    // CRC: 32 slices, combined pairwise
    const uint32_t L = (((n + 31u) / 32u) + 3u) & ~3u;
    uint32_t crc[32], cov[32];
    for (uint32_t lane = 0; lane < 32; ++lane) {
        const uint32_t s0 = lane * L, len = s0 < n ? (n - s0 < L ? n - s0 : L) : 0;
        crc[lane] = def_crc_slice(*T, in + (len ? s0 : 0), len);
        cov[lane] = len;
    }
    for (uint32_t s = 1; s < 32; s <<= 1)
        for (uint32_t lane = 0; lane < 32; lane += 2 * s) {
            crc[lane] = def_crc_combine(*T, crc[lane], crc[lane + s], cov[lane + s]);
            cov[lane] += cov[lane + s];
        }
    words[0] = 3u << 16;
    uint32_t bp = 19, carry = 0;
    for (uint32_t p0 = 0; p0 < n; p0 += 32) {
        uint32_t w[32], cand[32], len[32], dist[32];
        bool can[32];
        for (uint32_t lane = 0; lane < 32; ++lane) {
            const uint32_t pos = p0 + lane;
            can[lane] = pos + 4 <= n;
            w[lane] = can[lane] ? def_ld4(in + pos) : 0;
            cand[lane] = can[lane] ? head[DEFW_HASH(w[lane])] : 0xFFFFu;
        }
        for (uint32_t lane = 32; lane-- > 0;)  // of lanes with equal hashes the lowest wins, as in the kernel
            if (can[lane]) head[DEFW_HASH(w[lane])] = (uint16_t)(p0 + lane);
        for (uint32_t lane = 0; lane < 32; ++lane) {
            const uint32_t pos = p0 + lane;
            len[lane] = dist[lane] = 0;
            if (carry < 32 && cand[lane] != 0xFFFFu && pos - cand[lane] <= 32768u && def_ld4(in + cand[lane]) == w[lane]) {
                const uint32_t maxlen = n - pos < DEF_MAX_MATCH ? n - pos : DEF_MAX_MATCH;
                len[lane] = def_extend(in, cand[lane], pos, maxlen);
                dist[lane] = pos - cand[lane];
            }
        }
        const uint32_t lim = n - p0 < 32 ? n - p0 : 32;
        uint32_t cur = carry;
        while (cur < lim) {
            uint32_t nb = 0;
            const uint32_t bits = def_token(*T, in[p0 + cur], len[cur], dist[cur], nb);
            const uint32_t wi = bp >> 5, sh = bp & 31u;
            words[wi] |= bits << sh;
            if (sh + nb > 32) words[wi + 1] |= bits >> (32 - sh);
            bp += nb;
            cur += len[cur] ? len[cur] : 1;
        }
        carry = cur >= 32 ? cur - 32 : 0;
    }
    bp += 7;  // end of block: seven zero bits
    uint32_t payload = ((bp + 7) >> 3) - 2;
    memcpy(out + 16, words.data(), (size_t)payload + 2);
    if (payload >= n + 5) {
        uint8_t* p = out + 18;
        p[0] = 1;
        p[1] = (uint8_t)n;
        p[2] = (uint8_t)(n >> 8);
        p[3] = (uint8_t)~n;
        p[4] = (uint8_t)(~n >> 8);
        memcpy(p + 5, in, n);
        payload = n + 5;
    }
    uint8_t* ft = out + 18 + payload;
    for (int k = 0; k < 4; ++k) {
        ft[k] = (uint8_t)(crc[0] >> (8 * k));
        ft[4 + k] = (uint8_t)(n >> (8 * k));
    }
    const uint32_t bsize = 18 + payload + 8;
    out[16] = (uint8_t)(bsize - 1);
    out[17] = (uint8_t)((bsize - 1) >> 8);
    return (int64_t)bsize;
}

// The per-contig summary of a tabix index (inflated .tbi bytes): smallest chunk begin / largest chunk end over the
// bins (the metadata pseudo-bin 37450 aside) and where each contig's linear index sits in `data`.  A whole-genome
// index holds ~10^5 bins: walking them in Python cost the tool 0.6 s of start-up.
extern "C" int ugvc_tbi_summary(const uint8_t* data, size_t n, int32_t n_ref_capacity, uint64_t* out_lo, uint64_t* out_hi,
                                int64_t* out_linear_offset, int32_t* out_linear_count, int32_t* out_n_ref, int64_t* out_names_offset,
                                int32_t* out_names_bytes) {
    if (!data || n < 36 || memcmp(data, "TBI\1", 4) != 0) return UGVC_E_DATA;
    int32_t hdr[8];
    memcpy(hdr, data + 4, 32);
    const int32_t n_ref = hdr[0], l_nm = hdr[7];
    if (n_ref < 0 || l_nm < 0 || 36 + (size_t)l_nm > n) return UGVC_E_DATA;
    if (out_n_ref) *out_n_ref = n_ref;
    if (out_names_offset) *out_names_offset = 36;
    if (out_names_bytes) *out_names_bytes = l_nm;
    if (n_ref > n_ref_capacity) return UGVC_E_ARG;
    size_t p = 36 + (size_t)l_nm;
    for (int32_t r = 0; r < n_ref; ++r) {
        if (p + 4 > n) return UGVC_E_DATA;
        int32_t n_bin;
        memcpy(&n_bin, data + p, 4);
        p += 4;
        uint64_t lo = ~0ull, hi = 0;
        for (int32_t b = 0; b < n_bin; ++b) {
            if (p + 8 > n) return UGVC_E_DATA;
            uint32_t bin;
            int32_t n_chunk;
            memcpy(&bin, data + p, 4);
            memcpy(&n_chunk, data + p + 4, 4);
            p += 8;
            if (n_chunk < 0 || p + 16 * (size_t)n_chunk > n) return UGVC_E_DATA;
            if (bin != 37450u)
                for (int32_t c = 0; c < n_chunk; ++c) {
                    uint64_t cb, ce;
                    memcpy(&cb, data + p + 16 * (size_t)c, 8);
                    memcpy(&ce, data + p + 16 * (size_t)c + 8, 8);
                    lo = cb < lo ? cb : lo;
                    hi = ce > hi ? ce : hi;
                }
            p += 16 * (size_t)n_chunk;
        }
        if (p + 4 > n) return UGVC_E_DATA;
        int32_t n_intv;
        memcpy(&n_intv, data + p, 4);
        if (n_intv < 0 || p + 4 + 8 * (size_t)n_intv > n) return UGVC_E_DATA;
        out_lo[r] = lo;
        out_hi[r] = hi;
        out_linear_offset[r] = (int64_t)(p + 4);
        out_linear_count[r] = n_intv;
        p += 4 + 8 * (size_t)n_intv;
    }
    return UGVC_OK;
}
