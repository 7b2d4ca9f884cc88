// synth_kernel.cu -- device-side synthetic VCF generator (bench / test input only).
//
// Produces single-sample VCF data lines in the schema of SURVEY.md 8d (the CUDA twin of
// variantcalling_b200/synth.py; same tags and value shapes, its own counter-based random
// stream) directly in HBM, so the 50 M-record configuration never has to exist on the
// host.  Two passes over a deterministic per-record generator: lengths -> exclusive scan
// (cub) -> write.  Not part of the timed hot path.
#include <cub/device/device_scan.cuh>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <string>

#include "../../include/ugvc_b200.h"

int ugvc_ctx_device(const ugvc_ctx* ctx);
int ugvc_ctx_sm_count(const ugvc_ctx* ctx);
void ugvc_ctx_count_launches(ugvc_ctx* ctx, int n);
cudaStream_t ugvc_ctx_default_stream(ugvc_ctx* ctx);
int ugvc_ctx_fail(ugvc_ctx* ctx, int code, const char* msg);

#define N_CONTIGS 24
__constant__ long long c_contig_len[N_CONTIGS] = {
    248956422, 242193529, 198295559, 190214555, 181538259, 170805979, 159345973, 145138636,
    138394717, 133797422, 135086622, 133275309, 114364328, 107043718, 101991189, 90338345,
    83257441,  80373285,  58617616,  64444167,  46709983,  50818468,  156040895, 57227415};
static const long long h_contig_len[N_CONTIGS] = {
    248956422, 242193529, 198295559, 190214555, 181538259, 170805979, 159345973, 145138636,
    138394717, 133797422, 135086622, 133275309, 114364328, 107043718, 101991189, 90338345,
    83257441,  80373285,  58617616,  64444167,  46709983,  50818468,  156040895, 57227415};
#define GENOME_LEN 3088269832ll

struct Rng {
    uint64_t key;
    uint64_t ctr;
    __device__ uint64_t next() {
        uint64_t z = key + (++ctr) * 0x9E3779B97F4A7C15ull;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        return z ^ (z >> 31);
    }
    __device__ uint32_t below(uint32_t n) { return (uint32_t)(((next() >> 32) * (uint64_t)n) >> 32); }
    __device__ float uni() { return (float)(next() >> 40) * (1.0f / 16777216.0f); }
};

struct CountSink {
    unsigned n = 0;
    __device__ void put(char) { ++n; }
};
struct WriteSink {
    uint8_t* p;
    __device__ void put(char c) { *p++ = (uint8_t)c; }
};

template <class S>
__device__ void put_str(S& s, const char* t) {
    while (*t) s.put(*t++);
}
template <class S>
__device__ void put_uint(S& s, unsigned long long v) {
    char buf[20];
    int n = 0;
    do {
        buf[n++] = (char)('0' + v % 10);
        v /= 10;
    } while (v);
    while (n) s.put(buf[--n]);
}
// value = scaled / 10^decimals, printed with exactly `decimals` fraction digits
template <class S>
__device__ void put_fixed(S& s, long long scaled, int decimals) {
    if (scaled < 0) {
        s.put('-');
        scaled = -scaled;
    }
    long long p = 1;
    for (int i = 0; i < decimals; ++i) p *= 10;
    put_uint(s, (unsigned long long)(scaled / p));
    s.put('.');
    long long frac = scaled % p;
    for (int i = decimals - 1; i >= 0; --i) {
        long long q = 1;
        for (int j = 0; j < i; ++j) q *= 10;
        s.put((char)('0' + (frac / q) % 10));
    }
}
template <class S>
__device__ void put_custom_name(S& s, int j) {
    switch (j) {
        case 0: put_str(s, "LCR"); break;
        case 1: put_str(s, "MAP_UNIQUE"); break;
        case 2: put_str(s, "LONG_HMER"); break;
        case 3: put_str(s, "UG_HCR"); break;
        case 4: put_str(s, "EXOME"); break;
        default:
            put_str(s, "ANN");
            s.put((char)('0' + ((j - 5) / 10) % 10));
            s.put((char)('0' + (j - 5) % 10));
    }
}

__device__ __forceinline__ char base_of(unsigned i) { return "ACGT"[i & 3]; }

template <class S>
__device__ void gen_record(S& s, uint64_t seed, long long rec, long long total, int n_custom) {
    Rng r;
    r.key = seed ^ ((uint64_t)rec * 0xD6E8FEB86659FD93ull);
    r.ctr = 0;
    // contig by cumulative length, position jittered inside the record's own stratum (sorted)
    int c = 0;
    long long cum = 0, r0 = 0, r1 = 0;
    for (; c < N_CONTIGS; ++c) {
        r0 = (long long)(((__int128)total * cum) / GENOME_LEN);
        r1 = (long long)(((__int128)total * (cum + c_contig_len[c])) / GENOME_LEN);
        if (c == N_CONTIGS - 1) r1 = total;
        if (rec < r1) break;
        cum += c_contig_len[c];
    }
    if (c >= N_CONTIGS) c = N_CONTIGS - 1;  // rec >= total: keep generating on the last contig
    const long long n_c = r1 - r0 > 0 ? r1 - r0 : 1;
    const double step = (double)c_contig_len[c] / (double)n_c;
    long long pos = 1 + (long long)(((double)(rec - r0) + (double)r.uni()) * step);
    if (pos > c_contig_len[c]) pos = c_contig_len[c];
    put_str(s, "chr");
    if (c < 22) put_uint(s, (unsigned)(c + 1));
    else s.put(c == 22 ? 'X' : 'Y');
    s.put('\t');
    put_uint(s, (unsigned long long)pos);
    s.put('\t');
    if (r.below(100) < 85) s.put('.');
    else {
        put_str(s, "rs");
        put_uint(s, 1 + r.below(99999999));
    }
    s.put('\t');
    // alleles
    const unsigned kind = r.below(1000);
    char refb[12], altb[12];
    int ref_n = 1, alt_n = 1;
    const char* x_ic = "NA";
    int x_il = -1, x_hil = -1;
    char x_hin = '.';
    int vtype = 0;  // 0 snp, 1 h-indel, 2 non-h-indel
    refb[0] = base_of(r.below(4));
    if (kind < 800) {
        altb[0] = base_of((unsigned)(refb[0] == 'A' ? 0 : refb[0] == 'C' ? 1 : refb[0] == 'G' ? 2 : 3) + 1 + r.below(3));
    } else if (kind < 980) {
        const int ln = kind < 900 ? 1 : 2 + (int)r.below(9);
        char extra[10];
        for (int i = 0; i < ln; ++i) extra[i] = base_of(r.below(4));
        const bool ins = r.below(2) == 0;
        x_ic = ins ? "ins" : "del";
        x_il = ln;
        vtype = ln == 1 ? 1 : 2;
        if (ln == 1 || r.below(10) < 3) {
            x_hil = (int)r.below(21);
            x_hin = extra[0];
        }
        if (ins) {
            altb[0] = refb[0];
            for (int i = 0; i < ln; ++i) altb[1 + i] = extra[i];
            alt_n = 1 + ln;
        } else {
            altb[0] = refb[0];
            for (int i = 0; i < ln; ++i) refb[1 + i] = extra[i];
            ref_n = 1 + ln;
        }
    } else {
        const char* trip = r.below(2) ? "GGC" : "CCG";
        const bool ins = r.below(2) == 0;
        x_ic = ins ? "ins" : "del";
        x_il = 2;
        vtype = 2;
        if (ins) {
            refb[0] = trip[0];
            altb[0] = trip[0]; altb[1] = trip[1]; altb[2] = trip[2];
            alt_n = 3;
        } else {
            refb[0] = trip[0]; refb[1] = trip[1]; refb[2] = trip[2];
            ref_n = 3;
            altb[0] = trip[0];
        }
    }
    for (int i = 0; i < ref_n; ++i) s.put(refb[i]);
    s.put('\t');
    for (int i = 0; i < alt_n; ++i) s.put(altb[i]);
    s.put('\t');
    // QUAL: heavy right tail, two decimals
    {
        const float u = r.uni(), v = r.uni();
        const long long cents = 1000 + (long long)(u * u * v * 400000.0f);
        put_fixed(s, cents, 2);
    }
    s.put('\t');
    {
        const unsigned f = r.below(100);
        put_str(s, f < 90 ? "." : f < 97 ? "PASS" : "LowQual");
    }
    s.put('\t');
    // genotype first (AC / AF depend on it)
    const unsigned g = r.below(100);
    const int gt = g < 60 ? 0 : g < 98 ? 1 : 2;  // 0: 0/1, 1: 1/1, 2: 0/0
    const int dp = 12 + (int)r.below(16) + (int)r.below(16) + (int)r.below(16);
    put_str(s, gt == 0 ? "AC=1;AF=0.500;AN=2" : gt == 1 ? "AC=2;AF=1.00;AN=2" : "AC=0;AF=0.500;AN=2");
    if (r.below(10) >= 3) {
        put_str(s, ";BaseQRankSum=");
        put_fixed(s, (long long)r.below(6001) - 3000, 3);
    }
    put_str(s, ";DP=");
    put_uint(s, (unsigned)(dp + (int)r.below(4)));
    put_str(s, ";ExcessHet=3.0103;FS=");
    {
        const float u = r.uni();
        put_fixed(s, (long long)(-2000.0f * __logf(u + 1e-6f)), 3);
    }
    put_str(s, ";HAPCOMP=");
    put_uint(s, r.below(7));
    put_str(s, gt == 0 ? ";MLEAC=1;MLEAF=0.500;MQ=" : gt == 1 ? ";MLEAC=2;MLEAF=1.00;MQ=" : ";MLEAC=0;MLEAF=0.500;MQ=");
    {
        const float u = r.uni();
        long long mq = 6000 - (long long)(-150.0f * __logf(u + 1e-6f));
        if (mq < 2000) mq = 2000;
        put_fixed(s, mq, 2);
    }
    put_str(s, ";MQ0C=");
    put_uint(s, r.below(4));
    s.put(',');
    put_uint(s, r.below(4));
    if (r.below(10) >= 3) {
        put_str(s, ";MQRankSum=");
        put_fixed(s, (long long)r.below(6001) - 3000, 3);
    }
    put_str(s, ";QD=");
    put_fixed(s, 100 + (long long)r.below(3400), 2);
    if (r.below(10) >= 3) {
        put_str(s, ";ReadPosRankSum=");
        put_fixed(s, (long long)r.below(6001) - 3000, 3);
    }
    put_str(s, ";SCL=");
    put_uint(s, r.below(4));
    s.put(',');
    put_uint(s, r.below(4));
    put_str(s, ";SCR=");
    put_uint(s, r.below(4));
    s.put(',');
    put_uint(s, r.below(4));
    put_str(s, ";SOR=");
    {
        const float u = r.uni(), v = r.uni();
        put_fixed(s, (long long)(-600.0f * (__logf(u + 1e-6f) + __logf(v + 1e-6f))), 3);
    }
    put_str(s, ";VARIANT_TYPE=");
    put_str(s, vtype == 0 ? "snp" : vtype == 1 ? "h-indel" : "non-h-indel");
    put_str(s, ";XC=");
    put_uint(s, r.below(12));
    put_str(s, ";X_CSS=");
    {
        const unsigned k = r.below(3);
        put_str(s, k == 0 ? "non-skip" : k == 1 ? "possible-cycle-skip" : "cycle-skip");
    }
    put_str(s, ";X_GCC=");
    put_fixed(s, (long long)r.below(101), 2);
    put_str(s, ";X_HIL=");
    if (x_hil < 0) s.put('.');
    else put_uint(s, (unsigned)x_hil);
    put_str(s, ";X_HIN=");
    s.put(x_hin);
    put_str(s, ";X_IC=");
    put_str(s, x_ic);
    put_str(s, ";X_IL=");
    if (x_il < 0) s.put('.');
    else put_uint(s, (unsigned)x_il);
    put_str(s, ";X_LM=");
    for (int i = 0; i < 5; ++i) s.put(base_of(r.below(4)));
    put_str(s, ";X_RM=");
    for (int i = 0; i < 5; ++i) s.put(base_of(r.below(4)));
    for (int j = 0; j < n_custom; ++j) {
        if (r.below(100) < 15) {
            s.put(';');
            put_custom_name(s, j);
            if (j == 2) {
                s.put('=');
                put_uint(s, 7 + r.below(13));
            } else
                put_str(s, "=TRUE");
        }
    }
    put_str(s, "\tGT:AD:DP:GQ:PL\t");
    put_str(s, gt == 0 ? "0/1:" : gt == 1 ? "1/1:" : "0/0:");
    {
        int alt_reads = 0;
        const unsigned pct = gt == 1 ? 97 : 50;
        for (int i = 0; i < dp; ++i) alt_reads += r.below(100) < pct;
        put_uint(s, (unsigned)(dp - alt_reads));
        s.put(',');
        put_uint(s, (unsigned)alt_reads);
    }
    s.put(':');
    if (r.below(100) < 1) s.put('.');
    else put_uint(s, (unsigned)dp);
    s.put(':');
    put_uint(s, r.below(100));
    s.put(':');
    {
        const unsigned z = r.below(3);
        for (unsigned k = 0; k < 3; ++k) {
            if (k) s.put(',');
            put_uint(s, k == z ? 0u : 20u + r.below(1980));
        }
    }
    s.put('\n');
}

__global__ void synth_lengths(uint64_t seed, long long first, long long n, long long total, int n_custom,
                              unsigned long long* __restrict__ lens) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        CountSink s;
        gen_record(s, seed, first + i, total, n_custom);
        lens[i] = s.n;
    }
}

__global__ void synth_write(uint64_t seed, long long first, long long n, long long total, int n_custom,
                            const unsigned long long* __restrict__ offs, uint8_t* __restrict__ out,
                            unsigned long long capacity) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const unsigned long long o = offs[i], e = offs[i + 1];
        if (e > capacity) continue;
        WriteSink s;
        s.p = out + o;
        gen_record(s, seed, first + i, total, n_custom);
    }
}

extern "C" int ugvc_synth_device(ugvc_ctx* ctx, uint64_t seed, int64_t first_record, int64_t n_records,
                                 int64_t total_records, int n_custom, uint8_t* d_text, size_t capacity_bytes,
                                 size_t* out_bytes, void* stream) {
    if (!ctx || !d_text || n_records < 0 || total_records <= 0 || n_custom < 0 || n_custom > 100)
        return ugvc_ctx_fail(ctx, UGVC_E_ARG, "synth: bad argument");
    cudaSetDevice(ugvc_ctx_device(ctx));
    cudaStream_t st = (cudaStream_t)stream;
    unsigned long long* lens = nullptr;
    void* tmp = nullptr;
    size_t tmp_bytes = 0;
    cudaError_t e = cudaMalloc(&lens, (size_t)(n_records + 1) * 2 * sizeof(unsigned long long));
    if (e != cudaSuccess) return ugvc_ctx_fail(ctx, UGVC_E_CUDA, cudaGetErrorString(e));
    unsigned long long* offs = lens + (n_records + 1);
    cudaMemsetAsync(lens + n_records, 0, sizeof(unsigned long long), st);
    const int blocks = ugvc_ctx_sm_count(ctx) * 8;
    synth_lengths<<<blocks, 128, 0, st>>>(seed, first_record, n_records, total_records, n_custom, lens);
    cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, lens, offs, (int)(n_records + 1), st);
    e = cudaMalloc(&tmp, tmp_bytes ? tmp_bytes : 8);
    if (e != cudaSuccess) {
        cudaFree(lens);
        return ugvc_ctx_fail(ctx, UGVC_E_CUDA, cudaGetErrorString(e));
    }
    cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, lens, offs, (int)(n_records + 1), st);
    synth_write<<<blocks, 128, 0, st>>>(seed, first_record, n_records, total_records, n_custom, offs, d_text,
                                        (unsigned long long)capacity_bytes);
    unsigned long long total_bytes = 0;
    cudaMemcpyAsync(&total_bytes, offs + n_records, sizeof(total_bytes), cudaMemcpyDeviceToHost, st);
    e = cudaStreamSynchronize(st);
    cudaFree(tmp);
    cudaFree(lens);
    ugvc_ctx_count_launches(ctx, 4);
    if (e != cudaSuccess) return ugvc_ctx_fail(ctx, UGVC_E_CUDA, cudaGetErrorString(e));
    if (out_bytes) *out_bytes = (size_t)total_bytes;
    if (total_bytes > capacity_bytes) return ugvc_ctx_fail(ctx, UGVC_E_ARG, "synth: capacity_bytes too small");
    return UGVC_OK;
}

extern "C" int64_t ugvc_synth_header(int n_custom, char* out, size_t capacity) {
    std::string h;
    h += "##fileformat=VCFv4.2\n##FILTER=<ID=LowQual,Description=\"Low quality\">\n";
    struct T { const char* id; const char* num; const char* type; };
    const T info[] = {{"AC", "A", "Integer"}, {"AF", "A", "Float"}, {"AN", "1", "Integer"},
                      {"BaseQRankSum", "1", "Float"}, {"DP", "1", "Integer"}, {"ExcessHet", "1", "Float"},
                      {"FS", "1", "Float"}, {"HAPCOMP", "A", "Integer"}, {"MLEAC", "A", "Integer"},
                      {"MLEAF", "A", "Float"}, {"MQ", "1", "Float"}, {"MQ0C", "R", "Integer"},
                      {"MQRankSum", "1", "Float"}, {"QD", "1", "Float"}, {"ReadPosRankSum", "1", "Float"},
                      {"SCL", "R", "Integer"}, {"SCR", "R", "Integer"}, {"SOR", "1", "Float"},
                      {"VARIANT_TYPE", "1", "String"}, {"XC", "1", "Integer"}, {"X_CSS", "A", "String"},
                      {"X_GCC", "1", "Float"}, {"X_HIL", "A", "Integer"}, {"X_HIN", "A", "String"},
                      {"X_IC", "A", "String"}, {"X_IL", "A", "Integer"}, {"X_LM", "A", "String"},
                      {"X_RM", "A", "String"}};
    for (const T& t : info)
        h += std::string("##INFO=<ID=") + t.id + ",Number=" + t.num + ",Type=" + t.type + ",Description=\"synthetic " + t.id + "\">\n";
    const char* base[] = {"LCR", "MAP_UNIQUE", "LONG_HMER", "UG_HCR", "EXOME"};
    for (int j = 0; j < n_custom; ++j) {
        char name[16];
        if (j < 5) snprintf(name, sizeof(name), "%s", base[j]);
        else snprintf(name, sizeof(name), "ANN%02d", j - 5);
        h += std::string("##INFO=<ID=") + name + ",Number=1,Type=String,Description=\"synthetic annotation, " + name + "\">\n";
    }
    h += "##FORMAT=<ID=AD,Number=R,Type=Integer,Description=\"Allelic depths\">\n";
    h += "##FORMAT=<ID=DP,Number=1,Type=Integer,Description=\"Read depth\">\n";
    h += "##FORMAT=<ID=GQ,Number=1,Type=Integer,Description=\"Genotype quality\">\n";
    h += "##FORMAT=<ID=GT,Number=1,Type=String,Description=\"Genotype\">\n";
    h += "##FORMAT=<ID=PL,Number=G,Type=Integer,Description=\"Phred-scaled likelihoods\">\n";
    for (int c = 0; c < N_CONTIGS; ++c) {
        char name[8];
        if (c < 22) snprintf(name, sizeof(name), "chr%d", c + 1);
        else snprintf(name, sizeof(name), "chr%c", c == 22 ? 'X' : 'Y');
        h += std::string("##contig=<ID=") + name + ",length=" + std::to_string(h_contig_len[c]) + ">\n";
    }
    h += "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tSAMPLE1\n";
    if (out && capacity >= h.size()) memcpy(out, h.data(), h.size());
    else if (out) return UGVC_E_ARG;
    return (int64_t)h.size();
}
