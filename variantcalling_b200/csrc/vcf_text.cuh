// vcf_text.cuh -- device helpers over VCF line text shared by the low_af_ratio.cu and bridging_snvs.cu kernels.
#pragma once
#include <stdint.h>

#include "numparse.h"

__device__ __forceinline__ bool afr_eq(const uint8_t* a, int64_t na, const uint8_t* b, int64_t nb) {
    if (na != nb) return false;
    for (int64_t k = 0; k < na; ++k)
        if (a[k] != b[k]) return false;
    return true;
}

// the next `sep`-separated piece of [*p, e): [*p, q); *p moves past the separator (beyond e after the last piece)
__device__ __forceinline__ int64_t afr_piece(const uint8_t* s, int64_t* at, int64_t e, uint8_t sep) {
    int64_t q = *at;
    while (q < e && s[q] != sep) ++q;
    const int64_t n = q - *at;
    *at = q + 1;
    return n;
}

// One numeric element as pysam types it: 0 = a value in *v, 1 = None ("."), 2 = a literal the parser refuses.  Float:
// float32(strtod) widened (numparse.h); Integer: sign and digits.  The element is followed by a delimiter inside the line.
__device__ __forceinline__ int afr_number(const uint8_t* p, int64_t n, int integer, double* v) {
    if (n == 1 && p[0] == '.') return 1;
    if (n == 0) return 2;
    if (integer) {
        int64_t k = (p[0] == '-' || p[0] == '+') ? 1 : 0;
        if (k == n || n - k > 18) return 2;
        int64_t x = 0;
        for (int64_t j = k; j < n; ++j) {
            if (p[j] < '0' || p[j] > '9') return 2;
            x = x * 10 + (p[j] - '0');
        }
        *v = (double)(p[0] == '-' ? -x : x);
        return 0;
    }
    UgvcPtrSrc src{p};
    double d = 0.0;
    if (ugvc_parse_num(src, d) != NUM_OK || src.p != p + n) return 2;
    *v = (double)(float)d;
    return 0;
}

// A typed FORMAT value of one sample: None, a scalar number (Number=1) or a tuple of numbers / None
struct AfrVal {
    int kind;  // 0 None, 1 scalar, 2 tuple
    const uint8_t* p;
    int64_t n;
    int64_t len;  // tuple length
    int integer;
};

// value kind (0 absent / undeclared, 1 Number=1, 2 other Number), the sub-field text (present = the sample has the
// field).  *bad is set when an element is a literal the parser refuses.
__device__ __forceinline__ AfrVal afr_value(int kind, int integer, bool present, const uint8_t* p, int64_t n, bool* bad) {
    AfrVal v{0, p, n, 0, integer};
    if (kind == 0) return v;
    const bool dot = !present || (n == 1 && p[0] == '.');
    if (kind == 1) {
        if (dot || n == 0) return v;  // None
        double x;
        if (afr_number(p, n, integer, &x) == 2) *bad = true;
        v.kind = 1;
        return v;
    }
    v.kind = 2;
    if (dot) {  // (None,)
        v.p = nullptr;
        v.len = 1;
        return v;
    }
    if (n == 0) return v;  // ()
    int64_t at = 0;
    while (at <= n) {
        const int64_t b = at;
        const int64_t m = afr_piece(p, &at, n, ',');
        double x;
        if (afr_number(p + b, m, integer, &x) == 2) *bad = true;
        ++v.len;
    }
    return v;
}

// element k of a tuple: 0 value, 1 None
__device__ __forceinline__ int afr_elem(const AfrVal& v, int64_t k, double* x) {
    if (!v.p) return 1;
    int64_t at = 0;
    for (int64_t j = 0; j < k; ++j) afr_piece(v.p, &at, v.n, ',');
    const int64_t b = at;
    const int64_t m = afr_piece(v.p, &at, v.n, ',');
    return afr_number(v.p + b, m, v.integer, x) == 0 ? 0 : 1;
}
