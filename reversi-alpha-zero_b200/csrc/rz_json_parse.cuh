// rz_json_parse.cuh -- the play-JSON grammar and number conversion shared by the device parser (rz_ingest_json.cu,
// one warp per record) and its host twin (rz_ingest_json_host).  Everything here is __host__ __device__ and free of
// state, so both sides classify bytes, match the record skeleton and convert numbers with the same code.
//
// A play_*.json file (lib/data_helper.py:23-25) is one JSON array of records [[own, enemy], [p0, ..., p63], z]:
//   own, enemy  non-negative integer literals < 2^64 (bitboards; anything else is refused, never truncated)
//   p0..p63, z  JSON numbers, plus the NaN / Infinity / -Infinity tokens json.dump writes and json.load accepts
// Any JSON whitespace may sit between tokens.  A number becomes float32(float64(text)): Python's correctly rounded
// float(), then numpy's round-to-nearest-even cast.
#pragma once
#include <stdint.h>
#include "rz_pow10_table.cuh"

#define RZ_HD __host__ __device__ __forceinline__

namespace rz {
namespace json {

typedef unsigned long long u64;

constexpr u64 kNoError = ~0ull;  // "no error" in an error-offset slot; the first error is the smallest offset

// ---- byte classes ----------------------------------------------------------------------------------------------
enum : int { C_WS = 0, C_STRUCT = 1, C_NUM = 2, C_BAD = 3 };

RZ_HD int byte_class(unsigned char c) {
    if (c == ' ' || c == '\t' || c == '\n' || c == '\r') return C_WS;
    if (c == '[' || c == ']' || c == ',') return C_STRUCT;
    if ((c >= '0' && c <= '9') || c == '-' || c == '+' || c == '.' || c == 'e' || c == 'E') return C_NUM;
    // the letters of NaN and Infinity: a token made of them is checked by parse_number
    if (c == 'N' || c == 'a' || c == 'I' || c == 'n' || c == 'f' || c == 'i' || c == 't' || c == 'y') return C_NUM;
    return C_BAD;
}

// ---- record skeleton ----------------------------------------------------------------------------------------------
// The non-whitespace items of a record, in order: '[' '[' own ',' enemy ']' ',' '[' p0 ',' p1 ... ',' p63 ']' ',' z ']'
// -- 139 items, 67 of them numbers.  item_kind(i) is the byte expected at item i, or 'N' for a number.
constexpr int kItems = 139;
constexpr int kOwnItem = 2, kEnemyItem = 4, kFirstPolicyItem = 8, kZItem = 137;

RZ_HD char item_kind(int i) {
    if (i <= 1) return '[';
    if (i == 2 || i == 4) return 'N';
    if (i == 3 || i == 6) return ',';
    if (i == 5) return ']';
    if (i == 7) return '[';
    if (i <= 134) return ((i - kFirstPolicyItem) & 1) ? ',' : 'N';
    if (i == 135) return ']';
    if (i == 136) return ',';
    if (i == kZItem) return 'N';
    return ']';  // 138, the record's closing bracket
}

// ---- numbers ------------------------------------------------------------------------------------------------------
enum : int { NUM_OK = 0, NUM_EXACT_NEEDED = 1, NUM_BAD = 2 };

RZ_HD void mul64x64(u64 a, u64 b, u64* hi, u64* lo) {
#ifdef __CUDA_ARCH__
    *hi = __umul64hi(a, b);
    *lo = a * b;
#else
    const unsigned __int128 p = (unsigned __int128)a * b;
    *hi = (u64)(p >> 64);
    *lo = (u64)p;
#endif
}

RZ_HD int clz64(u64 x) {
#ifdef __CUDA_ARCH__
    return __clzll((long long)x);
#else
    return __builtin_clzll(x);
#endif
}

RZ_HD double bits_to_double(u64 b) {
#ifdef __CUDA_ARCH__
    return __longlong_as_double((long long)b);
#else
    double d;
    __builtin_memcpy(&d, &b, 8);
    return d;
#endif
}

// exact powers of ten for Clinger's fast path
#define RZ_EXACT_POW10_INIT {1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22}
static __device__ const double d_exact_pow10[23] = RZ_EXACT_POW10_INIT;
static const double h_exact_pow10[23] = RZ_EXACT_POW10_INIT;

RZ_HD double exact_pow10(int k) {
#ifdef __CUDA_ARCH__
    return d_exact_pow10[k];
#else
    return h_exact_pow10[k];
#endif
}

// Eisel-Lemire: w * 10^e10 (w != 0) correctly rounded to a normal double, from the 128-bit truncated mantissa of
// 10^e10.  Returns false when the 128-bit product cannot decide the rounding (the product sits too close to a
// halfway point) or the result is subnormal, infinite or outside the table; the caller then converts exactly.
RZ_HD bool eisel_lemire(u64 w, int e10, const u64 (*pow10)[2], u64* out_bits) {
    if (e10 < RZ_POW10_MIN_E || e10 > RZ_POW10_MAX_E) return false;
    const int lz = clz64(w);
    w <<= lz;
    // biased binary exponent of the result, before the normalisation of the product's top bit
    u64 exp2 = (u64)((long long)((217706ll * e10) >> 16) + 64 + 1023) - (u64)lz;
    const u64* t = pow10[e10 - RZ_POW10_MIN_E];
    u64 hi, lo;
    mul64x64(w, t[1], &hi, &lo);
    if ((hi & 0x1FF) == 0x1FF && lo + w < w) {  // the low half of the mantissa could still carry into the top 55 bits
        u64 yhi, ylo;
        mul64x64(w, t[0], &yhi, &ylo);
        u64 mhi = hi, mlo = lo + yhi;
        if (mlo < lo) ++mhi;
        if ((mhi & 0x1FF) == 0x1FF && mlo + 1 == 0 && ylo + w < w) return false;
        hi = mhi;
        lo = mlo;
    }
    const u64 msb = hi >> 63;
    u64 mant = hi >> (msb + 9);
    exp2 -= 1 ^ msb;
    if (lo == 0 && (hi & 0x1FF) == 0 && (mant & 3) == 1) return false;  // exactly halfway on the truncated product
    mant += mant & 1;
    mant >>= 1;
    if (mant >> 53) {
        mant >>= 1;
        ++exp2;
    }
    if (exp2 - 1 >= 0x7FF - 1) return false;  // subnormal, zero or infinite: the exact path decides
    *out_bits = (exp2 << 52) | (mant & 0x000FFFFFFFFFFFFFull);
    return true;
}

RZ_HD bool token_is(const unsigned char* s, u64 a, u64 b, const char* word) {
    u64 i = 0;
    for (; word[i]; ++i)
        if (a + i >= b || s[a + i] != (unsigned char)word[i]) return false;
    return a + i == b;
}

// Parses the number token s[a, b) (b = first byte after it whose class is not C_NUM).  NUM_OK: *value holds
// float64(text).  NUM_EXACT_NEEDED: the token is a valid number that the fast paths cannot round (more than 19
// significant digits, a subnormal, zero or infinite result, or an ambiguous product); *value is undefined and the
// host's exact conversion decides.  NUM_BAD: not a JSON number.
RZ_HD int parse_number(const unsigned char* s, u64 a, u64 b, const u64 (*pow10)[2], double* value) {
    const bool neg = s[a] == '-';
    u64 p = a + (neg ? 1 : 0);
    if (token_is(s, p, b, "Infinity")) {
        *value = bits_to_double(neg ? 0xFFF0000000000000ull : 0x7FF0000000000000ull);
        return NUM_OK;
    }
    if (!neg && token_is(s, p, b, "NaN")) {
        *value = bits_to_double(0x7FF8000000000000ull);  // float('nan')
        return NUM_OK;
    }
    // int: '0' | [1-9][0-9]*
    if (p >= b || s[p] < '0' || s[p] > '9') return NUM_BAD;
    u64 w = 0;
    int nd = 0;       // significant digits accumulated into w (at most 19)
    int dropped = 0;  // significant digits beyond the 19th
    long long e10 = 0;
    if (s[p] == '0') {
        ++p;
    } else {
        for (; p < b && s[p] >= '0' && s[p] <= '9'; ++p) {
            if (nd < 19) { w = w * 10 + (s[p] - '0'); ++nd; }
            else { ++dropped; ++e10; }
        }
    }
    bool is_int = true;  // an integer literal: json.load makes it a Python int, and int("-0") is 0
    if (p < b && s[p] == '.') {
        is_int = false;
        ++p;
        const u64 f0 = p;
        for (; p < b && s[p] >= '0' && s[p] <= '9'; ++p) {
            if (nd == 0 && s[p] == '0') { --e10; continue; }  // leading zeros are not significant
            if (nd < 19) { w = w * 10 + (s[p] - '0'); ++nd; --e10; }
            else ++dropped;
        }
        if (p == f0) return NUM_BAD;
    }
    if (p < b && (s[p] == 'e' || s[p] == 'E')) {
        is_int = false;
        ++p;
        bool eneg = false;
        if (p < b && (s[p] == '+' || s[p] == '-')) { eneg = s[p] == '-'; ++p; }
        const u64 x0 = p;
        long long x = 0;
        for (; p < b && s[p] >= '0' && s[p] <= '9'; ++p)
            if (x < 100000000ll) x = x * 10 + (s[p] - '0');  // saturates far beyond any double's range
        if (p == x0) return NUM_BAD;
        e10 += eneg ? -x : x;
    }
    if (p != b) return NUM_BAD;
    const u64 sign = neg ? 0x8000000000000000ull : 0;
    if (w == 0) {  // all digits zero ("0", "-0.0", "0e999"): zero, signed unless an integer literal
        *value = bits_to_double(is_int ? 0 : sign);
        return NUM_OK;
    }
    if (dropped) return NUM_EXACT_NEEDED;
    if (w <= (1ull << 53) && e10 >= -22 && e10 <= 22) {  // Clinger: one correctly rounded operation on exact operands
#ifdef __CUDA_ARCH__
        const double d = e10 < 0 ? __ddiv_rn((double)w, exact_pow10((int)-e10)) : __dmul_rn((double)w, exact_pow10((int)e10));
#else
        volatile double d = e10 < 0 ? (double)w / exact_pow10((int)-e10) : (double)w * exact_pow10((int)e10);
#endif
        *value = neg ? -d : d;
        return NUM_OK;
    }
    u64 bits;
    if (e10 < -400 || e10 > 400 || !eisel_lemire(w, (int)e10, pow10, &bits)) return NUM_EXACT_NEEDED;
    *value = bits_to_double(bits | sign);
    return NUM_OK;
}

// A bitboard: a decimal integer literal without sign, fraction or exponent, no leading zeros, value < 2^64.
RZ_HD bool parse_u64(const unsigned char* s, u64 a, u64 b, u64* out) {
    if (a >= b || (s[a] == '0' && b - a > 1)) return false;
    u64 v = 0;
    for (u64 p = a; p < b; ++p) {
        const unsigned c = s[p] - '0';
        if (c > 9) return false;
        if (v > (~0ull - c) / 10) return false;  // >= 2^64
        v = v * 10 + c;
    }
    *out = v;
    return true;
}

RZ_HD u64 token_end(const unsigned char* s, u64 p, u64 n) {
    while (p < n && byte_class(s[p]) == C_NUM) ++p;
    return p;
}

RZ_HD float to_float32(double d) {
#ifdef __CUDA_ARCH__
    return __double2float_rn(d);
#else
    return (float)d;
#endif
}

}  // namespace json
}  // namespace rz
