// Scalar pieces of the BVH MOTION-block parser and writer (bvh_text.cu), __host__ __device__ so that the CPU suite compiles the very
// same code for the host (tests/host/bvh_text_host.cu) and checks it against Python's float() and '%f'.
#pragma once
#include <stdint.h>

namespace zeggs {

#ifdef __CUDACC__
#define BVH_HD __host__ __device__ __forceinline__
#else
#define BVH_HD inline
#endif

// the ASCII whitespace of Python's str.split() / str.strip(): \t \n \v \f \r, \x1c-\x1f and space
BVH_HD bool bvh_is_space(unsigned c) { return c == ' ' || (c >= 9 && c <= 13) || (c >= 0x1c && c <= 0x1f); }
BVH_HD bool bvh_is_digit(unsigned c) { return c - '0' < 10u; }

// 10^k for 0 <= k <= 22 by binary powering: every factor (10, 1e2, 1e4, 1e8, 1e16) and every partial product is an exact double
BVH_HD double bvh_pow10(int k) {
  double p = 1.0, b = 10.0;
  for (; k; k >>= 1, b *= b)
    if (k & 1) p *= b;
  return p;
}

// One token [p, e) of the MOTION block.  Returns 1 and *out when the token is [+-]?(digits[.digits*]|.digits)([eE][+-]?digits)? with
// significant digits s <= 2^53 and a decimal exponent k in [-22, 22]: s * 10^k (or s / 10^-k) is then one correctly rounded IEEE
// operation on two exact operands, which is CPython's float() bit for bit (Clinger's fast path); the sign is applied afterwards, so
// "-0.000000" is -0.0.  Returns 0 for anything else (more digits, wider exponents, nan, inf, underscores, stray bytes): such a token
// is left to the host.
BVH_HD int bvh_parse_token(const unsigned char* p, const unsigned char* e, double* out) {
  const uint64_t lim = 1ull << 53;
  bool neg = false;
  if (p < e && (*p == '+' || *p == '-')) { neg = *p == '-'; ++p; }
  uint64_t s = 0;
  int k = 0, nd = 0;
  for (; p < e && bvh_is_digit(*p); ++p, ++nd) {
    s = s * 10 + (*p - '0');          // s <= 2^53 before the step: no wrap-around
    if (s > lim) return 0;
  }
  if (p < e && *p == '.') {
    for (++p; p < e && bvh_is_digit(*p); ++p, ++nd, --k) {
      s = s * 10 + (*p - '0');
      if (s > lim) return 0;
    }
  }
  if (nd == 0) return 0;
  if (p < e && (*p == 'e' || *p == 'E')) {
    ++p;
    bool eneg = false;
    if (p < e && (*p == '+' || *p == '-')) { eneg = *p == '-'; ++p; }
    int x = 0, ne = 0;
    for (; p < e && bvh_is_digit(*p); ++p, ++ne)
      if (x < 100000) x = x * 10 + (*p - '0');
    if (ne == 0) return 0;
    k += eneg ? -x : x;
  }
  if (p != e || k < -22 || k > 22) return 0;
  const double v = k >= 0 ? (double)s * bvh_pow10(k) : (double)s / bvh_pow10(-k);
  *out = neg ? -v : v;
  return 1;
}

// Longest "%f" text the writer produces for one value: sign, 33 integer digits (q = v * 10^6 < 2^128 has at most 39 digits), the point
// and 6 decimals.
constexpr int BVH_F_MAX_CHARS = 41;

// Python's / glibc's "%f" of v: v = m * 2^e exactly (m < 2^53), q = m * 10^6 * 2^e rounded half to even on the exact value in 128-bit
// integers, printed as q / 10^6 "." q % 10^6 with the sign of v ("-0.000000" for -0.0 and tiny negatives); nan, inf, -inf as Python
// writes them.  Writes the text to out (when not null) and returns its length, or -1 when m * 10^6 * 2^e does not fit in 128 bits.
BVH_HD int bvh_format_f(double v, char* out) {
  union { double d; uint64_t u; } cv;
  cv.d = v;
  const uint64_t bits = cv.u;
  const bool neg = bits >> 63;
  const int ex = (int)((bits >> 52) & 0x7ff);
  const uint64_t fr = bits & ((1ull << 52) - 1);
  if (ex == 0x7ff) {
    const char* t = fr ? "nan" : (neg ? "-inf" : "inf");
    int n = 0;
    for (; t[n]; ++n)
      if (out) out[n] = t[n];
    return n;
  }
  const uint64_t m = ex ? (fr | (1ull << 52)) : fr;
  const int e = ex ? ex - 1075 : -1074;
  typedef unsigned __int128 u128;
  const u128 N = (u128)m * 1000000u;        // < 2^73
  u128 q = 0;
  if (m != 0) {
    if (e >= 0) {
      if (e >= 128 || (e > 0 && (N >> (128 - e)) != 0)) return -1;
      q = N << e;
    } else if (-e < 74) {                   // for -e >= 74 the exact value is below 2^73 / 2^74 = 1/2: q = 0
      const int s = -e;
      q = N >> s;
      const u128 rem = N - (q << s), half = (u128)1 << (s - 1);
      if (rem > half || (rem == half && (q & 1))) ++q;
    }
  }
  // integer part (up to 33 digits) right to left, then the 6 decimals
  char dig[40];
  int nd = 0;
  const uint64_t frac = (uint64_t)(q % 1000000u);
  u128 ip = q / 1000000u;
  if (ip >> 64) {
    do { dig[nd++] = (char)('0' + (int)(ip % 10u)); ip /= 10u; } while (ip >> 64);
  }
  uint64_t ip64 = (uint64_t)ip;
  do { dig[nd++] = (char)('0' + (int)(ip64 % 10u)); ip64 /= 10u; } while (ip64);
  const int len = (neg ? 1 : 0) + nd + 7;
  if (out) {
    int o = 0;
    if (neg) out[o++] = '-';
    while (nd) out[o++] = dig[--nd];
    out[o++] = '.';
    uint64_t f = frac;
    for (int i = 6; i > 0; --i) { out[o + i - 1] = (char)('0' + (int)(f % 10u)); f /= 10u; }
  }
  return len;
}

}  // namespace zeggs
