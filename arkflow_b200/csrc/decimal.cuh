// decimal.cuh — decimal text → binary64, correctly rounded (round to nearest, ties to even), on the device.
//
// One routine serves every decoder that reads numbers from text: json_to_arrow (Float64 columns, List<Float64>
// elements, the float spellings of Int64 values) and the CSV `file` input.  Three steps, cheapest first:
//   1. Clinger's fast path: ≤ 19 significant digits with mantissa < 2^53 and |exp10| ≤ 22 → one IEEE mul / div.
//   2. Eisel–Lemire (D. Lemire, "Number Parsing at a Gigabyte per Second", 2021): the 64-bit decimal mantissa times
//      the 128-bit truncated mantissa of 10^q (pow10_table.h) gives a 192-bit product P that lies below the exact one
//      by less than 2^64.  Unless the bits under the rounding position fall inside that window just below the
//      halfway point, the rounding of P is the rounding of the exact value.  More than 19 significant digits: the
//      value lies in [w, w + 1) · 10^q for the first 19 digits w; it is decided when w and w + 1 round alike.
//   3. Otherwise (ties, near-ties, long inputs that straddle a halfway point) decimal_slow() compares the exact
//      decimal value with the halfway points around a candidate in big-integer arithmetic.  It is __noinline__ so
//      that the hot kernels' register allocation does not carry it.
#pragma once

#include <cstdint>

#include "pow10_table.h"

namespace ark {

// [+-]? digits? ('.' digits?)? ([eE] [+-]? digits)?, at least one mantissa digit, nothing else.
struct DecimalScan {
  unsigned long long mant;  // the first ≤ 19 significant digits
  int exp10;                // the value is mant · 10^exp10 when !truncated, else in (mant, mant + 1) · 10^exp10
  bool neg;
  bool truncated;           // a nonzero digit after the first 19 significant ones was dropped
};

__host__ __device__ inline bool decimal_scan(const uint8_t* s, int len, DecimalScan* d) {
  int i = 0;
  d->neg = false;
  if (i < len && (s[i] == '-' || s[i] == '+')) { d->neg = s[i] == '-'; ++i; }
  unsigned long long mant = 0;
  int digits = 0, exp10 = 0;
  bool any = false, truncated = false;
  for (; i < len && s[i] >= '0' && s[i] <= '9'; ++i) {
    any = true;
    if (digits < 19) { mant = mant * 10 + (s[i] - '0'); if (mant) ++digits; }
    else { ++exp10; truncated |= s[i] != '0'; }
  }
  if (i < len && s[i] == '.') {
    ++i;
    for (; i < len && s[i] >= '0' && s[i] <= '9'; ++i) {
      any = true;
      if (digits < 19) { mant = mant * 10 + (s[i] - '0'); if (mant) ++digits; --exp10; }
      else truncated |= s[i] != '0';
    }
  }
  if (!any) return false;
  if (i < len && (s[i] == 'e' || s[i] == 'E')) {
    ++i;
    bool eneg = false;
    if (i < len && (s[i] == '+' || s[i] == '-')) { eneg = s[i] == '-'; ++i; }
    int e = 0;
    bool eany = false;
    for (; i < len && s[i] >= '0' && s[i] <= '9'; ++i) { eany = true; if (e < 100000) e = e * 10 + (s[i] - '0'); }
    if (!eany) return false;
    exp10 += eneg ? -e : e;
  }
  if (i != len) return false;
  d->mant = mant;
  d->exp10 = exp10;
  d->truncated = truncated;
  return true;
}

constexpr unsigned long long kF64InfBits = 0x7FF0000000000000ull;

// Eisel–Lemire step for a nonzero w and q in [ARK_POW10_MIN, ARK_POW10_MAX].  *bits receives the bits of
// round(w · 10^q) and the result is true when that rounding is certain; when it is not, *bits is the
// truncated value, at most one ulp below the correct one.
__device__ __forceinline__ bool decimal_eisel_lemire(unsigned long long w, int q, unsigned long long* bits) {
  const int idx = q - ARK_POW10_MIN;
  const unsigned long long th = kPow10Mant[idx], tl = kPow10Lo[idx];
  const int lz = __clzll((long long)w);
  w <<= lz;
  // P = w · (th · 2^64 + tl) = p2:p1:p0, in [2^190, 2^192); the value is P · 2^b
  const unsigned long long p0 = w * tl, c0 = __umul64hi(w, tl);
  unsigned long long p1 = w * th, p2 = __umul64hi(w, th);
  p1 += c0;
  p2 += p1 < c0;
  const int b = (int)kPow10Exp2[idx] - 64 - lz;
  const int ex = (int)(p2 >> 63) + 190 + b;  // the value lies in [2^ex, 2^(ex + 1))
  if (ex > 1023) { *bits = kF64InfBits; return true; }
  // k = bits of P below the result's last mantissa bit: 52 below the top bit for a normal result, down to 2^-1074
  // for a subnormal one.  k ≥ 138, so the mantissa comes from p2 alone.
  const int k = ex >= -1022 ? ex - 52 - b : -1074 - b;
  const int s = k - 128;
  if (s > 64) { *bits = 0; return true; }  // below 2^-1075 by more than the error window
  const unsigned long long mant = s == 64 ? 0 : p2 >> s;
  const unsigned long long rtop = s == 64 ? p2 : p2 & ((1ull << s) - 1), half = 1ull << (s - 1);
  bool up = false;
  if (rtop > half || (rtop == half && (p1 | p0))) up = true;
  else if (rtop == half) up = (q < 0 || q > 55) || (mant & 1);  // P is exact for 0 ≤ q ≤ 55: a tie, to even
  // the exact value may still reach the halfway point when P lies less than 2^64 below it
  const bool decided = !(rtop == half - 1 && p1 == ~0ull && p0 != 0);
  const unsigned long long m = mant + (up ? 1 : 0);
  // normal: mant ∈ [2^52, 2^53] and a carry out of the mantissa moves into the exponent field by itself
  unsigned long long r = ex >= -1022 ? ((unsigned long long)(ex + 1022) << 52) + m : m;
  if (r > kF64InfBits) r = kF64InfBits;
  *bits = r;
  return decided;
}

// ---- slow path: exact comparison with halfway points ------------------------------------------------------------
constexpr int kDecimalMaxDigits = 780;  // significant digits kept; a halfway point has at most 767
constexpr int kDecimalLimbs = 46;       // 2944 bits: the scaled operands stay below 2^2650

struct DecimalBig {
  unsigned long long d[kDecimalLimbs];
  int n;
};

__device__ inline void big_mul_add(DecimalBig& x, unsigned long long m, unsigned long long a) {
  unsigned long long carry = a;
  for (int i = 0; i < x.n; ++i) {
    const unsigned long long lo = x.d[i] * m, hi = __umul64hi(x.d[i], m);
    x.d[i] = lo + carry;
    carry = hi + (x.d[i] < lo);
  }
  if (carry && x.n < kDecimalLimbs) x.d[x.n++] = carry;
}

__device__ inline void big_mul_pow5(DecimalBig& x, int e) {
  constexpr unsigned long long k5_27 = 7450580596923828125ull;
  for (; e >= 27; e -= 27) big_mul_add(x, k5_27, 0);
  unsigned long long r = 1;
  for (; e > 0; --e) r *= 5;
  if (r != 1) big_mul_add(x, r, 0);
}

// limb i of x · 2^sh
__device__ inline unsigned long long big_limb_shl(const DecimalBig& x, int sh, int i) {
  const int j = i - (sh >> 6), r = sh & 63;
  const unsigned long long lo = j >= 0 && j < x.n ? x.d[j] : 0;
  if (r == 0) return lo;
  const unsigned long long below = j - 1 >= 0 && j - 1 < x.n ? x.d[j - 1] : 0;
  return (lo << r) | (below >> (64 - r));
}

// sign of x · 2^sx − y · 2^sy
__device__ inline int big_cmp_shl(const DecimalBig& x, int sx, const DecimalBig& y, int sy) {
  const int m = sx < sy ? sx : sy;
  sx -= m;
  sy -= m;
  const int nx = x.n + (sx >> 6) + 1, ny = y.n + (sy >> 6) + 1;
  for (int i = (nx > ny ? nx : ny) - 1; i >= 0; --i) {
    const unsigned long long a = big_limb_shl(x, sx, i), b = big_limb_shl(y, sy, i);
    if (a != b) return a < b ? -1 : 1;
  }
  return 0;
}

// The correctly rounded magnitude of the decimal text s[0, len) (grammar of decimal_scan), whose first 19
// significant digits scale by 10^exp10; `cand` is a result at most a few ulps away.
static __device__ __noinline__ double decimal_slow(const uint8_t* s, int len, int exp10, unsigned long long cand) {
  DecimalBig x, y;
  x.n = 0;
  int i = (len > 0 && (s[0] == '-' || s[0] == '+')) ? 1 : 0;
  int n = 0, kept = 0, chunk_n = 0;
  unsigned long long chunk = 0;
  bool sticky = false;
  for (; i < len; ++i) {
    if (s[i] == '.') continue;
    if (s[i] < '0' || s[i] > '9') break;
    const unsigned dgt = s[i] - '0';
    if (n == 0 && dgt == 0) continue;  // leading zeros
    ++n;
    if (kept < kDecimalMaxDigits) {
      chunk = chunk * 10 + dgt;
      ++kept;
      if (++chunk_n == 19) { big_mul_add(x, 10000000000000000000ull, chunk); chunk = 0; chunk_n = 0; }
    } else if (dgt) sticky = true;
  }
  if (chunk_n) {
    unsigned long long p = 1;
    for (int k = 0; k < chunk_n; ++k) p *= 10;
    big_mul_add(x, p, chunk);
  }
  int e10 = exp10 - (n > 19 ? n - 19 : 0) + (n - kept);  // the value is x · 10^e10
  if (sticky) { big_mul_add(x, 10, 1); --e10; }          // a digit between the kept ones and the next
  if (e10 >= 0) big_mul_pow5(x, e10);
  // sign of (value − halfway point between b and b + 1), the halfway point being (2m + 1) · 2^(e − 1)
  auto cmp_half = [&](unsigned long long b) {
    const unsigned long long m = (b >> 52) ? (b & ((1ull << 52) - 1)) | (1ull << 52) : b;
    const int e = (b >> 52) ? (int)(b >> 52) - 1075 : -1074;
    y.d[0] = 2 * m + 1;
    y.n = 1;
    if (e10 >= 0) return big_cmp_shl(x, e10, y, e - 1);  // x·5^e10 · 2^e10 vs (2m + 1) · 2^(e − 1)
    big_mul_pow5(y, -e10);                                // x vs (2m + 1) · 5^−e10 · 2^(e − 1 − e10)
    return big_cmp_shl(x, 0, y, e - 1 - e10);
  };
  unsigned long long c = cand > kF64InfBits ? kF64InfBits : cand;
  for (int it = 0; it < 8; ++it) {
    if (c < kF64InfBits) { const int r = cmp_half(c); if (r > 0 || (r == 0 && (c & 1))) { ++c; continue; } }
    if (c > 0) { const int r = cmp_half(c - 1); if (r < 0 || (r == 0 && (c & 1))) { --c; continue; } }
    break;
  }
  return __longlong_as_double((long long)c);
}

static __constant__ double kDecimalPow10[23] = {1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11,
                                         1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};

// Steps 2 and 3 for a nonzero magnitude off Clinger's fast path.  Out of line, like the slow path, so that the
// decoders' kernels keep the register budget they had with the fast path alone.
static __device__ __noinline__ double decimal_general(const uint8_t* s, int len, unsigned long long mant, int exp10, bool truncated) {
  if (exp10 > ARK_POW10_MAX) return __longlong_as_double((long long)kF64InfBits);  // ≥ 10^309
  if (exp10 < ARK_POW10_MIN) return 0.0;                                           // < 10^-324
  unsigned long long bits, bits1;
  bool ok = decimal_eisel_lemire(mant, exp10, &bits);
  if (ok && truncated) ok = decimal_eisel_lemire(mant + 1, exp10, &bits1) && bits1 == bits;
  return ok ? __longlong_as_double((long long)bits) : decimal_slow(s, len, exp10, bits);
}

// The correctly rounded double of a scanned decimal s[0, len).
__device__ __forceinline__ double decimal_value(const uint8_t* s, int len, const DecimalScan& d) {
  double v;
  if (d.mant == 0) v = 0.0;
  else if (!d.truncated && d.mant < (1ull << 53) && d.exp10 >= -22 && d.exp10 <= 22) {
    v = (double)d.mant;
    v = d.exp10 < 0 ? v / kDecimalPow10[-d.exp10] : v * kDecimalPow10[d.exp10];
  } else v = decimal_general(s, len, d.mant, d.exp10, d.truncated);
  return d.neg ? -v : v;
}

// decimal text → correctly rounded f64; false when s[0, len) is not in decimal_scan's grammar
__device__ __forceinline__ bool decimal_to_f64(const uint8_t* s, int len, double* out) {
  DecimalScan d;
  if (!decimal_scan(s, len, &d)) return false;
  *out = decimal_value(s, len, d);
  return true;
}

}  // namespace ark
