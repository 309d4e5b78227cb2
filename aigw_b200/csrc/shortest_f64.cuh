// Is a 16- or 17-significant-digit decimal the text Go prints for the float64 it parses to?
//
// The request translators decode a JSON number into float64 and encode it again with strconv's shortest round-trip formatting
// (encoding/json and sonic agree on it).  For decimals of at most 15 significant digits that is the identity (canon_number in
// chat_walk_impl.cuh); a 16- or 17-digit decimal — 0.30000000000000004, 0.7000000000000001: what a client gets from float arithmetic —
// is reproduced ONLY when it already is that shortest form, which this function decides exactly, in integer arithmetic:
//   1. x = the double nearest to D = M / 10^k (round half to even), from a 128-bit quotient;
//   2. no decimal with one digit less lies in x's rounding interval (else the formatter prints the shorter one);
//   3. D is the closest decimal of its own length to x (else the formatter prints that neighbour).
// Domain: plain decimals with a fraction, last digit non-zero, at most 19 fraction digits (values down to about 1e-4); anything else
// returns false and the caller declines the body.  Plain C++ on purpose: tools/shortest_f64_check.cpp compiles it for the host and
// checks it against a reference formatter on random doubles.
#pragma once
#include <stdint.h>

#ifndef AIGW_SF64_HD
#ifdef __CUDACC__
// inlined into the walk kernels: around an out-of-line call their live registers follow the call ABI, which costs spills
#define AIGW_SF64_HD __host__ __device__ __attribute__((always_inline))
#else
#define AIGW_SF64_HD
#endif
#endif

namespace aigw {

typedef unsigned __int128 u128_t;

// p[0, n): optional '-', digits, '.', digits — already checked to be a JSON number without exponent
AIGW_SF64_HD inline bool shortest_f64_decimal(const uint8_t* p, uint32_t n) {
  uint32_t i = 0;
  if (i < n && p[i] == '-') i++;
  uint64_t M = 0; uint32_t sig = 0, k = 0; bool dot = false;
  for (; i < n; i++) {
    const uint32_t c = p[i];
    if (c == '.') { if (dot) return false; dot = true; continue; }
    if (c - '0' > 9u) return false;
    if (sig == 0 && c == '0') { if (dot) k++; continue; }   // leading zeros carry no significance
    if (sig >= 17) return false;
    M = M * 10u + (c - '0'); sig++;
    if (dot) k++;
  }
  if (!dot || k == 0 || k > 19 || sig < 16 || M % 10u == 0) return false;
  uint64_t P = 1; for (uint32_t j = 0; j < k; j++) P *= 10u;   // 10^k < 2^64
  // 1. nearest double f * 2^e: Q = floor(M * 2^s / P) with at least 54 bits
  const u128_t one = 1;
  int s = 0; u128_t Q = 0, R = 0;
  for (;; s++) {
    if (s > 70) return false;
    const u128_t N = (u128_t)M << s;
    Q = N / P; R = N % P;
    if ((Q >> 53) != 0) break;
  }
  int b = 0; while ((Q >> (53 + b + 1)) != 0) b++;            // Q has 54 + b bits; keep 53, drop b + 1
  const int drop = b + 1;
  uint64_t f = (uint64_t)(Q >> drop);
  const u128_t low = Q & ((one << drop) - 1), half = one << (drop - 1);
  const bool sticky = R != 0;
  if (low > half || (low == half && (sticky || (f & 1u)))) f++;
  int e = drop - s;
  if (f == (1ull << 53)) { f >>= 1; e++; }
  if (e > 1) return false;
  const int t = 1 - e;                                           // everything below is scaled by 10^k * 2^t
  if (t > 70) return false;
  // rounding interval of x, scaled: [(2f - 1) * P, (2f + 1) * P] (the lower half-ulp is half as wide at a power of two); closed iff f is even
  const u128_t hi = (u128_t)(2 * f + 1) * P;
  u128_t lo;
  if (f == (1ull << 52)) { if (t + 1 > 70) return false; lo = ((u128_t)(4 * f - 1) * P); }   // in units of half the scale (see below)
  else lo = (u128_t)(2 * f - 1) * P;
  const bool pow2 = f == (1ull << 52);
  const bool closed = (f & 1u) == 0;
  auto inside = [&](uint64_t c10) -> bool {   // is c10 / 10^k inside the interval?
    const u128_t A = (u128_t)c10 << t;
    const bool below_hi = closed ? A <= hi : A < hi;
    bool above_lo;
    if (pow2) { const u128_t A2 = A << 1; above_lo = closed ? A2 >= lo : A2 > lo; }
    else above_lo = closed ? A >= lo : A > lo;
    return below_hi && above_lo;
  };
  if (!inside(M)) return false;                                  // cannot happen for the nearest double; kept as a guard
  // 2. no neighbour with one digit less
  const uint64_t c_lo = (M / 10u) * 10u, c_hi = c_lo + 10u;
  if (inside(c_lo) || inside(c_hi)) return false;
  // 3. D is the closest decimal of its length: |D - x| < 10^-k / 2, i.e. |M * 2^t - 2f * P| < 2^(t-1) in the scaled units (a tie, or a
  //    farther neighbour that the formatter keeps because the closer one left the interval, is left to the caller's stock path)
  const u128_t a = (u128_t)M << t, x2 = (u128_t)(2 * f) * P;
  const u128_t diff = a > x2 ? a - x2 : x2 - a;
  return t == 0 ? diff == 0 : (diff >> (t - 1)) == 0;
}

}  // namespace aigw
