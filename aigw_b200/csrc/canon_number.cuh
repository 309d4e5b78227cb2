// The canonical-number test shared by the translate pass's walk (chat_walk_impl.cuh) and the large chat scan
// (chat_large_kernel.cu).  sm_90a only.
#pragma once
#include <stdint.h>

#include "shortest_f64.cuh"

namespace aigw {

__device__ __forceinline__ bool canon_digit(uint32_t c) { return c - '0' < 10u; }

// ------------------------------------------------------------------ canonical scalars
// A JSON number literal that strconv would print back digit-for-digit once trailing fractional
// zeros are dropped: -?(0|[1-9]\d*)(\.\d+)? , ≤ 15 significant digits, |v| ≥ 1e-6 unless zero.
// Returns the emitted length (a prefix of the literal), 0 when not canonical.
static __device__ uint32_t canon_number(const uint8_t* p, uint32_t n, bool integer_only) {
  uint32_t i = 0;
  bool neg = false;
  if (p[0] == '-') { neg = true; i = 1; }
  const uint32_t int_start = i;
  while (i < n && canon_digit(p[i])) i++;
  const uint32_t int_digits = i - int_start;
  if (int_digits == 0) return 0;
  const bool int_zero = (int_digits == 1 && p[int_start] == '0');
  if (i == n) {
    if (integer_only) { if (int_digits > 18) return 0; if (neg && int_zero) return 0; return n; }
    if (int_digits > 15) return 0;
    return n;  // "-0" prints "-0" for a float64
  }
  if (integer_only || p[i] != '.') return 0;
  const uint32_t dot = i; i++;
  const uint32_t frac_start = i;
  while (i < n && canon_digit(p[i])) i++;
  if (i != n) return 0;
  uint32_t fe = n;
  while (fe > frac_start && p[fe - 1] == '0') fe--;
  const uint32_t frac_digits = fe - frac_start;
  if (frac_digits == 0) return dot;  // "1.0" → "1", "-0.0" → "-0"
  uint32_t sig;
  if (int_zero) {
    uint32_t z = 0; while (frac_start + z < fe && p[frac_start + z] == '0') z++;
    if (z > 5) return 0;  // < 1e-6 switches strconv to exponent form
    sig = frac_digits - z;
  } else sig = int_digits + frac_digits;
  if (sig > 15) return (sig <= 17u && shortest_f64_decimal(p, fe)) ? fe : 0;   // 16 / 17 digits: only when the text is already the float64's shortest form
  return fe;
}

}  // namespace aigw
