// Pieces shared by the one-CTA-per-request streaming scans (emb_kernel.cu, rerank_large_kernel.cu): the in-thread prefix xor of
// the string parity scan, the JSON scalar grammar and the raw key compare.
#pragma once
#include <stdint.h>

namespace aigw {

// bit i of the result = xor of bits 0..i of x
__device__ __forceinline__ uint32_t prefix_xor32(uint32_t x) { x ^= x << 1; x ^= x << 2; x ^= x << 4; x ^= x << 8; x ^= x << 16; return x; }

// JSON scalar in [p, p+n): 0 invalid, 1 null, 2 true / false, 3 integer (-?digits, at most 18), 4 other number
static __device__ int scan_scalar_kind(const uint8_t* p, uint32_t n) {
  if (n == 4 && p[0] == 'n' && p[1] == 'u' && p[2] == 'l' && p[3] == 'l') return 1;
  if (n == 4 && p[0] == 't' && p[1] == 'r' && p[2] == 'u' && p[3] == 'e') return 2;
  if (n == 5 && p[0] == 'f' && p[1] == 'a' && p[2] == 'l' && p[3] == 's' && p[4] == 'e') return 2;
  uint32_t i = 0;
  if (i < n && p[i] == '-') i++;
  const uint32_t d0 = i;
  if (i >= n) return 0;
  if (p[i] == '0') i++;
  else if (p[i] >= '1' && p[i] <= '9') { while (i < n && p[i] >= '0' && p[i] <= '9') i++; }
  else return 0;
  const uint32_t nd = i - d0;
  if (i == n) return nd <= 18 ? 3 : 4;
  if (p[i] == '.') { i++; const uint32_t f0 = i; while (i < n && p[i] >= '0' && p[i] <= '9') i++; if (i == f0) return 0; }
  if (i < n && (p[i] == 'e' || p[i] == 'E')) { i++; if (i < n && (p[i] == '+' || p[i] == '-')) i++; const uint32_t e0 = i; while (i < n && p[i] >= '0' && p[i] <= '9') i++; if (i == e0) return 0; }
  return i == n ? 4 : 0;
}

// the raw bytes [p, p+n) equal the key k of length kl
__device__ __forceinline__ bool scan_key_is(const uint8_t* p, uint32_t n, const char* k, uint32_t kl) {
  if (n != kl) return false;
  for (uint32_t i = 0; i < n; i++) if (p[i] != (uint8_t)k[i]) return false;
  return true;
}

}  // namespace aigw
