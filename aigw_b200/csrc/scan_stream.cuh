// Pieces shared by the one-CTA-per-request streaming translators (rerank_large_kernel.cu, emb_large_kernel.cu): the token types
// of the scan, the odd-backslash-run rule of the escape stage, the token view the serial member walks read and grammar-check
// through, and the realigned 16-byte load of the emit copies.
#pragma once
#include <stdint.h>

#include "scan_common.cuh"

namespace aigw {

enum : uint32_t { T_QOPEN = '"', T_QCLOSE = '\'', T_SCALAR = 's' };
static constexpr uint32_t kNone = 0xffffffffu;

__device__ __forceinline__ void raise_min(int& fail, int r) { if (!fail || r < fail) fail = r; }

__device__ __forceinline__ bool is_hex(uint32_t c) { return (c >= '0' && c <= '9') || ((c | 0x20u) >= 'a' && (c | 0x20u) <= 'f'); }

// the escaped bytes of a thread's 32 bytes: bs = its backslashes, cin = its byte 0 is escaped (the carry-in)
__device__ __forceinline__ uint32_t escaped_mask(uint32_t bs, uint32_t cin) {
  const uint32_t even = 0x55555555u;
  bs &= ~cin;                                    // a leading backslash that is itself escaped starts no run
  const uint32_t follows = (bs << 1) | cin;
  const uint32_t odd_starts = bs & ~even & ~follows;
  const uint32_t seq_even = odd_starts + bs;     // runs that start on even bits carry through to the bit after their end
  return (even ^ (seq_even << 1)) & follows;
}

// Token view of one request for the serial walks.
struct ScanToks {
  const uint32_t* tok; uint32_t ntok; const uint8_t* body; uint32_t len;
  __device__ uint32_t ty(uint32_t k) const { return k < ntok ? tok[k] >> 24 : 0u; }
  __device__ uint32_t ps(uint32_t k) const { return tok[k] & 0xffffffu; }
  __device__ uint32_t scalar_end(uint32_t k) const {
    uint32_t e = k + 1 < ntok ? ps(k + 1) : len;
    const uint32_t b = ps(k);
    while (e > b && (body[e - 1] == ' ' || body[e - 1] == '\n' || body[e - 1] == '\r' || body[e - 1] == '\t')) e--;
    return e;
  }
  __device__ int scalar_kind(uint32_t k) const { const uint32_t b = ps(k); return scan_scalar_kind(body + b, scalar_end(k) - b); }
  // a scalar the depth pass found valid is null exactly when it starts with 'n'
  __device__ bool is_null(uint32_t k) const { return body[ps(k)] == 'n'; }
  __device__ bool has_backslash(uint32_t b, uint32_t e) const { for (uint32_t q = b; q < e; q++) if (body[q] == '\\') return true; return false; }
  // Go int64 member: digits only (a fraction or an exponent is the decoder's type error), exact int64 range
  __device__ bool int64_ok(uint32_t k) const {
    const uint32_t o = ps(k), e = scalar_end(k), i = o + (body[o] == '-' ? 1u : 0u);
    for (uint32_t q = i; q < e; q++) if (body[q] < '0' || body[q] > '9') return false;
    if (e - i < 19u) return true;
    if (e - i > 19u) return false;
    const char* lim = "9223372036854775808";   // -2^63; the positive bound is one less
    int c = 0;
    for (uint32_t q = 0; q < 19u && !c; q++) c = (int)body[i + q] - (int)lim[q];
    return !(c > 0 || (c == 0 && i == o));
  }
  // Grammar-check the value starting at token j and return the token after it, or kNone on a syntax error.  With `elems`, the
  // value is an array and bad_elem is set when one of its elements is neither a string nor null.  Depth ≤ 48 and the grammar of
  // every scalar are known here (the depth pass checks both in parallel), so a token costs a load and a few compares.
  __device__ uint32_t skip_value(uint32_t j, bool elems, bool& bad_elem) const {
    uint64_t stack = 0;   // bit d: the container at depth d + 1 is an object
    uint32_t depth = 0;
    bool want_key = false;
    for (;;) {
      uint32_t t = ty(j);
      if (want_key) {
        if (t != T_QOPEN || ty(j + 1) != T_QCLOSE || ty(j + 2) != ':') return kNone;
        j += 3; want_key = false; t = ty(j);
      }
      if (elems && depth == 1 && !(t == T_QOPEN || (t == T_SCALAR && is_null(j)))) bad_elem = true;
      if (t == '{' || t == '[') {
        if (ty(j + 1) == (t == '{' ? '}' : ']')) j += 2;
        else {
          if (depth >= 63u) return kNone;
          stack = (stack & ~(1ull << depth)) | ((uint64_t)(t == '{') << depth);
          depth++; j++; want_key = t == '{';
          continue;
        }
      } else if (t == T_QOPEN) { if (ty(j + 1) != T_QCLOSE) return kNone; j += 2; }
      else if (t == T_SCALAR) j++;
      else return kNone;
      for (;;) {   // after a value: a comma, or the close of the enclosing container
        if (depth == 0) return j;
        const bool obj = (stack >> (depth - 1)) & 1u;
        const uint32_t u = ty(j);
        if (u == ',') { j++; want_key = obj; break; }
        if (u != (obj ? '}' : ']')) return kNone;
        depth--; j++;
      }
    }
  }
};

// 16 bytes of body from src (any alignment): five aligned words, realigned with funnel shifts
__device__ __forceinline__ uint4 load16_unaligned(const uint8_t* src) {
  const uint32_t* a = (const uint32_t*)((uintptr_t)src & ~(uintptr_t)3);
  const uint32_t sh = ((uint32_t)(uintptr_t)src & 3u) * 8u;
  const uint32_t w0 = __ldg(a), w1 = __ldg(a + 1), w2 = __ldg(a + 2), w3 = __ldg(a + 3), w4 = sh ? __ldg(a + 4) : 0u;
  return make_uint4(__funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh), __funnelshift_r(w2, w3, sh), __funnelshift_r(w3, w4, sh));
}

}  // namespace aigw
