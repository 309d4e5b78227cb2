// aigw_b200 — SHA-256 of translated bodies for SigV4 (SURVEY §8f rank 1), sm_90a.
//
// Replaces `payloadHash := sha256.Sum256(body)` in the AWS request signer (internal/backendauth/aws.go:93-117), which today
// rescans every Bedrock-bound body on the CPU right after the translator produced it.  SHA-256 is sequential inside one message
// (Merkle–Damgård), so the parallelism is across messages: one THREAD per message, 32 messages per warp.  A thread reads its
// message with aligned 4-byte loads (17 per 64-byte block, funnel-shifted when the body starts at an odd address, as bodies
// inside `[path][body]` records do), keeps the 16-word schedule window and the eight working variables in registers and
// writes the 32-byte digest.  Integer-pipe bound: ≈ 2.9 k instructions per 64-byte block.
#include <cuda_runtime.h>
#include <stdint.h>

#include "sha256_kernel.cuh"

namespace aigw {
namespace {

__constant__ uint32_t kK[64] = {
  0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174,
  0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967,
  0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85, 0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070,
  0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};

__device__ __forceinline__ uint32_t rotr(uint32_t x, int r) { return __funnelshift_r(x, x, r); }
__device__ __forceinline__ uint32_t bswap(uint32_t x) { return __byte_perm(x, 0, 0x0123); }

__device__ __forceinline__ void compress(uint32_t h[8], uint32_t w[16]) {
  uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
#pragma unroll
  for (int i = 0; i < 64; i++) {
    if (i >= 16) {
      const uint32_t w15 = w[(i + 1) & 15], w2 = w[(i + 14) & 15];
      const uint32_t s0 = rotr(w15, 7) ^ rotr(w15, 18) ^ (w15 >> 3), s1 = rotr(w2, 17) ^ rotr(w2, 19) ^ (w2 >> 10);
      w[i & 15] += s0 + w[(i + 9) & 15] + s1;
    }
    const uint32_t S1 = rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25), ch = (e & f) ^ (~e & g), t1 = hh + S1 + ch + kK[i] + w[i & 15];
    const uint32_t S0 = rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22), mj = (a & b) ^ (a & c) ^ (b & c), t2 = S0 + mj;
    hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
  }
  h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
}

// message i = bytes[off[i] .. off[i]+len[i]); when `results` is given the span is the body of translate record i
__global__ void __launch_bounds__(128) sha256_kernel(const uint8_t* bytes, const uint64_t* off, const uint32_t* len, const aigw_doc_result* results, uint32_t n, uint8_t* digests) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t o; uint32_t l;
  if (results) {
    const aigw_doc_result r = results[i];
    if (r.status != AIGW_OK || r.body_kind != AIGW_BODY_BYTES) { uint4* d = (uint4*)(digests + 32ull * i); d[0] = make_uint4(0, 0, 0, 0); d[1] = make_uint4(0, 0, 0, 0); return; }
    o = r.out_off + r.path_len; l = r.body_len;
  } else { o = off[i]; l = len[i]; }
  const uint8_t* p = bytes + o;
  const uint32_t mis = (uint32_t)((uintptr_t)p & 3u), sh = mis * 8u;
  const uint32_t* wp = (const uint32_t*)(p - mis);   // aligned words; reads stay inside the words that hold message bytes
  uint32_t h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
  uint32_t w[16];
  const uint32_t full = l >> 6;
  for (uint32_t b = 0; b < full; b++) {
    const uint32_t* q = wp + 16u * b;
    uint32_t x[17];
#pragma unroll
    for (int k = 0; k < 16; k++) x[k] = __ldg(q + k);
    x[16] = mis ? __ldg(q + 16) : 0u;
#pragma unroll
    for (int k = 0; k < 16; k++) w[k] = bswap(__funnelshift_r(x[k], x[k + 1], sh));
    compress(h, w);
  }
  // tail: remaining r bytes, 0x80, zeros, 64-bit big-endian bit length (one or two blocks)
  const uint32_t r = l & 63u;
  const uint8_t* t = p + (full << 6);
  for (int pass = 0; pass < 2; pass++) {
#pragma unroll
    for (int k = 0; k < 16; k++) {
      uint32_t v = 0;
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const uint32_t idx = (uint32_t)pass * 64u + 4u * k + j;
        uint32_t c = 0;
        if (idx < r) c = t[idx]; else if (idx == r) c = 0x80u;
        v = (v << 8) | c;
      }
      w[k] = v;
    }
    const bool last = pass == 1 || r + 9u <= 64u;
    if (last) { const unsigned long long bits = (unsigned long long)l * 8ull; w[14] = (uint32_t)(bits >> 32); w[15] = (uint32_t)bits; }
    compress(h, w);
    if (last) break;
  }
  uint4* d = (uint4*)(digests + 32ull * i);
  d[0] = make_uint4(bswap(h[0]), bswap(h[1]), bswap(h[2]), bswap(h[3]));
  d[1] = make_uint4(bswap(h[4]), bswap(h[5]), bswap(h[6]), bswap(h[7]));
}

}  // namespace

cudaError_t launch_sha256(const uint8_t* bytes, const uint64_t* off, const uint32_t* len, const aigw_doc_result* results, uint32_t n, uint8_t* digests, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  sha256_kernel<<<(n + 127) / 128, 128, 0, st>>>(bytes, off, len, results, n, digests);
  return cudaGetLastError();
}

}  // namespace aigw
