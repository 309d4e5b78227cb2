// BASELINE config 3: large /v1/embeddings requests (1024 inputs of 64 characters, about 68.7 KB of JSON, above the 64 KiB
// ceiling of the warp-per-document translate pass) — EmbeddingsEndpointSpec.ParseBody (internal/endpointspec/endpointspec.go:231-240)
// over the input union's []string / string forms (internal/apischema/openai/union.go:71-147, openai.go:316-375) fused with the
// text table the BPE count kernel (bpe_kernel.cu) reads IN PLACE from the request bytes.  sm_90a only.
//
// Mapping: one CTA of 256 threads per request, persistent CTAs pulling requests from a counter; the body streams through in
// 8 KB tiles (32 bytes per thread, two coalesced 16-byte loads), nothing of it is kept on chip:
//   scan      bit-sliced classification of the thread's 32 bytes (classify.cuh), in-string parity by a prefix-xor inside the
//             thread and an exclusive xor-scan over the CTA (ballot + 8 shared-memory words), tokens = structural bytes outside
//             strings, both quotes of every string, the first byte of every scalar; token words (position | type << 24) are
//             compacted into a per-CTA slice of the workspace with a block-wide prefix sum
//   validate  the accepted shape is regular — a root object whose only container is the "input" array of strings — so the
//             array interior is checked in parallel (token j of the interior must be quote / quote / comma by j mod 3), the
//             handful of top-level members sequentially by one thread (key set, duplicates, scalar grammar, value types)
//   texts     input k of the request = the bytes between the quotes of interior tokens 3k and 3k+1: (offset, length) rows of
//             the text table, allocated by one atomicAdd per request
// Everything outside that shape is DECLINED (the stock path decides): any backslash (the counted text would need decoding),
// nested containers, members other than model / input / encoding_format / dimensions / user, non-string array elements, raw
// control bytes in strings.  Definite decode errors of the known members are reported as 400, as ParseBody would.
#include "emb_kernel.cuh"

#include "classify.cuh"

namespace aigw {

static constexpr int kEmbThreads = 256;
static constexpr uint32_t kTile = kEmbThreads * 32;
enum : uint32_t { T_QOPEN = '"', T_QCLOSE = '\'', T_SCALAR = 's' };
static constexpr uint32_t kNoFail = 0xffffffffu;

__device__ __forceinline__ uint32_t prefix_xor32(uint32_t x) { x ^= x << 1; x ^= x << 2; x ^= x << 4; x ^= x << 8; x ^= x << 16; return x; }

struct EmbShared {
  uint32_t wpar[2][8], wlast[2][8], wcnt[2][8];
  uint32_t doc; uint32_t fail;   // lowest reason code raised by any thread (declines, below 32, win over the definite errors); kNoFail = none
  uint32_t n_lc, n_rc, n_lb, n_rb, lb, rb;
  uint32_t text_base, n_inputs, str_open, str_close;
};

// JSON scalar in [p, p+n): 0 invalid, 1 null, 2 true / false, 3 integer (-?digits, at most 18), 4 other number
__device__ int emb_scalar_kind(const uint8_t* p, uint32_t n) {
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

__device__ __forceinline__ bool emb_key_is(const uint8_t* p, uint32_t n, const char* k, uint32_t kl) {
  if (n != kl) return false;
  for (uint32_t i = 0; i < n; i++) if (p[i] != (uint8_t)k[i]) return false;
  return true;
}

__global__ void __launch_bounds__(kEmbThreads, 4) emb_scan_kernel(const EmbScanParams P) {
  __shared__ EmbShared S;
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const uint32_t lt = (1u << lane) - 1u;
  uint32_t* tok = P.tok_ws + (size_t)blockIdx.x * P.tok_cap;
  for (;;) {
    __syncthreads();
    if (tid == 0) { S.doc = atomicAdd(P.next, 1u); S.fail = kNoFail; S.n_lc = S.n_rc = S.n_lb = S.n_rb = 0; S.lb = 0xffffffffu; S.rb = 0; S.n_inputs = 0; S.text_base = 0; S.str_open = S.str_close = 0; }
    __syncthreads();
    const uint32_t doc = S.doc;
    if (doc >= P.n) break;
    const uint64_t boff = P.offsets[doc];
    const uint8_t* body = P.bodies + boff;
    const uint32_t len = P.lens[doc];
    aigw_emb_count_result res;
    res.status = AIGW_DECLINED; res.reason = 0; res.model_len = 0; res.model_off = 0; res.n_inputs = 0; res.tokens = 0; res.first_text = 0; res.in_len = len; res.declined_inputs = 0; res.reserved = 0;
    int fail = 0;
    uint32_t ntok = 0;
    if (len >= (1u << 24) || len == 0) fail = len ? AIGW_R_TOO_LARGE : AIGW_R_E400_SYNTAX;
    else if (((uintptr_t)body) & 15u) fail = AIGW_R_ARGS;   // the arena convention: every request starts 16-byte aligned
    uint32_t in_str = 0, prev_sc = 0;   // carries across tiles (uniform over the CTA)
    // the next tile's 32 bytes are requested before the current tile is classified (two tiles of loads in flight per thread)
    uint4 na = make_uint4(0, 0, 0, 0), nb = na;
    if (!fail && tid * 32u + 32u <= len) { na = __ldg((const uint4*)(body + tid * 32u)); nb = __ldg((const uint4*)(body + tid * 32u + 16)); }
    if (!fail) for (uint32_t base = 0, it = 0; base < len; base += kTile, it ^= 1u) {
      const uint32_t pos0 = base + tid * 32u;
      uint32_t w[8];
      if (pos0 + 32u <= len) {
        w[0] = na.x; w[1] = na.y; w[2] = na.z; w[3] = na.w; w[4] = nb.x; w[5] = nb.y; w[6] = nb.z; w[7] = nb.w;
        if (pos0 + kTile + 32u <= len) { na = __ldg((const uint4*)(body + pos0 + kTile)); nb = __ldg((const uint4*)(body + pos0 + kTile + 16)); }
      } else {
#pragma unroll
        for (int k = 0; k < 8; k++) {
          uint32_t v = 0x20202020u;
          const uint32_t p = pos0 + 4u * k;
          if (p + 4u <= len) v = __ldg((const uint32_t*)(body + p));
          else if (p < len) { v = 0; for (uint32_t q = 0; q < 4; q++) v |= (uint32_t)(p + q < len ? body[p + q] : 0x20u) << (8u * q); }
          w[k] = v;
        }
      }
      const ByteClasses c = classify32(w);
      if (c.bslash) fail = AIGW_R_ESCAPE;
      const uint32_t par = __popc(c.quote) & 1u;
      const uint32_t bal = __ballot_sync(0xffffffffu, par != 0);
      if (lane == 0) S.wpar[it][warp] = __popc(bal) & 1u;
      __syncthreads();
      uint32_t pre = 0, tot = 0;
#pragma unroll
      for (uint32_t k = 0; k < 8; k++) { const uint32_t v = S.wpar[it][k]; tot ^= v; if (k < warp) pre ^= v; }
      const uint32_t in0 = in_str ^ pre ^ (__popc(bal & lt) & 1u);
      const uint32_t ps = prefix_xor32(c.quote) ^ (in0 ? 0xffffffffu : 0u);   // bit i: inside a string after byte i (the opening quote counts, the closing one does not)
      const uint32_t inside = ps & ~c.quote;
      const uint32_t out = ~ps & ~c.quote;
      if (c.ctl & inside) fail = AIGW_R_CTRL_IN_STRING;
      if (c.ctl & out & ~c.ws) fail = AIGW_R_SYNTAX;
      const uint32_t sc = out & ~c.op & ~c.ws;
      if (lane == 31) S.wlast[it][warp] = sc >> 31;
      uint32_t prev = __shfl_up_sync(0xffffffffu, sc >> 31, 1);
      __syncthreads();
      if (lane == 0) prev = warp == 0 ? prev_sc : S.wlast[it][warp - 1];
      const uint32_t sc_start = sc & ~((sc << 1) | prev);
      uint32_t tk = (c.op & out) | c.quote | sc_start;
      const uint32_t cnt = __popc(tk);
      uint32_t incl = cnt;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d); if ((int)lane >= d) incl += v; }
      if (lane == 31) S.wcnt[it][warp] = incl;
      const uint32_t last_sc_tile = S.wlast[it][7];
      __syncthreads();
      uint32_t wpre = 0, wtot = 0;
#pragma unroll
      for (uint32_t k = 0; k < 8; k++) { const uint32_t v = S.wcnt[it][k]; wtot += v; if (k < warp) wpre += v; }
      uint32_t off = ntok + wpre + incl - cnt;
      while (tk) {
        const uint32_t i = __ffs(tk) - 1u; tk &= tk - 1u;
        const uint32_t p = pos0 + i;
        const uint32_t bit = 1u << i;
        const uint32_t ty = (c.quote & bit) ? ((ps & bit) ? T_QOPEN : T_QCLOSE) : (c.op & bit) ? (uint32_t)body[p] : T_SCALAR;
        if (off < P.tok_cap) tok[off] = p | (ty << 24);
        off++;
      }
      ntok += wtot; in_str ^= tot; prev_sc = last_sc_tile;
    }
    if (!fail && in_str) fail = AIGW_R_E400_SYNTAX;     // unterminated string
    if (!fail && ntok > P.tok_cap) fail = AIGW_R_TOKENS;
    if (!fail && ntok < 2) fail = ntok ? AIGW_R_ROOT : AIGW_R_E400_SYNTAX;   // a lone scalar (null decodes to the zero request) is left to the stock path
    if (fail) atomicMin(&S.fail, (uint32_t)fail);
    __syncthreads();
    // ---- brackets: exactly one object (the root), at most one array
    if (S.fail == kNoFail) {
      for (uint32_t j = tid; j < ntok; j += kEmbThreads) {
        const uint32_t ty = tok[j] >> 24;
        if (ty == '{') atomicAdd(&S.n_lc, 1u); else if (ty == '}') atomicAdd(&S.n_rc, 1u);
        else if (ty == '[') { atomicAdd(&S.n_lb, 1u); atomicMin(&S.lb, j); } else if (ty == ']') { atomicAdd(&S.n_rb, 1u); atomicMax(&S.rb, j); }
      }
    }
    __syncthreads();
    if (S.fail == kNoFail && tid == 0) {
      int f = 0;
      if ((tok[0] >> 24) != '{') f = (tok[0] >> 24) == '[' || (tok[0] >> 24) == T_QOPEN || (tok[0] >> 24) == T_SCALAR ? AIGW_R_ROOT : AIGW_R_E400_SYNTAX;
      else if ((tok[ntok - 1] >> 24) != '}' || S.n_rc != S.n_lc) f = S.n_lc > 1 || S.n_rc > 1 ? AIGW_R_DEPTH : AIGW_R_E400_SYNTAX;
      else if (S.n_lc != 1 || S.n_lb > 1 || S.n_rb > 1) f = AIGW_R_DEPTH;
      else if (S.n_lb != S.n_rb || (S.n_lb == 1 && S.lb >= S.rb)) f = AIGW_R_E400_SYNTAX;
      if (f) S.fail = (uint32_t)f;
    }
    __syncthreads();
    // ---- interior of the array: quote, quote, comma, quote, quote, comma, ..., quote, quote
    if (S.fail == kNoFail && S.n_lb == 1) {
      const uint32_t lb = S.lb, rb = S.rb, nint = rb - lb - 1u;
      if (nint != 0 && nint % 3u != 2u) { if (tid == 0) atomicMin(&S.fail, (uint32_t)AIGW_R_UNSUPPORTED_FIELD); }
      else for (uint32_t r = tid; r < nint; r += kEmbThreads) {
        const uint32_t ty = tok[lb + 1u + r] >> 24, m = r % 3u;
        const uint32_t want = m == 0 ? T_QOPEN : m == 1 ? T_QCLOSE : (uint32_t)',';
        if (ty != want) atomicMin(&S.fail, (uint32_t)AIGW_R_UNSUPPORTED_FIELD);   // a non-string element, a missing comma: outside the decided shape
      }
    }
    __syncthreads();
    // ---- the top-level members, sequentially
    if (S.fail == kNoFail && tid == 0) {
      int f = 0, st400 = 0;
      uint32_t j = 1, seen = 0, model_o = 0, model_l = 0, n_inputs = 0, s_open = 0, s_close = 0;
      auto ty = [&](uint32_t k) -> uint32_t { return k < ntok ? tok[k] >> 24 : 0u; };
      auto ps = [&](uint32_t k) -> uint32_t { return tok[k] & 0xffffffu; };
      if (ty(1) == '}') { if (ntok != 2) f = AIGW_R_E400_SYNTAX; }
      else for (;;) {
        if (ty(j) != T_QOPEN || ty(j + 1) != T_QCLOSE || ty(j + 2) != ':') { f = AIGW_R_E400_SYNTAX; break; }
        const uint8_t* kp = body + ps(j) + 1u; const uint32_t kl = ps(j + 1) - ps(j) - 1u;
        int id = emb_key_is(kp, kl, "model", 5) ? 0 : emb_key_is(kp, kl, "input", 5) ? 1 : emb_key_is(kp, kl, "encoding_format", 15) ? 2 : emb_key_is(kp, kl, "dimensions", 10) ? 3 : emb_key_is(kp, kl, "user", 4) ? 4 : -1;
        if (id < 0) { f = AIGW_R_UNSUPPORTED_FIELD; break; }
        if (seen & (1u << id)) { f = AIGW_R_DUP_KEY; break; }
        seen |= 1u << id;
        const uint32_t v = j + 3, tv = ty(v);
        uint32_t next;
        int kind;   // 0 string, 1 null, 2 bool, 3 integer, 4 other number, 5 the array
        if (tv == T_QOPEN) { if (ty(v + 1) != T_QCLOSE) { f = AIGW_R_E400_SYNTAX; break; } kind = 0; next = v + 2; }
        else if (tv == T_SCALAR) {
          if (v + 1 >= ntok) { f = AIGW_R_E400_SYNTAX; break; }
          uint32_t e = ps(v + 1); const uint32_t b = ps(v);
          while (e > b && (body[e - 1] == ' ' || body[e - 1] == '\n' || body[e - 1] == '\r' || body[e - 1] == '\t')) e--;
          const int sk = emb_scalar_kind(body + b, e - b);
          if (!sk) { f = AIGW_R_E400_SYNTAX; break; }
          kind = sk; next = v + 1;
        }
        else if (tv == '[') { if (id != 1) { f = AIGW_R_UNSUPPORTED_FIELD; break; } kind = 5; next = S.rb + 1u; }
        else { f = AIGW_R_E400_SYNTAX; break; }
        if (id == 0) { if (kind == 0) { model_o = ps(v) + 1u; model_l = ps(v + 1) - ps(v) - 1u; } else if (kind != 1) st400 = 1; }
        else if (id == 1) {
          if (kind == 0) { n_inputs = 1; s_open = ps(v); s_close = ps(v + 1); }
          else if (kind == 5) { const uint32_t nint = S.rb - S.lb - 1u; n_inputs = (nint + 1u) / 3u; }
          else st400 = 1;   // null included (the union's UnmarshalJSON runs on null too): "invalid input type (must be string, object, or array)"
        }
        else if (id == 3) { if (kind != 1 && kind != 3) st400 = 1; }
        else { if (kind > 1) st400 = 1; }
        const uint32_t t2 = ty(next);
        if (t2 == ',') { j = next + 1; continue; }
        if (t2 == '}' && next == ntok - 1) break;
        f = AIGW_R_E400_SYNTAX; break;
      }
      if (!f && S.n_lb == 1 && !(seen & 2u)) f = AIGW_R_UNSUPPORTED_FIELD;   // cannot happen: the only array is input's
      if (!f && st400) f = AIGW_R_E400_TYPE;
      if (!f && model_l > 0xffffu) f = AIGW_R_TOO_LARGE;
      if (!f && n_inputs) {
        const uint32_t b = atomicAdd(P.text_used, n_inputs);
        if ((uint64_t)b + n_inputs > P.text_cap) f = AIGW_R_ARENA_FULL; else S.text_base = b;
      }
      if (f) S.fail = (uint32_t)f;
      else { res.model_off = model_o; res.model_len = (uint16_t)model_l; S.n_inputs = n_inputs; S.str_open = s_open; S.str_close = s_close; }
    }
    __syncthreads();
    if (S.fail == kNoFail) {
      const uint32_t n = S.n_inputs, tb = S.text_base;
      if (S.n_lb == 1) {
        const uint32_t lb = S.lb;
        for (uint32_t k = tid; k < n; k += kEmbThreads) {
          const uint32_t o = tok[lb + 1u + 3u * k] & 0xffffffu, cpos = tok[lb + 2u + 3u * k] & 0xffffffu;
          P.text_off[tb + k] = boff + o + 1u; P.text_len[tb + k] = cpos - o - 1u;
        }
      } else if (n == 1 && tid == 0) { P.text_off[tb] = boff + S.str_open + 1u; P.text_len[tb] = S.str_close - S.str_open - 1u; }
    }
    if (tid == 0) {
      const int f = S.fail == kNoFail ? 0 : (int)S.fail;
      if (!f) { res.status = AIGW_OK; res.n_inputs = S.n_inputs; res.first_text = S.text_base; }
      else { res.reason = (uint8_t)f; res.status = f >= 48 ? AIGW_INTERNAL : f >= 40 ? AIGW_INVALID_422 : f >= 32 ? AIGW_MALFORMED_400 : AIGW_DECLINED; }
      P.results[doc] = res;
    }
  }
}

// tokens of a request = sum over its inputs; an input the BPE kernel declined (0xFFFFFFFF) is counted in declined_inputs
__global__ void __launch_bounds__(256) emb_sum_kernel(aigw_emb_count_result* results, uint32_t n, const uint32_t* counts) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t doc = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (doc >= n) return;
  const aigw_emb_count_result r = results[doc];
  if (r.status != AIGW_OK) return;
  uint32_t sum = 0, decl = 0;
  for (uint32_t k = lane; k < r.n_inputs; k += 32) { const uint32_t c = counts[r.first_text + k]; if (c == 0xffffffffu) decl++; else sum += c; }
  sum = __reduce_add_sync(0xffffffffu, sum); decl = __reduce_add_sync(0xffffffffu, decl);
  if (lane == 0) { results[doc].tokens = sum; results[doc].declined_inputs = decl; }
}

int emb_scan_grid(int sm_count) { return sm_count * 4; }

cudaError_t launch_emb_scan(const EmbScanParams& P, int sm_count, cudaStream_t st) {
  const unsigned grid = (unsigned)emb_scan_grid(sm_count);
  emb_scan_kernel<<<P.n < grid ? (P.n ? P.n : 1u) : grid, kEmbThreads, 0, st>>>(P);
  return cudaGetLastError();
}
cudaError_t launch_emb_sum(aigw_emb_count_result* results, uint32_t n, const uint32_t* counts, cudaStream_t st) {
  if (!n) return cudaSuccess;
  emb_sum_kernel<<<(n + 7) / 8, 256, 0, st>>>(results, n, counts);
  return cudaGetLastError();
}

}  // namespace aigw
