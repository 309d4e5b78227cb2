// Cohere /v2/rerank requests above the translate pass's 64 KiB ceiling (and below it): RerankEndpointSpec.ParseBody over
// cohere.RerankV2Request and cohereToCohereTranslatorV2Rerank.RequestBody, with the semantics plan_rerank (chat_walk_impl.cuh)
// gives AIGW_SCHEMA_RERANK_COHERE.  sm_90a only.
//
// rerank_scan_kernel: one CTA of 256 threads per request, persistent CTAs pulling requests from a counter; the body streams
// through in 8 KB tiles (32 bytes per thread) with the next tile's loads in flight, as in emb_scan_kernel:
//   escapes   a thread's escaped bytes follow odd backslash runs (the odd-run rule from a carry-in bit).  Its carry-out is the
//             parity of its trailing run, or its carry-in when all 32 bytes are backslashes, so its carry-in comes from the
//             nearest preceding thread that is not all backslashes (one ballot and shuffles inside the warp, 8 shared words
//             across warps, the tile carry before the first).  Escaped bytes must be one of "\/bfnrtu, \u takes 4 hex digits
//             (read from global memory: they may lie in the next thread or tile); anything else DECLINES (AIGW_R_ESCAPE), as
//             the translate pass does.  Lone surrogates and invalid UTF-8 pass, as in Go.
//   strings   in-string parity of the unescaped quotes: prefix xor inside the thread, xor-scan over the CTA
//   tokens    structural bytes outside strings, both unescaped quotes of every string, the first byte of every scalar, compacted
//             into the CTA's workspace slice (position | type << 24) with a block-wide prefix sum
//   depth     bracket depth after every token by a block-wide prefix sum: a negative or non-zero final depth is a syntax error,
//             depth above 48 DECLINES (AIGW_R_DEPTH); the same pass checks the grammar of every scalar and finds the root's first
//             "documents" array
//   documents its interior is checked in parallel by a local neighbour rule (each element a string or a scalar, commas between):
//             null elements decode, numbers and bools are the decoder's type error; an object or array element sends the whole
//             array to the serial walk below
//   members   one thread walks the root's members in body order with plan_rerank's checks, and grammar-checks and skips the
//             values of unknown members (containers too, with a 48-level bit stack).  Its cost is linear in the tokens outside
//             the documents array: the other members of a real rerank request are a few scalars and small objects.
// The failure that counts: a decline of the scan (control byte in a string, bad escape, tokens, depth) first, then a syntax
// error anywhere (Go checks the whole body before it decodes), then the first problem of the member walk in body order.
//
// rerank_emit_kernel: one CTA per request with a record.  It bump-allocates the record (16-byte aligned, AIGW_R_OUT_SPACE when it
// does not fit) and writes [":path"][body]: a streaming copy with one splice, 16-byte stores, source words realigned with funnel
// shifts; only the 16-byte chunks that straddle the path, the splice or the end are assembled byte by byte.
#include "rerank_large_kernel.cuh"

#include "classify.cuh"
#include "scan_common.cuh"
#include "scan_stream.cuh"

namespace aigw {

static constexpr int kRrThreads = 256;
static constexpr uint32_t kRrTile = kRrThreads * 32;
static constexpr uint32_t FULL = 0xffffffffu;
// the request's workspace: at most 512 MiB for the whole grid
static constexpr uint64_t kRrWorkspace = 512ull << 20;

struct RrShared {
  uint32_t wesc[2][8], wpar[2][8], wlast[2][8], wcnt[2][8];
  int wsum[2][8];
  uint32_t doc, fail;        // fail: lowest reason raised by the scan / structure passes (declines, below 32, win); kNone = none
  uint32_t dlb, drb;         // tokens of the first documents array of the root and of its closing bracket
  uint32_t dnest, dsyn, dtype;
};

__global__ void __launch_bounds__(kRrThreads, 4) rerank_scan_kernel(const RerankLargeParams P) {
  __shared__ RrShared S;
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const uint32_t lt = (1u << lane) - 1u;
  uint32_t* tok = P.tok_ws + (size_t)blockIdx.x * P.tok_cap;
  uint8_t* dep = P.dep_ws + (size_t)blockIdx.x * P.tok_cap;
  for (;;) {
    __syncthreads();
    if (tid == 0) { S.doc = atomicAdd(P.next_scan, 1u); S.fail = kNone; S.dlb = S.drb = kNone; S.dnest = S.dsyn = S.dtype = 0; }
    __syncthreads();
    const uint32_t doc = S.doc;
    if (doc >= P.n) break;
    const uint8_t* body = P.bodies + P.offsets[doc];
    const uint32_t len = P.lens[doc];
    const uint32_t cap = min(rerank_tok_cap(len), P.tok_cap);
    int fail = 0;
    uint32_t ntok = 0;
    if (P.call_reason) fail = (int)P.call_reason;
    else if (len >= (1u << 24) || len == 0) fail = len ? AIGW_R_TOO_LARGE : AIGW_R_E400_SYNTAX;
    else if (((uintptr_t)body) & 15u) fail = AIGW_R_ARGS;   // the arena convention: every request starts 16-byte aligned
    uint32_t in_str = 0, prev_sc = 0, esc_c = 0;   // carries across tiles (uniform over the CTA)
    uint4 na = make_uint4(0, 0, 0, 0), nb = na;
    if (!fail && tid * 32u + 32u <= len) { na = __ldg((const uint4*)(body + tid * 32u)); nb = __ldg((const uint4*)(body + tid * 32u + 16)); }
    if (!fail) for (uint32_t base = 0, it = 0; base < len; base += kRrTile, it ^= 1u) {
      const uint32_t pos0 = base + tid * 32u;
      uint32_t w[8];
      if (pos0 + 32u <= len) {
        w[0] = na.x; w[1] = na.y; w[2] = na.z; w[3] = na.w; w[4] = nb.x; w[5] = nb.y; w[6] = nb.z; w[7] = nb.w;
        if (pos0 + kRrTile + 32u <= len) { na = __ldg((const uint4*)(body + pos0 + kRrTile)); nb = __ldg((const uint4*)(body + pos0 + kRrTile + 16)); }
      } else {
#pragma unroll
        for (int k = 0; k < 8; k++) {   // past the end: spaces, which are no token and no escape
          uint32_t v = 0x20202020u;
          const uint32_t p = pos0 + 4u * k;
          if (p + 4u <= len) v = __ldg((const uint32_t*)(body + p));
          else if (p < len) { v = 0; for (uint32_t q = 0; q < 4; q++) v |= (uint32_t)(p + q < len ? body[p + q] : 0x20u) << (8u * q); }
          w[k] = v;
        }
      }
      const ByteClasses c = classify32(w);
      // ---- escapes: carry-in from the nearest preceding thread that is not all backslashes
      const uint32_t bsm = c.bslash;
      const bool allbs = bsm == FULL;
      const uint32_t tpar = __clz(~bsm) & 1u;   // parity of the trailing backslash run (not all backslashes)
      const uint32_t nbm = __ballot_sync(FULL, !allbs);
      const uint32_t below = nbm & lt;
      const uint32_t lane_c = __shfl_sync(FULL, tpar, below ? 31u - __clz(below) : 0u);
      const uint32_t warp_c = __shfl_sync(FULL, tpar, nbm ? 31u - __clz(nbm) : 0u);
      if (lane == 0) S.wesc[it][warp] = nbm ? 2u | warp_c : 0u;
      __syncthreads();
      uint32_t cin_w = esc_c, cout_t = esc_c;
#pragma unroll
      for (uint32_t k = 0; k < 8; k++) { const uint32_t e = S.wesc[it][k]; if (e) { if (k < warp) cin_w = e & 1u; cout_t = e & 1u; } }
      const uint32_t cin = below ? lane_c : cin_w;
      const uint32_t esc = bsm | cin ? escaped_mask(bsm, cin) & (pos0 >= len ? 0u : pos0 + 32u <= len ? FULL : (1u << (len - pos0)) - 1u) : 0u;
      // ---- string parity of the unescaped quotes
      const uint32_t uq = c.quote & ~esc;
      const uint32_t bal = __ballot_sync(FULL, (__popc(uq) & 1u) != 0);
      if (lane == 0) S.wpar[it][warp] = __popc(bal) & 1u;
      __syncthreads();
      uint32_t pre = 0, tot = 0;
#pragma unroll
      for (uint32_t k = 0; k < 8; k++) { const uint32_t v = S.wpar[it][k]; tot ^= v; if (k < warp) pre ^= v; }
      const uint32_t in0 = in_str ^ pre ^ (__popc(bal & lt) & 1u);
      const uint32_t ps = prefix_xor32(uq) ^ (in0 ? FULL : 0u);   // bit i: inside a string after byte i (the opening quote counts)
      const uint32_t inside = ps & ~uq;
      const uint32_t out = ~ps & ~uq;
      if (c.ctl & inside) raise_min(fail, AIGW_R_CTRL_IN_STRING);
      if ((c.ctl & out & ~c.ws) || (bsm & out)) raise_min(fail, AIGW_R_E400_SYNTAX);
      for (uint32_t e = esc & inside; e;) {
        const uint32_t i = __ffs(e) - 1u; e &= e - 1u;
        const uint32_t p = pos0 + i, ch = body[p];
        const bool ok = ch == '"' || ch == '\\' || ch == '/' || ch == 'b' || ch == 'f' || ch == 'n' || ch == 'r' || ch == 't' ||
                        (ch == 'u' && p + 4u < len && is_hex(body[p + 1]) && is_hex(body[p + 2]) && is_hex(body[p + 3]) && is_hex(body[p + 4]));
        if (!ok) raise_min(fail, AIGW_R_ESCAPE);
      }
      // ---- tokens
      const uint32_t sc = out & ~c.op & ~c.ws;
      if (lane == 31) S.wlast[it][warp] = sc >> 31;
      uint32_t prev = __shfl_up_sync(FULL, sc >> 31, 1);
      __syncthreads();
      if (lane == 0) prev = warp == 0 ? prev_sc : S.wlast[it][warp - 1];
      const uint32_t sc_start = sc & ~((sc << 1) | prev);
      uint32_t tk = (c.op & out) | uq | sc_start;
      const uint32_t cnt = __popc(tk);
      uint32_t incl = cnt;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, d); if ((int)lane >= d) incl += v; }
      if (lane == 31) S.wcnt[it][warp] = incl;
      const uint32_t last_sc_tile = S.wlast[it][7];
      __syncthreads();
      uint32_t wpre = 0, wtot = 0;
#pragma unroll
      for (uint32_t k = 0; k < 8; k++) { const uint32_t v = S.wcnt[it][k]; wtot += v; if (k < warp) wpre += v; }
      uint32_t off = ntok + wpre + incl - cnt;
      while (tk) {
        const uint32_t i = __ffs(tk) - 1u; tk &= tk - 1u;
        const uint32_t p = pos0 + i, bit = 1u << i;
        const uint32_t ty = (uq & bit) ? ((ps & bit) ? T_QOPEN : T_QCLOSE) : (c.op & bit) ? (uint32_t)body[p] : T_SCALAR;
        if (off < cap) tok[off] = p | (ty << 24);
        off++;
      }
      ntok += wtot; in_str ^= tot; prev_sc = last_sc_tile; esc_c = cout_t;
    }
    if (!fail && in_str) fail = AIGW_R_E400_SYNTAX;   // unterminated string
    if (ntok > cap) raise_min(fail, AIGW_R_TOKENS);
    if (!fail && ntok == 0) fail = AIGW_R_E400_SYNTAX;   // white space only
    if (fail) atomicMin(&S.fail, (uint32_t)fail);
    __syncthreads();
    // ---- bracket depth after every token (block-wide prefix sum); the first "documents" array of the root
    if (S.fail == kNone) {
      int carry = 0;
      uint32_t it = 0;
      for (uint32_t b0 = 0; b0 < ntok; b0 += kRrThreads, it ^= 1u) {
        const uint32_t j = b0 + tid;
        const uint32_t ty = j < ntok ? tok[j] >> 24 : 0u;
        const int d = (ty == '{' || ty == '[') ? 1 : (ty == '}' || ty == ']') ? -1 : 0;
        int incl = d;
#pragma unroll
        for (int s = 1; s < 32; s <<= 1) { const int v = __shfl_up_sync(FULL, incl, s); if ((int)lane >= s) incl += v; }
        if (lane == 31) S.wsum[it][warp] = incl;
        __syncthreads();
        int pre = 0, tot = 0;
#pragma unroll
        for (uint32_t k = 0; k < 8; k++) { const int v = S.wsum[it][k]; tot += v; if (k < warp) pre += v; }
        const int da = carry + pre + incl;
        carry += tot;
        if (j < ntok) {
          if (da < 0) atomicMin(&S.fail, (uint32_t)AIGW_R_E400_SYNTAX);
          else if (da > (int)kRerankMaxDepth) atomicMin(&S.fail, (uint32_t)AIGW_R_DEPTH);
          dep[j] = (uint8_t)(da < 0 ? 0 : da > 255 ? 255 : da);
          if (ty == T_SCALAR && !ScanToks{tok, ntok, body, len}.scalar_kind(j)) atomicMin(&S.fail, (uint32_t)AIGW_R_E400_SYNTAX);
          if (ty == '[' && da == 2 && j >= 4 && (tok[j - 1] >> 24) == ':' && (tok[j - 2] >> 24) == T_QCLOSE && (tok[j - 3] >> 24) == T_QOPEN) {
            const uint32_t o = (tok[j - 3] & 0xffffffu) + 1u;
            if (scan_key_is(body + o, (tok[j - 2] & 0xffffffu) - o, "documents", 9)) atomicMin(&S.dlb, j);
          }
        }
      }
      if (carry != 0 && tid == 0) atomicMin(&S.fail, (uint32_t)AIGW_R_E400_SYNTAX);
    }
    __syncthreads();
    // ---- the documents array: its closing bracket, then its interior by the neighbour rule
    const uint32_t dlb = S.dlb;
    if (S.fail == kNone && dlb != kNone) {
      for (uint32_t j = dlb + 1u + tid; j < ntok; j += kRrThreads) {
        const uint32_t ty = tok[j] >> 24;
        if ((ty == ']' || ty == '}') && dep[j] == 1) atomicMin(&S.drb, j);
      }
      __syncthreads();
      const uint32_t drb = S.drb;
      if (drb == kNone || (tok[drb] >> 24) != ']') { if (tid == 0) S.dnest = 1; }
      else for (uint32_t j = dlb + 1u + tid; j < drb; j += kRrThreads) {
        const uint32_t ty = tok[j] >> 24, pv = tok[j - 1] >> 24, nx = tok[j + 1] >> 24;
        bool syn = false;
        if (ty == '{' || ty == '[' || ty == '}' || ty == ']') { S.dnest = 1; continue; }
        if (ty == T_QOPEN) syn = !(pv == '[' || pv == ',') || nx != T_QCLOSE;
        else if (ty == T_QCLOSE) syn = !(nx == ',' || nx == ']');
        else if (ty == T_SCALAR) {
          syn = !(pv == '[' || pv == ',') || !(nx == ',' || nx == ']');
          if (!syn) {
            const ScanToks W{tok, ntok, body, len};
            const int k = W.scalar_kind(j);
            if (!k) syn = true; else if (k != 1) S.dtype = 1;   // a number or a bool where []string decodes
          }
        } else if (ty == ',') syn = !(pv == T_QCLOSE || pv == T_SCALAR) || !(nx == T_QOPEN || nx == T_SCALAR);
        else syn = true;   // ':'
        if (syn) S.dsyn = 1;
      }
      __syncthreads();
      if (tid == 0 && !S.dnest && S.dsyn) atomicMin(&S.fail, (uint32_t)AIGW_R_E400_SYNTAX);
    }
    __syncthreads();
    // ---- the root's members, in body order (plan_rerank)
    if (tid == 0) {
      aigw_doc_result res;
      res.out_off = 0; res.body_len = 0; res.path_len = 0; res.status = AIGW_DECLINED; res.reason = 0; res.model_off = 0; res.model_len = 0;
      res.body_kind = AIGW_BODY_UNCHANGED; res.flags = 0; res.in_len = len; res._pad = 0;
      RerankSplice sp{0, 0, 0, 0, 0};
      int f = S.fail == kNone ? 0 : (int)S.fail;
      if (!f) {
        const ScanToks W{tok, ntok, body, len};
        int prob = 0;            // first problem of the walk: a decline or the decoder's type error
        bool syn = false;
        uint32_t model_v = kNone;
        bool dummy = false;
        if (W.ty(0) != '{') {
          // a root that is not an object: the decoder's type error once the body is valid JSON; a null root declines
          if (W.skip_value(0, false, dummy) != ntok) syn = true;
          else prob = W.ty(0) == T_SCALAR && W.scalar_kind(0) == 1 ? AIGW_R_ROOT : AIGW_R_E400_TYPE;
        } else {
          uint32_t seen = 0, j = 1;
          if (W.ty(1) == '}') j = 2;
          else for (;;) {
            if (W.ty(j) != T_QOPEN || W.ty(j + 1) != T_QCLOSE || W.ty(j + 2) != ':') { syn = true; break; }
            const uint32_t ko = W.ps(j) + 1u, kl = W.ps(j + 1) - ko;
            const bool kesc = W.has_backslash(ko, ko + kl);
            const uint8_t* kp = body + ko;
            const int id = kesc ? -1 : scan_key_is(kp, kl, "model", 5) ? 0 : scan_key_is(kp, kl, "query", 5) ? 1 : scan_key_is(kp, kl, "documents", 9) ? 2
                                    : scan_key_is(kp, kl, "top_n", 5) ? 3 : scan_key_is(kp, kl, "max_tokens_per_doc", 18) ? 4 : -1;
            int p = kesc ? AIGW_R_ESCAPE : 0;
            if (id >= 0) { if (seen & (1u << id)) p = AIGW_R_DUP_KEY; seen |= 1u << id; }
            const uint32_t v = j + 3, tv = W.ty(v);
            uint32_t e;
            if (id == 2 && v == dlb && !S.dnest) { e = S.drb + 1u; if (!p && S.dtype) p = AIGW_R_E400_TYPE; }
            else {
              bool bad = false;
              e = W.skip_value(v, id == 2 && tv == '[', bad);
              if (e == kNone) { syn = true; break; }
              if (!p && id >= 0 && !(tv == T_SCALAR && W.scalar_kind(v) == 1)) {   // null is a no-op for every member
                if (id <= 1) { if (tv != T_QOPEN) p = AIGW_R_E400_TYPE; }
                else if (id == 2) { if (tv != '[' || bad) p = AIGW_R_E400_TYPE; }
                else if (tv != T_SCALAR || W.scalar_kind(v) < 3 || !W.int64_ok(v)) p = AIGW_R_E400_TYPE;
              }
            }
            if (!p && id == 0) model_v = v;
            if (p && !prob) prob = p;
            const uint32_t t2 = W.ty(e);
            j = e + 1u;
            if (t2 == ',') continue;
            if (t2 != '}') syn = true;
            break;
          }
          if (!syn && j != ntok) syn = true;   // bytes after the root
        }
        f = syn ? AIGW_R_E400_SYNTAX : prob;
        if (!f && model_v != kNone && W.ty(model_v) == T_QOPEN) {
          const uint32_t mo = W.ps(model_v) + 1u, ml = W.ps(model_v + 1) - mo;
          if (W.has_backslash(mo, mo + ml)) f = AIGW_R_ESCAPE;
          else if (ml > 0xffffu) f = AIGW_R_TOO_LARGE;   // model_len is 16 bits
          else { res.model_off = mo; res.model_len = (uint16_t)ml; }
        }
        if (!f && P.override_len && !P.override_ok) f = AIGW_R_UNSUPPORTED_FIELD;
        if (!f) {
          res.path_len = (uint16_t)P.path_len;
          if (P.override_len) {
            // sjson set of "model": the value spliced in place, or the member appended before the root's '}' (the bytes outside
            // the root are dropped then)
            if (model_v != kNone) {
              const uint32_t b = W.ps(model_v);
              sp = RerankSplice{0, b, W.ty(model_v) == T_QOPEN ? W.ps(model_v + 1) + 1u : b + 4u, len, 1};
            } else {
              const uint32_t rc = W.ps(ntok - 1);
              sp = RerankSplice{W.ps(0), rc, rc, rc + 1u, ntok == 2 ? 3u : 2u};
            }
          } else if (P.force_mutation) sp = RerankSplice{0, len, len, len, 0};
          if (P.override_len || P.force_mutation) {
            const uint32_t lit = sp.lit == 0 ? 0u : P.override_len + 2u + (sp.lit == 1 ? 0u : sp.lit == 2 ? 9u : 8u);
            res.body_kind = AIGW_BODY_BYTES;
            res.body_len = (sp.keep_e - sp.keep_b) - (sp.cut_e - sp.cut_b) + lit;
          }
        }
      }
      if (!f) res.status = AIGW_OK;
      else { res.reason = (uint8_t)f; res.status = f >= 48 ? AIGW_INTERNAL : f >= 40 ? AIGW_INVALID_422 : f >= 32 ? AIGW_MALFORMED_400 : AIGW_DECLINED; }
      P.results[doc] = res;
      P.splice[doc] = sp;
    }
  }
}

// byte o of a record: [path][body[keep_b, cut_b)][literal][body[cut_e, keep_e)], zero past its end
__device__ __forceinline__ uint32_t rec_byte(uint32_t o, const uint8_t* head, uint32_t pl, const uint8_t* lit, uint32_t nl, const uint8_t* body,
                                             const RerankSplice& sp, uint32_t total) {
  if (o < pl) return head[o];
  o -= pl;
  const uint32_t n1 = sp.cut_b - sp.keep_b;
  if (o < n1) return body[sp.keep_b + o];
  o -= n1;
  if (o < nl) return lit[o];
  o -= nl;
  return o < total - pl - n1 - nl ? body[sp.cut_e + o] : 0u;
}

__global__ void __launch_bounds__(kRrThreads) rerank_emit_kernel(const RerankLargeParams P) {
  // s_lit = ,"model":"<override>": a record's literal is a suffix of it (the quoted override from byte 9, the member with or
  // without its comma from byte 0 or 1)
  __shared__ uint8_t s_head[128], s_lit[160];
  // the record in hand, read and allocated by thread 0 alone and handed to the CTA through the barrier
  __shared__ uint32_t s_doc, s_pl, s_total;
  __shared__ unsigned long long s_off;
  __shared__ RerankSplice s_sp;
  const uint32_t tid = threadIdx.x;
  for (uint32_t k = tid; k < P.path_len; k += kRrThreads) s_head[k] = (uint8_t)P.path[k];
  const uint32_t lit_all = 11u + P.override_len;
  if (tid < lit_all) {
    const char* mm = ",\"model\":\"";
    s_lit[tid] = tid < 10u ? (uint8_t)mm[tid] : tid == lit_all - 1u ? (uint8_t)'"' : (uint8_t)P.override_model[tid - 10u];
  }
  for (;;) {
    __syncthreads();   // the previous record is written: the shared record state may change
    if (tid == 0) {
      const uint32_t doc = atomicAdd(P.next_emit, 1u);
      s_doc = doc; s_off = ~0ull;
      if (doc < P.n) {
        const aigw_doc_result r = P.results[doc];
        if (r.status == AIGW_OK) {
          s_sp = P.splice[doc];
          s_pl = r.path_len; s_total = (uint32_t)r.path_len + r.body_len;
          const unsigned long long size = ((unsigned long long)s_total + 15u) & ~15ull;
          const unsigned long long o = atomicAdd(P.out_used, size);
          if (o + size > P.out_capacity) {
            aigw_doc_result d = r;
            d.status = AIGW_DECLINED; d.reason = AIGW_R_OUT_SPACE; d.path_len = 0; d.body_len = 0; d.body_kind = AIGW_BODY_UNCHANGED;
            P.results[doc] = d;
          } else { P.results[doc].out_off = o; s_off = o; }
        }
      }
    }
    __syncthreads();
    const uint32_t doc = s_doc;
    if (doc >= P.n) break;
    if (s_off == ~0ull) continue;   // not OK, or no room: no record
    const RerankSplice sp = s_sp;
    const uint32_t pl = s_pl, total = s_total;
    const uint8_t* lit = s_lit + (sp.lit == 1 ? 9u : sp.lit == 3 ? 1u : 0u);
    const uint32_t nl = sp.lit == 0 ? 0u : sp.lit == 1 ? P.override_len + 2u : sp.lit == 3 ? lit_all - 1u : lit_all;
    const uint8_t* body = P.bodies + P.offsets[doc];
    uint4* dst = (uint4*)(P.out + s_off);
    const uint32_t n1 = sp.cut_b - sp.keep_b, b2 = pl + n1 + nl;   // output offsets of the two body segments: [pl, pl+n1), [b2, total)
    const uint32_t nchunk = (total + 15u) >> 4;
    for (uint32_t c = tid; c < nchunk; c += kRrThreads) {
      const uint32_t o0 = c << 4;
      uint4 v;
      if (o0 >= pl && o0 + 16u <= pl + n1) v = load16_unaligned(body + sp.keep_b + (o0 - pl));
      else if (o0 >= b2 && o0 + 16u <= total) v = load16_unaligned(body + sp.cut_e + (o0 - b2));
      else {
        uint32_t x[4] = {0, 0, 0, 0};
#pragma unroll
        for (uint32_t b = 0; b < 16; b++) x[b >> 2] |= rec_byte(o0 + b, s_head, pl, lit, nl, body, sp, total) << (8u * (b & 3u));
        v = make_uint4(x[0], x[1], x[2], x[3]);
      }
      dst[c] = v;
    }
  }
}

int rerank_scan_grid(int sm_count, uint32_t tok_cap) {
  const uint64_t per_cta = (uint64_t)tok_cap * 5u;
  uint64_t g = kRrWorkspace / per_cta;
  if (g > (uint64_t)sm_count * 4u) g = (uint64_t)sm_count * 4u;
  return g < 1 ? 1 : (int)g;
}

cudaError_t launch_rerank_large(const RerankLargeParams& P, int sm_count, cudaStream_t st) {
  const unsigned grid = (unsigned)rerank_scan_grid(sm_count, P.tok_cap);
  rerank_scan_kernel<<<P.n < grid ? (P.n ? P.n : 1u) : grid, kRrThreads, 0, st>>>(P);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const unsigned egrid = (unsigned)sm_count * 8u;
  rerank_emit_kernel<<<P.n < egrid ? (P.n ? P.n : 1u) : egrid, kRrThreads, 0, st>>>(P);
  return cudaGetLastError();
}

}  // namespace aigw
