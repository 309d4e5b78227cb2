// The stages that chat_large_kernel (chat_large_kernel.cu), responses_large_kernel (responses_large_kernel.cu) and
// completions_large_kernel (completions_large_kernel.cu) share: one CTA of 256 threads streams one request, persistent CTAs pulling
// requests from a counter.  Each kernel supplies only its walk and plan (thread 0); the scan, the depth pass, the grammar check
// and the emit are this file's, and so is the flat-array stage that only a walker with kFlatArrays compiles in.
//   scan      the body streams through in 8 KB tiles (32 bytes per thread), as in emb_large_kernel: escapes by the odd-run rule with
//             a carry across threads and tiles, escape validation, in-string parity, token compaction.  Every token also gets the
//             number of escaped bytes, and of escapes the encoder re-spells (\/ \b \f \u), in front of it: a string holds a
//             backslash (or a re-spelled escape) exactly when the counts of its two quotes differ.  A lone surrogate anywhere
//             declines (AIGW_R_ESCAPE): the translate pass declines one only in the strings it echoes.
//   depth     bracket depth after every token by a block-wide prefix sum (depth above 48 declines), the grammar of every scalar,
//             escaped keys (declined: AIGW_R_ESCAPE)
//   flat      (kFlatArrays walkers only) every thread: each '[' whose tokens up to its ']' alternate scalar, ',', scalar, ... gets
//             its jump and a flag byte (CL_FLAT, and CL_ALL_INT64 when every element is null or an int64 literal), by two
//             block-wide max-scans; the grammar check steps over such an array in one move
//   grammar   thread 0 checks the token grammar and writes the jump table (every bracket to its partner)
//   walk      thread 0: the kernel's walker (cl_request_loop's Walk) checks the members over the jump table in the translate
//             pass's order, and the kernel's cl_plan lays out the record as at most 12 copy ops (body spans and literals)
//   emit      16-byte output chunks with every thread busy: a chunk inside one body span is one realigned 16-byte load, the others
//             are assembled byte by byte.
#pragma once
#include "chat_large_kernel.cuh"
#include "classify.cuh"
#include "scan_common.cuh"
#include "scan_stream.cuh"

namespace aigw {
// internal linkage: both kernels' translation units include these definitions
namespace {

static constexpr int kClThreads = 256;
static constexpr uint32_t kClTile = kClThreads * 32;
static constexpr uint32_t FULL = 0xffffffffu;
// the workspace of the whole grid: at most 1 GiB
static constexpr uint64_t kClWorkspace = 1ull << 30;
static constexpr int kClOps = 12;
enum : uint32_t { OP_BODY = 0, OP_LIT = 1 };

struct ClShared {
  uint32_t wesc[2][8], wpar[2][8], wlast[2][8], wem[2][8];
  unsigned long long wcnt[2][8];
  uint32_t wsum[2][8];
  uint32_t doc, fail;
  uint32_t stk[kChatLargeMaxDepth];     // thread 0: the open brackets of the grammar check, then emit_any's containers
  uint32_t path_len, total, flags, body_kind, model_off, model_len;
  unsigned long long off;
  uint32_t op_kind[kClOps], op_src[kClOps], op_end[kClOps];
  uint8_t lits[512];
  uint16_t lit_off[CL_COUNT], lit_len[CL_COUNT];
};

__device__ __forceinline__ uint32_t hex4v(const uint8_t* p) {
  uint32_t h = 0;
  for (int k = 0; k < 4; k++) { const uint32_t c = p[k]; h = h * 16u + (c <= '9' ? c - '0' : (c | 0x20u) - 'a' + 10u); }
  return h;
}

// the escaped 'u' at p (four hex digits inside the body) is half of a surrogate pair that has no partner.  `prev_esc(q)`: byte q
// is escaped (q >= p - 6).
template <class PrevEsc>
__device__ __forceinline__ bool lone_surrogate(const uint8_t* body, uint32_t len, uint32_t p, PrevEsc prev_esc) {
  const uint32_t cp = hex4v(body + p + 1);
  if (cp >= 0xD800u && cp < 0xDC00u) {
    if (!(p + 10u < len && body[p + 5] == '\\' && body[p + 6] == 'u' && is_hex(body[p + 7]) && is_hex(body[p + 8]) && is_hex(body[p + 9]) &&
          is_hex(body[p + 10]))) return true;
    const uint32_t lo = hex4v(body + p + 7);
    return lo < 0xDC00u || lo >= 0xE000u;
  }
  if (cp >= 0xDC00u && cp < 0xE000u) {
    if (!(p >= 7u && body[p - 7] == '\\' && body[p - 6] == 'u' && prev_esc(p - 6u))) return true;
    const uint32_t hi = hex4v(body + p - 5);
    return hi < 0xD800u || hi >= 0xDC00u;
  }
  return false;
}

// the flat-array stage's flag byte of a '[' token
enum : uint8_t { CL_FLAT = 1, CL_ALL_INT64 = 2 };
static constexpr uint32_t kClFlatPer = 8;                          // consecutive tokens per thread
static constexpr uint32_t kClFlatTile = kClThreads * kClFlatPer;   // tokens per round of the stage

// ---------------------------------------------------------------- token view with a jump table
// tw: position (24) | type (8) as the scan writes it; cum: escaped bytes / re-spelled escapes in front of the token; jmp: the
// partner of every bracket.  ty() answers as the translate pass's Doc does: '"' for both quotes, a scalar's first byte.
struct LDoc {
  const uint8_t* s; uint32_t len; const uint32_t* tw; const uint2* cum; uint32_t* jmp; uint32_t nt;
  __device__ uint32_t ty(uint32_t i) const {
    if (i >= nt) return 0u;
    const uint32_t t = tw[i] >> 24;
    return t == T_QOPEN || t == T_QCLOSE ? (uint32_t)'"' : t == T_SCALAR ? (uint32_t)s[tw[i] & 0xffffffu] : t;
  }
  __device__ uint32_t tok(uint32_t i) const { return tw[i] & 0xffffffu; }
  __device__ uint32_t next(uint32_t i) const { const uint32_t b = ty(i); return b == '{' || b == '[' ? jmp[i] + 1u : b == '"' ? i + 2u : i + 1u; }
  __device__ uint32_t after(uint32_t v) const { uint32_t nx = next(v); if (ty(nx) == ',') nx++; return nx; }
  __device__ uint32_t str_off(uint32_t i) const { return tok(i) + 1u; }
  __device__ uint32_t str_len(uint32_t i) const { return tok(i + 1) - tok(i) - 1u; }
  __device__ bool str_has_backslash(uint32_t i) const { return cum[i + 1].x != cum[i].x; }
  __device__ bool str_nc(uint32_t i) const { return cum[i + 1].y != cum[i].y; }
  __device__ uint32_t scalar_end(uint32_t i) const {
    uint32_t e = i + 1 < nt ? tok(i + 1) : len;
    const uint32_t b = tok(i);
    while (e > b && (s[e - 1] == ' ' || s[e - 1] == '\n' || s[e - 1] == '\r' || s[e - 1] == '\t')) e--;
    return e;
  }
  __device__ bool raw_is(uint32_t i, const char* k, uint32_t kl) const { return scan_key_is(s + str_off(i), str_len(i), k, kl); }
};

// validate_tokens (chat_walk_impl.cuh) over an LDoc: the grammar of the token list and its jump table.  0, AIGW_R_SYNTAX or
// AIGW_R_DEPTH.  `scalars`: check each scalar's grammar here (the body's were checked by the depth pass).  kSkipFlat: a '[' that
// cl_flat_arrays flagged CL_FLAT in `flat` is a whole value, its jump already written (flags are read at '[' tokens only).  Such an
// array holds scalars and commas in the only order the grammar takes, and the depth pass has declined nesting above 48, so the
// step gives the answer the token-by-token check would.
template <bool kSkipFlat = false>
__device__ int cl_validate(LDoc& d, uint32_t* open_idx, bool scalars, const uint8_t* flat = nullptr) {
  uint64_t isobj = 0;
  uint32_t depth = 0, i = 0;
  int st = 0;   // 0 value expected, 1 key or '}', 2 key, 3 ':', 4 ',' or close, 5 value or ']', 6 done
  const uint32_t nt = d.nt;
  while (i < nt) {
    const uint32_t b = d.ty(i);
    if (st == 6) return AIGW_R_SYNTAX;
    if (b == '"') {
      if (i + 1 >= nt || d.ty(i + 1) != '"') return AIGW_R_SYNTAX;
      if (st == 1 || st == 2) st = 3;
      else if (st == 0 || st == 5) st = depth ? 4 : 6;
      else return AIGW_R_SYNTAX;
      i += 2; continue;
    }
    if (b == '{' || b == '[') {
      if (!(st == 0 || st == 5)) return AIGW_R_SYNTAX;
      if constexpr (kSkipFlat) if (b == '[' && (flat[i] & CL_FLAT)) { i = d.jmp[i] + 1u; st = depth ? 4 : 6; continue; }
      if (depth >= kChatLargeMaxDepth) return AIGW_R_DEPTH;
      open_idx[depth] = i;
      if (b == '{') { isobj |= 1ull << depth; st = 1; } else { isobj &= ~(1ull << depth); st = 5; }
      depth++; i++; continue;
    }
    if (b == '}' || b == ']') {
      if (depth == 0) return AIGW_R_SYNTAX;
      const bool obj = (isobj >> (depth - 1)) & 1u;
      if (b == '}') { if (!obj || !(st == 1 || st == 4)) return AIGW_R_SYNTAX; }
      else { if (obj || !(st == 5 || st == 4)) return AIGW_R_SYNTAX; }
      depth--;
      d.jmp[open_idx[depth]] = i;
      st = depth ? 4 : 6; i++; continue;
    }
    if (b == ':') { if (st != 3) return AIGW_R_SYNTAX; st = 0; i++; continue; }
    if (b == ',') { if (st != 4) return AIGW_R_SYNTAX; st = ((isobj >> (depth - 1)) & 1u) ? 2 : 0; i++; continue; }
    if (!(st == 0 || st == 5)) return AIGW_R_SYNTAX;
    if (scalars) { const uint32_t o = d.tok(i); if (!scan_scalar_kind(d.s + o, d.scalar_end(i) - o)) return AIGW_R_SYNTAX; }
    st = depth ? 4 : 6; i++;
  }
  return st == 6 ? 0 : AIGW_R_SYNTAX;
}

// ---------------------------------------------------------------- the record's copy ops (thread 0)
struct ClRec {
  ClShared& S;
  uint32_t n = 0, olen = 0;
  bool full = false;
  __device__ explicit ClRec(ClShared& s) : S(s) {}
  __device__ void push(uint32_t kind, uint32_t src, uint32_t len) {
    if (!len) return;
    if (n >= (uint32_t)kClOps) { full = true; return; }
    olen += len;
    S.op_kind[n] = kind; S.op_src[n] = src; S.op_end[n] = olen; n++;
  }
  __device__ void body(uint32_t b, uint32_t e) { push(OP_BODY, b, e - b); }
  __device__ void lit(uint32_t id) { push(OP_LIT, S.lit_off[id], S.lit_len[id]); }
};

// openai_request_result (chat_walk_impl.cuh) after the model span and the stream flag, for the passthroughs whose ParseBody returns
// no mutated body (/v1/responses, /v1/completions): ":path", then the body, its original bytes, or the model override spliced in.
// Edit B of chat_large_kernel's cl_plan without edit A.  Walk::Top has model_raw: the "model" value token, null included (the
// splice point), kNone when absent.  0 or the reason.
template <class Walk>
__device__ __forceinline__ int cl_openai_plan(const ChatLargeParams& P, Walk& W, const typename Walk::Top& t, ClRec& R) {
  const LDoc& d = W.d;
  const uint32_t len = d.len;
  R.lit(CL_OPENAI_PATH);
  R.S.path_len = R.olen;
  if (P.override_len == 0) {
    if (P.force_mutation) { R.body(0, len); R.S.body_kind = AIGW_BODY_BYTES; } else R.S.body_kind = AIGW_BODY_UNCHANGED;
    return 0;
  }
  if (!P.override_ok) return AIGW_R_UNSUPPORTED_FIELD;
  R.S.body_kind = AIGW_BODY_BYTES;
  if (t.model_raw != kNone) {   // replace the value
    R.body(0, d.tok(t.model_raw));
    R.lit(CL_QUOTE); R.lit(CL_OVERRIDE); R.lit(CL_QUOTE);
    R.body(W.is_str(t.model_raw) ? d.tok(t.model_raw + 1) + 1u : d.scalar_end(t.model_raw), len);
  } else {                      // append at the root: sjson rebuilds it, so the bytes outside its braces go
    const uint32_t root_close = d.jmp[0];
    R.body(d.tok(0), d.tok(root_close));
    if (root_close != 1u) R.lit(CL_COMMA);
    R.lit(CL_MODEL_MEMBER); R.lit(CL_QUOTE); R.lit(CL_OVERRIDE); R.lit(CL_QUOTE);
    R.body(d.tok(root_close), d.tok(root_close) + 1u);
  }
  return 0;
}

// ---------------------------------------------------------------- flat arrays (every thread)
// The scalar at body[o] is an integer literal within int64, cp_int64's rule: an optional '-', digits only, and at most
// 9223372036854775807 (…808 with the sign).  The depth pass has checked the scalar's grammar, so the digits end the number unless a
// fraction or an exponent follows them.
__device__ __forceinline__ bool cl_int64_literal(const uint8_t* s, uint32_t len, uint32_t o) {
  const uint32_t i = o + (s[o] == '-' ? 1u : 0u);
  uint32_t e = i;
  while (e < len && e - i < 20u && s[e] - '0' < 10u) e++;
  if (e == i || e - i > 19u) return false;
  if (e < len && (s[e] == '.' || (s[e] | 0x20u) == 'e')) return false;
  if (e - i < 19u) return true;
  const char* lim = "9223372036854775808";   // -2^63; the positive bound is one less
  int c = 0;
  for (uint32_t q = 0; q < 19u && !c; q++) c = (int)s[i + q] - (int)lim[q];
  return c < 0 || (c == 0 && i != o);
}

// Finds every flat array: a '[' at token a whose tokens up to its ']' at b alternate scalar, ',', scalar, ..., scalar (or none:
// "[]").  A token is a stop when it is neither a scalar nor a comma, or breaks the alternation with its predecessor (scalar
// scalar, ',' ',', '[' ','); a ']' whose predecessor is ',' is not flat.  An exclusive max-scan over the CTA, carried across
// rounds of kClFlatTile tokens, gives each ']' the last stop before it; when that stop is a '[', the array is flat: the ']' thread
// writes jmp[a] = b and flag[a] = CL_FLAT, with CL_ALL_INT64 when a second max-scan (the last scalar that is neither null nor an
// int64 literal) lies before a.  The stage only accepts: an array it does not flag is checked token by token as before.  It
// writes the flag of every '[' of the request (0 in the round of the '[', then the ']' thread's flag after that round's barrier),
// so no flag of an earlier request survives in the reused slice.  Called by every thread after the depth pass has passed.
__device__ __forceinline__ void cl_flat_arrays(const uint32_t* tokw, uint32_t* jmp, uint8_t* flag, const uint8_t* body, uint32_t len,
                                               uint32_t ntok) {
  __shared__ uint32_t s_stop[2][8], s_bad[2][8];
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  // carried across rounds: 2 * (1 + the index of the last stop) + (that stop is a '['), and 1 + the index of the last element
  // that is neither null nor an int64 literal; 0 for none
  uint32_t c_stop = 0, c_bad = 0, it = 0;
  for (uint32_t t0 = 0; t0 < ntok; t0 += kClFlatTile, it ^= 1u) {
    const uint32_t j0 = t0 + tid * kClFlatPer;
    uint32_t w[kClFlatPer];
    if (j0 + kClFlatPer <= ntok) {   // 32-byte aligned: the slice is, and j0 is a multiple of 8
      const uint4 a = *(const uint4*)(tokw + j0), b = *(const uint4*)(tokw + j0 + 4);
      w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w; w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
    } else {
#pragma unroll
      for (uint32_t k = 0; k < kClFlatPer; k++) w[k] = j0 + k < ntok ? tokw[j0 + k] : 0u;
    }
    const uint32_t pt0 = j0 && j0 <= ntok ? tokw[j0 - 1] >> 24 : 0u;
    uint32_t stopm = 0, badm = 0, lstop = 0, lbad = 0, pt = pt0;
#pragma unroll
    for (uint32_t k = 0; k < kClFlatPer; k++) {
      const uint32_t j = j0 + k, t = w[k] >> 24;
      if (j < ntok) {
        const bool stop = (t != T_SCALAR && t != ',') || (t == T_SCALAR && pt == T_SCALAR) || (t == ',' && (pt == ',' || pt == '['));
        if (stop) { stopm |= 1u << k; lstop = 2u * (j + 1u) + (t == '[' ? 1u : 0u); }
        if (t == '[') flag[j] = 0;
        if (t == T_SCALAR) {
          const uint32_t o = w[k] & 0xffffffu;
          if (body[o] != 'n' && !cl_int64_literal(body, len, o)) { badm |= 1u << k; lbad = j + 1u; }
        }
      }
      pt = t;
    }
    // block-wide exclusive max-scans of (lstop, lbad) over the threads, carried in from the earlier rounds
    uint32_t is = lstop, ib = lbad;
#pragma unroll
    for (int dd = 1; dd < 32; dd <<= 1) {
      const uint32_t xs = __shfl_up_sync(FULL, is, dd), xb = __shfl_up_sync(FULL, ib, dd);
      if ((int)lane >= dd) { is = max(is, xs); ib = max(ib, xb); }
    }
    if (lane == 31) { s_stop[it][warp] = is; s_bad[it][warp] = ib; }
    const uint32_t us = __shfl_up_sync(FULL, is, 1), ub = __shfl_up_sync(FULL, ib, 1);
    __syncthreads();
    uint32_t rs = c_stop, rb = c_bad;
#pragma unroll
    for (uint32_t k = 0; k < 8; k++) {
      const uint32_t vs = s_stop[it][k], vb = s_bad[it][k];
      if (k < warp) { rs = max(rs, vs); rb = max(rb, vb); }
      c_stop = max(c_stop, vs); c_bad = max(c_bad, vb);
    }
    if (lane) { rs = max(rs, us); rb = max(rb, ub); }
    pt = pt0;
#pragma unroll
    for (uint32_t k = 0; k < kClFlatPer; k++) {
      const uint32_t j = j0 + k, t = w[k] >> 24;
      if (j < ntok) {
        if (t == ']' && (rs & 1u) && pt != ',') {
          const uint32_t a = (rs >> 1) - 1u;
          jmp[a] = j;
          flag[a] = CL_FLAT | (rb <= a ? CL_ALL_INT64 : 0);
        }
        if ((stopm >> k) & 1u) rs = 2u * (j + 1u) + (t == '[' ? 1u : 0u);
        if ((badm >> k) & 1u) rb = j + 1u;
      }
      pt = t;
    }
  }
}

// A walker with `static constexpr bool kOwnRecord = true` takes over after the depth pass (and the flat-array stage):
//   static void record(P, S, LDoc d, Scratch args, uint32_t doc)   called by every thread: the grammar check, its walk and plan,
//                                                                  the request's result and its record
template <class W, class = void> struct cl_own_record { static constexpr bool value = false; };
template <class W> struct cl_own_record<W, decltype((void)W::kOwnRecord)> { static constexpr bool value = W::kOwnRecord; };

// The request loop of a large-request kernel, one CTA per request.  Walk is the kernel's walker (thread 0):
//   Scratch, static Scratch scratch(uint2* rest)   its scratch, in the part of the CTA's slice past the escape counts
//   LDoc d; Scratch A; uint32_t* stk;               the request's tokens, the scratch, kChatLargeMaxDepth words of shared memory
//   int reason, pending; decline(r); bad()          the first decline; a pending 422 / 500 (declined as AIGW_R_CONTENT)
//   Top, bool scan_top(Top&)                        the top-level members: t.model (a string, or kNone), t.stream (kNone: absent)
//   void check(const Top&)                          every further check, in the translate pass's order
//   static constexpr bool kFlatArrays               run cl_flat_arrays after the depth pass and let the grammar check step over
//                                                   the arrays it flags; Scratch then has `uint8_t* flag`, one byte per token
// and cl_plan(P, W, t, stream, R) plans the record (0 or the reason).  Only requests whose grammar check passed reach scan_top.
template <class Walk>
__device__ __forceinline__ void cl_request_loop(const ChatLargeParams& P, ClShared& S) {
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const uint32_t lt = (1u << lane) - 1u;
  uint8_t* slice = P.ws + (size_t)blockIdx.x * P.slice;
  const size_t tcap = P.tok_cap;
  uint32_t* tokw = (uint32_t*)slice;
  uint32_t* jmp = tokw + tcap;
  uint2* cum = (uint2*)(jmp + tcap);   // 8-byte aligned: the slice is, and the two word arrays hold an even count
  const typename Walk::Scratch args = Walk::scratch(cum + tcap + 1);   // the rest of the slice: the walk's own
  for (uint32_t k = tid; k < sizeof S.lits; k += kClThreads) S.lits[k] = (uint8_t)P.lits[k];
  for (uint32_t k = tid; k < CL_COUNT; k += kClThreads) { S.lit_off[k] = P.lit_off[k]; S.lit_len[k] = P.lit_len[k]; }
  for (;;) {
    __syncthreads();
    if (tid == 0) { S.doc = atomicAdd(P.next, 1u); S.fail = kNone; S.path_len = 0; S.total = 0; S.flags = 0; S.body_kind = AIGW_BODY_UNCHANGED; S.model_off = 0; S.model_len = 0; S.off = ~0ull; }
    __syncthreads();
    const uint32_t doc = S.doc;
    if (doc >= P.n) break;
    const uint8_t* body = P.bodies + P.offsets[doc];
    const uint32_t len = P.lens[doc];
    const uint32_t cap = min(chat_large_tok_cap(len), P.tok_cap);
    int fail = 0;
    uint32_t ntok = 0, ecum = 0, ncum = 0;
    if (P.call_reason) fail = (int)P.call_reason;
    else if (len >= (1u << 24) || len == 0) fail = len ? AIGW_R_TOO_LARGE : AIGW_R_E400_SYNTAX;
    else if (((uintptr_t)body) & 15u) fail = AIGW_R_ARGS;   // the arena convention: every request starts 16-byte aligned
    uint32_t in_str = 0, prev_sc = 0, esc_c = 0, prev_em = 0;   // carries across tiles (uniform over the CTA)
    uint4 na = make_uint4(0, 0, 0, 0), nb = na;
    if (!fail && tid * 32u + 32u <= len) { na = __ldg((const uint4*)(body + tid * 32u)); nb = __ldg((const uint4*)(body + tid * 32u + 16)); }
    // ================================================================ scan
    // The tile loop of emb_large_kernel with a different per-token payload: escape counts in front of every token (one 64-bit
    // prefix sum of three counts) instead of escape entries compacted beside the tokens.  A shared form would take the payload as
    // a callback inside the prefix-sum and compaction steps, which changes emb_large_kernel's register allocation and SASS; the
    // pieces that are the same (classification, the odd-run rule, the realigned load) are shared through classify.cuh and
    // scan_stream.cuh.
    if (!fail) for (uint32_t base = 0, it = 0; base < len; base += kClTile, it ^= 1u) {
      const uint32_t pos0 = base + tid * 32u;
      uint32_t w[8];
      if (pos0 + 32u <= len) {
        w[0] = na.x; w[1] = na.y; w[2] = na.z; w[3] = na.w; w[4] = nb.x; w[5] = nb.y; w[6] = nb.z; w[7] = nb.w;
        if (pos0 + kClTile + 32u <= len) { na = __ldg((const uint4*)(body + pos0 + kClTile)); nb = __ldg((const uint4*)(body + pos0 + kClTile + 16)); }
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
      const uint32_t tpar = __clz(~bsm) & 1u;
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
      if (lane == 31) S.wem[it][warp] = esc;   // the escaped bytes of the warp's last thread: the next thread's low-surrogate check
      __syncthreads();
      uint32_t pre = 0, tot = 0;
#pragma unroll
      for (uint32_t k = 0; k < 8; k++) { const uint32_t v = S.wpar[it][k]; tot ^= v; if (k < warp) pre ^= v; }
      const uint32_t in0 = in_str ^ pre ^ (__popc(bal & lt) & 1u);
      const uint32_t ps = prefix_xor32(uq) ^ (in0 ? FULL : 0u);
      const uint32_t inside = ps & ~uq;
      const uint32_t out = ~ps & ~uq;
      if (c.ctl & inside) raise_min(fail, AIGW_R_CTRL_IN_STRING);
      if ((c.ctl & out & ~c.ws) || (bsm & out)) raise_min(fail, AIGW_R_E400_SYNTAX);
      const uint32_t up_esc = __shfl_up_sync(FULL, esc, 1);
      const uint32_t pesc = lane ? up_esc : warp ? S.wem[it][warp - 1] : prev_em;   // the previous thread's escaped bytes
      auto is_esc = [&](uint32_t q) -> bool { return q >= pos0 ? (esc >> (q - pos0)) & 1u : q + 32u >= pos0 ? (pesc >> (q + 32u - pos0)) & 1u : false; };
      const uint32_t ebits = esc & inside;
      uint32_t nc = 0;
      for (uint32_t e = ebits; e;) {
        const uint32_t i = __ffs(e) - 1u; e &= e - 1u;
        const uint32_t p = pos0 + i, ch = body[p];
        const bool ok = ch == '"' || ch == '\\' || ch == '/' || ch == 'b' || ch == 'f' || ch == 'n' || ch == 'r' || ch == 't' ||
                        (ch == 'u' && p + 4u < len && is_hex(body[p + 1]) && is_hex(body[p + 2]) && is_hex(body[p + 3]) && is_hex(body[p + 4]));
        if (!ok) raise_min(fail, AIGW_R_ESCAPE);
        else if (ch == '/' || ch == 'b' || ch == 'f' || ch == 'u') {
          nc |= 1u << i;
          if (ch == 'u' && lone_surrogate(body, len, p, is_esc)) raise_min(fail, AIGW_R_ESCAPE);
        }
      }
      // ---- tokens, with the escaped bytes and re-spelled escapes in front of each
      const uint32_t sc = out & ~c.op & ~c.ws;
      if (lane == 31) S.wlast[it][warp] = sc >> 31;
      uint32_t prev = __shfl_up_sync(FULL, sc >> 31, 1);
      const uint32_t last_em_tile = S.wem[it][7];
      __syncthreads();
      if (lane == 0) prev = warp == 0 ? prev_sc : S.wlast[it][warp - 1];
      const uint32_t sc_start = sc & ~((sc << 1) | prev);
      uint32_t tk = (c.op & out) | uq | sc_start;
      // three counts in one 64-bit scan: tokens (bits 0-20), escaped bytes (21-41), re-spelled escapes (42-62)
      const unsigned long long cnt = (unsigned long long)__popc(tk) | ((unsigned long long)__popc(ebits) << 21) | ((unsigned long long)__popc(nc) << 42);
      unsigned long long incl = cnt;
#pragma unroll
      for (int dd = 1; dd < 32; dd <<= 1) { const unsigned long long v = __shfl_up_sync(FULL, incl, dd); if ((int)lane >= dd) incl += v; }
      if (lane == 31) S.wcnt[it][warp] = incl;
      const uint32_t last_sc_tile = S.wlast[it][7];
      __syncthreads();
      unsigned long long wpre = 0, wtot = 0;
#pragma unroll
      for (uint32_t k = 0; k < 8; k++) { const unsigned long long v = S.wcnt[it][k]; wtot += v; if (k < warp) wpre += v; }
      const unsigned long long ex = wpre + incl - cnt;
      uint32_t off = ntok + (uint32_t)(ex & 0x1fffffu);
      const uint32_t e0 = ecum + (uint32_t)((ex >> 21) & 0x1fffffu), n0 = ncum + (uint32_t)(ex >> 42);
      while (tk) {
        const uint32_t i = __ffs(tk) - 1u; tk &= tk - 1u;
        const uint32_t p = pos0 + i, bit = 1u << i;
        const uint32_t ty = (uq & bit) ? ((ps & bit) ? T_QOPEN : T_QCLOSE) : (c.op & bit) ? (uint32_t)body[p] : T_SCALAR;
        if (off < cap) { tokw[off] = p | (ty << 24); cum[off] = make_uint2(e0 + __popc(ebits & (bit - 1u)), n0 + __popc(nc & (bit - 1u))); }
        off++;
      }
      ntok += (uint32_t)(wtot & 0x1fffffu); ecum += (uint32_t)((wtot >> 21) & 0x1fffffu); ncum += (uint32_t)(wtot >> 42);
      in_str ^= tot; prev_sc = last_sc_tile; esc_c = cout_t; prev_em = last_em_tile;
    }
    if (!fail && in_str) fail = AIGW_R_E400_SYNTAX;   // unterminated string
    if (ntok > cap) raise_min(fail, AIGW_R_TOKENS);
    if (!fail && ntok == 0) fail = AIGW_R_E400_SYNTAX;   // white space only
    if (fail) atomicMin(&S.fail, (uint32_t)fail);
    __syncthreads();
    // ================================================================ depth, escaped keys
    if (S.fail == kNone) {
      if (tid == 0) cum[ntok] = make_uint2(ecum, ncum);
      int carry = 0;
      uint32_t it = 0;
      for (uint32_t b0 = 0; b0 < ntok; b0 += kClThreads, it ^= 1u) {
        const uint32_t j = b0 + tid;
        const uint32_t ty = j < ntok ? tokw[j] >> 24 : 0u;
        const int d = (ty == '{' || ty == '[') ? 1 : (ty == '}' || ty == ']') ? -1 : 0;
        // block-wide exclusive prefix sum of d
        int incl = d;
#pragma unroll
        for (int s = 1; s < 32; s <<= 1) { const int x = __shfl_up_sync(FULL, incl, s); if ((int)lane >= s) incl += x; }
        if (lane == 31) S.wsum[it][warp] = (uint32_t)incl;
        __syncthreads();
        int wp = 0, tot = 0;
#pragma unroll
        for (uint32_t k = 0; k < 8; k++) { const int x = (int)S.wsum[it][k]; tot += x; if (k < warp) wp += x; }
        const int da = carry + wp + incl;
        carry += tot;
        if (j < ntok) {
          if (da < 0) atomicMin(&S.fail, (uint32_t)AIGW_R_E400_SYNTAX);
          else if (da > (int)kChatLargeMaxDepth) atomicMin(&S.fail, (uint32_t)AIGW_R_DEPTH);
          if (ty == T_SCALAR) { const uint32_t o = tokw[j] & 0xffffffu, e = j + 1 < ntok ? tokw[j + 1] & 0xffffffu : len; uint32_t q = e; while (q > o && (body[q - 1] == ' ' || body[q - 1] == '\n' || body[q - 1] == '\r' || body[q - 1] == '\t')) q--; if (!scan_scalar_kind(body + o, q - o)) atomicMin(&S.fail, (uint32_t)AIGW_R_E400_SYNTAX); }
          if (ty == T_QOPEN && j + 2 < ntok && (tokw[j + 2] >> 24) == ':' && cum[j + 1].x != cum[j].x) atomicMin(&S.fail, (uint32_t)AIGW_R_ESCAPE);
        }
      }
      if (carry != 0 && tid == 0) atomicMin(&S.fail, (uint32_t)AIGW_R_E400_SYNTAX);
    }
    __syncthreads();
    // ================================================================ flat arrays (every thread; kFlatArrays walkers only)
    if constexpr (Walk::kFlatArrays) {
      if (S.fail == kNone) cl_flat_arrays(tokw, jmp, args.flag, body, len, ntok);
      __syncthreads();
    }
    if constexpr (cl_own_record<Walk>::value) {
      Walk::record(P, S, LDoc{body, len, tokw, cum, jmp, ntok}, args, doc);   // grammar, walk, plan and emit of its own
    } else {
      // ================================================================ grammar, then the kernel's walk and plan (thread 0)
      if (tid == 0) {
        int f = S.fail == kNone ? 0 : (int)S.fail;
        Walk W;
        W.d = LDoc{body, len, tokw, cum, jmp, ntok};
        W.A = args; W.stk = S.stk;
        ClRec R(S);
        if (!f) {
          int vr;
          if constexpr (Walk::kFlatArrays) vr = cl_validate<true>(W.d, S.stk, false, args.flag); else vr = cl_validate(W.d, S.stk, false);
          if (vr) f = vr == AIGW_R_SYNTAX ? AIGW_R_E400_SYNTAX : vr;
        }
        if (!f) {
          typename Walk::Top t;
          if (W.scan_top(t)) {
            const bool stream = t.stream != kNone && W.d.ty(t.stream) == 't';
            if (t.model != kNone) {
              const uint32_t ml = W.d.str_len(t.model);
              if (ml > 0xffffu) W.decline(AIGW_R_TOO_LARGE);   // model_len is 16 bits
              else { S.model_off = W.d.str_off(t.model); S.model_len = ml; }
            }
            S.flags = stream ? 1u : 0u;
            if (!W.bad()) W.check(t);
            if (!W.bad() && W.pending) W.decline(AIGW_R_CONTENT);   // a 422 / internal error of another translator: outside the fast path
            if (!W.bad()) { if (const int r = cl_plan(P, W, t, stream, R)) W.decline(r); }
          }
          f = W.reason;
          if (!f && (R.full || R.n == 0)) f = AIGW_R_OPS;
        }
        S.total = R.olen;
        S.fail = f ? (uint32_t)f : kNone;
        aigw_doc_result res;
        res.out_off = 0; res.body_len = 0; res.path_len = 0; res.status = AIGW_DECLINED; res.reason = 0; res.model_off = 0; res.model_len = 0;
        res.body_kind = AIGW_BODY_UNCHANGED; res.flags = 0; res.in_len = len; res._pad = 0;
        if (f) {
          res.reason = (uint8_t)f; res.status = f >= 48 ? AIGW_INTERNAL : f >= 40 ? AIGW_INVALID_422 : f >= 32 ? AIGW_MALFORMED_400 : AIGW_DECLINED;
        } else {
          const unsigned long long size = ((unsigned long long)R.olen + 15u) & ~15ull;
          const unsigned long long o = atomicAdd(P.out_used, size);
          if (o + size > P.out_capacity) { res.reason = AIGW_R_OUT_SPACE; res.body_len = R.olen; }   // the record length this request needs
          else {
            S.off = o;
            res.out_off = o; res.path_len = (uint16_t)S.path_len; res.body_len = R.olen - S.path_len; res.status = AIGW_OK;
            res.model_off = S.model_off; res.model_len = (uint16_t)S.model_len; res.body_kind = (uint8_t)S.body_kind; res.flags = (uint8_t)S.flags;
          }
        }
        P.results[doc] = res;
      }
      __syncthreads();
      if (S.off == ~0ull) continue;
      // ================================================================ emit: 16-byte chunks, every thread busy
      const uint32_t total = S.total, nchunk = (total + 15u) >> 4;
      uint4* dst = (uint4*)(P.out + S.off);
      for (uint32_t ch = tid; ch < nchunk; ch += kClThreads) {
        const uint32_t o0 = ch << 4;
        uint32_t k = 0;
        while (S.op_end[k] <= o0) k++;
        const uint32_t start = k ? S.op_end[k - 1] : 0u;
        uint4 v;
        if (S.op_kind[k] == OP_BODY && o0 + 16u <= S.op_end[k]) v = load16_unaligned(body + S.op_src[k] + (o0 - start));
        else {
          unsigned long long lo = 0, hi = 0;   // zero past the record's end
          uint32_t kk = k, st = start;
          for (uint32_t b = 0; b < 16u && o0 + b < total; b++) {
            const uint32_t o = o0 + b;
            while (o >= S.op_end[kk]) { st = S.op_end[kk]; kk++; }
            const uint32_t src = S.op_src[kk] + (o - st);
            const unsigned long long x = S.op_kind[kk] == OP_BODY ? body[src] : S.lits[src];
            if (b < 8u) lo |= x << (8u * b); else hi |= x << (8u * (b - 8u));
          }
          v = make_uint4((uint32_t)lo, (uint32_t)(lo >> 32), (uint32_t)hi, (uint32_t)(hi >> 32));
        }
        dst[ch] = v;
      }
    }
  }
}

}  // namespace
}  // namespace aigw
