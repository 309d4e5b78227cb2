// The record phase of the large-request chat kernels that rebuild the body (chat_bedrock_large_kernel.cu,
// chat_anthropic_large_kernel.cu), after the scan and depth pass of large_request.cuh:
//   grammar   thread 0 checks the token grammar and writes the jump table
//   walk      thread 0 runs the planner's top-level scan and the planner over the emitting walk (ClWalkT<ClOut>, chat_bedrock_walk.cuh): its
//             checks in the translate pass's order, and the record as copy ops in the CTA's slice.  A string with an escape the
//             encoder re-spells (\/ \b \f \u) keeps its other stretches as body spans, its re-spelled runs go into scratch; a tool
//             call's "arguments" are unescaped, checked and re-serialised into scratch.
//   emit      every op's output end by a block-wide 64-bit prefix sum, one bump allocation, then 16-byte output chunks with every
//             thread busy: a chunk inside one body span is one realigned 16-byte load, the others are assembled byte by byte.
// The emit differs from emb_large_kernel's, whose cursor also walks escape entries inside its string ops; this record has none.
//
// A kernel is cl_request_loop<ClRecordRequest<Plan>>, where Plan has
//   using Top = …                                  the top-level members its scan keeps, with `model` and `stream` (value tokens,
//                                                  kNone when absent or null)
//   static bool scan(RecWalk& W, Top& t)           the top-level scan: true when it passed (the chat planners: ClChatTop, scan_top)
//   static void plan(const ChatLargeParams&, ClShared&, RecWalk& W, const Top& t, bool stream)
// plan is called by thread 0 after the scan has passed, with the model span, the stream flag and body_kind already set: it records
// the ":path" (and sets S.path_len), then the body, or declines through W.
#pragma once
#include "chat_bedrock_walk.cuh"
#include "chat_large_record.cuh"

namespace aigw {
namespace {

enum : uint32_t { REC_BODY = 0, REC_LIT = 1, REC_SCR = 2 };

static __device__ const LitTable g_rec_lits = make_lit_table();

// the record sink of the emitting walk: ops (kind, source offset, length, output end) in the slice, the op being extended in
// registers
struct ClOut {
  static constexpr bool kEmit = true;
  uint4* ops; uint32_t n, cap;
  uint4 cur; bool has;
  uint8_t* scr; uint32_t rs_n, rs_cap, ao_n, ao_end;   // re-spelled strings in [0, rs_cap), arguments in [rs_cap, ao_end)
  bool capturing; uint32_t cap0;
  unsigned long long olen;
  int err;

  __device__ void push(uint32_t kind, uint32_t src, uint32_t len) {
    if (!len || err) return;
    olen += len;
    if (has && cur.x == kind && cur.y + cur.z == src) { cur.z += len; return; }
    if (has) { if (n >= cap) { err = AIGW_R_OPS; return; } ops[n++] = cur; }
    cur = make_uint4(kind, src, len, 0); has = true;
  }
  __device__ void flush() { if (has && !err) { if (n >= cap) err = AIGW_R_OPS; else ops[n++] = cur; } has = false; }
  __device__ void put_ao(const uint8_t* p, uint32_t l) {
    if (err) return;
    if (ao_n + l > ao_end) { err = AIGW_R_SCRATCH; return; }
    for (uint32_t i = 0; i < l; i++) scr[ao_n + i] = p[i];
    ao_n += l;
  }
  __device__ void lit(uint32_t id) {
    const uint32_t o = g_rec_lits.off[id], l = g_rec_lits.off[id + 1] - o;
    if (capturing) put_ao((const uint8_t*)g_rec_lits.bytes + o, l); else push(REC_LIT, o, l);
  }
  __device__ void span(const LDoc& d, uint32_t b, uint32_t e) { if (capturing) put_ao(d.s + b, e - b); else push(REC_BODY, b, e - b); }
  // the arguments text is copied as it is re-serialised, then recorded as one scratch span
  __device__ void capture(bool on) {
    if (on) { cap0 = ao_n; capturing = true; }
    else { capturing = false; push(REC_SCR, cap0, ao_n - cap0); }
  }
  // a re-spelled byte run into scratch: room for `need` more bytes
  __device__ bool room(uint32_t need) { if (rs_n + need > rs_cap) { err = AIGW_R_SCRATCH; return false; } return true; }

  // emit_str / emit_str_respelled of a body string v, quotes included (kInner: without them).  The scan has checked every \u
  // escape's hex digits and declined lone surrogates, so every escape here decodes.
  template <bool kInner>
  __device__ __forceinline__ void str_q(const LDoc& d, uint32_t v) {
    const uint32_t q0 = d.tok(v), q1 = d.tok(v + 1);
    if (!d.str_nc(v)) { push(REC_BODY, kInner ? q0 + 1u : q0, kInner ? q1 - q0 - 1u : q1 + 1u - q0); return; }
    const uint8_t* s = d.s;
    uint32_t seg = kInner ? q0 + 1u : q0, i = q0 + 1, run = 0;
    bool in_run = false;
    while (i < q1) {
      const uint32_t c = s[i];
      const uint32_t e = c == '\\' ? s[i + 1] : 0u;
      if (c != '\\' || e == '"' || e == '\\' || e == 'n' || e == 'r' || e == 't') {
        if (in_run) { push(REC_SCR, run, rs_n - run); in_run = false; seg = i; }
        i += c == '\\' ? 2u : 1u;
        continue;
      }
      if (!in_run) { push(REC_BODY, seg, i - seg); in_run = true; run = rs_n; }
      if (!room(6)) return;
      uint8_t* o = scr + rs_n;
      uint32_t cp, used;
      if (e == '/') { cp = '/'; used = 2; }
      else if (e == 'b') { cp = 8; used = 2; }
      else if (e == 'f') { cp = 12; used = 2; }
      else {
        cp = hex4v(s + i + 2); used = 6;
        if (cp >= 0xD800u && cp < 0xDC00u) { cp = 0x10000u + ((cp - 0xD800u) << 10) + (hex4v(s + i + 8) - 0xDC00u); used = 12; }
      }
      uint32_t w;
      if (cp == '"' || cp == '\\') { o[0] = '\\'; o[1] = (uint8_t)cp; w = 2; }
      else if (cp == 10u || cp == 13u || cp == 9u) { o[0] = '\\'; o[1] = cp == 10u ? 'n' : cp == 13u ? 'r' : 't'; w = 2; }
      else if (cp < 0x20u) { const char* hx = "0123456789abcdef"; o[0] = '\\'; o[1] = 'u'; o[2] = '0'; o[3] = '0'; o[4] = hx[cp >> 4]; o[5] = hx[cp & 15u]; w = 6; }
      else if (cp < 0x80u) { o[0] = (uint8_t)cp; w = 1; }
      else if (cp < 0x800u) { o[0] = (uint8_t)(0xC0u | (cp >> 6)); o[1] = (uint8_t)(0x80u | (cp & 63u)); w = 2; }
      else if (cp < 0x10000u) { o[0] = (uint8_t)(0xE0u | (cp >> 12)); o[1] = (uint8_t)(0x80u | ((cp >> 6) & 63u)); o[2] = (uint8_t)(0x80u | (cp & 63u)); w = 3; }
      else { o[0] = (uint8_t)(0xF0u | (cp >> 18)); o[1] = (uint8_t)(0x80u | ((cp >> 12) & 63u)); o[2] = (uint8_t)(0x80u | ((cp >> 6) & 63u)); o[3] = (uint8_t)(0x80u | (cp & 63u)); w = 4; }
      rs_n += w; i += used;
    }
    if (in_run) { push(REC_SCR, run, rs_n - run); seg = q1; }
    push(REC_BODY, seg, (kInner ? q1 : q1 + 1u) - seg);
  }
  __device__ void str(const LDoc& d, uint32_t v) { str_q<false>(d, v); }
  // emit_str_inner: the string's bytes as the encoder spells them, without the quotes (text blocks concatenated into one string)
  __device__ void str_inner(const LDoc& d, uint32_t v) { str_q<true>(d, v); }
};

using RecWalk = ClWalkT<ClOut>;

struct RecSlice { uint4* ops; uint8_t* scr; };
__device__ __forceinline__ RecSlice rec_carve(uint2* rest, uint32_t max_len) {
  const uintptr_t a = (uintptr_t)rest + (uintptr_t)(kChatArgMax + 2u) * 16u + kChatArgMax + 16u;
  RecSlice s;
  s.ops = (uint4*)((a + 15u) & ~(uintptr_t)15u);
  s.scr = (uint8_t*)(s.ops + rec_op_cap(max_len));
  return s;
}

// The model of the ":path" (the override, or the request's model): url.PathEscape'd (kEscape) or raw.  A model that needs no
// escaping is a body span; an escaped one, or the override, goes into scratch.
template <bool kEscape, class Top = RecWalk::Top>
__device__ __forceinline__ void rec_path_model(const ChatLargeParams& P, const ClShared& S, RecWalk& W, const Top& t) {
  const LDoc& d = W.d;
  const bool ov = P.override_len != 0;
  const uint8_t* mp = ov ? S.lits + S.lit_off[CL_OVERRIDE] : t.model != kNone ? d.s + d.str_off(t.model) : nullptr;
  const uint32_t ml = ov ? P.override_len : t.model != kNone ? d.str_len(t.model) : 0u;
  auto keep = [](uint32_t c) {
    return !kEscape || (c - 'a' < 26u) || (c - 'A' < 26u) || (c - '0' < 10u) || c == '-' || c == '_' || c == '.' || c == '~' || c == '$' ||
           c == '&' || c == '+' || c == ':' || c == '=' || c == '@';
  };
  bool clean = true;
  for (uint32_t i = 0; i < ml && clean; i++) clean = keep(mp[i]);
  if (clean && !ov) { if (ml) W.o.span(d, d.str_off(t.model), d.str_off(t.model) + ml); }
  else if (W.o.room(3u * ml)) {
    const uint32_t at = W.o.rs_n;
    uint32_t w = at;
    for (uint32_t i = 0; i < ml; i++) {
      const uint32_t c = mp[i];
      if (keep(c)) W.o.scr[w++] = (uint8_t)c;
      else { const char* hx = "0123456789ABCDEF"; W.o.scr[w++] = '%'; W.o.scr[w++] = hx[c >> 4]; W.o.scr[w++] = hx[c & 15u]; }
    }
    W.o.rs_n = w;
    W.o.push(REC_SCR, at, w - at);
  }
}

// exclusive prefix sum of v over the CTA; wsum: 8 shared words per round (double-buffered by `it`)
__device__ __forceinline__ unsigned long long rec_excl(unsigned long long v, unsigned long long (*wsum)[8], uint32_t it, unsigned long long& tot) {
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  unsigned long long incl = v;
#pragma unroll
  for (int s = 1; s < 32; s <<= 1) { const unsigned long long x = __shfl_up_sync(FULL, incl, s); if ((int)lane >= s) incl += x; }
  if (lane == 31) wsum[it][warp] = incl;
  __syncthreads();
  unsigned long long pre = 0; tot = 0;
#pragma unroll
  for (uint32_t k = 0; k < 8; k++) { const unsigned long long x = wsum[it][k]; tot += x; if (k < warp) pre += x; }
  return pre + incl - v;
}

// the top-level scan of the /v1/chat/completions planners: ParseBody's checks (scan_top)
struct ClChatTop {
  using Top = RecWalk::Top;
  static __device__ __forceinline__ bool scan(RecWalk& W, Top& t) { return W.scan_top(t); }
};

template <class Plan>
struct ClRecordRequest {
  using Scratch = uint2*;
  static constexpr bool kFlatArrays = false;
  static constexpr bool kOwnRecord = true;
  static __device__ __forceinline__ uint2* scratch(uint2* rest) { return rest; }

  static __device__ void record(const ChatLargeParams& P, ClShared& S, const LDoc& d, uint2* rest, uint32_t doc) {
    __shared__ unsigned long long s_w64[2][8];
    __shared__ uint32_t s_nops;
    __shared__ unsigned long long s_total;
    const uint32_t tid = threadIdx.x;
    const RecSlice sl = rec_carve(rest, P.max_len);
    const uint32_t len = d.len;
    // ================================================================ grammar, walk and plan (thread 0)
    if (tid == 0) {
      int f = S.fail == kNone ? 0 : (int)S.fail;
      RecWalk W;
      W.d = d; W.A = RecWalk::scratch(rest); W.stk = S.stk;
      ClOut& o = W.o;
      o.ops = sl.ops; o.n = 0; o.cap = min(rec_op_cap(len), rec_op_cap(P.max_len)); o.has = false;
      o.scr = sl.scr; o.rs_n = 0; o.rs_cap = min(rec_rs_cap(len), rec_rs_cap(P.max_len));
      o.ao_n = rec_rs_cap(P.max_len); o.ao_end = o.ao_n + kRecArgOut;
      o.capturing = false; o.cap0 = 0; o.olen = 0; o.err = 0;
      if (!f) {
        const int vr = cl_validate(W.d, S.stk, false);
        if (vr) f = vr == AIGW_R_SYNTAX ? AIGW_R_E400_SYNTAX : vr;
      }
      if (!f) {
        typename Plan::Top t;
        if (Plan::scan(W, t)) {
          const bool stream = t.stream != kNone && W.d.ty(t.stream) == 't';
          if (t.model != kNone) {
            const uint32_t ml = W.d.str_len(t.model);
            if (ml > 0xffffu) W.decline(AIGW_R_TOO_LARGE);   // model_len is 16 bits
            else { S.model_off = W.d.str_off(t.model); S.model_len = ml; }
          }
          S.flags = stream ? 1u : 0u;
          S.body_kind = AIGW_BODY_BYTES;
          Plan::plan(P, S, W, t, stream);
        }
        o.flush();
        // the translate pass's order: a decline of the walk, then the plan's capacity, then a pending 422 / 500
        f = W.reason ? W.reason : o.err ? o.err : W.pending;
      }
      s_nops = f ? 0u : o.n;
      S.fail = f ? (uint32_t)f : kNone;
    }
    __syncthreads();
    // ================================================================ op ends: a block-wide prefix sum, saturated above the ceiling
    const uint32_t nops = s_nops;
    {
      unsigned long long run = 0;
      uint32_t it = 0;
      for (uint32_t b0 = 0; b0 < nops; b0 += kClThreads, it ^= 1u) {
        const uint32_t k = b0 + tid;
        const unsigned long long n = k < nops ? sl.ops[k].z : 0u;
        unsigned long long tot;
        const unsigned long long ex = rec_excl(n, s_w64, it, tot);
        if (k < nops) sl.ops[k].w = (uint32_t)min(run + ex + n, (unsigned long long)kRecOutCeiling + 1u);
        run += tot;
      }
      if (tid == 0) s_total = run;
    }
    __syncthreads();
    // ================================================================ the result, the record's place
    if (tid == 0) {
      aigw_doc_result res;
      res.out_off = 0; res.body_len = 0; res.path_len = 0; res.status = AIGW_DECLINED; res.reason = 0; res.model_off = 0; res.model_len = 0;
      res.body_kind = AIGW_BODY_UNCHANGED; res.flags = 0; res.in_len = len; res._pad = 0;
      const int f = S.fail == kNone ? 0 : (int)S.fail;
      const unsigned long long total = s_total;
      if (f) res.reason = (uint8_t)f, res.status = f >= 48 ? AIGW_INTERNAL : f >= 40 ? AIGW_INVALID_422 : f >= 32 ? AIGW_MALFORMED_400 : AIGW_DECLINED;
      else if (total > kRecOutCeiling) res.reason = AIGW_R_OUT_SPACE;   // body_len stays 0: no arena takes it
      else {
        const unsigned long long size = (total + 15u) & ~15ull;
        const unsigned long long o = atomicAdd(P.out_used, size);
        if (o + size > P.out_capacity) { res.reason = AIGW_R_OUT_SPACE; res.body_len = (uint32_t)total; }   // the record length this request needs
        else {
          S.off = o; S.total = (uint32_t)total;
          res.out_off = o; res.path_len = (uint16_t)S.path_len; res.body_len = (uint32_t)total - S.path_len; res.status = AIGW_OK;
          res.model_off = S.model_off; res.model_len = (uint16_t)S.model_len; res.body_kind = (uint8_t)S.body_kind; res.flags = (uint8_t)S.flags;
        }
      }
      P.results[doc] = res;
    }
    __syncthreads();
    if (S.off == ~0ull) return;
    // ================================================================ emit: 16-byte chunks, every thread busy
    const uint32_t total = S.total, nchunk = (total + 15u) >> 4;
    const uint8_t* body = d.s;
    const uint8_t* lits = (const uint8_t*)g_rec_lits.bytes;
    uint4* dst = (uint4*)(P.out + S.off);
    for (uint32_t ch = tid; ch < nchunk; ch += kClThreads) {
      const uint32_t o0 = ch << 4;
      uint32_t lo = 0, hi = nops;   // the op holding output byte o0: the first whose end is past it
      while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (sl.ops[m].w <= o0) lo = m + 1; else hi = m; }
      uint4 op = sl.ops[lo];
      uint4 v;
      if (op.x == REC_BODY && o0 + 16u <= op.w) v = load16_unaligned(body + op.y + (o0 - (op.w - op.z)));
      else {
        unsigned long long x0 = 0, x1 = 0;   // zero past the record's end
        uint32_t k = lo;
        for (uint32_t b = 0; b < 16u && o0 + b < total; b++) {
          const uint32_t o = o0 + b;
          while (o >= op.w) op = sl.ops[++k];
          const uint32_t src = op.y + (o - (op.w - op.z));
          const unsigned long long x = op.x == REC_BODY ? body[src] : op.x == REC_LIT ? lits[src] : sl.scr[src];
          if (b < 8u) x0 |= x << (8u * b); else x1 |= x << (8u * (b - 8u));
        }
        v = make_uint4((uint32_t)x0, (uint32_t)(x0 >> 32), (uint32_t)x1, (uint32_t)(x1 >> 32));
      }
      dst[ch] = v;
    }
  }
};

}  // namespace
}  // namespace aigw
