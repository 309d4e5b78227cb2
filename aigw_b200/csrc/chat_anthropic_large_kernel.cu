// /v1/chat/completions requests above the translate pass's 64 KiB ceiling (and below it) to the Anthropic Messages API behind GCP
// Vertex AI and AWS Bedrock: ParseBody's verdict, the ":path" and the Messages body, with the semantics group 2 of the translate
// pass gives them (scan_top and plan_anthropic in chat_walk_impl.cuh).  sm_90a only.
//
// chat_anthropic_large_kernel: one CTA of 256 threads per request, the scan and depth pass of large_request.cuh, then the record
// phase of chat_large_record_impl.cuh with this planner (thread 0), in plan_anthropic's order:
//   dry plan  the Bedrock plan over the sink that records nothing (ClWalkT<ClNoOut>), as plan_anthropic first runs plan_bedrock
//             with pl.dry: its declines stand, its pending 422 / 500 does not apply
//   checks    thinking, a non-empty "tools", a "stop" that is not a string or a non-empty array of strings, a non-empty
//             reasoning_effort
//   record    ":path", then the Messages body over the emitting walk: system and developer messages are checked in the message
//             pass and recorded after stop_sequences by a second pass; a run of tool messages becomes one user message of
//             tool_result blocks, each string content parsed for its is_error flag in the "arguments in hand" buffer
#include "chat_anthropic_large_kernel.cuh"

#include "chat_large_record_impl.cuh"

namespace aigw {
namespace {

// unit_range of the translate pass: a canonical decimal (canon_number's output, float form) against [0, 1]: -1 below, +1 above,
// 0 inside
__device__ __forceinline__ int an_unit_range(const uint8_t* p, uint32_t l) {
  uint32_t i = 0; bool neg = false;
  if (l && p[0] == '-') { neg = true; i = 1; }
  uint32_t iv = 0; bool nz = false;
  for (; i < l && p[i] != '.'; i++) { const uint32_t dg = p[i] - '0'; if (iv < 100u) iv = iv * 10u + dg; if (dg) nz = true; }
  bool fnz = false;
  for (i++; i < l; i++) if (p[i] != '0') fnz = true;
  if (neg) return (nz || fnz) ? -1 : 0;
  return (iv >= 2u || (iv == 1u && fnz)) ? 1 : 0;
}

// an_text_block: {"text":S[,"cache_control":{"type":"ephemeral"}],"type":"text"}; an empty text has no pinned layout and declines
__device__ __forceinline__ void an_text(RecWalk& W, uint32_t v, bool cache) {
  if (W.d.str_len(v) == 0) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
  W.lit(L_TEXT_OPEN); W.str(v); W.lit(cache ? L_AN_TEXT_CACHE_CLOSE : L_AN_TEXT_CLOSE);
}

// cache_simple: cache_control limited to {"type":…}; a ttl has no pinned position.  The dry plan has declined a cache_control
// that is not an object.
__device__ __forceinline__ bool an_cache_simple(RecWalk& W, uint32_t cc) {
  if (cc == kNone) return false;
  const LDoc& d = W.d;
  for (uint32_t m = cc + 1; d.ty(m) != '}'; m = d.after(m + 3))
    if (W.key(m, "ttl") && !W.is_null(m + 3)) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
  return W.cache_enabled(cc);
}

// an_is_error: a string tool content is an error when it decodes to a JSON object with an "error" member.  A content that cannot
// be an object (its first non-space byte is neither '{' nor a backslash) is not parsed.  The others are unescaped into the
// "arguments in hand" buffer and parsed there: a syntax error is false, an escape or control byte the tokenizer refuses, nesting
// deeper than 48 and an escaped key before "error" decline.  Above kChatArgMax unescaped bytes it declines AIGW_R_SCRATCH.  This
// is linear work: it does not count against kChatArgTotal.
__device__ __forceinline__ bool an_is_error(RecWalk& W, uint32_t v) {
  const LDoc& d = W.d;
  if (d.str_nc(v)) { W.decline(AIGW_R_ESCAPE); return false; }
  const uint8_t* p = d.s + d.str_off(v);
  const uint32_t n = d.str_len(v);
  uint32_t k = 0;
  while (k < n && p[k] == ' ') k++;
  if (k >= n || (p[k] != '{' && p[k] != '\\')) return false;
  uint32_t w = 0;
  for (uint32_t i = 0; i < n; i++, w++) {
    uint32_t c = p[i];
    if (c == '\\') { const uint32_t e = p[++i]; c = e == 'n' ? '\n' : e == 'r' ? '\r' : e == 't' ? '\t' : e; }
    if (w < kChatArgMax) W.A.s[w] = (uint8_t)c;
  }
  if (w > kChatArgMax) { W.decline(AIGW_R_SCRATCH); return false; }
  const int nt = cl_tokenize(W.A.s, w, W.A.tw, W.A.cum);
  if (nt == 0 || nt == -AIGW_R_SYNTAX) return false;
  if (nt < 0) { W.decline(-nt); return false; }
  LDoc a{W.A.s, w, W.A.tw, W.A.cum, W.A.jmp, (uint32_t)nt};
  const int vr = cl_validate(a, W.stk, true);
  if (vr == AIGW_R_SYNTAX) return false;
  if (vr) { W.decline(vr); return false; }
  if (a.ty(0) != '{') return false;
  for (uint32_t m = 1; a.ty(m) != '}'; m = a.after(m + 3)) {
    if (a.str_has_backslash(m)) { W.decline(AIGW_R_ESCAPE); return false; }
    if (a.raw_is(m, "error", 5)) return true;
  }
  return false;
}

// a system or developer message: one text block, its parts' raw text concatenated.  kE = false: the checks, in the message pass;
// kE = true: the record, in the second pass after stop_sequences (`first`: no block yet, so the opening literal goes first)
template <bool kE>
__device__ __forceinline__ void an_system(RecWalk& W, const RecWalk::Msg& g, bool& first) {
  const LDoc& d = W.d;
  const uint32_t c = g.content;
  if (c == kNone) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
  if constexpr (kE) { W.lit(first ? L_SYSTEM_OPEN : L_COMMA); first = false; }
  if (W.is_str(c)) {
    if constexpr (kE) an_text(W, c, false);
    else if (d.str_len(c) == 0) W.decline(AIGW_R_UNSUPPORTED_FIELD);
    return;
  }
  bool cache = false;
  uint32_t total = 0;
  if constexpr (kE) { W.lit(L_TEXT_OPEN); W.lit(L_QUOTE); }
  for (uint32_t q = c + 1; d.ty(q) != ']'; q = d.after(q)) {
    RecWalk::Part p; if (!W.scan_part(q, p)) return;
    if (p.text != kNone) {
      if (d.str_nc(p.text)) { W.decline(AIGW_R_ESCAPE); return; }   // the raw text is concatenated: a re-spelled escape has no place
      if constexpr (kE) W.o.span(d, d.str_off(p.text), d.str_off(p.text) + d.str_len(p.text));
      total += d.str_len(p.text);
    }
    if (an_cache_simple(W, p.cache)) cache = true;
    if (W.bad()) return;
  }
  if (total == 0) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
  if constexpr (kE) { W.lit(L_QUOTE); W.lit(cache ? L_AN_TEXT_CACHE_CLOSE : L_AN_TEXT_CLOSE); }
}

__device__ __forceinline__ void an_user(RecWalk& W, const RecWalk::Msg& g) {
  const LDoc& d = W.d;
  const uint32_t c = g.content;
  if (c == kNone) W.pend(AIGW_R_E500_ARGS);   // "unsupported OpenAI content type: <nil>"
  else if (W.is_null(c)) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
  else if (W.is_str(c)) an_text(W, c, false);
  else {
    if (d.ty(c + 1) == ']') { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
    bool first = true;
    for (uint32_t q = c + 1; d.ty(q) != ']'; q = d.after(q)) {
      RecWalk::Part p; if (!W.scan_part(q, p)) return;
      if (p.text == kNone) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
      const bool cache = an_cache_simple(W, p.cache);
      if (W.bad()) return;
      if (!first) W.lit(L_COMMA);
      first = false;
      an_text(W, p.text, cache);
      if (W.bad()) return;
    }
  }
  if (W.bad()) return;
  W.lit(L_USER_CLOSE);
}

__device__ __forceinline__ void an_assistant(RecWalk& W, const RecWalk::Msg& g) {
  const LDoc& d = W.d;
  bool first = true;
  const uint32_t c = g.content;
  if (c != kNone && !W.is_null(c)) {
    if (W.is_str(c)) { if (d.str_len(c) > 0) { an_text(W, c, false); first = false; } }
    else {
      const bool arr = W.is_arr(c);   // an object is one part
      for (uint32_t q = arr ? c + 1 : c; arr ? d.ty(q) != ']' : q == c; q = arr ? d.after(q) : kNone) {
        RecWalk::Part p; if (!W.scan_part(q, p)) return;
        if (p.type == kNone) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
        uint32_t src = kNone;
        bool cache = false;
        if (W.val(p.type, "text")) { src = p.text; cache = an_cache_simple(W, p.cache); }
        else if (W.val(p.type, "refusal")) src = p.refusal;
        else { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }   // thinking blocks, unknown types
        if (W.bad()) return;
        if (src != kNone) { if (!first) W.lit(L_COMMA); first = false; an_text(W, src, cache); if (W.bad()) return; }
        if (!arr) break;
      }
    }
  }
  const uint32_t tcs = g.tool_calls;
  if (tcs != kNone && !W.is_null(tcs)) {
    for (uint32_t q = tcs + 1; d.ty(q) != ']'; q = d.after(q)) {
      const uint32_t id = W.find(q, "id"), fn = W.find(q, "function");
      if (W.cache_enabled(W.find(q, "cache_control"))) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
      uint32_t name = kNone, args = kNone;
      if (fn != kNone) { name = W.find(fn, "name"); args = W.find(fn, "arguments"); }
      if (W.bad()) return;
      if (id == kNone) { W.decline(AIGW_R_TOOL); return; }
      if (args == kNone) W.pend(AIGW_R_E500_ARGS);
      if (!first) W.lit(L_COMMA);
      first = false;
      W.lit(L_AN_TOOLUSE_OPEN); W.str(id); W.lit(L_TOOLUSE_INPUT);
      if (args != kNone) W.arguments(args); else W.lit(L_NULL);
      if (W.bad()) return;
      W.lit(L_AN_NAME); if (name != kNone) W.str(name); else W.lit(L_EMPTY_STR);
      W.lit(L_AN_TOOLUSE_CLOSE);
    }
  }
  if (first) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }   // empty content: layout not pinned
  W.lit(L_ASST_CLOSE);
}

// one tool_result block
__device__ __forceinline__ void an_tool_result(RecWalk& W, const RecWalk::Msg& tm) {
  const LDoc& d = W.d;
  const uint32_t c = tm.content;
  W.lit(L_AN_TR_OPEN);
  uint32_t id = tm.tool_call_id;
  if (id != kNone && W.is_null(id)) id = kNone;
  if (id != kNone) W.str(id); else W.lit(L_EMPTY_STR);
  if (c == kNone) { W.pend(AIGW_R_E500_ARGS); W.lit(L_AN_TR_ERR_F); }
  else if (W.is_str(c)) {
    const bool ie = an_is_error(W, c);
    if (W.bad()) return;
    W.lit(ie ? L_AN_TR_ERR_T : L_AN_TR_ERR_F);
    an_text(W, c, false);
  } else {
    W.lit(L_AN_TR_ERR_F);
    if (d.ty(c + 1) == ']') { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
    bool first = true;
    for (uint32_t q = c + 1; d.ty(q) != ']'; q = d.after(q)) {
      RecWalk::Part p; if (!W.scan_part(q, p)) return;
      if (p.text == kNone || W.cache_enabled(p.cache)) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
      if (!first) W.lit(L_COMMA);
      first = false;
      an_text(W, p.text, false);
      if (W.bad()) return;
    }
  }
  if (W.bad()) return;
  W.lit(L_AN_TR_CLOSE);
}

// plan_anthropic after ParseBody's top-level checks
struct AnPlan : ClChatTop {
  static __device__ __forceinline__ void plan(const ChatLargeParams& P, ClShared& S, RecWalk& W, const RecWalk::Top& t, bool stream) {
    const LDoc& d = W.d;
    const bool gcp = P.gcp != 0;
    if (W.bad()) return;
    {
      ClWalkT<ClNoOut> D;
      D.d = d; D.A = W.A; D.stk = W.stk;
      D.check(t);
      if (D.reason) { W.decline(D.reason); return; }
    }
    if (t.thinking != kNone) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
    if (t.tools != kNone && d.ty(t.tools + 1) != ']') { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
    if (t.stop != kNone) {   // a string or a non-empty array of strings; anything else is not pinned (openai-go union decode)
      const uint32_t s = t.stop;
      if (W.is_arr(s)) {
        if (d.ty(s + 1) == ']') { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
        for (uint32_t e = s + 1; d.ty(e) != ']'; e = d.after(e)) if (!W.is_str(e)) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
      } else if (!W.is_str(s)) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
    }
    {   // scan_top has checked its type (a string) and declined a duplicate; only this planner reads it
      const uint32_t re = W.find(0, "reasoning_effort");
      if (re != kNone && d.str_len(re) > 0) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
    }
    // ":path": GCP publishers/anthropic/models/{model}:rawPredict | :streamRawPredict, AWS /model/{PathEscape(model)}/invoke[-with-response-stream]
    if (gcp) { W.lit(L_AN_GCP_PATH); rec_path_model<false>(P, S, W, t); W.lit(stream ? L_AN_STREAMRAWPREDICT : L_AN_RAWPREDICT); }
    else { W.lit(L_PATH_MODEL); rec_path_model<true>(P, S, W, t); W.lit(stream ? L_AN_INVOKE_STREAM : L_AN_INVOKE); }
    if (W.o.olen > 0xffffu) W.decline(AIGW_R_TOO_LARGE);   // path_len is 16 bits
    S.path_len = (uint32_t)W.o.olen;
    if (W.bad()) return;
    W.lit(L_AN_OPEN);
    const uint32_t mt = t.mct != kNone ? t.mct : t.max_tokens;
    if (mt != kNone) W.num_field(mt, true); else W.lit(L_ZERO);
    W.lit(L_AN_MSGS);
    bool mfirst = true, any_sys = false;
    if (t.messages != kNone) {
      uint32_t e = t.messages + 1;
      while (d.ty(e) != ']') {
        RecWalk::Msg g; const int role = W.scan_message(e, g);
        if (W.bad()) return;
        uint32_t nx = d.after(e);
        if (role == 2 || role == 3) { bool f = true; an_system<false>(W, g, f); any_sys = true; if (W.bad()) return; e = nx; continue; }
        if (!mfirst) W.lit(L_COMMA);
        mfirst = false;
        W.lit(L_MSG_CONTENT_OPEN);
        if (role == 0) an_user(W, g);
        else if (role == 1) an_assistant(W, g);
        else {   // consecutive tool messages aggregate into one user message
          an_tool_result(W, g);
          while (!W.bad() && d.ty(nx) != ']') {
            RecWalk::Msg g2; const int r2 = W.scan_message(nx, g2);
            if (W.bad() || r2 != 4) break;
            nx = d.after(nx);
            W.lit(L_COMMA);
            an_tool_result(W, g2);
          }
          if (W.bad()) return;
          W.lit(L_USER_CLOSE);
        }
        if (W.bad()) return;
        e = nx;
      }
    }
    if (mfirst) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }   // no messages: layout not pinned
    W.lit(L_RBRACK);
    // sampling parameters in MessageNewParams' declaration order; a temperature outside 0..1 is the translator's 422, found after
    // the message errors
    if (t.temperature != kNone) {
      W.lit(L_COMMA); W.lit(L_TEMP);
      W.num_field(t.temperature, false);
      if (W.bad()) return;
      const uint32_t tk = d.tok(t.temperature);
      if (an_unit_range(d.s + tk, canon_number(d.s + tk, d.scalar_end(t.temperature) - tk, false)) != 0) W.pend(AIGW_R_E422_TEMPERATURE);
    }
    if (t.top_p != kNone) { W.lit(L_AN_TOPP); W.num_field(t.top_p, false); if (W.bad()) return; }
    if (t.stop != kNone) {
      W.lit(L_AN_STOPSEQ);
      if (W.is_str(t.stop)) W.str(t.stop);
      else for (uint32_t e = t.stop + 1; d.ty(e) != ']'; e = d.after(e)) { if (e != t.stop + 1) W.lit(L_COMMA); W.str(e); }
      W.lit(L_RBRACK);
    }
    // "system" after the sampling parameters: a second pass over the messages records what the first one checked
    if (any_sys) {
      bool first = true;
      for (uint32_t e = t.messages + 1; d.ty(e) != ']'; e = d.after(e)) {
        RecWalk::Msg g; const int role = W.scan_message(e, g);
        if (role == 2 || role == 3) an_system<true>(W, g, first);
      }
      W.lit(L_RBRACK);
    }
    if (gcp && stream) W.lit(L_AN_STREAM);
    W.lit(L_AN_VERSION);
    if (const uint32_t vl = S.lit_len[CL_VERSION]) {
      const uint8_t* vp = S.lits + S.lit_off[CL_VERSION];
      for (uint32_t i = 0; i < vl; i++) { const uint32_t c = vp[i]; if (c < 0x20 || c > 0x7f || c == '"' || c == '\\') { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; } }
      if (W.o.room(vl)) {
        const uint32_t at = W.o.rs_n;
        for (uint32_t i = 0; i < vl; i++) W.o.scr[at + i] = vp[i];
        W.o.rs_n = at + vl;
        W.o.push(REC_SCR, at, vl);
      }
    } else W.lit(gcp ? L_AN_VER_GCP : L_AN_VER_AWS);
    W.lit(L_AN_END);
  }
};

__global__ void __launch_bounds__(kClThreads, 2) chat_anthropic_large_kernel(const __grid_constant__ ChatLargeParams P) {
  __shared__ ClShared S;
  cl_request_loop<ClRecordRequest<AnPlan>>(P, S);
}

}  // namespace

cudaError_t launch_chat_anthropic_large(const ChatLargeParams& P, int grid, cudaStream_t st) {
  chat_anthropic_large_kernel<<<P.n < (uint32_t)grid ? (P.n ? P.n : 1u) : (uint32_t)grid, kClThreads, 0, st>>>(P);
  return cudaGetLastError();
}

}  // namespace aigw
