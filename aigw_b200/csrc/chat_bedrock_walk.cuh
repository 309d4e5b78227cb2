// The OpenAI → AWS Bedrock Converse walk of a /v1/chat/completions request of any size (thread 0 of a large-request CTA):
// ParseBody's top-level checks (scan_top) and plan_bedrock of the translate pass (chat_walk_impl.cuh), over the jump table of
// large_request.cuh.  One walker, two instantiations:
//   ClWalkT<ClNoOut>   the dry plan: every check in the translate pass's order, nothing recorded.  chat_large_kernel runs it
//                      before a passthrough, as the translate pass runs plan_bedrock with pl.dry.
//   ClWalkT<ClOut>     the emitting plan: the same walk, and the Converse record as an unbounded list of copy ops in the CTA's
//                      slice (chat_large_record_impl.cuh, chat_bedrock_large_kernel.cu).  chat_anthropic_large_kernel.cu runs
//                      the dry plan first and records the Anthropic Messages body with this walker's pieces.
// A restatement of the translate pass, not a reuse: its Walker reads a 16-bit token word with key ids from its index stage and is
// compiled once per schema group into its own kernels.  This one reads 24-bit positions and compares keys by their bytes.  A change
// to ParseBody's checks or to plan_bedrock has to be made here too; test_chat_large_gpu.py, test_chat_bedrock_large_gpu.py and
// test_chat_anthropic_large_gpu.py compare the two on the translate pass's corpora.
#pragma once
#include "canon_number.cuh"
#include "chat_kernel.cuh"
#include "large_request.cuh"

namespace aigw {
namespace {

static constexpr int kAnyDepth = 24;   // emit_any's container limit in the translate pass

// tokenize_seq (chat_walk_impl.cuh) of an unescaped "arguments" text: tokens as the scan writes them, a string's backslashes
// counted in cum.x.  Returns the token count or -reason.
__device__ int cl_tokenize(const uint8_t* s, uint32_t len, uint32_t* tw, uint2* cum) {
  int nt = 0; uint32_t i = 0, nesc = 0;
  while (i < len) {
    const uint32_t c = s[i];
    if (c == ' ' || c == '\n' || c == '\r' || c == '\t') { i++; continue; }
    if (c == '"') {
      cum[nt] = make_uint2(nesc, 0); tw[nt++] = i | (T_QOPEN << 24); i++;
      for (;;) {
        if (i >= len) return -AIGW_R_SYNTAX;
        const uint32_t ch = s[i];
        if (ch == '"') break;
        if (ch < 0x20) return -AIGW_R_CTRL_IN_STRING;
        if (ch == '\\') {
          if (i + 1 >= len) return -AIGW_R_SYNTAX;
          const uint32_t e = s[i + 1];
          if (!(e == '"' || e == '\\' || e == 'n' || e == 'r' || e == 't')) return -AIGW_R_ESCAPE;
          nesc++; i += 2; continue;
        }
        i++;
      }
      cum[nt] = make_uint2(nesc, 0); tw[nt++] = i | (T_QCLOSE << 24); i++; continue;
    }
    cum[nt] = make_uint2(nesc, 0);
    if (c == '{' || c == '}' || c == '[' || c == ']' || c == ':' || c == ',') { tw[nt++] = i | (c << 24); i++; continue; }
    tw[nt++] = i | (T_SCALAR << 24);
    while (i < len) { const uint32_t x = s[i]; if (x == ' ' || x == '\n' || x == '\r' || x == '\t' || x == '{' || x == '}' || x == '[' || x == ']' || x == ':' || x == ',' || x == '"') break; i++; }
  }
  cum[nt] = make_uint2(nesc, 0);   // read by str_has_backslash of nothing; keeps cum[nt] defined
  return nt;
}

// byte order of two keys; the bytes it reads are added to `work`
__device__ int cmp_keys(const LDoc& d, uint32_t a, uint32_t b, uint32_t& work) {
  const uint8_t* pa = d.s + d.str_off(a); const uint32_t la = d.str_len(a);
  const uint8_t* pb = d.s + d.str_off(b); const uint32_t lb = d.str_len(b);
  const uint32_t m = la < lb ? la : lb;
  uint32_t k = 0;
  while (k < m && pa[k] == pb[k]) k++;
  work += k + 1u;
  if (k < m) return pa[k] < pb[k] ? -1 : 1;
  return la == lb ? 0 : (la < lb ? -1 : 1);
}

// ---------------------------------------------------------------- record sinks
// The dry sink: the walk's checks alone.
struct ClNoOut {
  static constexpr bool kEmit = false;
  __device__ __forceinline__ void lit(uint32_t) {}
  __device__ __forceinline__ void span(const LDoc&, uint32_t, uint32_t) {}
  __device__ __forceinline__ void str(const LDoc&, uint32_t) {}
  __device__ __forceinline__ void capture(bool) {}
};

// emit_any (chat_walk_impl.cuh): the order of the walk and every check it makes, the canonical re-serialisation (compact, keys in
// byte order, numbers as canon_number spells them) into `o`.  0 or the reason.  `work` counts, over the request, the member visits
// of its key-order search (quadratic in an object's members) and the key bytes its compares read; past kChatAnyWork the request
// declines with AIGW_R_SCRATCH.
template <class Out>
__device__ int cl_any(const LDoc& d, uint32_t* stk, uint32_t root, uint32_t& work, Out& o) {
  int sp = 0;
  int open = -1, state = 0;
  auto pop = [&]() { const int child = open; if (--sp) { open = (int)stk[sp - 1]; state = d.ty(open) == '[' ? child : child - 3; } };
  uint32_t vi = root;
  bool need_value = true;
  for (;;) {
    if (need_value) {
      need_value = false;
      const uint32_t c = d.ty(vi);
      if (c == '"') { if (d.str_nc(vi)) return AIGW_R_ESCAPE; o.span(d, d.tok(vi), d.tok(vi + 1) + 1u); }
      else if (c == '[') {
        o.span(d, d.tok(vi), d.tok(vi) + 1u);
        if (d.ty(vi + 1) != ']') {
          if (sp >= kAnyDepth) return AIGW_R_DEPTH;
          stk[sp++] = vi; open = (int)vi; state = (int)vi + 1;
          vi = vi + 1; need_value = true; continue;
        }
        o.span(d, d.tok(vi + 1), d.tok(vi + 1) + 1u);
      } else if (c == '{') {
        o.span(d, d.tok(vi), d.tok(vi) + 1u);
        if (sp >= kAnyDepth) return AIGW_R_DEPTH;
        stk[sp++] = vi; open = (int)vi; state = -1;
      } else if (!(c == 't' || c == 'f' || c == 'n')) {
        const uint32_t t = d.tok(vi);
        const uint32_t l = canon_number(d.s + t, d.scalar_end(vi) - t, false);
        if (!l) return AIGW_R_NUMBER;
        o.span(d, t, t + l);
      } else o.span(d, d.tok(vi), d.scalar_end(vi));
    }
    if (sp == 0) return 0;
    if (d.ty(open) == '[') {
      const uint32_t nx = d.next(state);
      o.span(d, d.tok(nx), d.tok(nx) + 1u);   // ',' or ']'
      if (d.ty(nx) == ',') { state = (int)nx + 1; vi = nx + 1; need_value = true; }
      else pop();
    } else {
      const int last = state;
      int best = -1, cnt = 0;
      for (uint32_t m = open + 1; d.ty(m) != '}'; m = d.after(m + 3)) {
        if (++work > kChatAnyWork) return AIGW_R_SCRATCH;
        if (d.str_has_backslash(m)) return AIGW_R_ESCAPE;
        const int c1 = last < 0 ? 1 : cmp_keys(d, m, last, work);
        if (c1 == 0 && (int)m != last) return AIGW_R_DUP_KEY;
        if (c1 > 0 && (best < 0 || cmp_keys(d, m, best, work) < 0)) best = (int)m;
        if (++cnt > 64) return AIGW_R_UNSUPPORTED_FIELD;
      }
      if (best < 0) { const uint32_t cl = d.tok(d.jmp[open]); o.span(d, cl, cl + 1u); pop(); continue; }
      if (last >= 0) o.lit(L_COMMA);
      const uint32_t ko = d.tok(best), kc = d.tok(best + 1), colon = d.tok(best + 2);
      if (colon == kc + 1u) o.span(d, ko, colon + 1u);
      else { o.span(d, ko, kc + 1u); o.lit(L_COLON); }
      state = best;
      vi = best + 3; need_value = true;
    }
  }
}

struct ClArgs { uint8_t* s; uint32_t* tw; uint2* cum; uint32_t* jmp; };

// the member names of openai.ChatCompletionRequest the translate pass gives a top-level id (K_model .. K_guided_json, in order)
__device__ const char* const kClTop[] = {
    "model", "messages", "max_tokens", "max_completion_tokens", "modalities", "temperature", "top_p", "tools", "tool_choice", "thinking",
    "top_logprobs", "stop", "stream", "stream_options", "service_tier", "seed", "safetySettings", "frequency_penalty", "logit_bias",
    "logprobs", "n", "presence_penalty", "parallel_tool_calls", "prediction", "response_format", "reasoning_effort", "verbosity", "user",
    "audio", "web_search_options", "generationConfig", "guided_choice", "guided_regex", "guided_json"};
enum ClTop : int {
  T_model, T_messages, T_max_tokens, T_mct, T_modalities, T_temperature, T_top_p, T_tools, T_tool_choice, T_thinking, T_top_logprobs,
  T_stop, T_stream, T_stream_options, T_service_tier, T_seed, T_safety, T_frequency_penalty, T_logit_bias, T_logprobs, T_n,
  T_presence_penalty, T_parallel_tool_calls, T_prediction, T_response_format, T_reasoning_effort, T_verbosity, T_user, T_audio,
  T_web_search, T_generation_config, T_guided_choice, T_guided_regex, T_guided_json, T_COUNT
};

__device__ __forceinline__ uint32_t clen(const char* k) { uint32_t n = 0; while (k[n]) n++; return n; }

// the top-level members scan_top keeps (value tokens, kNone when absent or null); one type for every instantiation of the walk, so
// that a dry walk and an emitting walk read the same scan
struct ClTopMembers {
  uint32_t model, messages, temperature, top_p, max_tokens, mct, stop, stream, stream_options, tools, tool_choice, thinking, service_tier, model_raw, so_raw;
};

// ---------------------------------------------------------------- the walk (thread 0)
template <class Out>
struct ClWalkT {
  using Scratch = ClArgs;
  static constexpr bool kFlatArrays = false;
  LDoc d;
  LDoc a;          // the "arguments" text in hand
  ClArgs A;
  uint32_t* stk;
  int reason = 0, pending = 0;
  uint32_t arg_total = 0, any_work = 0;
  Out o;

  // the "arguments" text in hand: its words, escape counts, jump table and bytes, each for kChatArgMax bytes
  static __device__ __forceinline__ ClArgs scratch(uint2* rest) {
    ClArgs args;
    args.cum = rest;
    args.tw = (uint32_t*)(args.cum + kChatArgMax + 2);
    args.jmp = args.tw + kChatArgMax + 2;
    args.s = (uint8_t*)(args.jmp + kChatArgMax + 2);
    return args;
  }
  __device__ void decline(int r) { if (!reason) reason = r; }
  __device__ void pend(int r) { if (!pending) pending = r; }
  __device__ bool bad() const { return reason != 0; }
  __device__ bool is_str(uint32_t v) const { return d.ty(v) == '"'; }
  __device__ bool is_obj(uint32_t v) const { return d.ty(v) == '{'; }
  __device__ bool is_arr(uint32_t v) const { return d.ty(v) == '['; }
  __device__ bool is_bool(uint32_t v) const { const uint32_t c = d.ty(v); return c == 't' || c == 'f'; }
  __device__ bool is_num(uint32_t v) const { const uint32_t c = d.ty(v); return c == '-' || c - '0' < 10u; }
  __device__ bool is_null(uint32_t v) const { return d.ty(v) == 'n'; }
  // keys hold no backslash here (the depth pass declined escaped keys), so their raw bytes are their decoded value
  __device__ bool key(uint32_t m, const char* k) const { return d.raw_is(m, k, clen(k)); }
  // an enumerated string value; an escaped one declines (the translate pass decodes it before the lookup)
  __device__ bool val(uint32_t v, const char* k) { if (d.str_has_backslash(v)) { decline(AIGW_R_ESCAPE); return false; } return d.raw_is(v, k, clen(k)); }
  __device__ void str(uint32_t v) { o.str(d, v); }
  __device__ void lit(uint32_t id) { o.lit(id); }

  // value token of member `k` in object `obj`, kNone when absent or null; duplicates decline
  __device__ uint32_t find(uint32_t obj, const char* k) {
    uint32_t r = kNone;
    const uint32_t kl = clen(k);
    for (uint32_t m = obj + 1; d.ty(m) != '}'; m = d.after(m + 3)) {
      if (d.raw_is(m, k, kl)) { if (r != kNone) { decline(AIGW_R_DUP_KEY); return kNone; } r = m + 3; }
    }
    if (r != kNone && is_null(r)) return kNone;
    return r;
  }
  __device__ bool cache_enabled(uint32_t cc) {
    if (cc == kNone) return false;
    if (!is_obj(cc)) { decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
    uint32_t t = kNone, ttl = kNone;
    for (uint32_t m = cc + 1; d.ty(m) != '}'; m = d.after(m + 3)) {
      if (key(m, "type")) { if (t != kNone) { decline(AIGW_R_DUP_KEY); return false; } t = m + 3; }
      else if (key(m, "ttl")) { if (ttl != kNone) { decline(AIGW_R_DUP_KEY); return false; } ttl = m + 3; }
    }
    if (ttl != kNone && !is_null(ttl) && !is_str(ttl)) { decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
    if (t == kNone || is_null(t)) return false;
    if (!is_str(t)) { decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
    return val(t, "ephemeral");
  }
  // emit_num_field: the canonical spelling of a number, a prefix of its bytes
  __device__ void num_field(uint32_t v, bool integer) {
    if (!is_num(v)) { decline(AIGW_R_E400_TYPE); return; }
    const uint32_t t = d.tok(v);
    const uint32_t l = canon_number(d.s + t, d.scalar_end(v) - t, integer);
    if (!l) decline(AIGW_R_NUMBER);
    else o.span(d, t, t + l);
  }
  __device__ bool check_scalar_type(uint32_t v, int kind /*0 str,1 bool,2 int,3 float*/) {
    if (v == kNone) return true;
    bool ok;
    if (kind == 0) ok = is_str(v);
    else if (kind == 1) ok = is_bool(v);
    else {
      ok = is_num(v);
      if (ok && kind == 2) {
        const uint32_t e = d.scalar_end(v), t = d.tok(v);
        ok = canon_number(d.s + t, e - t, true) != 0;
        if (!ok) {
          bool frac = false; for (uint32_t i = t; i < e; i++) { const uint32_t c = d.s[i]; if (c == '.' || c == 'e' || c == 'E') frac = true; }
          decline(frac ? AIGW_R_E400_TYPE : AIGW_R_NUMBER); return false;
        }
      }
    }
    if (!ok) decline(AIGW_R_E400_TYPE);
    return ok;
  }

  struct Part { uint32_t type, text, cache, refusal, signature, redacted; };
  __device__ bool scan_part(uint32_t e, Part& p) {
    p.type = p.text = p.cache = p.refusal = p.signature = p.redacted = kNone;
    uint32_t seen = 0;
    for (uint32_t m = e + 1; d.ty(m) != '}'; m = d.after(m + 3)) {
      const int slot = key(m, "type") ? 0 : key(m, "text") ? 1 : key(m, "cache_control") ? 2 : key(m, "refusal") ? 3 : key(m, "signature") ? 4
                     : key(m, "redactedContent") ? 5 : -1;
      if (slot < 0) continue;
      if (seen & (1u << slot)) { decline(AIGW_R_DUP_KEY); return false; }
      seen |= 1u << slot;
      const uint32_t v = is_null(m + 3) ? kNone : m + 3;
      switch (slot) { case 0: p.type = v; break; case 1: p.text = v; break; case 2: p.cache = v; break; case 3: p.refusal = v; break; case 4: p.signature = v; break; default: p.redacted = v; }
    }
    return true;
  }
  // emit_text_parts: system / developer (with cachePoint) and tool-result parts.  kE: record them (the system messages' second
  // pass); `first`: no separator yet (for the system list, its opening literal goes first)
  template <bool kE>
  __device__ void text_parts(uint32_t arr, bool with_cache, bool sys, bool& first) {
    for (uint32_t e = arr + 1; d.ty(e) != ']'; e = d.after(e)) {
      if (!is_obj(e)) { decline(is_null(e) ? AIGW_R_CONTENT : AIGW_R_E400_TYPE); return; }
      Part p; if (!scan_part(e, p)) return;
      if ((p.text != kNone && !is_str(p.text)) || (p.type != kNone && !is_str(p.type))) { decline(AIGW_R_E400_TYPE); return; }
      const bool cache = cache_enabled(p.cache);
      if (bad()) return;
      if constexpr (kE) {
        if (!first) lit(L_COMMA); else if (sys) lit(L_SYSTEM_OPEN);
        first = false;
        lit(L_TEXT_OPEN);
        if (p.text != kNone) str(p.text); else lit(L_EMPTY_STR);
        lit(L_RBRACE);
        if (with_cache && cache) { lit(L_COMMA); lit(L_CACHEPOINT); }
      }
    }
  }

  struct Msg { uint32_t role_v, content, name, tool_calls, tool_call_id, refusal, audio; };
  // role: 0 user 1 assistant 2 system 3 developer 4 tool
  __device__ int scan_message(uint32_t m, Msg& g) {
    g.role_v = g.content = g.name = g.tool_calls = g.tool_call_id = g.refusal = g.audio = kNone;
    if (!is_obj(m)) { decline(AIGW_R_E400_ROLE); return -1; }
    uint32_t seen = 0;
    for (uint32_t k = m + 1; d.ty(k) != '}'; k = d.after(k + 3)) {
      const uint32_t v = k + 3;
      const int which = key(k, "role") ? 0 : key(k, "content") ? 1 : key(k, "name") ? 2 : key(k, "tool_calls") ? 3 : key(k, "tool_call_id") ? 4
                      : key(k, "refusal") ? 5 : key(k, "audio") ? 6 : -1;
      if (which < 0) continue;
      if (seen & (1u << which)) { decline(AIGW_R_DUP_KEY); return -1; }
      seen |= 1u << which;
      switch (which) { case 0: g.role_v = v; break; case 1: g.content = v; break; case 2: g.name = v; break; case 3: g.tool_calls = v; break;
        case 4: g.tool_call_id = v; break; case 5: g.refusal = v; break; default: g.audio = v; }
    }
    if (g.role_v == kNone || !is_str(g.role_v)) { decline(AIGW_R_E400_ROLE); return -1; }
    if (d.str_has_backslash(g.role_v)) { decline(AIGW_R_ESCAPE); return -1; }
    if (val(g.role_v, "user")) return 0;
    if (val(g.role_v, "assistant")) return 1;
    if (val(g.role_v, "system")) return 2;
    if (val(g.role_v, "developer")) return 3;
    if (val(g.role_v, "tool")) return 4;
    decline(AIGW_R_E400_ROLE); return -1;
  }

  // bedrock_tool_result: one toolResult block
  __device__ void tool_result(const Msg& g) {
    lit(L_TOOLRESULT_OPEN);
    if (g.content == kNone) pend(AIGW_R_E422_CONTENT);
    else if (is_str(g.content)) { lit(L_TEXT_OPEN); str(g.content); lit(L_RBRACE); }
    else if (is_arr(g.content)) { bool first = true; text_parts<Out::kEmit>(g.content, false, false, first); }
    else { decline(AIGW_R_E400_CONTENT); return; }
    if (bad()) return;
    lit(L_TOOLRESULT_MID);
    uint32_t id = g.tool_call_id;
    if (id != kNone && is_null(id)) id = kNone;
    if (id != kNone && !is_str(id)) { decline(AIGW_R_E400_TYPE); return; }
    if (id != kNone) str(id); else lit(L_EMPTY_STR);
    lit(L_TOOLRESULT_CLOSE);
  }

  // emit_arguments: the JSON text inside the string → map[string]any, checked and re-serialised as the translate pass's emit_any
  // walks it (the record gets it through the sink's capture)
  __device__ void arguments(uint32_t v) {
    if (d.str_nc(v)) { decline(AIGW_R_ESCAPE); return; }
    const uint32_t off = d.str_off(v), n = d.str_len(v);
    if (n > kChatArgMax || arg_total + n > kChatArgTotal) { decline(AIGW_R_SCRATCH); return; }
    arg_total += n;
    const uint8_t* p = d.s + off;
    uint32_t w = 0;
    for (uint32_t i = 0; i < n; i++) {
      uint32_t c = p[i];
      if (c == '\\') { const uint32_t e = p[++i]; c = e == 'n' ? '\n' : e == 'r' ? '\r' : e == 't' ? '\t' : e; }
      A.s[w++] = (uint8_t)c;
    }
    const int nt = cl_tokenize(A.s, w, A.tw, A.cum);
    if (nt == 0 || nt == -AIGW_R_SYNTAX) { pend(AIGW_R_E500_ARGS); lit(L_NULL); return; }
    if (nt < 0) { decline(-nt); return; }
    a = LDoc{A.s, w, A.tw, A.cum, A.jmp, (uint32_t)nt};
    { const int vr = cl_validate(a, stk, true); if (vr == AIGW_R_SYNTAX) { pend(AIGW_R_E500_ARGS); lit(L_NULL); return; } if (vr) { decline(vr); return; } }
    const uint32_t c0 = a.ty(0);
    if (c0 == 'n') { lit(L_NULL); return; }
    if (c0 != '{') { pend(AIGW_R_E500_ARGS); lit(L_NULL); return; }
    o.capture(true);
    const int r = cl_any(a, stk, 0, any_work, o);
    o.capture(false);
    if (r) decline(r);
  }

  // bedrock_asst_part
  __device__ void asst_part(uint32_t e, bool& first) {
    if (!is_obj(e)) { decline(is_null(e) ? AIGW_R_CONTENT : AIGW_R_E400_CONTENT); return; }
    Part p; if (!scan_part(e, p)) return;
    if ((p.type != kNone && !is_str(p.type)) || (p.text != kNone && !is_str(p.text)) || (p.refusal != kNone && !is_str(p.refusal)) ||
        (p.signature != kNone && !is_str(p.signature))) { decline(AIGW_R_E400_TYPE); return; }
    if (p.redacted != kNone) { decline(AIGW_R_UNSUPPORTED_FIELD); return; }
    const bool cache = cache_enabled(p.cache);
    if constexpr (Out::kEmit) {
      if (bad() || p.type == kNone) return;   // type "" matches no case
      bool emitted = false;
      if (val(p.type, "text")) { if (p.text != kNone) { if (!first) lit(L_COMMA); first = false; lit(L_TEXT_OPEN); str(p.text); lit(L_RBRACE); emitted = true; } }
      else if (val(p.type, "refusal")) { if (p.refusal != kNone) { if (!first) lit(L_COMMA); first = false; lit(L_TEXT_OPEN); str(p.refusal); lit(L_RBRACE); emitted = true; } }
      else if (val(p.type, "thinking")) {
        if (p.text != kNone) {
          if (!first) lit(L_COMMA); first = false;
          lit(L_REASON_OPEN); str(p.text);
          if (p.signature != kNone && d.str_len(p.signature) > 0) { lit(L_REASON_SIG); str(p.signature); }
          lit(L_REASON_CLOSE); emitted = true;
        }
      }
      if (emitted && cache) { lit(L_COMMA); lit(L_CACHEPOINT); }
    }
  }

  __device__ void assistant(const Msg& g) {
    lit(L_MSG_CONTENT_OPEN);
    bool first = true;
    const uint32_t c = g.content;
    if (c != kNone && !is_null(c)) {
      if (is_str(c)) { if (d.str_len(c) > 0) { lit(L_TEXT_OPEN); str(c); lit(L_RBRACE); first = false; } }
      else if (is_arr(c)) { for (uint32_t e = c + 1; d.ty(e) != ']'; e = d.after(e)) { asst_part(e, first); if (bad()) return; } }
      else if (is_obj(c)) { asst_part(c, first); if (bad()) return; }
      else { decline(AIGW_R_E400_CONTENT); return; }
    }
    if (g.audio != kNone && !is_null(g.audio)) { decline(AIGW_R_UNSUPPORTED_FIELD); return; }
    if (g.name != kNone && !is_null(g.name) && !is_str(g.name)) { decline(AIGW_R_E400_TYPE); return; }
    if (g.refusal != kNone && !is_null(g.refusal) && !is_str(g.refusal)) { decline(AIGW_R_E400_TYPE); return; }
    const uint32_t tcs = g.tool_calls;
    if (tcs != kNone && !is_null(tcs)) {
      if (!is_arr(tcs)) { decline(AIGW_R_E400_TYPE); return; }
      for (uint32_t e = tcs + 1; d.ty(e) != ']'; e = d.after(e)) {
        if (!is_obj(e)) { decline(is_null(e) ? AIGW_R_TOOL : AIGW_R_E400_TYPE); return; }
        const uint32_t id = find(e, "id"), fn = find(e, "function"), ty = find(e, "type");
        (void)cache_enabled(find(e, "cache_control"));
        if (bad()) return;
        if (id == kNone) { decline(AIGW_R_TOOL); return; }
        if (!is_str(id)) { decline(AIGW_R_E400_TYPE); return; }
        if (ty != kNone && !is_str(ty)) { decline(AIGW_R_E400_TYPE); return; }
        uint32_t name = kNone, args = kNone;
        if (fn != kNone) { if (!is_obj(fn)) { decline(AIGW_R_E400_TYPE); return; } name = find(fn, "name"); args = find(fn, "arguments"); }
        if (bad()) return;
        if ((name != kNone && !is_str(name)) || (args != kNone && !is_str(args))) { decline(AIGW_R_E400_TYPE); return; }
        if (!first) lit(L_COMMA);
        first = false;
        lit(L_TOOLUSE_OPEN);
        if (name != kNone) str(name); else lit(L_EMPTY_STR);
        lit(L_TOOLUSE_INPUT);
        if (args == kNone) { pend(AIGW_R_E500_ARGS); lit(L_NULL); }
        else arguments(args);
        if (bad()) return;
        lit(L_TOOLUSE_ID); str(id);
        lit(L_TOOLRESULT_CLOSE);
      }
    }
    lit(L_ASST_CLOSE);
  }

  __device__ void user(const Msg& g) {
    const uint32_t c = g.content;
    if (g.name != kNone && !is_null(g.name) && !is_str(g.name)) { decline(AIGW_R_E400_TYPE); return; }
    if (c == kNone) { pend(AIGW_R_E422_CONTENT); return; }
    if (is_null(c)) { lit(L_MSG_TEXT_OPEN); lit(L_EMPTY_STR); lit(L_USER_CLOSE1); return; }
    if (is_str(c)) { lit(L_MSG_TEXT_OPEN); str(c); lit(L_USER_CLOSE1); return; }
    if (!is_arr(c)) { decline(AIGW_R_E400_CONTENT); return; }
    lit(L_MSG_CONTENT_OPEN);
    bool first = true;
    for (uint32_t e = c + 1; d.ty(e) != ']'; e = d.after(e)) {
      if (!is_obj(e)) { decline(AIGW_R_E400_CONTENT); return; }
      Part p; if (!scan_part(e, p)) return;
      if (p.type == kNone || !is_str(p.type)) { decline(AIGW_R_E400_CONTENT); return; }
      if (d.str_has_backslash(p.type)) { decline(AIGW_R_CONTENT); return; }
      if (!val(p.type, "text")) {
        decline((val(p.type, "image_url") || val(p.type, "input_audio") || val(p.type, "file")) ? AIGW_R_CONTENT : AIGW_R_E400_CONTENT); return;
      }
      if (p.text != kNone && !is_str(p.text)) { decline(AIGW_R_E400_TYPE); return; }
      const bool cache = cache_enabled(p.cache);
      if (bad()) return;
      if (!first) lit(L_COMMA);
      first = false;
      lit(L_TEXT_OPEN); if (p.text != kNone) str(p.text); else lit(L_EMPTY_STR); lit(L_RBRACE);
      if (cache) { lit(L_COMMA); lit(L_CACHEPOINT); }
    }
    lit(L_USER_CLOSE);
  }

  // bedrock_system: checked in the first pass over the messages, recorded (kE) in a second one, after the messages list
  template <bool kE>
  __device__ void system(const Msg& g, bool& first) {
    const uint32_t c = g.content;
    if (g.name != kNone && !is_null(g.name) && !is_str(g.name)) { decline(AIGW_R_E400_TYPE); return; }
    if (c == kNone) { pend(AIGW_R_E422_CONTENT); return; }
    if (is_str(c)) {
      if constexpr (kE) { lit(first ? L_SYSTEM_OPEN : L_COMMA); first = false; lit(L_TEXT_OPEN); str(c); lit(L_RBRACE); }
      return;
    }
    if (is_arr(c)) text_parts<kE>(c, true, true, first);
    else decline(AIGW_R_E400_CONTENT);
  }

  using Top = ClTopMembers;

  __device__ int top_id(uint32_t m) const {
    const uint32_t n = d.str_len(m);
    if (n < 1 || n > 21) return -1;
    for (int k = 0; k < T_COUNT; k++) if (d.raw_is(m, kClTop[k], clen(kClTop[k]))) return k;
    return -1;
  }

  // scan_top: the top-level members with the type checks of ParseBody
  __device__ bool scan_top(Top& t) {
    t.model = t.messages = t.temperature = t.top_p = t.max_tokens = t.mct = t.stop = t.stream = t.stream_options = t.tools = t.tool_choice = t.thinking = t.service_tier = t.model_raw = t.so_raw = kNone;
    if (d.nt == 0 || !is_obj(0)) { decline(d.nt && is_null(0) ? AIGW_R_ROOT : AIGW_R_E400_TYPE); return false; }
    uint64_t seen = 0;
    for (uint32_t k = 1; d.ty(k) != '}'; k = d.after(k + 3)) {
      const uint32_t v = k + 3;
      const int id = top_id(k);
      if (id < 0) continue;
      if (seen & (1ull << id)) { decline(AIGW_R_DUP_KEY); return false; }
      seen |= 1ull << id;
      if (id == T_model) t.model_raw = v; else if (id == T_stream_options) t.so_raw = v;
      if (is_null(v)) continue;
      switch (id) {
        case T_model: t.model = v; break; case T_messages: t.messages = v; break; case T_max_tokens: t.max_tokens = v; break; case T_mct: t.mct = v; break;
        case T_temperature: t.temperature = v; break; case T_top_p: t.top_p = v; break; case T_tools: t.tools = v; break; case T_tool_choice: t.tool_choice = v; break;
        case T_thinking: t.thinking = v; break; case T_stop: t.stop = v; break; case T_stream: t.stream = v; break; case T_stream_options: t.stream_options = v; break;
        case T_service_tier: t.service_tier = v; break;
        case T_reasoning_effort: case T_verbosity: case T_user: case T_guided_regex: if (!check_scalar_type(v, 0)) return false; break;
        case T_logprobs: case T_parallel_tool_calls: if (!check_scalar_type(v, 1)) return false; break;
        case T_top_logprobs: case T_seed: case T_n: if (!check_scalar_type(v, 2)) return false; break;
        case T_frequency_penalty: case T_presence_penalty: if (!check_scalar_type(v, 3)) return false; break;
        case T_guided_json: break;
        default: decline(AIGW_R_UNSUPPORTED_FIELD); return false;
      }
    }
    if (t.model != kNone && (!is_str(t.model) || d.str_has_backslash(t.model))) { decline(is_str(t.model) ? AIGW_R_ESCAPE : AIGW_R_E400_TYPE); return false; }
    if (t.messages != kNone && !is_arr(t.messages)) { decline(AIGW_R_E400_TYPE); return false; }
    if (t.stream != kNone && !is_bool(t.stream)) { decline(AIGW_R_E400_TYPE); return false; }
    if (t.service_tier != kNone && !is_str(t.service_tier)) { decline(AIGW_R_E400_TYPE); return false; }
    if (t.tools != kNone && !is_arr(t.tools)) { decline(AIGW_R_E400_TYPE); return false; }
    if (t.stream_options != kNone) {
      if (!is_obj(t.stream_options)) { decline(AIGW_R_E400_TYPE); return false; }
      const uint32_t iu = find(t.stream_options, "include_usage");
      if (iu != kNone && !is_bool(iu)) { decline(AIGW_R_E400_TYPE); return false; }
    }
    if (t.temperature != kNone && !is_num(t.temperature)) { decline(AIGW_R_E400_TYPE); return false; }
    if (t.top_p != kNone && !is_num(t.top_p)) { decline(AIGW_R_E400_TYPE); return false; }
    if (t.max_tokens != kNone && !check_scalar_type(t.max_tokens, 2)) return false;
    if (t.mct != kNone && !check_scalar_type(t.mct, 2)) return false;
    return !bad();
  }

  // the model contains `needle` (its raw bytes: scan_top declined an escaped model)
  __device__ bool model_contains(uint32_t mv, const char* needle) const {
    if (mv == kNone) return false;
    const uint8_t* p = d.s + d.str_off(mv); const uint32_t L = d.str_len(mv), n = clen(needle);
    for (uint32_t i = 0; i + n <= L; i++) { uint32_t k = 0; while (k < n && p[i + k] == (uint8_t)needle[k]) k++; if (k == n) return true; }
    return false;
  }

  // the dry plan, as cl_request_loop calls it
  __device__ void check(const Top& t) { plan(t); }

  // plan_bedrock after the ":path" (the sink records that): every check in the same order, the body's ops into the sink.  Inlined
  // into its caller, so that the walker and its sink stay in registers
  __device__ __forceinline__ void plan(const Top& t) {
    lit(L_LBRACE);
    if (t.thinking != kNone) {
      const uint32_t th = t.thinking;
      if (!is_obj(th)) { decline(AIGW_R_E400_TYPE); return; }
      const uint32_t ty = find(th, "type");
      if (ty == kNone || !is_str(ty)) { decline(AIGW_R_E400_TYPE); return; }
      if (val(ty, "enabled")) {
        const uint32_t bt = find(th, "budget_tokens"), it = find(th, "includeThoughts");
        if (it != kNone && !is_bool(it)) { decline(AIGW_R_E400_TYPE); return; }
        lit(L_ADDL_EN_PRE);
        if (bt != kNone) num_field(bt, true); else lit(L_ZERO);
        lit(L_ADDL_EN_POST);
      } else if (val(ty, "disabled")) lit(L_ADDL_DIS);
      else if (val(ty, "adaptive")) {}
      else { decline(AIGW_R_E400_TYPE); return; }
      if (bad()) return;
    }
    lit(L_INF_OPEN);
    bool f = true;
    const uint32_t mt = t.mct != kNone ? t.mct : t.max_tokens;
    if (mt != kNone) { lit(L_MAXTOK); num_field(mt, true); f = false; }
    if (t.stop != kNone) {
      const uint32_t s = t.stop;
      if (is_str(s)) { if (!f) lit(L_COMMA); f = false; lit(L_STOPSEQ); str(s); lit(L_RBRACK); }
      else if (is_arr(s)) {
        if (Out::kEmit && d.ty(s + 1) != ']') { if (!f) lit(L_COMMA); f = false; lit(L_STOPSEQ); }
        for (uint32_t e = s + 1; d.ty(e) != ']'; e = d.after(e)) {
          if (!is_str(e)) { decline(AIGW_R_UNSUPPORTED_FIELD); return; }
          if (e != s + 1) lit(L_COMMA);
          str(e);
        }
        if (Out::kEmit && d.ty(s + 1) != ']') lit(L_RBRACK);
      }
      else { decline(AIGW_R_UNSUPPORTED_FIELD); return; }
    }
    if (t.temperature != kNone) { if (!f) lit(L_COMMA); f = false; lit(L_TEMP); num_field(t.temperature, false); }
    if (t.top_p != kNone) { if (!f) lit(L_COMMA); f = false; lit(L_TOPP); num_field(t.top_p, false); }
    if (bad()) return;
    lit(L_INF_CLOSE_MSGS);
    bool any_sys = false;
    if (t.messages != kNone) {
      // a run of consecutive tool messages becomes one user message (openai_awsbedrock.go:559-575); a system message ends it
      bool mfirst = true, in_run = false;
      for (uint32_t e = t.messages + 1; d.ty(e) != ']'; e = d.after(e)) {
        Msg g; const int role = scan_message(e, g);
        if (bad()) return;
        if (role != 4 && in_run) { lit(L_USER_CLOSE); in_run = false; }
        if (role == 2 || role == 3) { bool first = true; system<false>(g, first); any_sys = true; }
        else {
          if (role == 4 && in_run) lit(L_COMMA);
          else { if (!mfirst) lit(L_COMMA); mfirst = false; }
          if (role == 0) user(g);
          else if (role == 1) assistant(g);
          else { if (!in_run) lit(L_MSG_CONTENT_OPEN); in_run = true; tool_result(g); }
        }
        if (bad()) return;
      }
      if (in_run) lit(L_USER_CLOSE);
    }
    lit(L_RBRACK);
    if constexpr (Out::kEmit) {
      // "system" goes after "messages": a second pass over the messages records what the first one checked
      if (any_sys) {
        bool first = true;
        for (uint32_t e = t.messages + 1; d.ty(e) != ']'; e = d.after(e)) {
          Msg g; const int role = scan_message(e, g);
          if (role == 2 || role == 3) system<true>(g, first);
        }
        if (!first) lit(L_RBRACK);
      }
      if (t.service_tier != kNone && d.str_len(t.service_tier) > 0) { lit(L_SERVICE_TIER); str(t.service_tier); lit(L_RBRACE); }
    } else (void)any_sys;
    // tool_choice decodes (and can fail) whether or not tools are present (openai.go:1194-1210)
    int tc_kind = 0;   // 1 auto, 2 any, 3 tool{name}
    uint32_t tc_name = kNone;
    if (t.tool_choice != kNone) {
      const uint32_t tc = t.tool_choice;
      if (is_str(tc)) {
        if constexpr (Out::kEmit) {
          if (val(tc, "auto")) tc_kind = 1;
          else if (val(tc, "required")) tc_kind = 2;
          else if (model_contains(t.model, "anthropic") && model_contains(t.model, "claude")) { tc_kind = 3; tc_name = tc; }
          if (bad()) return;
        }
      }
      else if (is_obj(tc)) {
        const uint32_t ty = find(tc, "type"), fn = find(tc, "function");
        if (ty != kNone && !is_str(ty)) { decline(AIGW_R_E400_TYPE); return; }
        if (fn != kNone) {
          if (!is_obj(fn)) { decline(AIGW_R_E400_TYPE); return; }
          tc_name = find(fn, "name");
          if (tc_name != kNone && !is_str(tc_name)) { decline(AIGW_R_E400_TYPE); return; }
        }
        if (bad()) return;
        tc_kind = 3;
      } else { decline(AIGW_R_E400_TYPE); return; }
    }
    if (t.tools != kNone && d.ty(t.tools + 1) != ']') {
      lit(L_TOOLCFG_OPEN);
      if (tc_kind == 1) lit(L_TOOLCHOICE_AUTO);
      else if (tc_kind == 2) lit(L_TOOLCHOICE_ANY);
      else if (tc_kind == 3) { lit(L_TOOLCHOICE_TOOL); if (tc_name != kNone) str(tc_name); else lit(L_EMPTY_STR); lit(L_TOOLCHOICE_TOOL_END); }
      lit(L_TOOLS_OPEN);
      bool tf = true;
      for (uint32_t e = t.tools + 1; d.ty(e) != ']'; e = d.after(e)) {
        if (!is_obj(e)) { decline(is_null(e) ? AIGW_R_TOOL : AIGW_R_E400_TYPE); return; }
        const uint32_t ty = find(e, "type"), fn = find(e, "function"), gs = find(e, "google_search");
        if (ty != kNone && !is_str(ty)) { decline(AIGW_R_E400_TYPE); return; }
        if (gs != kNone) { decline(AIGW_R_UNSUPPORTED_FIELD); return; }
        if (bad()) return;
        if (fn != kNone) {
          if (!is_obj(fn)) { decline(AIGW_R_E400_TYPE); return; }
          const uint32_t nm = find(fn, "name"), ds = find(fn, "description"), st = find(fn, "strict"), pr = find(fn, "parameters");
          const bool cache = cache_enabled(find(fn, "cache_control"));
          if (bad()) return;
          if ((nm != kNone && !is_str(nm)) || (ds != kNone && !is_str(ds)) || (st != kNone && !is_bool(st))) { decline(AIGW_R_E400_TYPE); return; }
          if (!tf) lit(L_COMMA);
          tf = false;
          lit(L_TOOLSPEC_OPEN);
          if (ds != kNone && d.str_len(ds) > 0) { lit(L_DESC); str(ds); lit(L_COMMA); }
          lit(L_INPUTSCHEMA);
          if (pr != kNone) { if (const int r = cl_any(d, stk, pr, any_work, o)) { decline(r); return; } }
          else lit(L_NULL);
          lit(L_NAME); if (nm != kNone) str(nm); else lit(L_EMPTY_STR); lit(L_RBRACE);
          if (cache) lit(L_TOOL_CACHE);
          lit(L_RBRACE);
        }
      }
      lit(L_TOOLS_CLOSE);
    }
    lit(L_RBRACE);
  }
};

using ClWalk = ClWalkT<ClNoOut>;

}  // namespace
}  // namespace aigw
