// /v1/chat/completions requests above the translate pass's 64 KiB ceiling (and below it) to the OpenAI and Azure OpenAI
// passthroughs: ChatCompletionsEndpointSpec.ParseBody's verdict, the ":path" and at most two sjson edits, with the semantics group
// 1 of the translate pass gives them (scan_top, passthrough_accepts, plan_passthrough / plan_azure in chat_walk_impl.cuh).
// sm_90a only.
//
// chat_large_kernel: one CTA of 256 threads per request, the stages of large_request.cuh (scan, depth, grammar, emit) around this
// file's walk and plan:
//   walk      thread 0 runs scan_top and the dry Bedrock plan over the jump table: the same checks in the same order, so the
//             first problem decides as in the translate pass (ParseBody's 400s, then a pending 422 / 500 as AIGW_R_CONTENT).  A
//             tool call's "arguments" string is unescaped into the CTA's slice, tokenized and checked there.
//   plan      the record as at most 12 copy ops: ":path" from literals (and the Azure deployment from the body), then the body
//             with edit A (stream_options.include_usage) and edit B (the model override) spliced in body order
#include "chat_large_kernel.cuh"

#include <string.h>

#include "canon_number.cuh"
#include "large_request.cuh"

namespace aigw {

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

// emit_any (chat_walk_impl.cuh) in the dry plan: the order of the walk and every check it makes, nothing emitted.  0 or the reason.
// `work` counts, over the request, the member visits of its key-order search (quadratic in an object's members) and the key
// bytes its compares read; past kChatAnyWork the request declines with AIGW_R_SCRATCH.
__device__ int cl_any(const LDoc& d, uint32_t* stk, uint32_t root, uint32_t& work) {
  int sp = 0;
  int open = -1, state = 0;
  auto pop = [&]() { const int child = open; if (--sp) { open = (int)stk[sp - 1]; state = d.ty(open) == '[' ? child : child - 3; } };
  uint32_t vi = root;
  bool need_value = true;
  for (;;) {
    if (need_value) {
      need_value = false;
      const uint32_t c = d.ty(vi);
      if (c == '"') { if (d.str_nc(vi)) return AIGW_R_ESCAPE; }
      else if (c == '[') {
        if (d.ty(vi + 1) != ']') {
          if (sp >= kAnyDepth) return AIGW_R_DEPTH;
          stk[sp++] = vi; open = (int)vi; state = (int)vi + 1;
          vi = vi + 1; need_value = true; continue;
        }
      } else if (c == '{') {
        if (sp >= kAnyDepth) return AIGW_R_DEPTH;
        stk[sp++] = vi; open = (int)vi; state = -1;
      } else if (!(c == 't' || c == 'f' || c == 'n')) {
        const uint32_t o = d.tok(vi);
        if (!canon_number(d.s + o, d.scalar_end(vi) - o, false)) return AIGW_R_NUMBER;
      }
    }
    if (sp == 0) return 0;
    if (d.ty(open) == '[') {
      const uint32_t nx = d.next(state);
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
      if (best < 0) { pop(); continue; }
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

// ---------------------------------------------------------------- the walk (thread 0): the translate pass's Walker, dry
// A restatement, not a reuse: the translate pass's Walker (chat_walk_impl.cuh) reads a 16-bit token word with key ids from its
// index stage and is compiled once per schema group into its own kernels.  This one reads 24-bit positions and compares keys by
// their bytes.  A change to ParseBody's checks or to the dry Bedrock plan has to be made in both; test_chat_large_gpu.py compares
// the two on the translate pass's corpora under every OpenAI / Azure configuration.
struct ClWalk {
  using Scratch = ClArgs;
  static constexpr bool kFlatArrays = false;
  LDoc d;
  LDoc a;          // the "arguments" text in hand
  ClArgs A;
  uint32_t* stk;
  int reason = 0, pending = 0;
  uint32_t arg_total = 0, any_work = 0;

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
  __device__ void num_field(uint32_t v, bool integer) {
    if (!is_num(v)) { decline(AIGW_R_E400_TYPE); return; }
    const uint32_t o = d.tok(v);
    if (!canon_number(d.s + o, d.scalar_end(v) - o, integer)) decline(AIGW_R_NUMBER);
  }
  __device__ bool check_scalar_type(uint32_t v, int kind /*0 str,1 bool,2 int,3 float*/) {
    if (v == kNone) return true;
    bool ok;
    if (kind == 0) ok = is_str(v);
    else if (kind == 1) ok = is_bool(v);
    else {
      ok = is_num(v);
      if (ok && kind == 2) {
        const uint32_t e = d.scalar_end(v), o = d.tok(v);
        ok = canon_number(d.s + o, e - o, true) != 0;
        if (!ok) {
          bool frac = false; for (uint32_t i = o; i < e; i++) { const uint32_t c = d.s[i]; if (c == '.' || c == 'e' || c == 'E') frac = true; }
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
  __device__ void text_parts(uint32_t arr) {
    for (uint32_t e = arr + 1; d.ty(e) != ']'; e = d.after(e)) {
      if (!is_obj(e)) { decline(is_null(e) ? AIGW_R_CONTENT : AIGW_R_E400_TYPE); return; }
      Part p; if (!scan_part(e, p)) return;
      if ((p.text != kNone && !is_str(p.text)) || (p.type != kNone && !is_str(p.type))) { decline(AIGW_R_E400_TYPE); return; }
      cache_enabled(p.cache);
      if (bad()) return;
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

  __device__ void tool_result(const Msg& g) {
    if (g.content == kNone) pend(AIGW_R_E422_CONTENT);
    else if (is_str(g.content)) {}
    else if (is_arr(g.content)) text_parts(g.content);
    else { decline(AIGW_R_E400_CONTENT); return; }
    if (bad()) return;
    uint32_t id = g.tool_call_id;
    if (id != kNone && is_null(id)) id = kNone;
    if (id != kNone && !is_str(id)) decline(AIGW_R_E400_TYPE);
  }

  // emit_arguments: the JSON text inside the string → map[string]any, checked as the translate pass's emit_any walks it
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
    if (nt == 0 || nt == -AIGW_R_SYNTAX) { pend(AIGW_R_E500_ARGS); return; }
    if (nt < 0) { decline(-nt); return; }
    a = LDoc{A.s, w, A.tw, A.cum, A.jmp, (uint32_t)nt};
    { const int vr = cl_validate(a, stk, true); if (vr == AIGW_R_SYNTAX) { pend(AIGW_R_E500_ARGS); return; } if (vr) { decline(vr); return; } }
    const uint32_t c0 = a.ty(0);
    if (c0 == 'n') return;
    if (c0 != '{') { pend(AIGW_R_E500_ARGS); return; }
    if (const int r = cl_any(a, stk, 0, any_work)) decline(r);
  }

  __device__ void asst_part(uint32_t e) {
    if (!is_obj(e)) { decline(is_null(e) ? AIGW_R_CONTENT : AIGW_R_E400_CONTENT); return; }
    Part p; if (!scan_part(e, p)) return;
    if ((p.type != kNone && !is_str(p.type)) || (p.text != kNone && !is_str(p.text)) || (p.refusal != kNone && !is_str(p.refusal)) ||
        (p.signature != kNone && !is_str(p.signature))) { decline(AIGW_R_E400_TYPE); return; }
    if (p.redacted != kNone) { decline(AIGW_R_UNSUPPORTED_FIELD); return; }
    cache_enabled(p.cache);
  }

  __device__ void assistant(const Msg& g) {
    const uint32_t c = g.content;
    if (c != kNone && !is_null(c)) {
      if (is_str(c)) {}
      else if (is_arr(c)) { for (uint32_t e = c + 1; d.ty(e) != ']'; e = d.after(e)) { asst_part(e); if (bad()) return; } }
      else if (is_obj(c)) { asst_part(c); if (bad()) return; }
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
        if (args == kNone) pend(AIGW_R_E500_ARGS);
        else arguments(args);
        if (bad()) return;
      }
    }
  }

  __device__ void user(const Msg& g) {
    const uint32_t c = g.content;
    if (g.name != kNone && !is_null(g.name) && !is_str(g.name)) { decline(AIGW_R_E400_TYPE); return; }
    if (c == kNone) { pend(AIGW_R_E422_CONTENT); return; }
    if (is_null(c) || is_str(c)) return;
    if (!is_arr(c)) { decline(AIGW_R_E400_CONTENT); return; }
    for (uint32_t e = c + 1; d.ty(e) != ']'; e = d.after(e)) {
      if (!is_obj(e)) { decline(AIGW_R_E400_CONTENT); return; }
      Part p; if (!scan_part(e, p)) return;
      if (p.type == kNone || !is_str(p.type)) { decline(AIGW_R_E400_CONTENT); return; }
      if (d.str_has_backslash(p.type)) { decline(AIGW_R_CONTENT); return; }
      if (!val(p.type, "text")) {
        decline((val(p.type, "image_url") || val(p.type, "input_audio") || val(p.type, "file")) ? AIGW_R_CONTENT : AIGW_R_E400_CONTENT); return;
      }
      if (p.text != kNone && !is_str(p.text)) { decline(AIGW_R_E400_TYPE); return; }
      cache_enabled(p.cache);
      if (bad()) return;
    }
  }

  __device__ void system(const Msg& g) {
    const uint32_t c = g.content;
    if (g.name != kNone && !is_null(g.name) && !is_str(g.name)) { decline(AIGW_R_E400_TYPE); return; }
    if (c == kNone) { pend(AIGW_R_E422_CONTENT); return; }
    if (is_str(c)) return;
    if (is_arr(c)) text_parts(c);
    else decline(AIGW_R_E400_CONTENT);
  }

  struct Top { uint32_t model, messages, temperature, top_p, max_tokens, mct, stop, stream, stream_options, tools, tool_choice, thinking, service_tier, model_raw, so_raw; };

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

  // plan_bedrock in dry mode: every check, in the same order, nothing planned
  __device__ void check(const Top& t) {
    if (t.thinking != kNone) {
      const uint32_t th = t.thinking;
      if (!is_obj(th)) { decline(AIGW_R_E400_TYPE); return; }
      const uint32_t ty = find(th, "type");
      if (ty == kNone || !is_str(ty)) { decline(AIGW_R_E400_TYPE); return; }
      if (val(ty, "enabled")) {
        const uint32_t bt = find(th, "budget_tokens"), it = find(th, "includeThoughts");
        if (it != kNone && !is_bool(it)) { decline(AIGW_R_E400_TYPE); return; }
        if (bt != kNone) num_field(bt, true);
      } else if (val(ty, "disabled") || val(ty, "adaptive")) {}
      else { decline(AIGW_R_E400_TYPE); return; }
      if (bad()) return;
    }
    const uint32_t mt = t.mct != kNone ? t.mct : t.max_tokens;
    if (mt != kNone) num_field(mt, true);
    if (t.stop != kNone) {
      const uint32_t s = t.stop;
      if (is_str(s)) {}
      else if (is_arr(s)) { for (uint32_t e = s + 1; d.ty(e) != ']'; e = d.after(e)) if (!is_str(e)) { decline(AIGW_R_UNSUPPORTED_FIELD); return; } }
      else { decline(AIGW_R_UNSUPPORTED_FIELD); return; }
    }
    if (t.temperature != kNone) num_field(t.temperature, false);
    if (t.top_p != kNone) num_field(t.top_p, false);
    if (bad()) return;
    if (t.messages != kNone) {
      for (uint32_t e = t.messages + 1; d.ty(e) != ']'; e = d.after(e)) {
        Msg g; const int role = scan_message(e, g);
        if (bad()) return;
        if (role == 2 || role == 3) system(g);
        else if (role == 0) user(g);
        else if (role == 1) assistant(g);
        else tool_result(g);
        if (bad()) return;
      }
    }
    if (t.tool_choice != kNone) {
      const uint32_t tc = t.tool_choice;
      if (is_str(tc)) {}
      else if (is_obj(tc)) {
        const uint32_t ty = find(tc, "type"), fn = find(tc, "function");
        if (ty != kNone && !is_str(ty)) { decline(AIGW_R_E400_TYPE); return; }
        if (fn != kNone) {
          if (!is_obj(fn)) { decline(AIGW_R_E400_TYPE); return; }
          const uint32_t nm = find(fn, "name");
          if (nm != kNone && !is_str(nm)) { decline(AIGW_R_E400_TYPE); return; }
        }
        if (bad()) return;
      } else { decline(AIGW_R_E400_TYPE); return; }
    }
    if (t.tools != kNone && d.ty(t.tools + 1) != ']') {
      for (uint32_t e = t.tools + 1; d.ty(e) != ']'; e = d.after(e)) {
        if (!is_obj(e)) { decline(is_null(e) ? AIGW_R_TOOL : AIGW_R_E400_TYPE); return; }
        const uint32_t ty = find(e, "type"), fn = find(e, "function"), gs = find(e, "google_search");
        if (ty != kNone && !is_str(ty)) { decline(AIGW_R_E400_TYPE); return; }
        if (gs != kNone) { decline(AIGW_R_UNSUPPORTED_FIELD); return; }
        if (bad()) return;
        if (fn != kNone) {
          if (!is_obj(fn)) { decline(AIGW_R_E400_TYPE); return; }
          const uint32_t nm = find(fn, "name"), ds = find(fn, "description"), st = find(fn, "strict"), pr = find(fn, "parameters");
          cache_enabled(find(fn, "cache_control"));
          if (bad()) return;
          if ((nm != kNone && !is_str(nm)) || (ds != kNone && !is_str(ds)) || (st != kNone && !is_bool(st))) { decline(AIGW_R_E400_TYPE); return; }
          if (pr != kNone) { if (const int r = cl_any(d, stk, pr, any_work)) { decline(r); return; } }
        }
      }
    }
  }
};

// plan_passthrough / plan_azure after passthrough_accepts: the record's ops, flags and body kind.  0 or the reason.
__device__ int cl_plan(const ChatLargeParams& P, ClWalk& W, const ClWalk::Top& t, bool stream, ClRec& R) {
  const LDoc& d = W.d;
  const uint32_t len = d.len;
  const bool need_model = P.override_len != 0;
  uint32_t iu_raw = kNone;
  if (t.stream_options != kNone)
    for (uint32_t m = t.stream_options + 1; d.ty(m) != '}'; m = d.after(m + 3)) if (W.key(m, "include_usage")) { iu_raw = m + 3; break; }
  const bool inc_true = iu_raw != kNone && d.ty(iu_raw) == 't';
  const bool need_usage = stream && P.cost_configured && !inc_true;
  if (P.azure) {
    if (need_usage) R.S.flags |= 2u;
    R.lit(CL_AZ_PREFIX);
    if (need_model) R.lit(CL_OVERRIDE); else if (t.model != kNone) R.body(d.str_off(t.model), d.str_off(t.model) + d.str_len(t.model));
    R.lit(CL_AZ_SUFFIX); R.lit(CL_VERSION);
    if (R.olen > 0xffffu) return AIGW_R_TOO_LARGE;   // path_len is 16 bits
    R.S.path_len = R.olen; R.S.body_kind = AIGW_BODY_UNCHANGED;
    return 0;
  }
  R.lit(CL_OPENAI_PATH);
  R.S.path_len = R.olen;
  if (need_model && !P.override_ok) return AIGW_R_UNSUPPORTED_FIELD;
  if (need_usage) R.S.flags |= 2u;
  if (!need_usage && !need_model) {
    if (P.force_mutation) { R.body(0, len); R.S.body_kind = AIGW_BODY_BYTES; } else R.S.body_kind = AIGW_BODY_UNCHANGED;
    return 0;
  }
  R.S.body_kind = AIGW_BODY_BYTES;
  const uint32_t root_close = d.jmp[0];
  const bool root_empty = root_close == 1;
  // edit A (usage): 1 replace with true, 2 append member in stream_options, 3 replace with an object, 4 append at the root
  uint32_t a_b = kNone, a_e = 0; int a_kind = 0; bool a_comma = false;
  if (need_usage) {
    if (iu_raw != kNone) { a_kind = 1; a_b = d.tok(iu_raw); a_e = d.scalar_end(iu_raw); }
    else if (t.stream_options != kNone) { a_kind = 2; const uint32_t cl = d.jmp[t.stream_options]; a_b = a_e = d.tok(cl); a_comma = cl != t.stream_options + 1; }
    else if (t.so_raw != kNone) { a_kind = 3; a_b = d.tok(t.so_raw); a_e = d.scalar_end(t.so_raw); }
    else { a_kind = 4; a_b = a_e = d.tok(root_close); a_comma = !root_empty; }
  }
  // edit B (model): 1 replace the value, 2 append at the root
  uint32_t b_b = kNone, b_e = 0; int b_kind = 0;
  if (need_model) {
    if (t.model_raw != kNone) { b_kind = 1; b_b = d.tok(t.model_raw); b_e = W.is_str(t.model_raw) ? d.tok(t.model_raw + 1) + 1u : d.scalar_end(t.model_raw); }
    else { b_kind = 2; b_b = b_e = d.tok(root_close); }
  }
  const bool drop_outside = a_kind == 4 || b_kind == 2;   // sjson rebuilds the root: the bytes outside its braces go
  uint32_t cur = drop_outside ? d.tok(0) : 0u;
  const uint32_t end = drop_outside ? d.tok(root_close) + 1u : len;
  for (int pass = 0; pass < 2; pass++) {
    // the earlier edit first; at equal positions (both root appends) usage goes first, as in the reference's call order
    const bool do_a = pass == 0 ? (a_kind && (!b_kind || a_b <= b_b)) : (a_kind && b_kind && a_b > b_b);
    const bool do_b = pass == 0 ? (b_kind && !do_a) : (b_kind && a_kind && a_b <= b_b);
    if (do_a) {
      R.body(cur, a_b); cur = a_e;
      if (a_kind == 1) R.lit(CL_TRUE);
      else if (a_kind == 2) { if (a_comma) R.lit(CL_COMMA); R.lit(CL_IU_MEMBER); }
      else if (a_kind == 3) R.lit(CL_IU_OBJ);
      else { if (a_comma) R.lit(CL_COMMA); R.lit(CL_SO_APPEND); }
    } else if (do_b) {
      R.body(cur, b_b); cur = b_e;
      if (b_kind == 2) { if (!root_empty || a_kind == 4) R.lit(CL_COMMA); R.lit(CL_MODEL_MEMBER); }
      R.lit(CL_QUOTE); R.lit(CL_OVERRIDE); R.lit(CL_QUOTE);
    }
  }
  R.body(cur, end);
  return 0;
}

__global__ void __launch_bounds__(kClThreads, 2) chat_large_kernel(const __grid_constant__ ChatLargeParams P) {
  __shared__ ClShared S;
  cl_request_loop<ClWalk>(P, S);
}

uint64_t chat_large_slice_bytes(uint32_t max_len) {
  const uint64_t tc = chat_large_tok_cap(max_len);
  const uint64_t toks = tc * 4u * 2u + 8u + (tc + 1u) * 8u;                             // words, jump table, escape counts
  const uint64_t args = (uint64_t)(kChatArgMax + 2u) * (8u + 4u + 4u) + kChatArgMax + 16u;   // the "arguments" text in hand
  return (toks + args + 255u) & ~255ull;
}

int chat_large_grid(int sm_count, uint32_t max_len) {
  uint64_t g = kClWorkspace / chat_large_slice_bytes(max_len);
  if (g > (uint64_t)sm_count * 2u) g = (uint64_t)sm_count * 2u;
  return g < 1 ? 1 : (int)g;
}

void chat_large_lits(ChatLargeParams& P, const char* openai_path, uint32_t path_len, const char* override_model, uint32_t override_len,
                     const char* version, uint32_t version_len) {
  static const char* const kText[CL_OPENAI_PATH] = {
      "true", ",", "\"", "\"include_usage\":true", "{\"include_usage\":true}", "\"stream_options\":{\"include_usage\":true}", "\"model\":",
      "/openai/deployments/", "/chat/completions?api-version="};
  uint32_t at = 0;
  auto put = [&](uint32_t id, const char* s, uint32_t n) { P.lit_off[id] = (uint16_t)at; P.lit_len[id] = (uint16_t)n; memcpy(P.lits + at, s, n); at += n; };
  memset(P.lits, 0, sizeof P.lits);
  for (uint32_t i = 0; i < CL_OPENAI_PATH; i++) put(i, kText[i], (uint32_t)strlen(kText[i]));
  put(CL_OPENAI_PATH, openai_path, path_len);
  put(CL_OVERRIDE, override_model, override_len);
  put(CL_VERSION, version, version_len);
}

cudaError_t launch_chat_large(const ChatLargeParams& P, int grid, cudaStream_t st) {
  chat_large_kernel<<<P.n < (uint32_t)grid ? (P.n ? P.n : 1u) : (uint32_t)grid, kClThreads, 0, st>>>(P);
  return cudaGetLastError();
}

}  // namespace aigw
