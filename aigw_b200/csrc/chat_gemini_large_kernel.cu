// /v1/chat/completions requests above the translate pass's 64 KiB ceiling (and below it) to Gemini on GCP Vertex AI: ParseBody's
// verdict, the ":path" and the GenerateContent body, with the semantics group 3 of the translate pass gives them (scan_top and
// plan_gemini in chat_walk_impl.cuh).  sm_90a only.
//
// chat_gemini_large_kernel: one CTA of 256 threads per request, the scan and depth pass of large_request.cuh, then the record
// phase of chat_large_record_impl.cuh with this planner (thread 0), in plan_gemini's order:
//   dry plan  the Bedrock plan over the sink that records nothing (ClWalkT<ClNoOut>), as plan_gemini first runs plan_bedrock with
//             pl.dry: its declines stand, its pending 422 / 500 does not apply
//   checks    tool_choice, thinking, a non-empty reasoning_effort
//   record    ":path", then "contents" (consecutive user messages merged into one), "tools", "generation_config" in genai's field
//             order, and "system_instruction": system and developer messages are checked in the message pass and recorded after
//             generation_config by a second pass
#include "chat_gemini_large_kernel.cuh"

#include "chat_large_record_impl.cuh"

namespace aigw {
namespace {

// the generation_config members scan_top checks but does not keep (value tokens, kNone when absent or null).  scan_top has checked
// their types and declined a duplicate; only this planner reads them, so ClTopMembers (and every other large kernel) stays as it is.
struct GemTop { uint32_t n, freq_pen, pres_pen, top_logprobs, logprobs, seed, reasoning_effort; };

__device__ __forceinline__ GemTop gem_top(RecWalk& W) {
  GemTop g;
  g.n = g.freq_pen = g.pres_pen = g.top_logprobs = g.logprobs = g.seed = g.reasoning_effort = kNone;
  const LDoc& d = W.d;
  for (uint32_t k = 1; d.ty(k) != '}'; k = d.after(k + 3)) {
    const uint32_t v = k + 3;
    if (W.is_null(v)) continue;
    if (W.key(k, "n")) g.n = v;
    else if (W.key(k, "frequency_penalty")) g.freq_pen = v;
    else if (W.key(k, "presence_penalty")) g.pres_pen = v;
    else if (W.key(k, "top_logprobs")) g.top_logprobs = v;
    else if (W.key(k, "logprobs")) g.logprobs = v;
    else if (W.key(k, "seed")) g.seed = v;
    else if (W.key(k, "reasoning_effort")) g.reasoning_effort = v;
  }
  return g;
}

// emit_i32_field of the translate pass: the canonical spelling of an int32 field, at most 9 digits.  Its length, or 0 after a
// decline with AIGW_R_NUMBER; `zero`: the value is 0 (omitted by the omitempty fields)
__device__ __forceinline__ uint32_t gem_i32(RecWalk& W, uint32_t v, bool& zero) {
  const LDoc& d = W.d;
  const uint32_t t = d.tok(v);
  const uint32_t l = canon_number(d.s + t, d.scalar_end(v) - t, true);
  if (!l || l > 9u + (d.s[t] == '-' ? 1u : 0u)) { W.decline(AIGW_R_NUMBER); return 0; }
  zero = l == 1u && d.s[t] == '0';
  return l;
}

// emit_f32_field of the translate pass: a float32 field echoes its canonical literal when that has at most 6 significant digits
// (float32 to the shortest decimal then gives it back); more decline with AIGW_R_NUMBER
__device__ __forceinline__ void gem_f32(RecWalk& W, uint32_t v) {
  const LDoc& d = W.d;
  const uint32_t t = d.tok(v);
  const uint32_t l = canon_number(d.s + t, d.scalar_end(v) - t, false);
  if (!l) { W.decline(AIGW_R_NUMBER); return; }
  uint32_t sig = 0; bool lead = true;
  for (uint32_t i = t; i < t + l; i++) { const uint32_t c = d.s[i]; if (c - '0' < 10u) { if (c != '0') lead = false; if (!lead) sig++; } }
  if (sig > 6u) { W.decline(AIGW_R_NUMBER); return; }
  W.o.span(d, t, t + l);
}

// rm_contains: the override when one is configured, else the request's model, contains `needle`
__device__ __forceinline__ bool gem_model_contains(const ChatLargeParams& P, const ClShared& S, const RecWalk& W, const RecWalk::Top& t, const char* needle) {
  if (!P.override_len) return W.model_contains(t.model, needle);
  const uint8_t* p = S.lits + S.lit_off[CL_OVERRIDE];
  const uint32_t L = P.override_len, n = clen(needle);
  for (uint32_t i = 0; i + n <= L; i++) { uint32_t k = 0; while (k < n && p[i + k] == (uint8_t)needle[k]) k++; if (k == n) return true; }
  return false;
}

// str_eq_lit of the translate pass: a string value that is `w`, unescaped
__device__ __forceinline__ bool gem_is(const RecWalk& W, uint32_t v, const char* w) { return !W.d.str_has_backslash(v) && W.d.raw_is(v, w, clen(w)); }

// gem_schema_ok: "parameters" in the subset whose conversion is a sorted re-marshal ({type, description: string; properties:
// {name: schema}; items: schema; required, enum: [string]}).  The translate pass's 24-entry stack (here W.stk, which cl_any fills
// only afterwards) and its 512 member visits per declaration, so that the answers agree below 64 KiB.
__device__ __forceinline__ bool gem_schema_ok(RecWalk& W, uint32_t root) {
  const LDoc& d = W.d;
  uint32_t* stack = W.stk;
  int sp = 0, guard = 0;
  stack[sp++] = root;
  while (sp) {
    const uint32_t o = stack[--sp];
    if (!W.is_obj(o)) return false;
    for (uint32_t m = o + 1; d.ty(m) != '}'; m = d.after(m + 3)) {
      if (++guard > 512 || d.str_has_backslash(m)) return false;
      const uint32_t v = m + 3;
      if (W.key(m, "type") || W.key(m, "description")) { if (!W.is_str(v)) return false; }
      else if (W.key(m, "properties")) {
        if (!W.is_obj(v)) return false;
        for (uint32_t q = v + 1; d.ty(q) != '}'; q = d.after(q + 3)) { if (sp >= 24) return false; stack[sp++] = q + 3; }
      } else if (W.key(m, "items")) { if (sp >= 24) return false; stack[sp++] = v; }
      else if (W.key(m, "required") || W.key(m, "enum")) {
        if (!W.is_arr(v)) return false;
        for (uint32_t q = v + 1; d.ty(q) != ']'; q = d.after(q)) if (!W.is_str(q)) return false;
      } else return false;
    }
  }
  return true;
}

// one {"text":S} part; `first`: no separator yet
__device__ __forceinline__ void gem_text(RecWalk& W, uint32_t v, bool& first) {
  if (!first) W.lit(L_COMMA);
  first = false;
  W.lit(L_TEXT_OPEN); W.str(v); W.lit(L_RBRACE);
}

// a system or developer message's non-empty texts.  kE = false: the check, in the message pass (a missing content is a pending
// 422; the dry plan has declined a null one and parts that are not text objects); kE = true: the record, in the second pass after
// generation_config.  Returns whether the message yields a part.
template <bool kE>
__device__ __forceinline__ bool gem_system(RecWalk& W, const RecWalk::Msg& g, bool& first) {
  const LDoc& d = W.d;
  const uint32_t c = g.content;
  if (c == kNone || W.is_null(c)) { if constexpr (!kE) W.pend(AIGW_R_E422_CONTENT); return false; }
  if (W.is_str(c)) {
    if (d.str_len(c) == 0) return false;
    if constexpr (kE) gem_text(W, c, first);
    return true;
  }
  bool any = false;
  for (uint32_t q = c + 1; d.ty(q) != ']'; q = d.after(q)) {
    RecWalk::Part p; if (!W.scan_part(q, p)) return false;
    if (p.text != kNone && d.str_len(p.text) > 0) { any = true; if constexpr (kE) gem_text(W, p.text, first); }
  }
  return any;
}

// plan_gemini after ParseBody's top-level checks
struct GemPlan : ClChatTop {
  static __device__ __forceinline__ void plan(const ChatLargeParams& P, ClShared& S, RecWalk& W, const RecWalk::Top& t, bool stream) {
    const LDoc& d = W.d;
    if (W.bad()) return;
    {
      ClWalkT<ClNoOut> D;
      D.d = d; D.A = W.A; D.stk = W.stk;
      D.check(t);
      if (D.reason) { W.decline(D.reason); return; }
    }
    if (t.tool_choice != kNone || t.thinking != kNone) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
    const GemTop g = gem_top(W);
    if (g.reasoning_effort != kNone && d.str_len(g.reasoning_effort) > 0) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
    // ":path": publishers/google/models/{model}:generateContent | :streamGenerateContent?alt=sse, the model raw
    W.lit(L_EM_GOOGLE_PATH); rec_path_model<false>(P, S, W, t); W.lit(stream ? L_GEM_STREAM : L_GEM_GENERATE);
    if (W.o.olen > 0xffffu) W.decline(AIGW_R_TOO_LARGE);   // path_len is 16 bits
    S.path_len = (uint32_t)W.o.olen;
    if (W.bad()) return;
    // "contents": a run of user messages is one user content (a system message does not end it), an assistant message one model
    // content
    W.lit(L_GEM_CONTENTS);
    bool any_content = false, user_open = false, ufirst = true, any_sys = false;
    auto content_sep = [&] { if (!any_content) { W.lit(L_LBRACK); any_content = true; } else W.lit(L_COMMA); };
    auto open_user = [&] { if (!user_open) { content_sep(); W.lit(L_GEM_PARTS_OPEN); user_open = true; } };
    if (t.messages != kNone) {
      for (uint32_t e = t.messages + 1; d.ty(e) != ']'; e = d.after(e)) {
        RecWalk::Msg m; const int role = W.scan_message(e, m);
        if (W.bad()) return;
        const uint32_t c = m.content;
        if (role == 2 || role == 3) { bool f = true; if (gem_system<false>(W, m, f)) any_sys = true; }
        else if (role == 0) {
          if (c == kNone || W.is_null(c)) { W.pend(AIGW_R_E422_CONTENT); continue; }
          if (W.is_str(c)) { if (d.str_len(c) > 0) { open_user(); gem_text(W, c, ufirst); } }
          else {
            for (uint32_t q = c + 1; d.ty(q) != ']'; q = d.after(q)) {
              RecWalk::Part p; if (!W.scan_part(q, p)) return;
              if (p.text == kNone || d.str_len(p.text) == 0) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }   // a Part{} layout
              open_user(); gem_text(W, p.text, ufirst);
            }
          }
        } else if (role == 4) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }   // a FunctionResponse part
        else {
          if (user_open) { W.lit(L_USER_CLOSE); user_open = false; ufirst = true; }
          if (m.tool_calls != kNone && !W.is_null(m.tool_calls) && d.ty(m.tool_calls + 1) != ']') { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }   // FunctionCall
          bool has_parts = false;
          if (c != kNone && !W.is_null(c)) {
            if (W.is_str(c)) has_parts = d.str_len(c) > 0;
            else if (W.is_arr(c)) {
              for (uint32_t q = c + 1; d.ty(q) != ']'; q = d.after(q)) {
                RecWalk::Part p; if (!W.scan_part(q, p)) return;
                if (p.type == kNone) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
                if (W.val(p.type, "text")) { if (p.text != kNone && d.str_len(p.text) > 0) has_parts = true; }
                else if (!W.val(p.type, "refusal")) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }   // thought parts, unknown types
              }
            } else { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }   // a single part object
          }
          content_sep();
          if (!has_parts) W.lit(L_GEM_MODEL_EMPTY);
          else {
            W.lit(L_GEM_PARTS_OPEN);
            bool first = true;
            if (W.is_str(c)) gem_text(W, c, first);
            else for (uint32_t q = c + 1; d.ty(q) != ']'; q = d.after(q)) {
              RecWalk::Part p; W.scan_part(q, p);
              if (gem_is(W, p.type, "text") && p.text != kNone && d.str_len(p.text) > 0) gem_text(W, p.text, first);
            }
            W.lit(L_GEM_MODEL_CLOSE);
          }
        }
        if (W.bad()) return;
      }
    }
    if (user_open) W.lit(L_USER_CLOSE);
    W.lit(any_content ? L_RBRACK : L_NULL);
    // "tools": one declaration per function tool
    W.lit(L_GEM_TOOLS);
    bool any_decl = false;
    if (t.tools != kNone) {
      const bool json_schema = gem_model_contains(P, S, W, t, "gemini") && (gem_model_contains(P, S, W, t, "2.5") || gem_model_contains(P, S, W, t, "3"));
      for (uint32_t e = t.tools + 1; d.ty(e) != ']'; e = d.after(e)) {
        const uint32_t ty = W.find(e, "type"), fn = W.find(e, "function");
        if (W.bad()) return;
        if (ty == kNone || !gem_is(W, ty, "function")) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
        if (fn == kNone) continue;
        const uint32_t nm = W.find(fn, "name"), ds = W.find(fn, "description"), pr = W.find(fn, "parameters");
        if (W.bad()) return;
        W.lit(any_decl ? L_COMMA : L_GEM_DECLS_OPEN);
        any_decl = true;
        W.lit(L_LBRACE);
        bool f = true;
        if (ds != kNone && d.str_len(ds) > 0) { W.lit(L_DESC); W.str(ds); f = false; }
        if (nm != kNone && d.str_len(nm) > 0) { if (!f) W.lit(L_COMMA); W.lit(L_GEM_NAME); W.str(nm); f = false; }
        if (pr != kNone) {
          const bool empty_obj = W.is_obj(pr) && d.ty(pr + 1) == '}';
          bool emit = false;
          if (json_schema) emit = !empty_obj;
          else if (!W.is_obj(pr)) W.pend(AIGW_R_E422_CONTENT);
          else if (!empty_obj) {
            if (!gem_schema_ok(W, pr)) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; }
            emit = true;
          }
          if (emit) {
            if (!f) W.lit(L_COMMA);
            W.lit(json_schema ? L_GEM_PARAMS_JS : L_GEM_PARAMS);
            if (const int r = cl_any(d, W.stk, pr, W.any_work, W.o)) { W.decline(r); return; }
          }
        }
        W.lit(L_RBRACE);
      }
    }
    W.lit(any_decl ? L_GEM_DECLS_CLOSE : L_NULL);
    // "generation_config", genai.GenerationConfig's field order
    W.lit(L_GEM_GENCFG);
    bool gf = true, zero = false;
    auto sep = [&] { if (!gf) W.lit(L_COMMA); gf = false; };
    if (g.n != kNone) {
      const uint32_t l = gem_i32(W, g.n, zero); if (!l) return;
      if (!zero) { sep(); W.lit(L_GEM_CANDIDATES); W.o.span(d, d.tok(g.n), d.tok(g.n) + l); }
    }
    if (g.freq_pen != kNone) { sep(); W.lit(L_GEM_FREQ); gem_f32(W, g.freq_pen); }
    if (g.top_logprobs != kNone) {
      const uint32_t l = gem_i32(W, g.top_logprobs, zero); if (!l) return;
      sep(); W.lit(L_GEM_LOGPROBS); W.o.span(d, d.tok(g.top_logprobs), d.tok(g.top_logprobs) + l);   // an explicit 0 is its own spelling
    }
    {
      const uint32_t mt = t.mct != kNone ? t.mct : t.max_tokens;
      if (mt != kNone) {
        const uint32_t l = gem_i32(W, mt, zero); if (!l) return;
        if (!zero) { sep(); W.lit(L_GEM_MAXOUT); W.o.span(d, d.tok(mt), d.tok(mt) + l); }
      }
    }
    if (g.pres_pen != kNone) { sep(); W.lit(L_GEM_PRES); gem_f32(W, g.pres_pen); }
    if (g.logprobs != kNone && d.ty(g.logprobs) == 't') { sep(); W.lit(L_GEM_RESP_LOGPROBS); }
    if (g.seed != kNone) {
      const uint32_t l = gem_i32(W, g.seed, zero); if (!l) return;
      sep(); W.lit(L_GEM_SEED); W.o.span(d, d.tok(g.seed), d.tok(g.seed) + l);
    }
    if (t.stop != kNone) {   // the dry plan has declined anything but a string or an array of strings
      const uint32_t s = t.stop;
      if (W.is_str(s)) { sep(); W.lit(L_STOPSEQ); W.str(s); W.lit(L_RBRACK); }
      else if (d.ty(s + 1) != ']') {
        sep(); W.lit(L_STOPSEQ);
        for (uint32_t e = s + 1; d.ty(e) != ']'; e = d.after(e)) { if (e != s + 1) W.lit(L_COMMA); W.str(e); }
        W.lit(L_RBRACK);
      }
    }
    if (t.temperature != kNone) { sep(); W.lit(L_TEMP); gem_f32(W, t.temperature); }
    if (t.top_p != kNone) { sep(); W.lit(L_TOPP); gem_f32(W, t.top_p); }
    W.lit(L_RBRACE);
    if (W.bad()) return;
    // "system_instruction" last: a second pass over the messages records what the first one checked
    if (any_sys) {
      W.lit(L_GEM_SYS_OPEN);
      bool first = true;
      for (uint32_t e = t.messages + 1; d.ty(e) != ']'; e = d.after(e)) {
        RecWalk::Msg m; const int role = W.scan_message(e, m);
        if (role == 2 || role == 3) gem_system<true>(W, m, first);
      }
      W.lit(L_GEM_SYS_CLOSE);
    }
    W.lit(L_RBRACE);
  }
};

__global__ void __launch_bounds__(kClThreads, 2) chat_gemini_large_kernel(const __grid_constant__ ChatLargeParams P) {
  __shared__ ClShared S;
  cl_request_loop<ClRecordRequest<GemPlan>>(P, S);
}

}  // namespace

cudaError_t launch_chat_gemini_large(const ChatLargeParams& P, int grid, cudaStream_t st) {
  chat_gemini_large_kernel<<<P.n < (uint32_t)grid ? (P.n ? P.n : 1u) : (uint32_t)grid, kClThreads, 0, st>>>(P);
  return cudaGetLastError();
}

}  // namespace aigw
