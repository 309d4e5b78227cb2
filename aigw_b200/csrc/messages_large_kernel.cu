// /v1/messages requests above the translate pass's 64 KiB ceiling (and below it) to the backends that need a full re-map of the
// request: an OpenAI chat-completions request (AIGW_SCHEMA_MSG_OPENAI) or a Bedrock Converse request (AIGW_SCHEMA_MSG_AWS_BEDROCK),
// with the semantics group 9 of the translate pass gives them (plan_messages_full in chat_walk_impl.cuh).  sm_90a only.
//
// messages_large_kernel: one CTA of 256 threads per request, the scan and depth pass of large_request.cuh, then the record phase
// of chat_large_record_impl.cuh with this planner (thread 0), in plan_messages_full's order:
//   scan      mx_scan: the top-level members of anthropic.MessagesRequest with every block, tool and tool_choice checked, problems
//             in member order (the record phase reads the model and stream tokens it keeps)
//   checks    the model (a missing or empty one is the 422), the override's bytes
//   record    ":path", then the OpenAI body (mx_openai) or the Converse body (mx_bedrock).  A tool_use block's "input" becomes
//             the OpenAI "arguments" string: cl_any re-serialises it into a sink that escapes '"' and '\' by splitting each body
//             span before them and putting a one-byte backslash from scratch in front, so the escaped text costs copy ops, not
//             scratch.  The Converse body takes the input as JSON, straight from cl_any.
// A restatement of the translate pass, not a reuse: keys and enumerated values are compared by their bytes (an escaped value
// declines AIGW_R_ESCAPE, the depth pass has declined escaped keys), and the walk accepts whitespace between tokens, as group 9
// does, since it rebuilds the body.  A change to plan_messages_full has to be made here too; test_messages_large_gpu.py compares
// the two on the translate pass's corpus.
#include "messages_large_kernel.cuh"

#include "chat_large_record_impl.cuh"

namespace aigw {
namespace {

// the top-level members of anthropic.MessagesRequest the subset takes, in the translate pass's id order (MK_model .. MK_tool_choice)
__device__ const char* const kMxTopKeys[] = {"model", "max_tokens", "messages", "stream", "system", "temperature", "top_p", "top_k",
                                             "stop_sequences", "metadata", "tools", "tool_choice"};
enum MxTopId : int { MX_model, MX_max_tokens, MX_messages, MX_stream, MX_system, MX_temperature, MX_top_p, MX_top_k, MX_stop_sequences,
                     MX_metadata, MX_tools, MX_tool_choice, MX_COUNT };

// the members mx_scan keeps (value tokens, kNone when absent or null; system: the value token, null included)
struct MxTop { uint32_t model, max_tokens, temperature, top_p, top_k, stream, stop, system, messages, tools, tool_choice; };

__device__ __forceinline__ int mx_top_id(const RecWalk& W, uint32_t m) {
  const uint32_t n = W.d.str_len(m);
  if (n < 4 || n > 14) return -1;
  for (int k = 0; k < MX_COUNT; k++) if (W.key(m, kMxTopKeys[k])) return k;
  return -1;
}

// exactly {"type":"ephemeral"}
__device__ __forceinline__ bool mx_cache_ok(RecWalk& W, uint32_t v) {
  const LDoc& d = W.d;
  if (!W.is_obj(v)) return false;
  const uint32_t k = v + 1;
  return d.ty(k) != '}' && W.key(k, "type") && W.is_str(k + 3) && W.val(k + 3, "ephemeral") && d.ty(d.after(k + 3)) == '}';
}

// msg_text_block: {"type":"text","text":S[,"cache_control":{"type":"ephemeral"}]} in any order, nothing else
__device__ __forceinline__ bool msg_text_block(RecWalk& W, uint32_t b) {
  const LDoc& d = W.d;
  if (!W.is_obj(b)) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
  uint32_t seen = 0;
  for (uint32_t m = b + 1; d.ty(m) != '}'; m = d.after(m + 3)) {
    const uint32_t v = m + 3;
    uint32_t bit = 0; bool ok;
    if (W.key(m, "type")) { bit = 1; ok = !(seen & 1u) && W.is_str(v) && W.val(v, "text"); }
    else if (W.key(m, "text")) { bit = 2; ok = !(seen & 2u) && W.is_str(v); }
    else if (W.key(m, "cache_control")) ok = mx_cache_ok(W, v);
    else ok = false;
    if (!ok) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
    seen |= bit;
  }
  if ((seen & 3u) != 3u) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
  return true;
}

// mx_block: one content block of a message: 0 text, 1 tool_use, 2 tool_result, -1 declined
__device__ __forceinline__ int mx_block(RecWalk& W, uint32_t b) {
  const LDoc& d = W.d;
  if (!W.is_obj(b)) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return -1; }
  uint32_t ty = kNone;
  for (uint32_t m = b + 1; d.ty(m) != '}'; m = d.after(m + 3)) if (W.key(m, "type")) { if (ty != kNone) { W.decline(AIGW_R_DUP_KEY); return -1; } ty = m + 3; }
  if (ty == kNone || !W.is_str(ty)) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return -1; }
  if (W.val(ty, "text")) return msg_text_block(W, b) ? 0 : -1;
  const bool use = W.val(ty, "tool_use");
  if (!use && !W.val(ty, "tool_result")) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return -1; }
  // members by a bit each (the translate pass's ids); any other key declines, a repeated one too
  uint32_t seen = 0;
  for (uint32_t m = b + 1; d.ty(m) != '}'; m = d.after(m + 3)) {
    const uint32_t v = m + 3;
    const int id = W.key(m, "type") ? 0 : W.key(m, "cache_control") ? 1 : W.key(m, "id") ? 2 : W.key(m, "name") ? 3 : W.key(m, "input") ? 4
                 : W.key(m, "tool_use_id") ? 5 : W.key(m, "is_error") ? 6 : W.key(m, "content") ? 7 : -1;
    if (id < 0 || (seen & (1u << id))) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return -1; }
    seen |= 1u << id;
    bool ok = true;
    if (id == 0) continue;
    if (id == 1) ok = mx_cache_ok(W, v);
    else if (use) {
      if (id == 2 || id == 3) ok = W.is_str(v);
      else if (id == 4) ok = W.is_null(v) || W.is_obj(v);
      else ok = false;
    } else {
      if (id == 5) ok = W.is_str(v);
      else if (id == 6) ok = W.is_bool(v);
      else if (id == 7) {
        if (W.is_arr(v)) { for (uint32_t q = v + 1; d.ty(q) != ']'; q = d.after(q)) if (!msg_text_block(W, q)) return -1; }
        else ok = W.is_null(v) || W.is_str(v);
      } else ok = false;
    }
    if (!ok) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return -1; }
  }
  const uint32_t need = use ? (1u << 2) | (1u << 3) : (1u << 5);
  if ((seen & need) != need) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return -1; }
  return use ? 1 : 2;
}

// mx_plain_int: a non-negative integer literal of at most 15 digits, optionally followed by ".0…0" (a float64 field, int64()
// conversion): its digit count, or 0
__device__ __forceinline__ uint32_t mx_plain_int(const RecWalk& W, uint32_t v) {
  const LDoc& d = W.d;
  const uint32_t o = d.tok(v), e = d.scalar_end(v);
  uint32_t i = o; while (i < e && d.s[i] - '0' < 10u) i++;
  const uint32_t nd = i - o;
  if (nd == 0 || nd > 15 || (nd > 1 && d.s[o] == '0')) return 0;
  if (i < e) { if (d.s[i] != '.' || i + 1 == e) return 0; for (uint32_t k = i + 1; k < e; k++) if (d.s[k] != '0') return 0; }
  return nd;
}

// the members of an input_schema: type, properties and required checked, every other member dropped; a key twice declines.  The
// repeat check compares each member's key with the ones before it, so its key bytes count against kChatAnyWork
// (AIGW_R_SCRATCH above) as cl_any's key-order check does.
__device__ __forceinline__ bool mx_input_schema_ok(RecWalk& W, uint32_t tv) {
  const LDoc& d = W.d;
  for (uint32_t s = tv + 1; d.ty(s) != '}'; s = d.after(s + 3)) {
    if (d.str_has_backslash(s)) return false;
    for (uint32_t s2 = tv + 1; s2 != s; s2 = d.after(s2 + 3)) {
      if (++W.any_work > kChatAnyWork) { W.decline(AIGW_R_SCRATCH); return false; }
      if (cmp_keys(d, s, s2, W.any_work) == 0) return false;
    }
    const uint32_t sv = s + 3;
    if (W.key(s, "type")) { if (!W.is_str(sv)) return false; }
    else if (W.key(s, "properties")) { if (!(W.is_null(sv) || W.is_obj(sv))) return false; }
    else if (W.key(s, "required")) {
      if (!(W.is_null(sv) || W.is_arr(sv))) return false;
      if (W.is_arr(sv)) for (uint32_t e = sv + 1; d.ty(e) != ']'; e = d.after(e)) if (!W.is_str(e)) return false;
    }
  }
  return true;
}

// mx_scan: the top-level members in order, each checked as the decoder meets it
__device__ __forceinline__ bool mx_scan(RecWalk& W, MxTop& t) {
  const LDoc& d = W.d;
  t.model = t.max_tokens = t.temperature = t.top_p = t.top_k = t.stream = t.stop = t.system = t.messages = t.tools = t.tool_choice = kNone;
  if (W.is_null(0)) return true;
  if (!W.is_obj(0)) { W.decline(AIGW_R_E400_TYPE); return false; }
  uint32_t seen = 0;
  for (uint32_t m = 1; d.ty(m) != '}'; m = d.after(m + 3)) {
    const int id = mx_top_id(W, m);
    if (id < 0) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
    if (seen & (1u << id)) { W.decline(AIGW_R_DUP_KEY); return false; }
    seen |= 1u << id;
    const uint32_t v = m + 3; const bool nul = W.is_null(v);
    switch (id) {
      case MX_model: if (!nul) { if (!W.is_str(v)) { W.decline(AIGW_R_E400_TYPE); return false; } t.model = v; } break;
      case MX_max_tokens:
        if (!nul) {
          if (!W.is_num(v)) { W.decline(AIGW_R_E400_TYPE); return false; }
          if (!mx_plain_int(W, v)) { W.decline(AIGW_R_NUMBER); return false; }
          t.max_tokens = v;
        }
        break;
      case MX_temperature: if (!nul) { if (!W.is_num(v)) { W.decline(AIGW_R_E400_TYPE); return false; } t.temperature = v; } break;
      case MX_top_p: if (!nul) { if (!W.is_num(v)) { W.decline(AIGW_R_E400_TYPE); return false; } t.top_p = v; } break;
      case MX_top_k:
        if (!nul) {
          if (!W.is_num(v)) { W.decline(AIGW_R_E400_TYPE); return false; }
          const uint32_t o = d.tok(v), e = d.scalar_end(v);
          if (e - o > 9u) { W.decline(AIGW_R_NUMBER); return false; }
          for (uint32_t i = o; i < e; i++) if (d.s[i] - '0' >= 10u) { W.decline(AIGW_R_NUMBER); return false; }
          t.top_k = v;
        }
        break;
      case MX_stream: if (!nul) { if (!W.is_bool(v)) { W.decline(AIGW_R_E400_TYPE); return false; } t.stream = v; } break;
      case MX_stop_sequences:
        if (!nul) {
          if (!W.is_arr(v)) { W.decline(AIGW_R_E400_TYPE); return false; }
          for (uint32_t q = v + 1; d.ty(q) != ']'; q = d.after(q)) if (!W.is_str(q)) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
          t.stop = v;
        }
        break;
      case MX_metadata:
        if (!nul) {
          if (!W.is_obj(v)) { W.decline(AIGW_R_E400_TYPE); return false; }
          const uint32_t k = v + 1;
          if (d.ty(k) != '}') {
            if (d.ty(d.after(k + 3)) != '}') { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
            if (!W.key(k, "user_id") || !(W.is_str(k + 3) || W.is_null(k + 3))) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
          }
        }
        break;
      case MX_system:
        t.system = v;
        if (W.is_str(v)) break;
        if (!W.is_arr(v)) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
        for (uint32_t q = v + 1; d.ty(q) != ']'; q = d.after(q)) if (!msg_text_block(W, q)) return false;
        break;
      case MX_messages:
        if (nul) break;
        if (!W.is_arr(v)) { W.decline(AIGW_R_E400_TYPE); return false; }
        t.messages = v;
        for (uint32_t q = v + 1; d.ty(q) != ']'; q = d.after(q)) {
          if (!W.is_obj(q)) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
          uint32_t ms = 0;
          for (uint32_t k = q + 1; d.ty(k) != '}'; k = d.after(k + 3)) {
            const uint32_t cv = k + 3;
            if (W.key(k, "role")) { if ((ms & 1u) || !W.is_str(cv)) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; } ms |= 1u; }
            else if (W.key(k, "content")) {
              if (ms & 2u) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
              ms |= 2u;
              if (W.is_str(cv)) continue;
              if (!W.is_arr(cv)) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
              for (uint32_t b = cv + 1; d.ty(b) != ']'; b = d.after(b)) if (mx_block(W, b) < 0) return false;
            } else { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
          }
          if (ms != 3u) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
        }
        break;
      case MX_tools:
        if (nul) break;
        if (!W.is_arr(v)) { W.decline(AIGW_R_E400_TYPE); return false; }
        t.tools = v;
        for (uint32_t q = v + 1; d.ty(q) != ']'; q = d.after(q)) {
          if (!W.is_obj(q)) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
          uint32_t ts = 0;
          for (uint32_t k = q + 1; d.ty(k) != '}'; k = d.after(k + 3)) {
            const uint32_t tv = k + 3;
            const int kid = W.key(k, "type") ? 0 : W.key(k, "name") ? 1 : W.key(k, "description") ? 2 : W.key(k, "cache_control") ? 3
                          : W.key(k, "input_schema") ? 4 : -1;
            if (kid < 0 || (ts & (1u << kid))) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
            ts |= 1u << kid;
            bool ok;
            if (kid == 0) ok = W.is_str(tv) && (d.str_len(tv) == 0 || W.val(tv, "custom"));
            else if (kid == 1 || kid == 2) ok = W.is_str(tv);
            else if (kid == 3) ok = mx_cache_ok(W, tv);
            else ok = W.is_obj(tv) && mx_input_schema_ok(W, tv);
            if (!ok) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
          }
          if ((ts & 0x12u) != 0x12u) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }   // name and input_schema
        }
        break;
      case MX_tool_choice: {
        if (nul) break;
        if (!W.is_obj(v)) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
        uint32_t ty = kNone, nm = kNone, cs = 0;
        for (uint32_t k = v + 1; d.ty(k) != '}'; k = d.after(k + 3)) {
          const int kid = W.key(k, "type") ? 0 : W.key(k, "name") ? 1 : W.key(k, "disable_parallel_tool_use") ? 2 : -1;
          if (kid < 0 || (cs & (1u << kid))) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
          cs |= 1u << kid;
          if (kid == 0) ty = k + 3;
          else if (kid == 1) nm = k + 3;
          else if (!(W.is_bool(k + 3) || W.is_null(k + 3))) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
        }
        if (ty == kNone || !W.is_str(ty)) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
        const bool tool = W.val(ty, "tool");
        const bool known = tool || W.val(ty, "auto") || W.val(ty, "any") || W.val(ty, "none");
        if (!known || (tool ? (nm == kNone || !W.is_str(nm)) : nm != kNone)) { W.decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
        t.tool_choice = v;
        break;
      }
    }
  }
  return true;
}

// the literal `id` without its first `skip` bytes
__device__ __forceinline__ void mx_lit_tail(RecWalk& W, uint32_t id, uint32_t skip) {
  const uint32_t o = g_rec_lits.off[id], l = g_rec_lits.off[id + 1] - o;
  W.o.push(REC_LIT, o + skip, l - skip);
}

// configuration text (the OpenAI path, the override: checked to need no JSON escaping) into scratch, as one op
__device__ __forceinline__ void mx_cfg(RecWalk& W, const ClShared& S, uint32_t id, uint32_t n) {
  if (!n || !W.o.room(n)) return;
  const uint8_t* p = S.lits + S.lit_off[id];
  const uint32_t at = W.o.rs_n;
  for (uint32_t i = 0; i < n; i++) W.o.scr[at + i] = p[i];
  W.o.rs_n = at + n;
  W.o.push(REC_SCR, at, n);
}

// emit_escaped_json's sink: cl_any's output (body spans and the literals ',' and ':') inside a JSON string.  Every '"' and '\' of a
// span gets a backslash in front: the span is split before it and a one-byte scratch op holding a backslash goes between, about
// two ops per escaped byte.
struct MxEscOut {
  ClOut& o;
  uint32_t bs;   // the scratch offset of the backslash
  __device__ void lit(uint32_t id) { o.lit(id); }
  __device__ void span(const LDoc& d, uint32_t b, uint32_t e) {
    uint32_t seg = b;
    for (uint32_t i = b; i < e; i++) {
      const uint32_t c = d.s[i];
      if (c == '"' || c == '\\') { o.push(REC_BODY, seg, i - seg); o.push(REC_SCR, bs, 1); seg = i; }
    }
    o.push(REC_BODY, seg, e - seg);
  }
};

// json.Marshal of a tool_use "input" object embedded in a JSON string
__device__ __forceinline__ void mx_escaped_json(RecWalk& W, uint32_t v, uint32_t& bs) {
  if (bs == kNone) {
    if (!W.o.room(1)) return;
    bs = W.o.rs_n++;
    W.o.scr[bs] = '\\';
  }
  MxEscOut e{W.o, bs};
  if (const int r = cl_any(W.d, W.stk, v, W.any_work, e)) W.decline(r);
}

// the value of member `k` by the translate pass's find (kNone when absent or null); the scan has declined repeats wherever the
// record looks a member up
__device__ __forceinline__ bool mx_is(RecWalk& W, uint32_t obj, const char* k, const char* w) {
  const uint32_t v = W.find(obj, k);
  return v != kNone && W.is_str(v) && W.val(v, w);
}

// anthropicContentToText of an array content: its text blocks' concatenation is non-empty / its inner bytes
__device__ __forceinline__ bool mx_array_text_nonempty(RecWalk& W, uint32_t arr) {
  const LDoc& d = W.d;
  for (uint32_t b = arr + 1; d.ty(b) != ']'; b = d.after(b))
    if (mx_is(W, b, "type", "text")) { const uint32_t tx = W.find(b, "text"); if (tx != kNone && d.str_len(tx)) return true; }
  return false;
}
__device__ __forceinline__ void mx_array_text_inner(RecWalk& W, uint32_t arr) {
  const LDoc& d = W.d;
  for (uint32_t b = arr + 1; d.ty(b) != ']'; b = d.after(b))
    if (mx_is(W, b, "type", "text")) { const uint32_t tx = W.find(b, "text"); if (tx != kNone) W.o.str_inner(d, tx); }
}
// the text items of a tool_result's array content, inner bytes (toolResultToText)
__device__ __forceinline__ void mx_array_text_inner_items(RecWalk& W, uint32_t arr) {
  const LDoc& d = W.d;
  for (uint32_t q = arr + 1; d.ty(q) != ']'; q = d.after(q)) { const uint32_t tx = W.find(q, "text"); if (tx != kNone) W.o.str_inner(d, tx); }
}
// 0 text, 1 tool_use, 2 tool_result, -1 other
__device__ __forceinline__ int mx_block_kind(RecWalk& W, uint32_t b) {
  const uint32_t ty = W.find(b, "type");
  if (ty == kNone || !W.is_str(ty)) return -1;
  return W.val(ty, "text") ? 0 : W.val(ty, "tool_use") ? 1 : W.val(ty, "tool_result") ? 2 : -1;
}

// ToolInputSchema marshalled: {"type":T[,"properties":{…}][,"required":[…]]}
__device__ __forceinline__ void mx_schema(RecWalk& W, uint32_t sch) {
  const LDoc& d = W.d;
  const uint32_t ty = W.find(sch, "type"), pr = W.find(sch, "properties"), rq = W.find(sch, "required");
  W.lit(L_MX_SCHEMA_TYPE);
  if (ty != kNone) W.str(ty); else W.lit(L_EMPTY_STR);
  if (pr != kNone && d.ty(pr + 1) != '}') {
    W.lit(L_MX_PROPS);
    if (const int r = cl_any(d, W.stk, pr, W.any_work, W.o)) { W.decline(r); return; }
  }
  if (rq != kNone && d.ty(rq + 1) != ']') {
    W.lit(L_MX_REQUIRED);
    for (uint32_t e = rq + 1; d.ty(e) != ']'; e = d.after(e)) { if (e != rq + 1) W.lit(L_COMMA); W.str(e); }
    W.lit(L_RBRACK);
  }
  W.lit(L_RBRACE);
}
__device__ __forceinline__ void mx_str_array(RecWalk& W, uint32_t arr) {
  for (uint32_t e = arr + 1; W.d.ty(e) != ']'; e = W.d.after(e)) { if (e != arr + 1) W.lit(L_COMMA); W.str(e); }
}
__device__ __forceinline__ void mx_max_tokens(RecWalk& W, const MxTop& t) {
  if (t.max_tokens != kNone) { const uint32_t o = W.d.tok(t.max_tokens); W.o.span(W.d, o, o + mx_plain_int(W, t.max_tokens)); }
  else W.lit(L_ZERO);
}
// the role of a message (its value is a string: the scan checked it): 1 user, 2 assistant, 0 other
__device__ __forceinline__ int mx_role(RecWalk& W, uint32_t msg) {
  const uint32_t r = W.find(msg, "role");
  if (r == kNone) return 0;
  return W.val(r, "user") ? 1 : W.val(r, "assistant") ? 2 : 0;
}

// mx_openai: the chat-completions body, openai.ChatCompletionRequest's field order
__device__ __forceinline__ void mx_openai(const ChatLargeParams& P, const ClShared& S, RecWalk& W, const MxTop& t, bool stream) {
  const LDoc& d = W.d;
  // stop sequences: sjson marshals the []string with encoding/json; only spellings it shares with sonic are decided here
  if (t.stop != kNone) for (uint32_t e = t.stop + 1; d.ty(e) != ']'; e = d.after(e)) {
    if (d.str_nc(e)) { W.decline(AIGW_R_ESCAPE); return; }
    const uint32_t o = d.str_off(e), n = d.str_len(e);
    for (uint32_t i = 0; i < n; i++) { const uint32_t c = d.s[o + i]; if (c >= 0x7fu || c == '<' || c == '>' || c == '&') { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; } }
  }
  W.lit(L_MX_OPEN);
  bool any = false;
  auto sep = [&] { W.lit(any ? L_COMMA : L_LBRACK); any = true; };
  uint32_t bs = kNone;
  if (t.system != kNone) {
    const uint32_t sv = t.system;
    if (W.is_str(sv)) { if (d.str_len(sv)) { sep(); W.lit(L_MX_CONTENT_Q); W.o.str_inner(d, sv); W.lit(L_MX_SYS_CLOSE); } }
    else if (W.is_arr(sv)) {
      bool ne = false;
      for (uint32_t q = sv + 1; d.ty(q) != ']'; q = d.after(q)) { const uint32_t tx = W.find(q, "text"); if (tx != kNone && d.str_len(tx)) ne = true; }
      if (ne) {
        sep(); W.lit(L_MX_CONTENT_Q);
        for (uint32_t q = sv + 1; d.ty(q) != ']'; q = d.after(q)) { const uint32_t tx = W.find(q, "text"); if (tx != kNone) W.o.str_inner(d, tx); }
        W.lit(L_MX_SYS_CLOSE);
      }
    }
  }
  if (t.messages != kNone) for (uint32_t q = t.messages + 1; d.ty(q) != ']'; q = d.after(q)) {
    if (W.bad()) return;
    const int role = mx_role(W, q);
    const uint32_t c = W.find(q, "content");
    if (c == kNone) continue;
    if (role == 1) {
      if (W.is_arr(c)) for (uint32_t b = c + 1; d.ty(b) != ']'; b = d.after(b)) {
        if (mx_block_kind(W, b) != 2) continue;
        sep(); W.lit(L_MX_CONTENT_Q);
        const uint32_t rc = W.find(b, "content");
        if (rc != kNone) { if (W.is_str(rc)) W.o.str_inner(d, rc); else mx_array_text_inner_items(W, rc); }
        W.lit(L_MX_TOOL_MID); W.str(W.find(b, "tool_use_id")); W.lit(L_RBRACE);
      }
      if (W.is_str(c)) { if (d.str_len(c)) { sep(); W.lit(L_EM_CONTENT); W.str(c); mx_lit_tail(W, L_MX_USER_CLOSE_Q, 1); } }
      else if (mx_array_text_nonempty(W, c)) { sep(); W.lit(L_MX_CONTENT_Q); mx_array_text_inner(W, c); W.lit(L_MX_USER_CLOSE_Q); }
    } else if (role == 2) {
      sep(); W.lit(L_MX_ASST_OPEN);
      if (W.is_str(c)) { if (d.str_len(c)) W.str(c); else W.lit(L_NULL); }
      else if (mx_array_text_nonempty(W, c)) { W.lit(L_QUOTE); mx_array_text_inner(W, c); W.lit(L_QUOTE); }
      else W.lit(L_NULL);
      bool calls = false;
      if (W.is_arr(c)) for (uint32_t b = c + 1; d.ty(b) != ']'; b = d.after(b)) {
        if (mx_block_kind(W, b) != 1) continue;
        W.lit(L_COMMA); if (!calls) W.lit(L_R_TOOLCALLS);
        calls = true;
        W.lit(L_R_TC_ID); W.str(W.find(b, "id")); W.lit(L_R_TC_ARGS);
        const uint32_t in = W.find(b, "input");
        if (in != kNone) mx_escaped_json(W, in, bs); else W.lit(L_NULL);
        if (W.bad()) return;
        W.lit(L_R_TC_NAME); W.str(W.find(b, "name")); W.lit(L_R_TC_END);
      }
      if (calls) W.lit(L_RBRACK);
      W.lit(L_RBRACE);
    }
  }
  if (W.bad()) return;
  W.lit(any ? L_RBRACK : L_NULL);
  W.lit(L_R_MODEL_KEY);
  if (P.override_len) { W.lit(L_QUOTE); mx_cfg(W, S, CL_OVERRIDE, P.override_len); W.lit(L_QUOTE); } else W.str(t.model);
  W.lit(L_MX_MAXCT); mx_max_tokens(W, t);
  if (stream) { W.lit(L_AN_STREAM); W.lit(L_COMMA); W.lit(L_STREAMOPT_APPEND); }
  if (t.temperature != kNone) { W.lit(L_COMMA); W.lit(L_TEMP); W.num_field(t.temperature, false); }
  if (t.top_p != kNone) { W.lit(L_MX_TOPP); W.num_field(t.top_p, false); }
  if (t.tools != kNone && d.ty(t.tools + 1) != ']') {
    W.lit(L_MX_TOOLS);
    for (uint32_t q = t.tools + 1; d.ty(q) != ']'; q = d.after(q)) {
      if (W.bad()) return;
      if (q != t.tools + 1) W.lit(L_COMMA);
      W.lit(L_MX_TOOL_OPEN); W.str(W.find(q, "name"));
      const uint32_t ds = W.find(q, "description");
      if (ds != kNone && d.str_len(ds)) { W.lit(L_COMMA); W.lit(L_DESC); W.str(ds); }
      W.lit(L_COMMA); W.lit(L_GEM_PARAMS); mx_schema(W, W.find(q, "input_schema")); W.lit(L_R_RBRACE2);
    }
    W.lit(L_RBRACK);
    if (t.tool_choice != kNone) {
      const uint32_t ty = W.find(t.tool_choice, "type");
      if (W.val(ty, "auto")) W.lit(L_MX_TC_AUTO); else if (W.val(ty, "none")) W.lit(L_MX_TC_NONE); else if (W.val(ty, "any")) W.lit(L_MX_TC_REQUIRED);
      else { W.lit(L_MX_TC_NAMED); W.str(W.find(t.tool_choice, "name")); W.lit(L_R_RBRACE2); }
    }
  }
  if (t.stop != kNone && d.ty(t.stop + 1) != ']') { W.lit(L_MX_STOP); mx_str_array(W, t.stop); W.lit(L_RBRACK); }
  W.lit(L_RBRACE);
}

// convertToolResultBlock
__device__ __forceinline__ void mx_bedrock_tool_result(RecWalk& W, uint32_t b) {
  const LDoc& d = W.d;
  const uint32_t rc = W.find(b, "content"), ie = W.find(b, "is_error");
  if (rc != kNone && W.is_str(rc) && d.str_len(rc)) { W.lit(L_TOOLRESULT_OPEN); W.lit(L_TEXT_OPEN); W.str(rc); W.lit(L_RBRACE); W.lit(L_RBRACK); }
  else if (rc != kNone && W.is_arr(rc) && d.ty(rc + 1) != ']') {
    W.lit(L_TOOLRESULT_OPEN);
    for (uint32_t q = rc + 1; d.ty(q) != ']'; q = d.after(q)) { if (q != rc + 1) W.lit(L_COMMA); W.lit(L_TEXT_OPEN); W.str(W.find(q, "text")); W.lit(L_RBRACE); }
    W.lit(L_RBRACK);
  } else W.lit(L_MX_TR_NULL);
  if (ie != kNone && d.ty(ie) == 't') W.lit(L_MX_TR_STATUS_ERR); else mx_lit_tail(W, L_TOOLRESULT_MID, 1);
  W.str(W.find(b, "tool_use_id")); W.lit(L_TOOLRESULT_CLOSE);
}

// mx_bedrock: the Converse body
__device__ __forceinline__ void mx_bedrock(RecWalk& W, const MxTop& t) {
  const LDoc& d = W.d;
  W.lit(L_LBRACE);
  if (t.top_k != kNone) { W.lit(L_MX_TOPK); W.o.span(d, d.tok(t.top_k), d.scalar_end(t.top_k)); W.lit(L_RBRACE); W.lit(L_COMMA); }
  W.lit(L_INF_OPEN); W.lit(L_MAXTOK); mx_max_tokens(W, t);
  if (t.stop != kNone && d.ty(t.stop + 1) != ']') { W.lit(L_COMMA); W.lit(L_STOPSEQ); mx_str_array(W, t.stop); W.lit(L_RBRACK); }
  if (t.temperature != kNone) { W.lit(L_COMMA); W.lit(L_TEMP); W.num_field(t.temperature, false); }
  if (t.top_p != kNone) { W.lit(L_COMMA); W.lit(L_TOPP); W.num_field(t.top_p, false); }
  W.lit(L_INF_CLOSE_MSGS);
  bool first = true;
  if (t.messages != kNone) for (uint32_t q = t.messages + 1; d.ty(q) != ']'; q = d.after(q)) {
    if (W.bad()) return;
    const int role = mx_role(W, q);
    const uint32_t c = W.find(q, "content");
    if (role == 0) { W.pend(AIGW_R_E422_ROLE); return; }   // "unexpected role: …"
    const bool user = role == 1;
    if (!first) W.lit(L_COMMA);
    first = false;
    W.lit(L_MSG_CONTENT_OPEN);
    if (c != kNone && W.is_str(c)) { if (d.str_len(c)) { W.lit(L_TEXT_OPEN); W.str(c); W.lit(L_RBRACE); } }
    else if (c != kNone) {
      bool bf = true;
      for (uint32_t b = c + 1; d.ty(b) != ']'; b = d.after(b)) {
        const int k = mx_block_kind(W, b);
        if (!(k == 0 || (user && k == 2) || (!user && k == 1))) continue;
        if (!bf) W.lit(L_COMMA);
        bf = false;
        if (k == 0) { W.lit(L_TEXT_OPEN); W.str(W.find(b, "text")); W.lit(L_RBRACE); }
        else if (k == 2) mx_bedrock_tool_result(W, b);
        else {
          W.lit(L_TOOLUSE_OPEN); W.str(W.find(b, "name")); W.lit(L_TOOLUSE_INPUT);
          const uint32_t in = W.find(b, "input");
          if (in != kNone) { if (const int r = cl_any(d, W.stk, in, W.any_work, W.o)) { W.decline(r); return; } }
          else W.lit(L_NULL);
          W.lit(L_TOOLUSE_ID); W.str(W.find(b, "id")); W.lit(L_TOOLRESULT_CLOSE);
        }
      }
    }
    W.lit(user ? L_USER_CLOSE : L_ASST_CLOSE);
  }
  if (W.bad()) return;
  W.lit(L_RBRACK);
  if (t.system != kNone) {   // convertSystemPrompt; an empty slice is dropped by omitempty
    const uint32_t sv = t.system;
    if (W.is_str(sv)) { if (d.str_len(sv)) { W.lit(L_SYSTEM_OPEN); W.lit(L_TEXT_OPEN); W.str(sv); W.lit(L_RBRACE); W.lit(L_RBRACK); } }
    else if (W.is_arr(sv) && d.ty(sv + 1) != ']') {
      W.lit(L_SYSTEM_OPEN);
      for (uint32_t q = sv + 1; d.ty(q) != ']'; q = d.after(q)) { if (q != sv + 1) W.lit(L_COMMA); W.lit(L_TEXT_OPEN); W.str(W.find(q, "text")); W.lit(L_RBRACE); }
      W.lit(L_RBRACK);
    }
  }
  if (t.tools != kNone && d.ty(t.tools + 1) != ']') {   // convertTools
    W.lit(L_TOOLCFG_OPEN);
    if (t.tool_choice != kNone) {
      const uint32_t ty = W.find(t.tool_choice, "type");
      if (W.val(ty, "auto")) W.lit(L_TOOLCHOICE_AUTO); else if (W.val(ty, "any")) W.lit(L_TOOLCHOICE_ANY);
      else if (W.val(ty, "tool")) { W.lit(L_TOOLCHOICE_TOOL); W.str(W.find(t.tool_choice, "name")); W.lit(L_TOOLCHOICE_TOOL_END); }
    }
    W.lit(L_TOOLS_OPEN);
    for (uint32_t q = t.tools + 1; d.ty(q) != ']'; q = d.after(q)) {
      if (W.bad()) return;
      if (q != t.tools + 1) W.lit(L_COMMA);
      W.lit(L_TOOLSPEC_OPEN);
      const uint32_t ds = W.find(q, "description");
      if (ds != kNone && d.str_len(ds)) { W.lit(L_DESC); W.str(ds); W.lit(L_COMMA); }
      W.lit(L_INPUTSCHEMA); mx_schema(W, W.find(q, "input_schema")); W.lit(L_NAME); W.str(W.find(q, "name")); W.lit(L_R_RBRACE2);
    }
    W.lit(L_TOOLS_CLOSE);
  }
  W.lit(L_RBRACE);
}

// plan_messages_full: group 9's scan, the model and override checks, the ":path", then the body of the schema's target
struct MxPlan {
  using Top = MxTop;
  static __device__ __forceinline__ bool scan(RecWalk& W, Top& t) { return mx_scan(W, t) && !W.bad(); }
  static __device__ __forceinline__ void plan(const ChatLargeParams& P, ClShared& S, RecWalk& W, const Top& t, bool stream) {
    const LDoc& d = W.d;
    if (t.model == kNone || d.str_len(t.model) == 0) { W.decline(AIGW_R_E422_MODEL); return; }   // "model field is required"
    if (d.str_has_backslash(t.model)) { W.decline(AIGW_R_ESCAPE); return; }
    if (W.bad()) return;
    {
      const uint8_t* p = S.lits + S.lit_off[CL_OVERRIDE];
      for (uint32_t i = 0; i < P.override_len; i++) { const uint32_t c = p[i]; if (c < 0x20 || c > 0x7e || c == '"' || c == '\\') { W.decline(AIGW_R_UNSUPPORTED_FIELD); return; } }
    }
    if (!P.bedrock) {
      mx_cfg(W, S, CL_OPENAI_PATH, S.lit_len[CL_OPENAI_PATH]);   // path.Join("/", prefix, "chat/completions")
      S.path_len = (uint32_t)W.o.olen;
      mx_openai(P, S, W, t, stream);
    } else {
      W.lit(L_PATH_MODEL); rec_path_model<true>(P, S, W, t); W.lit(L_PATH_CONVERSE); if (stream) W.lit(L_PATH_STREAM);
      if (W.o.olen > 0xffffu) W.decline(AIGW_R_TOO_LARGE);   // path_len is 16 bits
      S.path_len = (uint32_t)W.o.olen;
      if (W.bad()) return;
      mx_bedrock(W, t);
    }
  }
};

__global__ void __launch_bounds__(kClThreads, 2) messages_large_kernel(const __grid_constant__ ChatLargeParams P) {
  __shared__ ClShared S;
  cl_request_loop<ClRecordRequest<MxPlan>>(P, S);
}

}  // namespace

cudaError_t launch_messages_large(const ChatLargeParams& P, int grid, cudaStream_t st) {
  messages_large_kernel<<<P.n < (uint32_t)grid ? (P.n ? P.n : 1u) : (uint32_t)grid, kClThreads, 0, st>>>(P);
  return cudaGetLastError();
}

}  // namespace aigw
