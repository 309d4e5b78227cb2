// T5, response direction for /v1/messages served by an OpenAI-schema backend (included by stream_kernel.cu inside its namespace):
//   AIGW_STREAM_MESSAGES_OPENAI           OpenAI chat-completion SSE chunks -> Anthropic SSE events, one ResponseBody call per step
//                                         (internal/translator/anthropic_openai.go:154-185; openAIStreamToAnthropicState,
//                                         internal/translator/openai_helper.go:436-766)
//   AIGW_STREAM_MESSAGES_OPENAI_BUFFERED  buffered ChatCompletionResponse -> anthropic.MessagesResponse
//                                         (anthropic_openai.go:112-152; openAIResponseToAnthropic, openai_helper.go:263-338)
// One thread per call, like the other kinds.  The typed walk decides what json.Unmarshal decides (a chunk that does not decode is
// skipped silently, a buffered body that does not decode is the reference's error); the members the translator reads are then
// found by a plain member navigation over the already-validated text.  Strings are copied only when the reference's encoder would
// re-emit their bytes unchanged (`canonical`); everything else DECLINES the stream, never approximates.
#pragma once

// ---- member navigation over a value the typed walk has accepted (well-formed; no escaped keys, no duplicate known keys)
__device__ __forceinline__ int jv_ws(const uint8_t* p, int i, int n) { while (i < n && ws(p[i])) i++; return i; }
// value start of member `key` of the object at p[o] == '{'; -1 when absent or null
__device__ int jv_member(const uint8_t* p, int n, int o, const char* key, int kl) {
  int i = jv_ws(p, o + 1, n);
  if (i >= n || p[i] != '"') return -1;
  for (;;) {
    bool e = false; const int j = scan_string(p, i, n, e); if (j < 0) return -1;
    const bool hit = (j - i - 2 == kl) && eq(p + i + 1, (uint32_t)kl, key, (uint32_t)kl);
    int v = jv_ws(p, j, n); if (v >= n || p[v] != ':') return -1;
    v = jv_ws(p, v + 1, n); if (v >= n) return -1;
    if (hit) return p[v] == 'n' ? -1 : v;
    const int end = skip_any(p, v, n); if (end < 0) return -1;
    i = jv_ws(p, end, n);
    if (i >= n || p[i] != ',') return -1;
    i = jv_ws(p, i + 1, n);
    if (i >= n || p[i] != '"') return -1;
  }
}
#define JV(p, n, o, key) jv_member(p, n, o, key, (int)sizeof(key) - 1)
__device__ int jv_first(const uint8_t* p, int n, int a) { const int i = jv_ws(p, a + 1, n); return (i < n && p[i] != ']') ? i : -1; }
__device__ int jv_next(const uint8_t* p, int n, int v) {
  const int e = skip_any(p, v, n); if (e < 0) return -1;
  int i = jv_ws(p, e, n);
  if (i < n && p[i] == ',') return jv_ws(p, i + 1, n);
  return -1;
}
// raw bytes between the quotes of the string at p[v] (v < 0: the empty string)
struct JStr { const uint8_t* p; uint32_t n; };
__device__ JStr jv_str(const uint8_t* p, int n, int v) {
  JStr s{p, 0u};
  if (v < 0 || p[v] != '"') return s;
  bool e = false; const int j = scan_string(p, v, n, e);
  if (j < 0) return s;
  s.p = p + v + 1; s.n = (uint32_t)(j - v - 2);
  return s;
}

struct O2aTools { uint32_t n; int32_t idx[15]; int32_t blk[15]; };   // activeTools (openai_helper.go:448): lives in StreamSlot::_pad
static_assert(sizeof(O2aTools) <= kStreamHdrBytes - 640, "tool map does not fit the slot header");
static constexpr uint32_t SF_O2A_CLOSED = 16u;   // closingEmitted; SF_SENT_FIRST = messageStarted, SF_TOOL_ACTIVE = hasOpenBlock

__device__ void o2a_event(Wr& w, const char* type, uint32_t tl) { WL(w, "event: "); w.lit(type, tl); WL(w, "\ndata: "); }
#define O2A_EVENT(w, text) o2a_event(w, text, (uint32_t)sizeof(text) - 1u)
__device__ void o2a_block_stop(StreamSlot& S, Wr& w) { O2A_EVENT(w, "content_block_stop"); WL(w, "{\"type\":\"content_block_stop\",\"index\":"); w.sdec(S.tool_index); WL(w, "}\n\n"); }

// emitClosingEvents (openai_helper.go:717-757)
__device__ void o2a_closing(StreamSlot& S, Wr& w) {
  if (S.flags & SF_O2A_CLOSED) return;
  S.flags |= SF_O2A_CLOSED;
  if (S.flags & SF_TOOL_ACTIVE) { o2a_block_stop(S, w); S.flags &= ~(uint32_t)SF_TOOL_ACTIVE; }
  O2A_EVENT(w, "message_delta"); WL(w, "{\"type\":\"message_delta\",\"delta\":{\"stop_reason\":\"");
  switch (S.stop_reason) { case 2: WL(w, "max_tokens"); break; case 3: WL(w, "tool_use"); break; case 4: WL(w, "refusal"); break; default: WL(w, "end_turn"); break; }
  WL(w, "\",\"stop_sequence\":null},\"usage\":{\"output_tokens\":"); w.dec(S.usage.output); WL(w, "}}\n\n");
  O2A_EVENT(w, "message_stop"); WL(w, "{\"type\":\"message_stop\"}\n\n");
}

// processEventBlock + handleChunk (openai_helper.go:492-589): 0 or AIGW_DECLINED
__device__ int o2a_block(StreamSlot& S, const uint8_t* blk, uint32_t bn, Wr& w) {
  const uint8_t* d = nullptr; uint32_t dl = 0;
  uint32_t pos = 0;
  for (;;) {   // the LAST non-empty "data: " line of the block
    uint32_t nl = pos; while (nl < bn && blk[nl] != '\n') nl++;
    const uint8_t* line = blk + pos; const uint32_t ll = nl - pos;
    if (prefix(line, ll, "data: ", 6)) { const uint8_t* q = line + 6; uint32_t ql = ll - 6; trim_space(q, ql); if (ql) { d = q; dl = ql; } }
    if (nl >= bn) break;
    pos = nl + 1;
  }
  if (!dl || EQ(d, dl, "[DONE]")) return 0;
  Capture cp; cap_reset(cp);
  const int n = (int)dl;
  const bool ok = walk(d, n, g_chunk_schema.nodes, g_chunk_schema.fields, g_chunk_schema.keys, N_ROOT, cp);
  if (cp.weird) return AIGW_DECLINED;
  if (!ok) return 0;                       // malformed chunks are skipped silently
  // the walk bounds each skipped value to skip_any's 64 levels from its own start; jv_member / jv_next below skip whole members
  // from the root, which can nest deeper than that: decline the chunk rather than read such a member as absent
  if (skip_any(d, 0, n) == -2) return AIGW_DECLINED;
  const int r = jv_ws(d, 0, n);
  if (d[r] != '{') return 0;               // `null`: the zero chunk
  {
    const JStr id = jv_str(d, n, JV(d, n, r, "id"));
    if (id.n && !S.id_len) { if (id.n > sizeof S.id || !canonical(id.p, id.n)) return AIGW_DECLINED; for (uint32_t k = 0; k < id.n; k++) S.id[k] = (char)id.p[k]; S.id_len = id.n; }
    const JStr md = jv_str(d, n, JV(d, n, r, "model"));
    if (md.n && !S.rmodel_len) { if (md.n > sizeof S.rmodel || !canonical(md.p, md.n)) return AIGW_DECLINED; for (uint32_t k = 0; k < md.n; k++) S.rmodel[k] = (char)md.p[k]; S.rmodel_len = md.n; }
  }
  const int chs = JV(d, n, r, "choices");
  const int c0 = chs >= 0 ? jv_first(d, n, chs) : -1;
  const bool has_usage = (cp.obj_seen >> C_OBJ_USAGE) & 1u;
  if (c0 < 0 && has_usage) {   // the usage-only chunk of stream_options.include_usage: ExtractTokenUsageFromExplicitCaching(in, out, &0, &0)
    if (cp.big) return AIGW_DECLINED;
    S.usage.input = cp.ints[C_PROMPT]; S.usage.output = cp.ints[C_COMPLETION]; S.usage.total = S.usage.input + S.usage.output;
    S.usage.cached = 0; S.usage.cache_creation = 0; S.usage.mask = 1u | 2u | 4u | 8u | 16u;
    o2a_closing(S, w);
    return 0;
  }
  if (c0 < 0 || d[c0] != '{') return 0;   // no choices, or a null first choice (the zero choice: no delta, no finish_reason)
  const int delta = JV(d, n, c0, "delta");
  if (!(S.flags & SF_SENT_FIRST) && delta >= 0) {   // emitMessageStart
    S.flags |= SF_SENT_FIRST;
    O2A_EVENT(w, "message_start"); WL(w, "{\"type\":\"message_start\",\"message\":{\"id\":\""); w.raw((const uint8_t*)S.id, S.id_len);
    WL(w, "\",\"type\":\"message\",\"role\":\"assistant\",\"content\":[],\"model\":\"");
    if (S.rmodel_len) w.raw((const uint8_t*)S.rmodel, S.rmodel_len); else w.raw((const uint8_t*)S.model, S.model_len);
    WL(w, "\",\"stop_reason\":null,\"stop_sequence\":null,\"usage\":{\"input_tokens\":0,\"output_tokens\":0}}}\n\n");
  }
  if (delta >= 0) {
    const JStr text = jv_str(d, n, JV(d, n, delta, "content"));
    if (text.n) {
      if (!canonical(text.p, text.n)) return AIGW_DECLINED;
      if (!(S.flags & SF_TOOL_ACTIVE)) {
        S.flags |= SF_TOOL_ACTIVE;
        O2A_EVENT(w, "content_block_start"); WL(w, "{\"type\":\"content_block_start\",\"index\":"); w.sdec(S.tool_index); WL(w, ",\"content_block\":{\"type\":\"text\",\"text\":\"\"}}\n\n");
      }
      O2A_EVENT(w, "content_block_delta"); WL(w, "{\"type\":\"content_block_delta\",\"index\":"); w.sdec(S.tool_index); WL(w, ",\"delta\":{\"type\":\"text_delta\",\"text\":\"");
      w.raw(text.p, text.n); WL(w, "\"}}\n\n");
    }
    const int tcs = JV(d, n, delta, "tool_calls");
    O2aTools& T = *(O2aTools*)S._pad;
    for (int e = tcs >= 0 ? jv_first(d, n, tcs) : -1; e >= 0; e = jv_next(d, n, e)) {   // handleToolCallDelta
      if (d[e] != '{') return AIGW_DECLINED;   // a null element is the zero tool call: stock path
      int32_t idx = 0;
      { const int iv = JV(d, n, e, "index"); if (iv >= 0) { bool ii; int ie; const int je = scan_number(d, iv, n, ii, ie); uint32_t lo; bool bg = false; if (je < 0 || !parse_i64(d, iv, je, lo, &bg) || bg) return AIGW_DECLINED; idx = (int32_t)lo; } }
      const JStr tid = jv_str(d, n, JV(d, n, e, "id"));
      const int fn = JV(d, n, e, "function");
      const JStr name = jv_str(d, n, fn >= 0 ? JV(d, n, fn, "name") : -1), args = jv_str(d, n, fn >= 0 ? JV(d, n, fn, "arguments") : -1);
      if (!canonical(tid.p, tid.n) || !canonical(name.p, name.n) || !canonical(args.p, args.n)) return AIGW_DECLINED;
      int32_t blk = -1;
      for (uint32_t k = 0; k < T.n; k++) if (T.idx[k] == idx) { blk = T.blk[k]; break; }
      if (blk < 0) {
        if (T.n >= 15u) return AIGW_DECLINED;
        if (S.flags & SF_TOOL_ACTIVE) { o2a_block_stop(S, w); S.tool_index++; }
        blk = S.tool_index; T.idx[T.n] = idx; T.blk[T.n] = blk; T.n++;
        S.flags |= SF_TOOL_ACTIVE;
        O2A_EVENT(w, "content_block_start"); WL(w, "{\"type\":\"content_block_start\",\"index\":"); w.sdec(blk); WL(w, ",\"content_block\":{\"type\":\"tool_use\",\"id\":\"");
        w.raw(tid.p, tid.n); WL(w, "\",\"name\":\""); w.raw(name.p, name.n); WL(w, "\",\"input\":{}}}\n\n");
      }
      if (args.n) {
        O2A_EVENT(w, "content_block_delta"); WL(w, "{\"type\":\"content_block_delta\",\"index\":"); w.sdec(blk); WL(w, ",\"delta\":{\"type\":\"input_json_delta\",\"partial_json\":\"");
        w.raw(args.p, args.n); WL(w, "\"}}\n\n");
      }
    }
  }
  const JStr fr = jv_str(d, n, JV(d, n, c0, "finish_reason"));
  if (fr.n) {
    for (uint32_t k = 0; k < fr.n; k++) if (fr.p[k] == '\\') return AIGW_DECLINED;
    S.stop_reason = EQ(fr.p, fr.n, "length") ? 2u : EQ(fr.p, fr.n, "tool_calls") ? 3u : EQ(fr.p, fr.n, "content_filter") ? 4u : 1u;
  }
  return 0;
}

// one ResponseBody(stream) call: processBuffer (openai_helper.go:460-490)
__device__ void step_messages_openai(StreamSlot& S, const StreamStep& st, uint8_t* out, aigw_chunk_result& R) {
  const uint8_t* b = S.buf; const uint32_t n = S.end;
  Wr w{out, 0, st.out_cap, 0};
  uint32_t pos = 0; int status = 0;
  for (;;) {
    uint32_t cut = pos; bool found = false;
    while (cut + 1 < n) { if (b[cut] == '\n' && b[cut + 1] == '\n') { found = true; break; } cut++; }
    if (!found) break;
    status = o2a_block(S, b + pos, cut - pos, w);
    if (status) break;
    pos = cut + 2;
  }
  if (!status && st.eos) {
    if (pos < n) { status = o2a_block(S, b + pos, n - pos, w); pos = n; }
    if (!status) o2a_closing(S, w);
  }
  const char* m = S.rmodel_len ? S.rmodel : S.model; const uint32_t ml = S.rmodel_len ? S.rmodel_len : S.model_len;   // cmp.Or(state.model, requestModel)
  if (!status && w.n + ml > st.out_cap) w.ovf = 1;   // the model follows the body in the same range
  if (!status && w.ovf) status = AIGW_DECLINED;
  if (status) { S.flags |= SF_DEAD; S.dead_status = (uint32_t)status; S.dead_reason = w.ovf ? AIGW_R_OUT_SPACE : AIGW_R_UNSUPPORTED_FIELD; R.status = (uint8_t)status; R.reason = (uint8_t)S.dead_reason; return; }
  S.beg = pos;
  R.usage = S.usage; R.out_len = w.n; R.body_kind = w.n ? AIGW_BODY_BYTES : AIGW_BODY_EMPTY;
  for (uint32_t k = 0; k < ml; k++) out[w.n + k] = (uint8_t)m[k];
  R.model_len = ml;
}

// ---- buffered: the tool-call `arguments` string becomes the tool_use `input` object (json.Unmarshal into map[string]any, then
// json.Marshal: keys sorted, compact).  Accepted without re-serialising: a string whose only escapes are \" and \\ and whose
// unescaped text is ALREADY that canonical form — an object, no white space outside strings, keys strictly ascending at every
// level, canonical strings, plain decimal numbers of at most 15 significant digits.  The text is unescaped straight into the
// output and checked there.  false: outside the fast path.
__device__ bool o2a_canon_number(const uint8_t* p, uint32_t l) {
  uint32_t i = 0; bool neg = false;
  if (i < l && p[i] == '-') { neg = true; i++; }
  const uint32_t is = i; while (i < l && dig(p[i])) i++;
  const uint32_t idg = i - is;
  if (!idg || (idg > 1 && p[is] == '0')) return false;
  const bool izero = idg == 1 && p[is] == '0';
  if (i == l) return !(neg && izero) && idg <= 15;
  if (p[i] != '.') return false;
  const uint32_t fs = ++i; while (i < l && dig(p[i])) i++;
  if (i != l || i == fs || p[l - 1] == '0') return false;          // no exponent, no trailing zeros
  uint32_t z = 0; if (izero) { while (fs + z < l && p[fs + z] == '0') z++; if (z > 5) return false; }
  return (izero ? (l - fs - z) : idg + (l - fs)) <= 15;
}
__device__ bool o2a_canon_object(const uint8_t* p, uint32_t n) {
  const int MAXD = 8;
  uint32_t prev_off[MAXD], prev_len[MAXD]; uint8_t is_obj[MAXD];
  int sp = 0; uint32_t i = 0;
  if (!n || p[0] != '{') return false;
  bool want_value = true;
  while (true) {
    if (want_value) {
      if (i >= n) return false;
      const uint32_t c = p[i];
      if (c == '{' || c == '[') {
        if (sp >= MAXD) return false;
        is_obj[sp] = c == '{'; prev_len[sp] = 0xffffffffu; prev_off[sp] = 0; sp++; i++;
        if (i < n && p[i] == (c == '{' ? '}' : ']')) { i++; sp--; want_value = false; continue; }
        if (c == '{') goto key;
        continue;
      }
      if (c == '"') { bool e = false; const int j = scan_string(p, (int)i, (int)n, e); if (j < 0 || !canonical(p + i + 1, (uint32_t)j - i - 2)) return false; i = (uint32_t)j; }
      else if (c == 't') { if (!lit(p, (int)i, (int)n, "true", 4)) return false; i += 4; }
      else if (c == 'f') { if (!lit(p, (int)i, (int)n, "false", 5)) return false; i += 5; }
      else if (c == 'n') { if (!lit(p, (int)i, (int)n, "null", 4)) return false; i += 4; }
      else { uint32_t j = i; while (j < n && p[j] != ',' && p[j] != '}' && p[j] != ']') j++; if (!o2a_canon_number(p + i, j - i)) return false; i = j; }
      want_value = false;
      continue;
    }
    if (sp == 0) return i == n;
    if (i >= n) return false;
    if (p[i] == ',') { i++; if (is_obj[sp - 1]) goto key; want_value = true; continue; }
    if (p[i] == (is_obj[sp - 1] ? '}' : ']')) { i++; sp--; continue; }
    return false;
  key: {
      if (i >= n || p[i] != '"') return false;
      bool e = false; const int j = scan_string(p, (int)i, (int)n, e);
      if (j < 0 || e) return false;
      const uint32_t ko = i + 1, kl = (uint32_t)j - i - 2;
      for (uint32_t k = 0; k < kl; k++) if (p[ko + k] < 0x20) return false;
      if (prev_len[sp - 1] != 0xffffffffu) {   // strictly ascending, bytewise
        const uint32_t po = prev_off[sp - 1], pl = prev_len[sp - 1]; uint32_t k = 0;
        while (k < pl && k < kl && p[po + k] == p[ko + k]) k++;
        const bool less = k < pl && k < kl ? p[po + k] < p[ko + k] : pl < kl;
        if (!less) return false;
      }
      prev_off[sp - 1] = ko; prev_len[sp - 1] = kl;
      i = (uint32_t)j;
      if (i >= n || p[i] != ':') return false;
      i++; want_value = true;
    }
  }
}
// writes the tool_use input of `args` (raw string body); false: outside the fast path
__device__ bool o2a_input(Wr& w, JStr args) {
  if (!args.n) { WL(w, "{}"); return true; }
  const uint32_t o0 = w.n;
  for (uint32_t k = 0; k < args.n; k++) {
    uint32_t c = args.p[k];
    if (c < 0x20) return false;
    if (c == '\\') { if (k + 1 >= args.n) return false; c = args.p[++k]; if (c != '"' && c != '\\') return false; }
    w.ch((char)c);
  }
  if (w.ovf) return true;   // reported as an overflow by the caller
  return o2a_canon_object(w.p + o0, w.n - o0);
}

// responseBodyNonStreaming (anthropic_openai.go:112-152): the body accumulates in the slot, the last call (eos) converts it
__device__ void step_messages_openai_buffered(StreamSlot& S, const StreamStep& st, uint8_t* out, aigw_chunk_result& R) {
  if (!st.eos) { R.body_kind = AIGW_BODY_EMPTY; return; }
  const uint8_t* b = S.buf; const int n = (int)S.end;
  Wr w{out, 0, st.out_cap, 0};
  Capture cp; cap_reset(cp);
  const bool ok = walk(b, n, g_o2a_resp_schema.nodes, g_o2a_resp_schema.fields, g_o2a_resp_schema.keys, R_ROOT, cp, /*allow_trailing=*/true);   // json.Decoder: one value
  int status = 0;
  if (cp.weird) status = AIGW_DECLINED;
  else if (!ok) status = AIGW_INTERNAL;   // "failed to unmarshal OpenAI response"
  else if (cp.big) status = AIGW_DECLINED;
  else if (skip_any(b, 0, n) == -2) status = AIGW_DECLINED;   // deeper than jv_member / jv_next can skip (see o2a_chunk)
  const uint8_t* mp = (const uint8_t*)S.model; uint32_t ml = S.model_len;
  if (!status) {
    const int r = jv_ws(b, 0, n);
    const bool obj = b[r] == '{';
    const JStr id = jv_str(b, n, obj ? JV(b, n, r, "id") : -1), md = jv_str(b, n, obj ? JV(b, n, r, "model") : -1);
    if (!canonical(id.p, id.n) || !canonical(md.p, md.n)) status = AIGW_DECLINED;
    if (md.n) { mp = md.p; ml = md.n; }
    const int chs = obj ? JV(b, n, r, "choices") : -1;
    const int c0 = chs >= 0 ? jv_first(b, n, chs) : -1;
    const uint32_t pt = cp.ints[C_PROMPT], ct = cp.ints[C_COMPLETION];
    WL(w, "{\"id\":\""); w.raw(id.p, id.n); WL(w, "\",\"type\":\"message\",\"role\":\"assistant\",\"content\":");
    bool any = false; uint32_t stop = 0;   // 0: no choice
    if (!status && c0 >= 0) {
      stop = 1;
      if (b[c0] == '{') {
        const int msg = JV(b, n, c0, "message");
        if (msg >= 0) {
          const JStr text = jv_str(b, n, JV(b, n, msg, "content"));
          if (text.n) { if (!canonical(text.p, text.n)) status = AIGW_DECLINED; WL(w, "[{\"type\":\"text\",\"text\":\""); w.raw(text.p, text.n); WL(w, "\"}"); any = true; }
          const int tcs = JV(b, n, msg, "tool_calls");
          for (int e = tcs >= 0 ? jv_first(b, n, tcs) : -1; e >= 0 && !status; e = jv_next(b, n, e)) {
            if (b[e] != '{') { status = AIGW_DECLINED; break; }
            const JStr tid = jv_str(b, n, JV(b, n, e, "id"));
            const int fn = JV(b, n, e, "function");
            const JStr name = jv_str(b, n, fn >= 0 ? JV(b, n, fn, "name") : -1), args = jv_str(b, n, fn >= 0 ? JV(b, n, fn, "arguments") : -1);
            if (!canonical(tid.p, tid.n) || !canonical(name.p, name.n)) { status = AIGW_DECLINED; break; }
            w.ch(any ? ',' : '['); any = true;
            WL(w, "{\"type\":\"tool_use\",\"id\":\""); w.raw(tid.p, tid.n); WL(w, "\",\"name\":\""); w.raw(name.p, name.n); WL(w, "\",\"input\":");
            if (!o2a_input(w, args)) { status = AIGW_DECLINED; break; }
            w.ch('}');
          }
        }
        const JStr fr = jv_str(b, n, JV(b, n, c0, "finish_reason"));
        for (uint32_t k = 0; k < fr.n; k++) if (fr.p[k] == '\\') status = AIGW_DECLINED;
        stop = EQ(fr.p, fr.n, "length") ? 2u : EQ(fr.p, fr.n, "tool_calls") ? 3u : EQ(fr.p, fr.n, "content_filter") ? 4u : 1u;
      }
    }
    if (any) w.ch(']'); else WL(w, "null");   // a nil []MessagesContentBlock
    WL(w, ",\"model\":\""); w.raw(mp, ml); w.ch('"');
    if (stop) { WL(w, ",\"stop_reason\":\""); switch (stop) { case 2: WL(w, "max_tokens"); break; case 3: WL(w, "tool_use"); break; case 4: WL(w, "refusal"); break; default: WL(w, "end_turn"); break; } w.ch('"'); }
    WL(w, ",\"usage\":{\"cache_creation_input_tokens\":0,\"cache_read_input_tokens\":0,\"input_tokens\":"); w.dec(pt); WL(w, ",\"output_tokens\":"); w.dec(ct); WL(w, "}}");
    if (!status && w.n + ml > st.out_cap) w.ovf = 1;   // the model follows the body in the same range
    if (!status && w.ovf) status = AIGW_DECLINED;
    if (!status) {
      R.usage.input = pt; R.usage.output = ct; R.usage.total = pt + ct; R.usage.mask = 7u;   // ExtractTokenUsageFromExplicitCaching(in, out, nil, nil)
      R.out_len = w.n; R.body_kind = AIGW_BODY_BYTES;
      for (uint32_t k = 0; k < ml; k++) out[w.n + k] = mp[k];
      R.model_len = ml;
      S.beg = S.end;
    }
  }
  if (status) { S.flags |= SF_DEAD; S.dead_status = (uint32_t)status; S.dead_reason = w.ovf ? AIGW_R_OUT_SPACE : AIGW_R_UNSUPPORTED_FIELD; R.status = (uint8_t)status; R.reason = (uint8_t)S.dead_reason; }
}
