// T5: streamed response of /v1/messages served by Anthropic on AWS Bedrock (included by stream_kernel.cu inside its namespace).
//   AIGW_STREAM_MESSAGES_AWS_ANTHROPIC   eventstream frames {"bytes": base64(MessagesStreamChunk JSON)} -> Anthropic SSE
//   (anthropicToAWSAnthropicTranslator.ResponseBody / convertMessagesEventWrappedInAmazonEventStreamEvent,
//    internal/translator/anthropic_awsanthropic.go:93-160; reflectStreamingEvent / updateTotalTokens, anthropic_anthropic.go:155-201;
//    MessagesStreamChunk.UnmarshalJSON and MessagesContentBlock.UnmarshalJSON, internal/apischema/anthropic/anthropic.go:1696-1748,1505-1557)
// A chunk that decodes is forwarded as "event: <type>\ndata: <decoded bytes>\n\n" and reflected into the usage; one that does not is
// dropped; outside the restated subset of the chunk decode (integer token counts, a message_start without content blocks, text / tool_use / thinking block types) the stream DECLINES.
// The frame walk, the base64 unwrap and the message_start / message_delta decode are the ones of the kinds above.
#pragma once

// an `index` member: 0 decodes, 1 outside the subset, 2 type error
__device__ int mc_index(const uint8_t* p, int vs, int ve) {
  if (vs < 0 || p[vs] == 'n') return 0;
  if (!(p[vs] == '-' || dig(p[vs]))) return 2;
  long long x; return n_count(p, vs, ve, x) ? 0 : 1;
}
// members of the object p[vs..ve) named in `names` (NUL-separated list, at most 9) must be strings or null and must not repeat:
// 0 ok, 1 escaped / repeated member, 2 type error
__device__ int mc_strings(const uint8_t* p, int vs, int ve, const char* names, int nnames) {
  int i = vs + 1, ks, kl, a, b; bool kesc; uint32_t seen = 0; int rc = 0;
  while (next_member(p, i, ve, ks, kl, kesc, a, b)) {
    if (kesc) return 1;
    const char* nm = names;
    for (int k = 0; k < nnames; k++) {
      int l = 0; while (nm[l]) l++;
      if (l == kl && eq(p + ks, (uint32_t)kl, nm, (uint32_t)l)) {
        if (seen & (1u << k)) return 1;
        seen |= 1u << k;
        if (!(p[a] == '"' || p[a] == 'n')) rc = 2;
        break;
      }
      nm += l + 1;
    }
  }
  return rc;
}
// json.Unmarshal(J, &MessagesStreamChunk{}) + reflectStreamingEvent: 0 decoded (et/etl = the event type), 1 outside the subset, 2 dropped
__device__ int mc_chunk(StreamSlot& S, const uint8_t* p, int n, const uint8_t*& et, uint32_t& etl) {
  int e = skip_any(p, 0, n);
  if (e == -2) return 1;                                  // nested beyond skip_any's levels
  if (e < 0 || skipws(p, e, n) != n) return 2;            // not one JSON value: json.Unmarshal fails
  const int r0 = skipws(p, 0, n);
  if (p[r0] != '{') return 1;
  int i = r0 + 1, ks, kl, a, b; bool kesc; uint32_t seen = 0;
  int ty_s = -1, ty_e = 0, ix_s = -1, ix_e = 0, dl_s = -1, dl_e = 0, cb_s = -1, cb_e = 0; bool has_msg = false;
  while (next_member(p, i, n, ks, kl, kesc, a, b)) {
    if (kesc) return 1;
    const uint8_t* k = p + ks; const uint32_t l = (uint32_t)kl;
    const uint32_t bit = EQ(k, l, "type") ? 1u : EQ(k, l, "message") ? 2u : EQ(k, l, "usage") ? 4u : EQ(k, l, "delta") ? 8u : EQ(k, l, "index") ? 16u : EQ(k, l, "content_block") ? 32u : 0u;
    if (!bit) continue;
    if (seen & bit) return 1;
    seen |= bit;
    if (bit == 1u) { ty_s = a; ty_e = b; } else if (bit == 2u) has_msg = true; else if (bit == 8u) { dl_s = a; dl_e = b; } else if (bit == 16u) { ix_s = a; ix_e = b; } else if (bit == 32u) { cb_s = a; cb_e = b; }
  }
  if (ty_s < 0 || p[ty_s] != '"') return 2;               // missing type / a type that names no event
  et = p + ty_s + 1; etl = (uint32_t)(ty_e - ty_s - 2);
  for (uint32_t k = 0; k < etl; k++) if (et[k] == '\\') return 1;
  if (EQ(et, etl, "message_start")) { if (!has_msg) return 2; return native_event(S, p, n) ? 1 : 0; }
  if (EQ(et, etl, "message_delta")) return native_event(S, p, n) ? 1 : 0;
  if (EQ(et, etl, "message_stop")) return 0;
  if (EQ(et, etl, "content_block_stop")) return mc_index(p, ix_s, ix_e);
  if (EQ(et, etl, "content_block_delta")) {
    const int r = mc_index(p, ix_s, ix_e); if (r) return r;
    if (dl_s < 0 || p[dl_s] == 'n') return 0;
    if (p[dl_s] != '{') return 2;
    return mc_strings(p, dl_s, dl_e, "type\0text\0partial_json\0thinking\0signature\0", 5);
  }
  if (EQ(et, etl, "content_block_start")) {
    const int r = mc_index(p, ix_s, ix_e); if (r) return r;
    if (cb_s < 0) return 0;
    if (p[cb_s] != '{') return 1;
    // the block's own type, then the members its struct reads
    int j = cb_s + 1; int ct_s = -1, ct_e = 0, cit_s = -1, in_s = -1; uint32_t cs = 0;
    while (next_member(p, j, cb_e, ks, kl, kesc, a, b)) {
      if (kesc) return 1;
      const uint8_t* k = p + ks; const uint32_t l = (uint32_t)kl;
      const uint32_t bit = EQ(k, l, "type") ? 1u : EQ(k, l, "citations") ? 2u : EQ(k, l, "input") ? 4u : 0u;
      if (!bit) continue;
      if (cs & bit) return 1;
      cs |= bit;
      if (bit == 1u) { ct_s = a; ct_e = b; } else if (bit == 2u) cit_s = a; else in_s = a;
    }
    if (ct_s < 0) return 2;                               // "missing type field in message content block"
    if (p[ct_s] != '"') return 1;
    const uint8_t* ct = p + ct_s + 1; const uint32_t ctl = (uint32_t)(ct_e - ct_s - 2);
    for (uint32_t k = 0; k < ctl; k++) if (ct[k] == '\\') return 1;
    const int sr = mc_strings(p, cb_s, cb_e, "type\0text\0id\0name\0thinking\0signature\0data\0", 7);
    if (sr == 1) return 1;
    auto bad = [&](const char* key, uint32_t kl2) -> bool {   // the member `key` of the block is present and neither string nor null
      int q = cb_s + 1, s2, l2, a2, b2; bool e2;
      while (next_member(p, q, cb_e, s2, l2, e2, a2, b2)) if ((uint32_t)l2 == kl2 && eq(p + s2, kl2, key, kl2)) return !(p[a2] == '"' || p[a2] == 'n');
      return false;
    };
    if (EQ(ct, ctl, "text")) { if (bad("text", 4)) return 2; return (cit_s < 0 || p[cit_s] == 'n') ? 0 : 1; }
    if (EQ(ct, ctl, "tool_use") || EQ(ct, ctl, "server_tool_use")) { if (bad("id", 2) || bad("name", 4)) return 2; return (in_s < 0 || p[in_s] == 'n' || p[in_s] == '{') ? 0 : 2; }
    if (EQ(ct, ctl, "thinking")) return (bad("thinking", 8) || bad("signature", 9)) ? 2 : 0;
    if (EQ(ct, ctl, "redacted_thinking")) return bad("data", 4) ? 2 : 0;
    if (EQ(ct, ctl, "web_search_tool_result")) return 1;
    return 0;                                             // unknown block types are ignored for forward compatibility
  }
  return 2;                                               // "unknown stream event type"
}

__device__ void step_messages_aws_anthropic(StreamSlot& S, const StreamStep& st, uint8_t* out, aigw_chunk_result& R) {
  uint8_t* b = S.buf; const uint32_t n = S.end;
  Wr w{out, 0, st.out_cap, 0};
  uint32_t pos = 0; int status = 0, reason = AIGW_R_UNSUPPORTED_FIELD;
  for (;;) {
    uint32_t total, hlen;
    const int fr = es_frame(b, n, pos, total, hlen);
    if (fr == 1) break;
    if (fr == 2) { status = AIGW_DECLINED; reason = AIGW_R_TOO_LARGE; break; }
    uint8_t* pl = b + pos + 12 + hlen; const int pn = (int)(total - hlen - 16u);
    pos += total;                                          // the frame is consumed whatever it holds
    int e = skip_any(pl, 0, pn);
    if (e == -2) { status = AIGW_DECLINED; break; }         // nested beyond skip_any's levels: not known to fail
    if (e < 0 || skipws(pl, e, pn) != pn) continue;        // json.Unmarshal error: the frame is skipped
    const int r0 = skipws(pl, 0, pn);
    if (pl[r0] != '{') continue;
    int i = r0 + 1, ks, kl, a, c; bool kesc; int bs = -1, be = 0; bool odd = false;
    while (next_member(pl, i, pn, ks, kl, kesc, a, c)) {
      if (kesc) { odd = true; break; }
      if (kl == 5) {
        const uint8_t* k = pl + ks;
        if (EQ(k, 5u, "bytes")) { if (bs >= 0) { odd = true; break; } bs = a; be = c; }
        else if ((k[0] | 32) == 'b' && (k[1] | 32) == 'y' && (k[2] | 32) == 't' && (k[3] | 32) == 'e' && (k[4] | 32) == 's') { odd = true; break; }   // case-insensitive field match: stock path
      }
    }
    if (odd) { status = AIGW_DECLINED; break; }
    if (bs < 0 || pl[bs] != '"') continue;                  // absent / null: no bytes; other types: unmarshal error
    uint8_t* t64 = pl + bs + 1; const int n64 = be - bs - 2;
    bool esc = false; for (int k = 0; k < n64; k++) if (t64[k] == '\\') esc = true;
    if (esc) { status = AIGW_DECLINED; break; }
    if (n64 == 0) continue;
    const int dl = b64_inplace(t64, n64);
    if (dl == -2) { status = AIGW_DECLINED; break; }
    if (dl < 0) continue;                                   // base64 error: skipped
    const uint8_t* et = nullptr; uint32_t etl = 0;
    const int rc = mc_chunk(S, t64, dl, et, etl);
    if (rc == 1) { status = AIGW_DECLINED; break; }
    if (rc == 2) continue;
    WL(w, "event: "); w.raw(et, etl); WL(w, "\ndata: "); w.raw(t64, (uint32_t)dl); WL(w, "\n\n");
  }
  const char* m = S.rmodel_len ? S.rmodel : S.model; const uint32_t ml = S.rmodel_len ? S.rmodel_len : S.model_len;
  if (!status && w.n + ml > st.out_cap) w.ovf = 1;   // the model follows the body in the same range
  if (!status && w.ovf) { status = AIGW_DECLINED; reason = AIGW_R_OUT_SPACE; }
  if (status) { S.flags |= SF_DEAD; S.dead_status = (uint32_t)status; S.dead_reason = (uint32_t)reason; R.status = (uint8_t)status; R.reason = (uint8_t)reason; return; }
  if (st.eos) {  // updateTotalTokens (anthropic_anthropic.go:176-201)
    aigw_usage& u = S.usage;
    const bool out_set = u.mask & 2u;
    if (out_set && !(u.mask & 1u)) { u.input = 0; u.mask |= 1u; }
    if (out_set) { if (!(u.mask & 8u)) { u.cached = 0; u.mask |= 8u; } if (!(u.mask & 16u)) { u.cache_creation = 0; u.mask |= 16u; } }
    if ((u.mask & 1u) && out_set) { u.total = u.input + u.output; u.mask |= 4u; }
  }
  S.beg = pos;
  R.usage = S.usage; R.out_len = w.n; R.body_kind = w.n ? AIGW_BODY_BYTES : AIGW_BODY_EMPTY;
  for (uint32_t k = 0; k < ml; k++) out[w.n + k] = (uint8_t)m[k];
  R.model_len = ml;
}
