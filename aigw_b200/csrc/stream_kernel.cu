// See stream_kernel.cuh.  sm_90a only.
#include <cstddef>
#include <cstring>

#include "bedrock_common.cuh"
#include "device_once.cuh"
#include "sse_schema.cuh"
#include "stream_kernel.cuh"

namespace aigw {
namespace {

// ------------------------------------------------------------------ device tables (one copy per device, uploaded on first use)
__device__ SchemaBlob g_chunk_schema;        // openai.ChatCompletionResponseChunk
__device__ SchemaBlob g_cmpl_schema;         // openai.CompletionResponse (legacy /v1/completions)
__device__ RespSchemaBlob g_o2a_resp_schema; // openai.ChatCompletionResponse (buffered /v1/messages response of an OpenAI backend)
__device__ RspSchemaBlob g_rsp_schema;       // openai.Response and its stream events (/v1/responses)
__device__ BedrockSchema g_conv_schema;      // awsbedrock.ConverseStreamEvent
__device__ uint32_t g_crc_tab[256];          // IEEE CRC-32

// ---- Anthropic stream events (anthropic-sdk-go v1.38.0 MessageStartEvent / ContentBlockStartEvent / ContentBlockDeltaEvent /
// MessageDeltaEvent / … as the reference reads them, internal/translator/anthropic_helper.go:944-1135): ONE union schema —
// every event type is an object whose members of interest have distinct names.
enum ASpan : uint8_t { AS_ID = 0, AS_CBTYPE, AS_CBID, AS_CBNAME, AS_INPUT, AS_DTYPE, AS_TEXT, AS_PARTIAL, AS_STOP, AS_COUNT };
enum AInt : uint8_t { AI_IN = 0, AI_OUT, AI_READ, AI_CREATE };
enum AObj : uint8_t { AO_MESSAGE = 0, AO_USAGE, AO_CB, AO_DELTA };
enum AN : uint8_t { A_ANY = 0, A_STR, A_ROOT, A_MESSAGE, A_USAGE, A_CB, A_DELTA, A_ID, A_CBTYPE, A_CBID, A_CBNAME, A_INPUT, A_DTYPE, A_TEXT, A_PARTIAL, A_STOP,
                  A_IN, A_OUT, A_READ, A_CREATE, A_COUNT };
const FieldDef kAnFields[] = {
  {A_ROOT, "type", A_STR}, {A_ROOT, "message", A_MESSAGE}, {A_ROOT, "content_block", A_CB}, {A_ROOT, "delta", A_DELTA}, {A_ROOT, "usage", A_USAGE},
  {A_MESSAGE, "id", A_ID}, {A_MESSAGE, "usage", A_USAGE},
  {A_USAGE, "input_tokens", A_IN}, {A_USAGE, "output_tokens", A_OUT}, {A_USAGE, "cache_read_input_tokens", A_READ}, {A_USAGE, "cache_creation_input_tokens", A_CREATE},
  {A_CB, "type", A_CBTYPE}, {A_CB, "id", A_CBID}, {A_CB, "name", A_CBNAME}, {A_CB, "input", A_INPUT},
  {A_DELTA, "type", A_DTYPE}, {A_DELTA, "text", A_TEXT}, {A_DELTA, "partial_json", A_PARTIAL}, {A_DELTA, "stop_reason", A_STOP},
};
constexpr int kNumAnFields = sizeof(kAnFields) / sizeof(kAnFields[0]);
struct alignas(16) AnSchema { Node nodes[A_COUNT]; Field fields[24]; char keys[256]; };
static_assert(kNumAnFields <= 24, "field table too small");
__device__ AnSchema g_an_schema;
using ACap = CaptureT<AS_COUNT>;

AnSchema build_an_schema() {
  AnSchema b; memset(&b, 0, sizeof b);
  auto set = [&](int n, uint8_t kind, uint8_t cap = 0xff, uint8_t elem = 0) { b.nodes[n].kind = kind; b.nodes[n].cap = cap; b.nodes[n].elem = elem; };
  set(A_ANY, K_ANY); set(A_STR, K_STR); set(A_ROOT, K_OBJ);
  set(A_MESSAGE, K_OBJ, AO_MESSAGE); set(A_USAGE, K_OBJ, AO_USAGE); set(A_CB, K_OBJ, AO_CB); set(A_DELTA, K_OBJ, AO_DELTA);
  set(A_ID, K_STR, AS_ID); set(A_CBTYPE, K_STR, AS_CBTYPE); set(A_CBID, K_STR, AS_CBID); set(A_CBNAME, K_STR, AS_CBNAME); set(A_INPUT, K_ANY, AS_INPUT);
  set(A_DTYPE, K_STR, AS_DTYPE); set(A_TEXT, K_STR, AS_TEXT); set(A_PARTIAL, K_STR, AS_PARTIAL); set(A_STOP, K_STR, AS_STOP);
  set(A_IN, K_INT, AI_IN); set(A_OUT, K_INT, AI_OUT); set(A_READ, K_INT, AI_READ); set(A_CREATE, K_INT, AI_CREATE);
  int ko = 0;
  for (int f = 0; f < kNumAnFields; f++) {
    const FieldDef& d = kAnFields[f];
    Node& o = b.nodes[d.owner];
    if (o.nf == 0) o.f0 = (uint8_t)f;
    o.nf++;
    const int kl = (int)strlen(d.key);
    b.fields[f].koff = (uint16_t)ko; b.fields[f].klen = (uint8_t)kl; b.fields[f].node = d.node;
    memcpy(b.keys + ko, d.key, kl); ko += kl;
  }
  return b;
}

// ------------------------------------------------------------------ bounded writer of one call's body mutation
struct Wr {
  uint8_t* p; uint32_t n, cap, ovf;
  __device__ __forceinline__ void ch(char c) { if (n < cap) p[n] = (uint8_t)c; else ovf = 1; n++; }
  __device__ void lit(const char* s, uint32_t l) { if (n + l <= cap) { for (uint32_t k = 0; k < l; k++) p[n + k] = (uint8_t)s[k]; } else ovf = 1; n += l; }
  __device__ void raw(const uint8_t* s, uint32_t l) { if (n + l <= cap) { for (uint32_t k = 0; k < l; k++) p[n + k] = s[k]; } else ovf = 1; n += l; }
  __device__ void dec(unsigned long long v) { char b[20]; int k = 0; do { b[k++] = (char)('0' + v % 10ull); v /= 10ull; } while (v); for (int t = k - 1; t >= 0; t--) ch(b[t]); }
  __device__ void sdec(long long v) { if (v < 0) { ch('-'); dec(0ull - (unsigned long long)v); } else dec((unsigned long long)v); }
};
#define WL(w, text) (w).lit(text, (uint32_t)sizeof(text) - 1u)

__device__ __forceinline__ bool go_space(uint32_t c) { return c == ' ' || c == '\t' || c == '\n' || c == '\v' || c == '\f' || c == '\r'; }
// bytes.TrimSpace: ASCII white space plus U+0085 / U+00A0 in UTF-8
__device__ void trim_space(const uint8_t*& p, uint32_t& n) {
  for (;;) {
    if (n && go_space(p[0])) { p++; n--; continue; }
    if (n >= 2 && p[0] == 0xC2 && (p[1] == 0x85 || p[1] == 0xA0)) { p += 2; n -= 2; continue; }
    break;
  }
  for (;;) {
    if (n && go_space(p[n - 1])) { n--; continue; }
    if (n >= 2 && p[n - 2] == 0xC2 && (p[n - 1] == 0x85 || p[n - 1] == 0xA0)) { n -= 2; continue; }
    break;
  }
}
__device__ __forceinline__ bool eq(const uint8_t* p, uint32_t l, const char* w, uint32_t wl) { if (l != wl) return false; for (uint32_t k = 0; k < l; k++) if (p[k] != (uint8_t)w[k]) return false; return true; }
#define EQ(p, l, text) eq(p, l, text, (uint32_t)sizeof(text) - 1u)
__device__ __forceinline__ bool prefix(const uint8_t* p, uint32_t l, const char* w, uint32_t wl) { if (l < wl) return false; for (uint32_t k = 0; k < wl; k++) if (p[k] != (uint8_t)w[k]) return false; return true; }

template <class CAP>
__device__ __forceinline__ void cap_reset(CAP& cp) {
  cp.int_set = 0; cp.obj_seen = 0; cp.span_set = 0; cp.span_esc = 0; cp.weird = 0; cp.big = 0;
#pragma unroll
  for (int k = 0; k < 8; k++) cp.ints[k] = 0;
}

// ------------------------------------------------------------------ S1: OpenAI SSE usage scan, one ResponseBody call
// (openAIToOpenAITranslatorV1ChatCompletion.ResponseBody stream branch + extractUsageFromBufferEvent,
//  internal/translator/openai_openai.go:131-145,179-215)
// `completions`: the legacy /v1/completions translator (openai_completions.go:80-96,157-203) — the same loop over
// openai.CompletionResponse chunks; responseModel is the stream's own model only (no fallback to the request model)
__device__ void step_openai(StreamSlot& S, const StreamStep& st, uint8_t* out, aigw_chunk_result& R, bool completions = false) {
  const SchemaBlob& sch = completions ? g_cmpl_schema : g_chunk_schema;
  const uint8_t* b = S.buf; const uint32_t n = S.end;
  uint32_t pos = 0;
  aigw_usage u; memset(&u, 0, sizeof u);
  int status = 0;
  for (;;) {
    uint32_t nl = pos; while (nl < n && b[nl] != '\n') nl++;
    if (nl >= n) break;
    const uint8_t* line = b + pos; const uint32_t ll = nl - pos;
    pos = nl + 1;
    if (!prefix(line, ll, "data: ", 6)) continue;
    Capture cp; cap_reset(cp);
    const bool ok = walk(line + 6, (int)ll - 6, sch.nodes, sch.fields, sch.keys, N_ROOT, cp);
    if (cp.weird || (cp.span_esc & 1u)) { status = AIGW_DECLINED; break; }
    if (!ok) continue;   // not a chunk (e.g. [DONE]): skipped silently
    if ((cp.span_set & 1u) && cp.span_len[0] > 0) {
      if (cp.span_len[0] > sizeof S.rmodel) { status = AIGW_DECLINED; break; }
      for (uint32_t k = 0; k < cp.span_len[0]; k++) S.rmodel[k] = (char)line[6 + cp.span_off[0] + k];
      S.rmodel_len = cp.span_len[0];
    }
    if (cp.obj_seen & (1u << C_OBJ_USAGE)) {
      u.input = cp.ints[C_PROMPT]; u.output = cp.ints[C_COMPLETION]; u.total = cp.ints[C_TOTAL]; u.mask |= 7u;
      if (cp.obj_seen & (1u << C_OBJ_PTD)) { u.cached = cp.ints[C_CACHED]; u.cache_creation = cp.ints[C_CACHE_CREATION]; u.mask |= 8u | 16u; }
      if (cp.obj_seen & (1u << C_OBJ_CTD)) { u.reasoning = cp.ints[C_REASONING]; u.mask |= 32u; }
    }
  }
  // responseModel = cmp.Or(streamingResponseModel, requestModel): placed after the (empty) body
  const char* m = S.rmodel_len ? S.rmodel : S.model; const uint32_t ml = S.rmodel_len ? S.rmodel_len : completions ? 0u : S.model_len;
  int reason = AIGW_R_UNSUPPORTED_FIELD;
  if (!status && ml > st.out_cap) { status = AIGW_DECLINED; reason = AIGW_R_OUT_SPACE; }
  if (status) { S.flags |= SF_DEAD; S.dead_status = (uint32_t)status; S.dead_reason = (uint32_t)reason; R.status = (uint8_t)status; R.reason = (uint8_t)reason; return; }
  S.beg = pos;
  R.usage = u; R.body_kind = AIGW_BODY_UNCHANGED; R.out_len = 0;
  for (uint32_t k = 0; k < ml; k++) out[k] = (uint8_t)m[k];
  R.model_len = ml;
}

// ------------------------------------------------------------------ S3: Anthropic SSE → OpenAI SSE
// serializeOpenAIChatCompletionChunk(constructOpenAIChatCompletionChunk(delta, finish)), anthropic_helper.go:1138-1162
struct AnDelta { const uint8_t* content; uint32_t content_len; bool has_content; int tool; /* 0 none, 1 start, 2 delta */ const uint8_t* a; uint32_t al; const uint8_t* b; uint32_t bl; };
__device__ void an_chunk(StreamSlot& S, Wr& w, const AnDelta& d, const char* finish, uint32_t finish_len) {
  bool role = false;
  if (!(S.flags & SF_SENT_FIRST) && (d.has_content || d.tool)) { role = true; S.flags |= SF_SENT_FIRST; }
  WL(w, "data: {");
  if (S.id_len) { WL(w, "\"id\":\""); w.raw((const uint8_t*)S.id, S.id_len); WL(w, "\","); }
  WL(w, "\"choices\":[{\"index\":0,\"delta\":{");
  bool f = true;
  if (d.has_content) { WL(w, "\"content\":\""); w.raw(d.content, d.content_len); w.ch('"'); f = false; }
  if (role) { if (!f) w.ch(','); WL(w, "\"role\":\"assistant\""); f = false; }
  if (d.tool) {
    if (!f) w.ch(',');
    WL(w, "\"tool_calls\":[{\"index\":"); w.sdec(S.tool_index);
    if (d.tool == 1) { WL(w, ",\"id\":\""); w.raw(d.a, d.al); WL(w, "\",\"function\":{\"arguments\":\"\",\"name\":\""); w.raw(d.b, d.bl); WL(w, "\"},\"type\":\"function\"}]"); }
    else { WL(w, ",\"id\":null,\"function\":{\"arguments\":\""); w.raw(d.a, d.al); WL(w, "\",\"name\":\"\"}}]"); }
  }
  w.ch('}');
  if (finish_len) { WL(w, ",\"finish_reason\":\""); w.lit(finish, finish_len); w.ch('"'); }
  WL(w, "}]");
  if (S.flags & SF_HAVE_CREATED) { WL(w, ",\"created\":"); w.sdec(S.created); }
  if (S.model_len) { WL(w, ",\"model\":\""); w.raw((const uint8_t*)S.model, S.model_len); w.ch('"'); }
  WL(w, ",\"object\":\"chat.completion.chunk\"}\n\n");
}

// one event block; 0, AIGW_INTERNAL (the reference returns an error) or AIGW_DECLINED
__device__ int an_event_core(StreamSlot& S, const uint8_t* et, uint32_t etl, const uint8_t* data, uint32_t dl, int ndata, Wr& w);
__device__ int an_event(StreamSlot& S, const uint8_t* blk, uint32_t bn, Wr& w) {
  const uint8_t* et = nullptr; uint32_t etl = 0; const uint8_t* data = nullptr; uint32_t dl = 0; int ndata = 0;
  uint32_t pos = 0;
  for (;;) {
    uint32_t nl = pos; while (nl < bn && blk[nl] != '\n') nl++;
    const uint8_t* line = blk + pos; const uint32_t ll = nl - pos;
    if (prefix(line, ll, "event: ", 7)) { et = line + 7; etl = ll - 7; trim_space(et, etl); }
    else if (prefix(line, ll, "data: ", 6)) { const uint8_t* q = line + 6; uint32_t ql = ll - 6; trim_space(q, ql); if (ql) { if (ndata == 0) { data = q; dl = ql; } ndata++; } }
    if (nl >= bn) break;
    pos = nl + 1;
  }
  return an_event_core(S, et, etl, data, dl, ndata, w);
}
// one event given as its (trimmed) type and data line
__device__ int an_event_core(StreamSlot& S, const uint8_t* et, uint32_t etl, const uint8_t* data, uint32_t dl, int ndata, Wr& w) {
  if (!etl || !dl) return 0;
  if (ndata > 1) return AIGW_DECLINED;   // concatenated data lines: stock path
  int ev;  // 1 message_start 2 content_block_start 3 message_delta 4 content_block_delta 5 content_block_stop 6 message_stop 7 error
  if (EQ(et, etl, "message_start")) ev = 1; else if (EQ(et, etl, "content_block_start")) ev = 2; else if (EQ(et, etl, "message_delta")) ev = 3;
  else if (EQ(et, etl, "content_block_delta")) ev = 4; else if (EQ(et, etl, "content_block_stop")) ev = 5; else if (EQ(et, etl, "message_stop")) ev = 6;
  else if (EQ(et, etl, "error")) ev = 7; else return 0;   // ping and unknown types are ignored before any decode
  ACap cp; cap_reset(cp);
  const bool ok = walk(data, (int)dl, g_an_schema.nodes, g_an_schema.fields, g_an_schema.keys, A_ROOT, cp);
  if (!ok) {  // syntax error ⇒ "unmarshal …" error; a well-formed value of another shape ⇒ unpinned, stock path
    int e = skip_any(data, 0, (int)dl);
    if (e == -2) return AIGW_DECLINED;   // nesting beyond skip_any's levels: the decoder may accept it
    if (e >= 0) { while (e < (int)dl && ws(data[e])) e++; }
    return (e < 0 || e != (int)dl) ? AIGW_INTERNAL : AIGW_DECLINED;
  }
  if (cp.weird || cp.big) return AIGW_DECLINED;
  if (ev == 7) return AIGW_INTERNAL;   // "anthropic stream error: …"
  auto has = [&](int s) { return (cp.span_set >> s) & 1u; };
  auto sp = [&](int s) { return data + cp.span_off[s]; };
  auto len = [&](int s) { return has(s) ? cp.span_len[s] : 0u; };
  auto clean = [&](int s) { return !has(s) || canonical(sp(s), cp.span_len[s]); };   // re-encoded byte for byte by the reference's encoder
  auto plain = [&](int s) { return !((cp.span_esc >> s) & 1u); };
  const unsigned long long in = cp.ints[AI_IN], o = cp.ints[AI_OUT], rd = cp.ints[AI_READ], cr = cp.ints[AI_CREATE];
  switch (ev) {
    case 1: {
      if (!clean(AS_ID) || len(AS_ID) > sizeof S.id) return AIGW_DECLINED;
      if (in + rd + cr >= 0x80000000ull) return AIGW_DECLINED;
      S.id_len = len(AS_ID); for (uint32_t k = 0; k < S.id_len; k++) S.id[k] = (char)sp(AS_ID)[k];
      S.flags |= SF_HAVE_CREATED;
      S.usage.input = (uint32_t)(in + rd + cr); S.usage.cached = (uint32_t)rd; S.usage.cache_creation = (uint32_t)cr; S.usage.mask |= 1u | 8u | 16u;
      S.tool_index = -1;
      return 0;
    }
    case 2: {
      if (!plain(AS_CBTYPE)) return AIGW_DECLINED;
      const uint8_t* t = sp(AS_CBTYPE); const uint32_t tl = len(AS_CBTYPE);
      if (EQ(t, tl, "tool_use") || EQ(t, tl, "server_tool_use")) {
        S.tool_index++;
        if (has(AS_INPUT)) {
          const uint8_t* q = sp(AS_INPUT); const uint32_t ql = cp.span_len[AS_INPUT];
          if (!EQ(q, ql, "null")) {
            if (q[0] != '{') return AIGW_INTERNAL;                     // "unexpected tool use input type"
            uint32_t k = 1; while (k < ql && ws(q[k])) k++;
            if (!(k < ql && q[k] == '}')) return AIGW_DECLINED;        // non-empty map: json.Marshal(map) layout left to the stock path
          }
        }
        if (!clean(AS_CBID) || !clean(AS_CBNAME)) return AIGW_DECLINED;
        S.flags |= SF_TOOL_ACTIVE; S.active_index = S.tool_index;
        AnDelta d{}; d.tool = 1; d.a = sp(AS_CBID); d.al = len(AS_CBID); d.b = sp(AS_CBNAME); d.bl = len(AS_CBNAME);
        an_chunk(S, w, d, nullptr, 0);
      } else if (EQ(t, tl, "thinking")) { AnDelta d{}; d.has_content = true; an_chunk(S, w, d, nullptr, 0); }
      return 0;
    }
    case 3: {
      if (!plain(AS_STOP) || len(AS_STOP) > 255u) return AIGW_DECLINED;
      S.usage.output += (uint32_t)o; S.usage.input += (uint32_t)rd; S.usage.cached += (uint32_t)rd; S.usage.input += (uint32_t)cr; S.usage.cache_creation += (uint32_t)cr;
      S.usage.mask |= 2u | 1u | 8u | 16u;
      if ((S.usage.input | S.usage.output) & 0x80000000u) return AIGW_DECLINED;
      if (len(AS_STOP)) {
        const uint8_t* q = sp(AS_STOP); const uint32_t ql = len(AS_STOP);
        S.stop_reason = EQ(q, ql, "end_turn") || EQ(q, ql, "stop_sequence") || EQ(q, ql, "pause_turn") ? 1u : EQ(q, ql, "max_tokens") ? 2u : EQ(q, ql, "tool_use") ? 3u : EQ(q, ql, "refusal") ? 4u : 5u;
      }
      return 0;
    }
    case 4: {
      if (!plain(AS_DTYPE)) return AIGW_DECLINED;
      const uint8_t* t = sp(AS_DTYPE); const uint32_t tl = len(AS_DTYPE);
      if (EQ(t, tl, "text_delta") || EQ(t, tl, "thinking_delta")) {
        if (!clean(AS_TEXT)) return AIGW_DECLINED;
        AnDelta d{}; d.has_content = true; d.content = sp(AS_TEXT); d.content_len = len(AS_TEXT);
        an_chunk(S, w, d, nullptr, 0);
      } else if (EQ(t, tl, "input_json_delta")) {
        if (!((S.flags & SF_TOOL_ACTIVE) && S.active_index == S.tool_index)) return AIGW_INTERNAL;   // "received input_json_delta for unknown tool"
        if (!clean(AS_PARTIAL)) return AIGW_DECLINED;
        AnDelta d{}; d.tool = 2; d.a = sp(AS_PARTIAL); d.al = len(AS_PARTIAL);
        an_chunk(S, w, d, nullptr, 0);
      }
      return 0;
    }
    case 5: if ((S.flags & SF_TOOL_ACTIVE) && S.active_index == S.tool_index) S.flags &= ~(uint32_t)SF_TOOL_ACTIVE; return 0;
    default: {  // message_stop
      if (S.stop_reason == 0) S.stop_reason = 1;
      AnDelta d{};
      switch (S.stop_reason) {
        case 1: an_chunk(S, w, d, "stop", 4); break; case 2: an_chunk(S, w, d, "length", 6); break;
        case 3: an_chunk(S, w, d, "tool_calls", 10); break; case 4: an_chunk(S, w, d, "content_filter", 14); break;
        default: return AIGW_INTERNAL;   // "received invalid stop reason"
      }
      return 0;
    }
  }
}

// end of stream: the final usage chunk and [DONE] (anthropic_helper.go:859-916)
__device__ int an_finish(StreamSlot& S, Wr& w) {
  if (S.flags & SF_TOOL_ACTIVE) return AIGW_DECLINED;   // an open tool call is replayed in the final chunk: stock path
  S.usage.total = S.usage.input + S.usage.output; S.usage.mask |= 4u;
  if (S.usage.input > 0 || S.usage.output > 0) {
    WL(w, "data: {");
    if (S.id_len) { WL(w, "\"id\":\""); w.raw((const uint8_t*)S.id, S.id_len); WL(w, "\","); }
    WL(w, "\"choices\":[]");
    if (S.flags & SF_HAVE_CREATED) { WL(w, ",\"created\":"); w.sdec(S.created); }
    if (S.model_len) { WL(w, ",\"model\":\""); w.raw((const uint8_t*)S.model, S.model_len); w.ch('"'); }
    WL(w, ",\"object\":\"chat.completion.chunk\",\"usage\":{");
    bool f = true;
    auto num = [&](const char* k, uint32_t kl, uint32_t v) { if (!v) return; if (!f) w.ch(','); f = false; w.lit(k, kl); w.dec(v); };
    num("\"prompt_tokens\":", 16, S.usage.input); num("\"completion_tokens\":", 20, S.usage.output); num("\"total_tokens\":", 15, S.usage.total);
    if (!f) w.ch(',');
    WL(w, "\"prompt_tokens_details\":{"); f = true;
    num("\"cached_tokens\":", 16, S.usage.cached); num("\"cache_creation_input_tokens\":", 30, S.usage.cache_creation);
    WL(w, "}}}\n\n");
  }
  WL(w, "data: [DONE]\n\n");
  return 0;
}

// anthropicStreamParser.Process, internal/translator/anthropic_helper.go:826-919
__device__ void step_anthropic(StreamSlot& S, const StreamStep& st, uint8_t* out, aigw_chunk_result& R) {
  const uint8_t* b = S.buf; const uint32_t n = S.end;
  Wr w{out, 0, st.out_cap, 0};
  uint32_t pos = 0; int status = 0;
  for (;;) {
    uint32_t cut = pos; bool found = false;
    while (cut + 1 < n) { if (b[cut] == '\n' && b[cut + 1] == '\n') { found = true; break; } cut++; }
    if (!found) break;
    status = an_event(S, b + pos, cut - pos, w);
    if (status) break;
    pos = cut + 2;
  }
  if (!status && st.eos && pos < n) { status = an_event(S, b + pos, n - pos, w); pos = n; }
  if (!status && st.eos) status = an_finish(S, w);
  if (!status && w.n + S.model_len > st.out_cap) w.ovf = 1;   // the model follows the body in the same range
  if (!status && w.ovf) status = AIGW_DECLINED;
  if (status) { S.flags |= SF_DEAD; S.dead_status = (uint32_t)status; S.dead_reason = w.ovf ? AIGW_R_OUT_SPACE : AIGW_R_UNSUPPORTED_FIELD; R.status = (uint8_t)status; R.reason = (uint8_t)S.dead_reason; return; }
  S.beg = pos;
  R.usage = S.usage; R.out_len = w.n; R.body_kind = w.n ? AIGW_BODY_BYTES : AIGW_BODY_EMPTY;
  for (uint32_t k = 0; k < S.model_len; k++) out[w.n + k] = (uint8_t)S.model[k];
  R.model_len = S.model_len;
}

// ------------------------------------------------------------------ S2: Bedrock eventstream → OpenAI SSE
// (ResponseBody stream branch, extractAmazonEventStreamEvents, convertEvent: internal/translator/openai_awsbedrock.go:695-732,829-852,858-1006)
__device__ uint32_t crc32_dev(const uint8_t* p, uint32_t n) { uint32_t c = 0xffffffffu; for (uint32_t k = 0; k < n; k++) c = g_crc_tab[(c ^ p[k]) & 0xffu] ^ (c >> 8); return ~c; }

__device__ void step_bedrock(StreamSlot& S, const StreamStep& st, uint8_t* out, aigw_chunk_result& R) {
  const uint8_t* b = S.buf; const uint32_t n = S.end;
  const uint8_t* base = (const uint8_t*)&S;                       // spans in records are offsets from the slot base
  const uint32_t buf_off = (uint32_t)offsetof(StreamSlot, buf), role_off = (uint32_t)offsetof(StreamSlot, role);
  uint32_t pos = 0, wn = 0; int status = 0, reason = 0;
  aigw_usage u; memset(&u, 0, sizeof u);
  for (;;) {
    if (n - pos < 12u) break;
    const uint8_t* f = b + pos;
    const uint32_t total = be32(f), hlen = be32(f + 4);
    if (crc32_dev(f, 8) != be32(f + 8)) break;                     // decoder error: this frame blocks the stream (as in the reference)
    if (hlen > 128u * 1024u || total < 16u || hlen > total - 16u || total - hlen - 16u > 16u * 1024u * 1024u) break;
    if (total > kStreamCarryCap) { status = AIGW_DECLINED; reason = AIGW_R_TOO_LARGE; break; }
    if (n - pos < total) break;                                    // incomplete frame: wait for more bytes
    if (crc32_dev(f, total - 4u) != be32(f + total - 4u)) break;
    const uint8_t* et = nullptr; uint32_t etl = 0; bool bad = false;
    {
      uint32_t h = 12; const uint32_t hend = 12 + hlen;
      while (h < hend) {
        const uint32_t nl = f[h]; h++;
        if (h + nl + 1 > hend) { bad = true; break; }
        const uint8_t* name = f + h; h += nl;
        const uint32_t type = f[h]; h++;
        int vs;
        switch (type) { case 0: case 1: vs = 0; break; case 2: vs = 1; break; case 3: vs = 2; break; case 4: vs = 4; break; case 5: case 8: vs = 8; break; case 9: vs = 16; break; case 6: case 7: vs = -1; break; default: vs = -2; }
        if (vs == -2) { bad = true; break; }
        if (vs == -1) { if (h + 2 > hend) { bad = true; break; } vs = (f[h] << 8) | f[h + 1]; h += 2; }
        if (h + (uint32_t)vs > hend) { bad = true; break; }
        if (type == 7 && same(name, nl, ":event-type", 11)) { et = f + h; etl = (uint32_t)vs; }
        h += (uint32_t)vs;
      }
    }
    if (bad) break;
    const uint8_t* pl = f + 12 + hlen; const int pn = (int)(total - hlen - 16u);
    const uint32_t pl_rel = buf_off + pos + 12u + hlen;
    BCap cp; cap_reset(cp);
    bool ok;
    if (pn == 4 && pl[0] == 'n' && pl[1] == 'u' && pl[2] == 'l' && pl[3] == 'l') ok = true;
    else ok = walk(pl, pn, g_conv_schema.nodes, g_conv_schema.fields, g_conv_schema.keys, B_ROOT, cp);
    if (cp.weird) { status = AIGW_DECLINED; reason = AIGW_R_UNSUPPORTED_FIELD; break; }
    uint32_t kind = KD_NONE, flags = 0; bool decl = false;
    BedrockRec rec; memset(&rec, 0, sizeof rec);
    if (ok) {
      auto has = [&](int sp) { return (cp.span_set >> sp) & 1u; };
      auto span_ok = [&](int sp) { return !has(sp) || canonical(pl + cp.span_off[sp], cp.span_len[sp]); };
      if (has(S_EVT)) { et = pl + cp.span_off[S_EVT]; etl = cp.span_len[S_EVT]; if ((cp.span_esc >> S_EVT) & 1u) decl = true; }
      if (same(et, etl, "metadata", 8)) {
        if (cp.obj_seen & (1u << O_USAGE)) {
          kind = KD_META;
          const bool hr = (cp.int_set >> I_READ) & 1u, hw = (cp.int_set >> I_WRITE) & 1u;
          const unsigned long long tin = (unsigned long long)cp.ints[I_IN] + (hr ? cp.ints[I_READ] : 0u) + (hw ? cp.ints[I_WRITE] : 0u);
          if (cp.big || tin + cp.ints[I_OUT] >= 0x80000000ull) decl = true;
          rec.a[0] = (uint32_t)tin; rec.a[1] = cp.ints[I_OUT]; rec.a[2] = cp.ints[I_READ]; rec.a[3] = cp.ints[I_WRITE];
          if (hr) flags |= F_HAS_READ; if (hw) flags |= F_HAS_WRITE;
          memset(&u, 0, sizeof u);
          u.input = (uint32_t)tin; u.output = cp.ints[I_OUT]; u.total = u.input + u.output; u.mask = 7u;
          if (hr) { u.cached = cp.ints[I_READ]; u.mask |= 8u; }
          if (hw) { u.cache_creation = cp.ints[I_WRITE]; u.mask |= 16u; }
          if ((cp.obj_seen & (1u << O_TIER)) && has(S_TIER) && cp.span_len[S_TIER]) { if (!span_ok(S_TIER)) decl = true; rec.a[4] = pl_rel + cp.span_off[S_TIER]; rec.a[5] = cp.span_len[S_TIER]; }
        }
      } else if (same(et, etl, "messageStart", 12)) {
        if (has(S_ROLE)) {
          kind = KD_MSGSTART;
          if (!span_ok(S_ROLE) || cp.span_len[S_ROLE] > sizeof S.role) decl = true;
          else { S.role_len = cp.span_len[S_ROLE]; for (uint32_t k = 0; k < S.role_len; k++) S.role[k] = (char)pl[cp.span_off[S_ROLE] + k]; }
        }
      } else if (same(et, etl, "contentBlockDelta", 17)) {
        if (cp.obj_seen & (1u << O_DELTA)) {
          if (has(S_TEXT)) { kind = KD_TEXT; if (!span_ok(S_TEXT)) decl = true; rec.a[0] = pl_rel + cp.span_off[S_TEXT]; rec.a[1] = cp.span_len[S_TEXT]; }
          else if (cp.obj_seen & (1u << O_DTOOL)) { kind = KD_TOOLDELTA; if (!span_ok(S_TOOLIN)) decl = true; if (has(S_TOOLIN)) { rec.a[0] = pl_rel + cp.span_off[S_TOOLIN]; rec.a[1] = cp.span_len[S_TOOLIN]; } }
          else if (cp.obj_seen & (1u << O_DREASON)) {
            kind = KD_REASON;
            if (!span_ok(S_RTEXT) || !span_ok(S_RSIG)) decl = true;
            if (has(S_RTEXT)) { rec.a[0] = pl_rel + cp.span_off[S_RTEXT]; rec.a[1] = cp.span_len[S_RTEXT]; }
            if (has(S_RSIG)) { rec.a[2] = pl_rel + cp.span_off[S_RSIG]; rec.a[3] = cp.span_len[S_RSIG]; }
            if (has(S_REDACT) && cp.span_len[S_REDACT]) decl = true;
          } else kind = KD_EMPTY;
        }
      } else if (same(et, etl, "contentBlockStart", 17)) {
        if (cp.obj_seen & (1u << O_START)) {
          if (cp.obj_seen & (1u << O_STOOL)) {
            kind = KD_TOOLSTART;
            if (!span_ok(S_NAME) || !span_ok(S_TUID)) decl = true;
            if (has(S_NAME)) { rec.a[0] = pl_rel + cp.span_off[S_NAME]; rec.a[1] = cp.span_len[S_NAME]; }
            if (has(S_TUID)) { rec.a[2] = pl_rel + cp.span_off[S_TUID]; rec.a[3] = cp.span_len[S_TUID]; }
          } else kind = KD_EMPTY;
        }
      } else if (same(et, etl, "messageStop", 11)) {
        if (has(S_STOP)) {
          kind = KD_STOP;
          if ((cp.span_esc >> S_STOP) & 1u) decl = true;
          const uint8_t* q = pl + cp.span_off[S_STOP]; const uint32_t ql = cp.span_len[S_STOP];
          if (same(q, ql, "max_tokens", 10)) flags |= 1u; else if (same(q, ql, "content_filtered", 16)) flags |= 2u; else if (same(q, ql, "tool_use", 8)) flags |= 3u;
        }
      } else if (same(et, etl, "contentBlockStop", 16)) kind = KD_BLOCKSTOP;
    }
    if (decl) { status = AIGW_DECLINED; reason = AIGW_R_UNSUPPORTED_FIELD; break; }
    // stream state in event order (convertEvent): the role of the latest messageStart, the tool-call index
    if (kind == KD_TOOLSTART) S.flags |= SF_TOOL_ACTIVE;
    rec.tool_index = (uint32_t)S.tool_index; rec.role_off = role_off; rec.role_len = S.role_len;
    if (kind == KD_BLOCKSTOP && (S.flags & SF_TOOL_ACTIVE)) { S.tool_index++; S.flags &= ~(uint32_t)SF_TOOL_ACTIVE; }
    if (kind != KD_NONE && kind != KD_BLOCKSTOP) {
      rec.kf = kind | (flags << 8);
      const uint32_t need = emit_chunk<false>(rec, S, nullptr, nullptr);
      if (wn + need > st.out_cap) { status = AIGW_DECLINED; reason = AIGW_R_OUT_SPACE; break; }
      emit_chunk<true>(rec, S, base, out + wn);
      wn += need;
    }
    pos += total;
  }
  if (!status && st.eos) { if (wn + 13u > st.out_cap) { status = AIGW_DECLINED; reason = AIGW_R_OUT_SPACE; } else { const char* dn = "data: [DONE]\n"; for (int k = 0; k < 13; k++) out[wn + k] = (uint8_t)dn[k]; wn += 13; } }
  if (!status && wn + S.model_len > st.out_cap) { status = AIGW_DECLINED; reason = AIGW_R_OUT_SPACE; }
  if (status) { S.flags |= SF_DEAD; S.dead_status = (uint32_t)status; S.dead_reason = (uint32_t)reason; R.status = (uint8_t)status; R.reason = (uint8_t)reason; return; }
  S.beg = pos;
  R.usage = u; R.out_len = wn; R.body_kind = wn ? AIGW_BODY_BYTES : AIGW_BODY_EMPTY;
  for (uint32_t k = 0; k < S.model_len; k++) out[wn + k] = (uint8_t)S.model[k];
  R.model_len = S.model_len;
}

// ------------------------------------------------------------------ S3 behind AWS: Anthropic events wrapped in eventstream frames
// (openAIToAWSAnthropicTranslatorV1ChatCompletion.ResponseBody + extractAnthropicSSEFromEventStream,
//  internal/translator/openai_awsanthropic.go:162-184,216-261): every frame's payload is {"bytes":"<base64 of the event JSON>"};
//  the reference decodes it, takes gjson "type" and hands "event: T\ndata: J\n\n" to the Anthropic stream parser.
__device__ __forceinline__ int skipws(const uint8_t* p, int i, int n);
__device__ bool next_member(const uint8_t* p, int& i, int n, int& ks, int& kl, bool& kesc, int& vs, int& ve);
// 0 frame at pos is complete and valid, 1 wait / blocked (decoder error), 2 too large for the carry
__device__ int es_frame(const uint8_t* b, uint32_t n, uint32_t pos, uint32_t& total, uint32_t& hlen) {
  if (n - pos < 12u) return 1;
  const uint8_t* f = b + pos;
  total = be32(f); hlen = be32(f + 4);
  if (crc32_dev(f, 8) != be32(f + 8)) return 1;
  if (hlen > 128u * 1024u || total < 16u || hlen > total - 16u || total - hlen - 16u > 16u * 1024u * 1024u) return 1;
  if (total > kStreamCarryCap) return 2;
  if (n - pos < total) return 1;
  if (crc32_dev(f, total - 4u) != be32(f + total - 4u)) return 1;
  uint32_t h = 12; const uint32_t hend = 12 + hlen;
  while (h < hend) {
    const uint32_t nl = f[h]; h++;
    if (h + nl + 1 > hend) return 1;
    h += nl;
    const uint32_t type = f[h]; h++;
    int vs;
    switch (type) { case 0: case 1: vs = 0; break; case 2: vs = 1; break; case 3: vs = 2; break; case 4: vs = 4; break; case 5: case 8: vs = 8; break; case 9: vs = 16; break; case 6: case 7: vs = -1; break; default: vs = -2; }
    if (vs == -2) return 1;
    if (vs == -1) { if (h + 2 > hend) return 1; vs = (f[h] << 8) | f[h + 1]; h += 2; }
    if (h + (uint32_t)vs > hend) return 1;
    h += (uint32_t)vs;
  }
  return 0;
}
__device__ __forceinline__ int b64v(uint32_t c) { return c - 'A' < 26u ? (int)(c - 'A') : c - 'a' < 26u ? (int)(c - 'a') + 26 : c - '0' < 10u ? (int)(c - '0') + 52 : c == '+' ? 62 : c == '/' ? 63 : -1; }
// base64.StdEncoding.DecodeString of p[0, n) written over p (the decoded text is shorter).  Returns the length, -1 = not decodable,
// -2 = a byte outside the alphabet that Go's decoder would skip or that needs the stock path (CR / LF)
__device__ int b64_inplace(uint8_t* p, int n) {
  if (n & 3) return -1;
  int w = 0;
  for (int i = 0; i < n; i += 4) {
    const uint32_t c0 = p[i], c1 = p[i + 1], c2 = p[i + 2], c3 = p[i + 3];
    if (c0 == '\r' || c0 == '\n' || c1 == '\r' || c1 == '\n' || c2 == '\r' || c2 == '\n' || c3 == '\r' || c3 == '\n') return -2;
    const int a = b64v(c0), b = b64v(c1);
    if (a < 0 || b < 0) return -1;
    const bool last = i + 4 == n;
    if (c2 == '=') { if (!last || c3 != '=') return -1; p[w++] = (uint8_t)((a << 2) | (b >> 4)); break; }
    const int c = b64v(c2);
    if (c < 0) return -1;
    if (c3 == '=') { if (!last) return -1; p[w++] = (uint8_t)((a << 2) | (b >> 4)); p[w++] = (uint8_t)(((b & 15) << 4) | (c >> 2)); break; }
    const int d = b64v(c3);
    if (d < 0) return -1;
    p[w++] = (uint8_t)((a << 2) | (b >> 4)); p[w++] = (uint8_t)(((b & 15) << 4) | (c >> 2)); p[w++] = (uint8_t)(((c & 3) << 6) | d);
  }
  return w;
}
__device__ void step_aws_anthropic(StreamSlot& S, const StreamStep& st, uint8_t* out, aigw_chunk_result& R) {
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
    if (pl[r0] != '{') continue;                           // null decodes to the zero struct, other roots fail: nothing to forward either way
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
    if (bs < 0 || pl[bs] != '"') continue;                  // absent / null: Bytes == "" ; other types: unmarshal error
    uint8_t* t64 = pl + bs + 1; const int n64 = be - bs - 2;
    bool esc = false; for (int k = 0; k < n64; k++) if (t64[k] == '\\') esc = true;
    if (esc) { status = AIGW_DECLINED; break; }
    if (n64 == 0) continue;
    const int dl = b64_inplace(t64, n64);
    if (dl == -2) { status = AIGW_DECLINED; break; }
    if (dl < 0) continue;                                   // base64 error: skipped
    const uint8_t* J = t64;
    bool nlc = false; for (int k = 0; k < dl; k++) if (J[k] == '\n') nlc = true;
    if (nlc) { status = AIGW_DECLINED; break; }              // a line break inside the event would split the SSE block
    int je = skip_any(J, 0, dl);
    if (je < 0 || skipws(J, je, dl) != dl) { status = AIGW_DECLINED; break; }   // gjson on malformed text: stock path
    const int j0 = skipws(J, 0, dl);
    const uint8_t* et = nullptr; uint32_t etl = 0;
    if (J[j0] == '{') {
      int j = j0 + 1; bool bad = false;
      while (next_member(J, j, dl, ks, kl, kesc, a, c)) {
        if (kesc) { bad = true; break; }
        if (!et && EQ(J + ks, (uint32_t)kl, "type")) {
          if (J[a] != '"') { bad = true; break; }
          et = J + a + 1; etl = (uint32_t)(c - a - 2);
          for (uint32_t k = 0; k < etl; k++) if (et[k] == '\\') bad = true;
          if (etl == 0) et = nullptr;
        }
      }
      if (bad) { status = AIGW_DECLINED; break; }
    }
    if (!et) continue;                                       // "event: \ndata: …": a block without an event type is ignored by the parser
    { const uint8_t* q = et; uint32_t ql = etl; trim_space(q, ql); et = q; etl = ql; }
    const uint8_t* dq = J; uint32_t dql = (uint32_t)dl; trim_space(dq, dql);
    status = an_event_core(S, et, etl, dq, dql, dql ? 1 : 0, w);
    if (status) break;
  }
  if (!status && st.eos) status = an_finish(S, w);
  if (!status && w.n + S.model_len > st.out_cap) w.ovf = 1;   // the model follows the body in the same range
  if (!status && w.ovf) { status = AIGW_DECLINED; reason = AIGW_R_OUT_SPACE; }
  if (status) { S.flags |= SF_DEAD; S.dead_status = (uint32_t)status; S.dead_reason = (uint32_t)reason; R.status = (uint8_t)status; R.reason = (uint8_t)reason; return; }
  S.beg = pos;
  R.usage = S.usage; R.out_len = w.n; R.body_kind = w.n ? AIGW_BODY_BYTES : AIGW_BODY_EMPTY;
  for (uint32_t k = 0; k < S.model_len; k++) out[w.n + k] = (uint8_t)S.model[k];
  R.model_len = S.model_len;
}

// ------------------------------------------------------------------ S4 / R1: Gemini GenerateContentResponse → OpenAI
// (handleStreamingResponse / parseGCPStreamingChunks / convertGCPChunkToOpenAI, internal/translator/openai_gcpvertexai.go:202-337,390-482;
//  buffered: ResponseBody :139-198, geminiCandidatesToOpenAIChoices gemini_helper.go:741-828; usage :942-958; finish reasons :836-868)
static constexpr int kGemCands = 2, kGemTexts = 8;
struct GemCand { uint32_t null_, has_content, ntext; uint32_t toff[kGemTexts], tlen[kGemTexts]; uint32_t tthought; uint32_t fin_off, fin_len; };
struct GemResp { uint32_t id_off, id_len, mv_off, mv_len, has_time, has_usage, ncand; long long created; uint32_t prompt, cand, total, cached, thoughts; GemCand c[kGemCands]; };

__device__ __forceinline__ int skipws(const uint8_t* p, int i, int n) { while (i < n && ws(p[i])) i++; return i; }
// object member iteration over syntactically valid JSON: i = position after '{' or after the previous value; false at '}'
__device__ bool next_member(const uint8_t* p, int& i, int n, int& ks, int& kl, bool& kesc, int& vs, int& ve) {
  i = skipws(p, i, n);
  if (p[i] == ',') i = skipws(p, i + 1, n);
  if (p[i] == '}') { i++; return false; }
  kesc = false; const int e = scan_string(p, i, n, kesc);
  ks = i + 1; kl = e - i - 2;
  i = skipws(p, e, n); i = skipws(p, i + 1, n);   // ':'
  vs = i; ve = skip_any(p, i, n); i = ve;
  return true;
}
__device__ bool next_elem(const uint8_t* p, int& i, int n, int& vs, int& ve) {
  i = skipws(p, i, n);
  if (p[i] == ',') i = skipws(p, i + 1, n);
  if (p[i] == ']') { i++; return false; }
  vs = i; ve = skip_any(p, i, n); i = ve;
  return true;
}
__device__ __forceinline__ bool is_null_at(const uint8_t* p, int vs) { return p[vs] == 'n'; }
// RFC 3339 → Unix seconds
__device__ bool rfc3339_unix(const uint8_t* s, int n, long long& out) {
  auto dig = [&](int i) { return i < n && s[i] - '0' < 10u; };
  auto num = [&](int i, int k, int& v) { v = 0; for (int t = 0; t < k; t++) { if (!dig(i + t)) return false; v = v * 10 + (s[i + t] - '0'); } return true; };
  int Y, M, D, h, m, sec;
  if (n < 20 || !num(0, 4, Y) || s[4] != '-' || !num(5, 2, M) || s[7] != '-' || !num(8, 2, D) || (s[10] != 'T' && s[10] != 't') || !num(11, 2, h) || s[13] != ':' || !num(14, 2, m) || s[16] != ':' || !num(17, 2, sec)) return false;
  int i = 19;
  if (i < n && s[i] == '.') { i++; if (!dig(i)) return false; while (dig(i)) i++; }
  int off = 0;
  if (i < n && (s[i] == 'Z' || s[i] == 'z')) i++;
  else { int oh, om; if (i + 6 > n || (s[i] != '+' && s[i] != '-') || !num(i + 1, 2, oh) || s[i + 3] != ':' || !num(i + 4, 2, om)) return false; off = (oh * 60 + om) * 60 * (s[i] == '-' ? -1 : 1); i += 6; }
  if (i != n || M < 1 || M > 12 || D < 1 || D > 31 || h > 23 || m > 59 || sec > 59) return false;
  const long long y = Y - (M <= 2); const long long era = (y >= 0 ? y : y - 399) / 400; const long long yoe = y - era * 400;
  const long long doy = (153 * (M + (M > 2 ? -3 : 9)) + 2) / 5 + D - 1; const long long doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
  out = (era * 146097 + doe - 719468) * 86400 + h * 3600 + m * 60 + sec - off;
  return true;
}
// 0 decoded, 1 not decodable (syntax / trailing bytes), 2 unpinned (stock path)
__device__ int gem_decode(const uint8_t* p, int n, GemResp& g, bool buffered) {
  memset(&g, 0, sizeof g);
  int i = skipws(p, 0, n);
  const int root_end = skip_any(p, i, n);
  if (root_end == -2) return 2;
  if (root_end < 0) return 1;
  if (!buffered && skipws(p, root_end, n) != n) return 1;
  if (p[i] == 'n') return 0;
  if (p[i] != '{') return 2;
  bool unp = false;
  auto str_span = [&](int vs, int ve, uint32_t& off, uint32_t& len) { if (is_null_at(p, vs)) return; if (p[vs] != '"') { unp = true; return; } off = vs + 1; len = ve - vs - 2; if (!canonical(p + off, len)) unp = true; };
  auto u31 = [&](int vs, int ve, uint32_t& out) { if (is_null_at(p, vs)) return; bool ii; int ie; if (!(p[vs] == '-' || dig(p[vs])) || scan_number(p, vs, n, ii, ie) != ve || !ii) { unp = true; return; } uint32_t v; bool big = false; if (!parse_i64(p, vs, ve, v, &big) || big) { unp = true; return; } out = v; };
  int ks, kl, vs, ve; bool kesc;
  i++;
  while (next_member(p, i, n, ks, kl, kesc, vs, ve)) {
    if (kesc) { unp = true; continue; }
    const uint8_t* k = p + ks;
    if (EQ(k, kl, "responseId")) str_span(vs, ve, g.id_off, g.id_len);
    else if (EQ(k, kl, "modelVersion")) str_span(vs, ve, g.mv_off, g.mv_len);
    else if (EQ(k, kl, "createTime")) { if (!is_null_at(p, vs)) { if (p[vs] != '"' || !rfc3339_unix(p + vs + 1, ve - vs - 2, g.created)) unp = true; else g.has_time = 1; } }
    else if (EQ(k, kl, "usageMetadata")) {
      if (is_null_at(p, vs)) continue;
      if (p[vs] != '{') { unp = true; continue; }
      g.has_usage = 1;
      int j = vs + 1, ks2, kl2, vs2, ve2; bool ke2;
      while (next_member(p, j, n, ks2, kl2, ke2, vs2, ve2)) {
        const uint8_t* q = p + ks2;
        if (EQ(q, kl2, "promptTokenCount")) u31(vs2, ve2, g.prompt); else if (EQ(q, kl2, "candidatesTokenCount")) u31(vs2, ve2, g.cand); else if (EQ(q, kl2, "totalTokenCount")) u31(vs2, ve2, g.total);
        else if (EQ(q, kl2, "cachedContentTokenCount")) u31(vs2, ve2, g.cached); else if (EQ(q, kl2, "thoughtsTokenCount")) u31(vs2, ve2, g.thoughts);
      }
    } else if (EQ(k, kl, "candidates")) {
      if (is_null_at(p, vs)) continue;
      if (p[vs] != '[') { unp = true; continue; }
      int j = vs + 1, cs, ce;
      while (next_elem(p, j, n, cs, ce)) {
        if (g.ncand >= (uint32_t)kGemCands) { unp = true; continue; }
        GemCand& c = g.c[g.ncand++];
        if (is_null_at(p, cs)) { c.null_ = 1; continue; }
        if (p[cs] != '{') { unp = true; continue; }
        int a = cs + 1, ks2, kl2, vs2, ve2; bool ke2;
        while (next_member(p, a, n, ks2, kl2, ke2, vs2, ve2)) {
          const uint8_t* q = p + ks2;
          if (EQ(q, kl2, "finishReason")) { str_span(vs2, ve2, c.fin_off, c.fin_len); }
          else if (buffered && (EQ(q, kl2, "safetyRatings") || EQ(q, kl2, "groundingMetadata") || EQ(q, kl2, "logprobsResult"))) { if (!is_null_at(p, vs2)) unp = true; }
          else if (EQ(q, kl2, "content")) {
            if (is_null_at(p, vs2)) continue;
            if (p[vs2] != '{') { unp = true; continue; }
            c.has_content = 1;
            int b = vs2 + 1, ks3, kl3, vs3, ve3; bool ke3;
            while (next_member(p, b, n, ks3, kl3, ke3, vs3, ve3)) {
              if (!EQ(p + ks3, kl3, "parts") || is_null_at(p, vs3)) continue;
              if (p[vs3] != '[') { unp = true; continue; }
              int e = vs3 + 1, ps, pe;
              while (next_elem(p, e, n, ps, pe)) {
                if (is_null_at(p, ps)) continue;
                if (p[ps] != '{') { unp = true; continue; }
                uint32_t toff = 0, tlen = 0; bool thought = false;
                int f = ps + 1, ks4, kl4, vs4, ve4; bool ke4;
                while (next_member(p, f, n, ks4, kl4, ke4, vs4, ve4)) {
                  const uint8_t* r = p + ks4;
                  if (EQ(r, kl4, "text")) str_span(vs4, ve4, toff, tlen);
                  else if (EQ(r, kl4, "thought")) { if (p[vs4] == 't') thought = true; else if (p[vs4] != 'f' && !is_null_at(p, vs4)) unp = true; }
                  else if (EQ(r, kl4, "functionCall") || EQ(r, kl4, "thoughtSignature")) { if (!is_null_at(p, vs4)) unp = true; }
                }
                if (tlen) { if (c.ntext >= (uint32_t)kGemTexts) unp = true; else { c.toff[c.ntext] = toff; c.tlen[c.ntext] = tlen; if (thought) c.tthought |= 1u << c.ntext; c.ntext++; } }
              }
            }
          }
        }
      }
    }
  }
  return unp ? 2 : 0;
}
__device__ void gem_finish(Wr& w, const uint8_t* p, const GemCand& c, bool always) {
  const uint8_t* q = p + c.fin_off; const uint32_t l = c.fin_len;
  const char* fr; uint32_t fl;
  if (l == 0) { fr = ""; fl = 0; }
  else if (EQ(q, l, "STOP")) { fr = "stop"; fl = 4; } else if (EQ(q, l, "MAX_TOKENS")) { fr = "length"; fl = 6; }
  else if (EQ(q, l, "SAFETY") || EQ(q, l, "BLOCKLIST") || EQ(q, l, "PROHIBITED_CONTENT") || EQ(q, l, "SPII") || EQ(q, l, "IMAGE_SAFETY") || EQ(q, l, "IMAGE_PROHIBITED_CONTENT")) { fr = "content_filter"; fl = 14; }
  else if (EQ(q, l, "RECITATION") || EQ(q, l, "IMAGE_RECITATION")) { fr = "recitation"; fl = 10; } else if (EQ(q, l, "MALFORMED_FUNCTION_CALL")) { fr = "malformed_function_call"; fl = 23; }
  else if (EQ(q, l, "UNEXPECTED_TOOL_CALL")) { fr = "unexpected_tool_call"; fl = 20; } else if (EQ(q, l, "LANGUAGE")) { fr = "language"; fl = 8; } else if (EQ(q, l, "NO_IMAGE")) { fr = "no_image"; fl = 8; }
  else { fr = "error"; fl = 5; }
  if (always) { WL(w, "{\"finish_reason\":\""); w.lit(fr, fl); w.ch('"'); }
  else if (fl) { WL(w, ",\"finish_reason\":\""); w.lit(fr, fl); w.ch('"'); }
}
__device__ void gem_usage(Wr& w, const GemResp& g) {
  bool f = true;
  auto num = [&](const char* k, uint32_t kl, uint32_t v) { if (!v) return; if (!f) w.ch(','); f = false; w.lit(k, kl); w.dec(v); };
  w.ch('{'); num("\"prompt_tokens\":", 16, g.prompt); num("\"completion_tokens\":", 20, g.cand + g.thoughts); num("\"total_tokens\":", 15, g.total);
  if (!f) w.ch(',');
  WL(w, "\"completion_tokens_details\":{"); if (g.thoughts) { WL(w, "\"reasoning_tokens\":"); w.dec(g.thoughts); }
  WL(w, "},\"prompt_tokens_details\":{"); if (g.cached) { WL(w, "\"cached_tokens\":"); w.dec(g.cached); }
  WL(w, "}}");
}
__device__ void gem_texts(Wr& w, const uint8_t* p, const GemCand& c, bool thought) { for (uint32_t k = 0; k < c.ntext; k++) if ((((c.tthought >> k) & 1u) != 0) == thought) w.raw(p + c.toff[k], c.tlen[k]); }
__device__ bool gem_has(const GemCand& c, bool thought) { for (uint32_t k = 0; k < c.ntext; k++) if ((((c.tthought >> k) & 1u) != 0) == thought) return true; return false; }

__device__ void gem_stream_chunk(StreamSlot& S, Wr& w, const uint8_t* p, const GemResp& g) {
  auto head = [&] { WL(w, "data: {"); if (g.id_len) { WL(w, "\"id\":\""); w.raw(p + g.id_off, g.id_len); WL(w, "\","); } };
  auto tail = [&] { if (g.has_time) { WL(w, ",\"created\":"); w.sdec(g.created); } if (S.model_len) { WL(w, ",\"model\":\""); w.raw((const uint8_t*)S.model, S.model_len); w.ch('"'); } WL(w, ",\"object\":\"chat.completion.chunk\""); };
  head(); WL(w, "\"choices\":[");
  bool cf = true;
  for (uint32_t ci = 0; ci < g.ncand; ci++) {
    const GemCand& c = g.c[ci];
    if (c.null_) continue;
    if (!cf) w.ch(','); cf = false;
    WL(w, "{\"index\":"); w.dec(ci); WL(w, ",\"delta\":{");
    if (c.has_content) {
      if (gem_has(c, false)) { WL(w, "\"content\":\""); gem_texts(w, p, c, false); WL(w, "\","); }
      WL(w, "\"role\":\"assistant\"");
      if (gem_has(c, true)) { WL(w, ",\"reasoning_content\":{\"text\":\""); gem_texts(w, p, c, true); WL(w, "\"}"); }
    }
    w.ch('}'); gem_finish(w, p, c, false); w.ch('}');
  }
  w.ch(']'); tail(); WL(w, "}\n\n");
  if (g.has_usage && g.prompt > 0) { head(); WL(w, "\"choices\":[]"); tail(); WL(w, ",\"usage\":"); gem_usage(w, g); WL(w, "}\n\n"); }
}

__device__ void step_gemini(StreamSlot& S, const StreamStep& st, uint8_t* out, aigw_chunk_result& R) {
  uint8_t* b = S.buf; const uint32_t n = S.end; const uint32_t old_len = S._r0;   // carry length before this call's append
  Wr w{out, 0, st.out_cap, 0};
  aigw_usage u; memset(&u, 0, sizeof u);
  int status = 0;
  if (n) {
    if (S.stop_reason == 0) {   // delimiter not detected yet: CRLFCRLF, LFLF, CRCR in that order of preference
      bool crlf = false, lf = false, cr = false;
      for (uint32_t i = 0; i + 1 < n; i++) { if (b[i] == '\n' && b[i + 1] == '\n') lf = true; if (b[i] == '\r' && b[i + 1] == '\r') cr = true; if (i + 3 < n && b[i] == '\r' && b[i + 1] == '\n' && b[i + 2] == '\r' && b[i + 3] == '\n') crlf = true; }
      S.stop_reason = crlf ? 1u : lf ? 2u : cr ? 3u : 0u;
    }
    const uint32_t dk = S.stop_reason, dl = dk == 1 ? 4u : dk ? 2u : 0u;
    uint32_t pos = 0; bool touched = false; uint32_t nb_off = 0, nb_len = old_len;   // the new bufferedBody as a span of b
    for (;;) {
      uint32_t cut = n; 
      if (dk) for (uint32_t i = pos; i + dl <= n; i++) { const bool m = dk == 1 ? (b[i] == '\r' && b[i + 1] == '\n' && b[i + 2] == '\r' && b[i + 3] == '\n') : dk == 2 ? (b[i] == '\n' && b[i + 1] == '\n') : (b[i] == '\r' && b[i + 1] == '\r'); if (m) { cut = i; break; } }
      const uint8_t* part = b + pos; uint32_t pl = cut - pos;
      trim_space(part, pl);
      if (pl) {
        if (prefix(part, pl, "data: ", 6)) { part += 6; pl -= 6; }
        GemResp g;
        const int rc = gem_decode(part, (int)pl, g, false);
        if (rc == 2) { status = AIGW_DECLINED; break; }
        touched = true;
        if (rc == 1) { nb_off = (uint32_t)(part - b); nb_len = pl; }
        else {
          nb_len = 0;
          gem_stream_chunk(S, w, part, g);
          if (g.has_usage && g.prompt > 0) { u.input = g.prompt; u.output = g.cand; u.total = g.total; u.cached = g.cached; u.reasoning = g.thoughts; u.mask = 1u | 2u | 4u | 8u | 32u; }
        }
      }
      if (cut >= n) break;
      pos = cut + dl;
    }
    if (!status) {
      if (!touched) { nb_off = 0; nb_len = old_len; }
      for (uint32_t k = 0; k < nb_len; k++) b[k] = b[nb_off + k];   // bufferedBody := the (trimmed, prefix-stripped) undecodable part; forward copy, nb_off ≥ 0
      S.beg = 0; S.end = nb_len;
    }
  }
  if (!status && st.eos) WL(w, "data: [DONE]\n");
  if (!status && w.n + S.model_len > st.out_cap) w.ovf = 1;   // the model follows the body in the same range
  if (!status && w.ovf) status = AIGW_DECLINED;
  if (status) { S.flags |= SF_DEAD; S.dead_status = (uint32_t)status; S.dead_reason = w.ovf ? AIGW_R_OUT_SPACE : AIGW_R_UNSUPPORTED_FIELD; R.status = (uint8_t)status; R.reason = (uint8_t)S.dead_reason; return; }
  R.usage = u; R.out_len = w.n; R.body_kind = w.n ? AIGW_BODY_BYTES : AIGW_BODY_EMPTY;
  for (uint32_t k = 0; k < S.model_len; k++) out[w.n + k] = (uint8_t)S.model[k];
  R.model_len = S.model_len;
}

// buffered response: the body accumulates in the slot; the last call (eos) converts it
__device__ void step_gemini_buffered(StreamSlot& S, const StreamStep& st, uint8_t* out, aigw_chunk_result& R) {
  if (!st.eos) { R.body_kind = AIGW_BODY_EMPTY; return; }
  const uint8_t* b = S.buf; const int n = (int)S.end;
  Wr w{out, 0, st.out_cap, 0};
  GemResp g;
  const int rc = gem_decode(b, n, g, true);
  int status = rc == 1 ? AIGW_INTERNAL : rc == 2 ? AIGW_DECLINED : 0;   // "error decoding GCP response"
  if (!status) for (uint32_t ci = 0; ci < g.ncand; ci++) if (!g.c[ci].null_ && !g.c[ci].has_content) status = AIGW_DECLINED;
  if (!status) {
    w.ch('{');
    if (g.id_len) { WL(w, "\"id\":\""); w.raw(b + g.id_off, g.id_len); WL(w, "\","); }
    WL(w, "\"choices\":[");
    bool cf = true;
    for (uint32_t ci = 0; ci < g.ncand; ci++) {
      const GemCand& c = g.c[ci];
      if (c.null_) continue;
      if (!cf) w.ch(','); cf = false;
      gem_finish(w, b, c, true); WL(w, ",\"index\":"); w.dec(ci); WL(w, ",\"message\":{");
      if (gem_has(c, false)) { WL(w, "\"content\":\""); gem_texts(w, b, c, false); WL(w, "\","); }
      WL(w, "\"role\":\"assistant\"");
      if (gem_has(c, true)) { WL(w, ",\"reasoning_content\":\""); gem_texts(w, b, c, true); w.ch('"'); }
      WL(w, "}}");
    }
    w.ch(']');
    if (g.has_time) { WL(w, ",\"created\":"); w.sdec(g.created); }
    const uint8_t* m = g.mv_len ? b + g.mv_off : (const uint8_t*)S.model; const uint32_t ml = g.mv_len ? g.mv_len : S.model_len;
    if (ml) { WL(w, ",\"model\":\""); w.raw(m, ml); w.ch('"'); }
    WL(w, ",\"object\":\"chat.completion\"");
    if (g.has_usage) { WL(w, ",\"usage\":"); gem_usage(w, g); }
    w.ch('}');
    if (!status && w.n + ml > st.out_cap) w.ovf = 1;   // the model follows the body in the same range
    if (w.ovf) status = AIGW_DECLINED;
    else {
      R.usage.input = g.prompt; R.usage.output = g.cand + g.thoughts; R.usage.total = g.total; R.usage.mask = 7u;
      if (g.has_usage) { R.usage.cached = g.cached; R.usage.reasoning = g.thoughts; R.usage.mask |= 8u | 32u; }
      R.out_len = w.n; R.body_kind = AIGW_BODY_BYTES;
      for (uint32_t k = 0; k < ml; k++) out[w.n + k] = m[k];
      R.model_len = ml;
      S.beg = S.end;
    }
  }
  if (status) { S.flags |= SF_DEAD; S.dead_status = (uint32_t)status; S.dead_reason = w.ovf ? AIGW_R_OUT_SPACE : AIGW_R_UNSUPPORTED_FIELD; R.status = (uint8_t)status; R.reason = (uint8_t)S.dead_reason; }
}

// ------------------------------------------------------------------ S1 variant: native Anthropic SSE, usage scan only
// (anthropicToAnthropicTranslator.ResponseBody stream branch, extractUsageFromBufferEvent / reflectStreamingEvent /
//  updateTotalTokens, internal/translator/anthropic_anthropic.go:86-101,133-201; MessagesStreamChunk.UnmarshalJSON,
//  internal/apischema/anthropic/anthropic.go:1696-1748).  The body passes through untouched.  Only message_start and
//  message_delta change the state; they are decoded over the subset include/aigw_b200.h names, anything else kills the
//  stream with DECLINED (the content-block unions are not restated here).
struct NUsage { long long in, out, rd, cr; };
// a token count: integer literal (optional '-'), magnitude below 2^31; null counts as 0.  false: outside the subset
__device__ bool n_count(const uint8_t* p, int vs, int ve, long long& out) {
  out = 0;
  if (p[vs] == 'n') return true;
  int i = vs; bool neg = false;
  if (p[i] == '-') { neg = true; i++; }
  if (i >= ve) return false;
  long long x = 0;
  for (; i < ve; i++) { const uint32_t c = p[i] - '0'; if (c > 9u) return false; x = x * 10 + c; if (x >= (1ll << 31)) return false; }
  out = neg ? -x : x;
  return true;
}
__device__ __forceinline__ bool n_str_or_null(const uint8_t* p, int vs) { return p[vs] == '"' || p[vs] == 'n'; }
__device__ bool n_usage(const uint8_t* p, int vs, int ve, NUsage& u) {
  if (p[vs] != '{') return false;
  int i = vs + 1, ks, kl, a, b; bool kesc; uint32_t seen = 0;
  while (next_member(p, i, ve, ks, kl, kesc, a, b)) {
    if (kesc) return false;
    const uint8_t* k = p + ks;
    const uint32_t bit = EQ(k, (uint32_t)kl, "input_tokens") ? 1u : EQ(k, (uint32_t)kl, "output_tokens") ? 2u : EQ(k, (uint32_t)kl, "cache_read_input_tokens") ? 4u
                         : EQ(k, (uint32_t)kl, "cache_creation_input_tokens") ? 8u : 0u;
    if (!bit) continue;
    if (seen & bit) return false;
    seen |= bit;
    long long x;
    if (!n_count(p, a, b, x)) return false;
    if (bit == 1u) u.in = x; else if (bit == 2u) u.out = x; else if (bit == 4u) u.rd = x; else u.cr = x;
  }
  return true;
}
// one `data: ` payload: 0 handled or ignored, 1 outside the subset
__device__ int native_event(StreamSlot& S, const uint8_t* p, int n) {
  int e = skip_any(p, 0, n);
  if (e == -2) return 1;
  if (e < 0) return 0;
  e = skipws(p, e, n);
  if (e != n) return 0;                                   // not one JSON value: the line is skipped
  int r0 = skipws(p, 0, n);
  if (p[r0] != '{') return 0;                             // no "type" to find
  int i = r0 + 1, ks, kl, a, b; bool kesc;
  int ty_s = -1, ty_e = 0, msg_s = -1, msg_e = 0, us_s = -1, us_e = 0, dl_s = -1, dl_e = 0; uint32_t seen = 0;
  while (next_member(p, i, n, ks, kl, kesc, a, b)) {
    if (kesc) return 1;
    const uint8_t* k = p + ks;
    const uint32_t bit = EQ(k, (uint32_t)kl, "type") ? 1u : EQ(k, (uint32_t)kl, "message") ? 2u : EQ(k, (uint32_t)kl, "usage") ? 4u : EQ(k, (uint32_t)kl, "delta") ? 8u : 0u;
    if (!bit) continue;
    if (seen & bit) { if (seen & 1u) return 1; seen |= 16u; continue; }   // a repeated member: decided below once the type is known
    seen |= bit;
    if (bit == 1u) { ty_s = a; ty_e = b; } else if (bit == 2u) { msg_s = a; msg_e = b; } else if (bit == 4u) { us_s = a; us_e = b; } else { dl_s = a; dl_e = b; }
  }
  if (ty_s < 0) return 0;                                 // "missing type field in stream event"
  if (p[ty_s] != '"') return 1;
  if (seen & 16u) return 1;
  const uint8_t* t = p + ty_s + 1; const uint32_t tl = (uint32_t)(ty_e - ty_s - 2);
  for (uint32_t k = 0; k < tl; k++) if (t[k] == '\\') return 1;
  if (EQ(t, tl, "message_start")) {
    if (msg_s < 0 || p[msg_s] == 'n') return 0;
    if (p[msg_s] != '{') return 1;
    int j = msg_s + 1; uint32_t ms = 0; int model_s = -1, model_e = 0, mus_s = -1, mus_e = 0;
    while (next_member(p, j, msg_e, ks, kl, kesc, a, b)) {
      if (kesc) return 1;
      const uint8_t* k = p + ks; const uint32_t l = (uint32_t)kl;
      const uint32_t bit = EQ(k, l, "id") ? 1u : EQ(k, l, "stop_reason") ? 2u : EQ(k, l, "stop_sequence") ? 4u : EQ(k, l, "model") ? 8u : EQ(k, l, "type") ? 16u : EQ(k, l, "role") ? 32u
                           : EQ(k, l, "content") ? 64u : EQ(k, l, "usage") ? 128u : 0u;
      if (!bit) continue;
      if (ms & bit) return 1;
      ms |= bit;
      if (bit <= 4u) { if (!n_str_or_null(p, a)) return 1; }
      else if (bit == 8u) { if (!n_str_or_null(p, a)) return 1; if (p[a] == '"') { model_s = a + 1; model_e = b - 1; } }
      else if (bit == 16u) { if (!(p[a] == '"' && EQ(p + a + 1, (uint32_t)(b - a - 2), "message"))) return 1; }
      else if (bit == 32u) { if (!(p[a] == '"' && EQ(p + a + 1, (uint32_t)(b - a - 2), "assistant"))) return 1; }
      else if (bit == 64u) { if (p[a] != 'n') { if (p[a] != '[') return 1; const int q = skipws(p, a + 1, b); if (p[q] != ']') return 1; } }
      else { if (p[a] != 'n') { mus_s = a; mus_e = b; } }
    }
    NUsage u{0, 0, 0, 0};
    if (mus_s >= 0 && !n_usage(p, mus_s, mus_e, u)) return 1;
    if (mus_s >= 0 && (u.in < 0 || u.out < 0 || u.rd < 0 || u.cr < 0 || u.in + u.rd + u.cr >= (1ll << 31) || u.in + u.rd + u.cr + u.out >= (1ll << 31))) return 1;
    if (model_s >= 0 && model_e > model_s) {
      const uint32_t ml = (uint32_t)(model_e - model_s);
      if (ml > sizeof S.rmodel) return 1;
      for (uint32_t k = 0; k < ml; k++) { if (p[model_s + k] == '\\') return 1; S.rmodel[k] = (char)p[model_s + k]; }
      S.rmodel_len = ml;
    }
    if (mus_s >= 0) {   // ExtractTokenUsageFromExplicitCaching + Override (metrics.go:292-307)
      S.usage.input = (uint32_t)(u.in + u.rd + u.cr); S.usage.output = (uint32_t)u.out; S.usage.total = S.usage.input + S.usage.output;
      S.usage.cached = (uint32_t)u.rd; S.usage.cache_creation = (uint32_t)u.cr; S.usage.mask |= 31u;
    }
    return 0;
  }
  if (EQ(t, tl, "message_delta")) {
    NUsage u{0, 0, 0, 0};
    if (us_s >= 0 && p[us_s] != 'n' && !n_usage(p, us_s, us_e, u)) return 1;
    if (dl_s >= 0 && p[dl_s] != 'n') {
      if (p[dl_s] != '{') return 1;
      int j = dl_s + 1; uint32_t ds = 0;
      while (next_member(p, j, dl_e, ks, kl, kesc, a, b)) {
        if (kesc) return 1;
        const uint32_t bit = EQ(p + ks, (uint32_t)kl, "stop_reason") ? 1u : EQ(p + ks, (uint32_t)kl, "stop_sequence") ? 2u : 0u;
        if (!bit) continue;
        if (ds & bit) return 1;
        ds |= bit;
        if (!n_str_or_null(p, a)) return 1;
      }
    }
    if (u.out >= 0) { S.usage.output = (uint32_t)u.out; S.usage.mask |= 2u; }
    return 0;
  }
  return 0;
}
__device__ void step_anthropic_native(StreamSlot& S, const StreamStep& st, uint8_t* out, aigw_chunk_result& R) {
  const uint8_t* b = S.buf; const uint32_t n = S.end;
  uint32_t pos = 0; int status = 0;
  for (;;) {
    uint32_t nl = pos; while (nl < n && b[nl] != '\n') nl++;
    if (nl >= n) break;
    const uint8_t* line = b + pos; const uint32_t ll = nl - pos;
    pos = nl + 1;
    if (!prefix(line, ll, "data: ", 6)) continue;
    if (native_event(S, line + 6, (int)ll - 6)) { status = AIGW_DECLINED; break; }
  }
  const char* m = S.rmodel_len ? S.rmodel : S.model; const uint32_t ml = S.rmodel_len ? S.rmodel_len : S.model_len;
  int reason = AIGW_R_UNSUPPORTED_FIELD;
  if (!status && ml > st.out_cap) { status = AIGW_DECLINED; reason = AIGW_R_OUT_SPACE; }
  if (status) { S.flags |= SF_DEAD; S.dead_status = (uint32_t)status; S.dead_reason = (uint32_t)reason; R.status = (uint8_t)status; R.reason = (uint8_t)reason; return; }
  {  // updateTotalTokens
    aigw_usage& u = S.usage;
    const bool out_set = u.mask & 2u;
    if (out_set && !(u.mask & 1u)) { u.input = 0; u.mask |= 1u; }
    if (out_set) { if (!(u.mask & 8u)) { u.cached = 0; u.mask |= 8u; } if (!(u.mask & 16u)) { u.cache_creation = 0; u.mask |= 16u; } }
    if ((u.mask & 1u) && out_set) { u.total = u.input + u.output; u.mask |= 4u; }
  }
  S.beg = pos;
  R.usage = S.usage; R.body_kind = AIGW_BODY_UNCHANGED; R.out_len = 0;
  for (uint32_t k = 0; k < ml; k++) out[k] = (uint8_t)m[k];
  R.model_len = ml;
}

// ------------------------------------------------------------------ S1 variant: /v1/responses, usage scan only
// (openAIToOpenAITranslatorV1Responses.ResponseBody stream branch: handleStreamingResponse + extractUsageFromBufferEvent,
//  internal/translator/openai_responses.go:102-114,146-192).  The reference keeps NO carry: every call splits only its own bytes into
//  lines (a line cut across two calls is lost) and parses the last one even without a newline, so the step reads the call's bytes in
//  place from the staged input and the slot holds only the stream's model.  A line counts when it starts with "data: " and its
//  first top-level "type" is response.created (model) or response.completed (all six counters, cache creation 0, last one of the
//  call wins); other events change nothing and are not validated.  A response.completed without usage DECLINES (the reference
//  dereferences the nil *ResponseUsage).  It runs in its own kernel (stream_responses_kernel): the shared step kernel's code and frame
//  stay as they were.
__device__ void step_openai_responses(StreamSlot& S, const StreamStep& st, const uint8_t* b, uint8_t* out, aigw_chunk_result& R) {
  const uint32_t n = st.len;
  aigw_usage u; memset(&u, 0, sizeof u);
  int status = 0;
  for (uint32_t pos = 0; pos < n && !status;) {
    uint32_t nl = pos; while (nl < n && b[nl] != '\n') nl++;
    const uint8_t* line = b + pos; const uint32_t ll = nl - pos;
    pos = nl + 1;
    if (!prefix(line, ll, "data: ", 6)) continue;
    const uint8_t* d = line + 6; const int dl = (int)ll - 6;
    const int r0 = skipws(d, 0, dl);
    if (r0 >= dl || d[r0] != '{') continue;   // empty data, [DONE], or no "type" to find
    int ts = 0, tl = 0; const int r = union_tag(d, r0, dl, ts, tl);
    if (r == -2) { status = AIGW_DECLINED; break; }
    if (r <= 0) continue;
    const bool created = EQ(d + ts, (uint32_t)tl, "response.created");
    if (!created && !EQ(d + ts, (uint32_t)tl, "response.completed")) continue;
    Capture cp; cap_reset(cp);
    const bool ok = walk<Capture, true>(d, dl, g_rsp_schema.nodes, g_rsp_schema.fields, g_rsp_schema.keys, X_EVENT, cp);
    if (cp.weird || (cp.span_esc & 1u)) { status = AIGW_DECLINED; break; }
    if (!ok) continue;   // a decode error skips the line
    if (created) {
      if ((cp.span_set & 1u) && cp.span_len[0] > 0) {
        if (cp.span_len[0] > sizeof S.rmodel) { status = AIGW_DECLINED; break; }
        for (uint32_t k = 0; k < cp.span_len[0]; k++) S.rmodel[k] = (char)d[cp.span_off[0] + k];
        S.rmodel_len = cp.span_len[0];
      }
    } else {
      if (!(cp.obj_seen & (1u << C_OBJ_RESPONSE)) || !(cp.obj_seen & (1u << C_OBJ_USAGE))) { status = AIGW_DECLINED; break; }
      u.input = cp.ints[C_PROMPT]; u.output = cp.ints[C_COMPLETION]; u.total = cp.ints[C_TOTAL];
      u.cached = cp.ints[C_CACHED]; u.cache_creation = 0; u.reasoning = cp.ints[C_REASONING]; u.mask = 63u;
    }
  }
  // responseModel = cmp.Or(streamingResponseModel, requestModel)
  const char* m = S.rmodel_len ? S.rmodel : S.model; const uint32_t ml = S.rmodel_len ? S.rmodel_len : S.model_len;
  int reason = AIGW_R_UNSUPPORTED_FIELD;
  if (!status && ml > st.out_cap) { status = AIGW_DECLINED; reason = AIGW_R_OUT_SPACE; }
  if (status) { S.flags |= SF_DEAD; S.dead_status = (uint32_t)status; S.dead_reason = (uint32_t)reason; R.status = (uint8_t)status; R.reason = (uint8_t)reason; return; }
  R.usage = u; R.body_kind = AIGW_BODY_UNCHANGED; R.out_len = 0;
  for (uint32_t k = 0; k < ml; k++) out[k] = (uint8_t)m[k];
  R.model_len = ml;
}

#include "stream_messages_openai.cuh"
#include "stream_messages_aws_anthropic.cuh"

#ifndef AIGW_HOST_HARNESS
// ------------------------------------------------------------------ kernels
__global__ void __launch_bounds__(128) stream_init_kernel(StreamSlot* slots, const uint32_t* slot_ids, uint32_t n, const uint8_t* tmpl) {
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n) return;
  uint4* dst = (uint4*)&slots[slot_ids[warp]]; const uint4* src = (const uint4*)tmpl;
  for (uint32_t i = lane; i < kStreamHdrBytes / 16; i += 32) dst[i] = src[i];
}

__global__ void __launch_bounds__(128) stream_append_kernel(const __grid_constant__ StreamParams P) {
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= P.n) return;
  const StreamStep st = P.steps[warp];
  StreamSlot& S = P.slots[st.slot];
  if (S.flags & SF_DEAD) return;
  if (S.kind == AIGW_STREAM_OPENAI_RESPONSES) return;   // no carry: the step reads the call's bytes in place (beg = end = 0 stays)
  const uint32_t beg = S.beg, end = S.end, n = end - beg;
  if (lane == 0) S._r0 = n;   // carry length before this call (the Gemini step restates bufferedBody from it)
  if (beg) {   // move the carry to the front (reads of one batch complete before its writes; later batches read further right)
    for (uint32_t i0 = 0; i0 < n; i0 += 32) {
      const uint32_t i = i0 + lane;
      uint8_t c = 0; if (i < n) c = S.buf[beg + i];
      __syncwarp();
      if (i < n) S.buf[i] = c;
      __syncwarp();
    }
  }
  if (n + st.len > kStreamCarryCap) {
    if (lane == 0) { S.flags |= SF_DEAD; S.dead_status = AIGW_DECLINED; S.dead_reason = AIGW_R_TOO_LARGE; S.beg = 0; S.end = n; }
    return;
  }
  const uint8_t* src = P.in + st.in_off;
  for (uint32_t i = lane; i < st.len; i += 32) S.buf[n + i] = src[i];
  __syncwarp();
  if (lane == 0) { S.beg = 0; S.end = n + st.len; }
}

__global__ void __launch_bounds__(64) stream_step_kernel(const __grid_constant__ StreamParams P) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P.n) return;
  const StreamStep st = P.steps[i];
  StreamSlot& S = P.slots[st.slot];
  aigw_chunk_result R; memset(&R, 0, sizeof R);
  R.out_off = st.out_off;
  if (S.flags & SF_DEAD) { R.status = (uint8_t)S.dead_status; R.reason = (uint8_t)S.dead_reason; }
  else {
    uint8_t* out = P.out + st.out_off;
    switch (S.kind) {
      case AIGW_STREAM_OPENAI: step_openai(S, st, out, R); break;
      case AIGW_STREAM_AWS_BEDROCK: step_bedrock(S, st, out, R); break;
      case AIGW_STREAM_GCP_ANTHROPIC: step_anthropic(S, st, out, R); break;
      case AIGW_STREAM_GCP_GEMINI: step_gemini(S, st, out, R); break;
      case AIGW_STREAM_GCP_GEMINI_BUFFERED: step_gemini_buffered(S, st, out, R); break;
      case AIGW_STREAM_ANTHROPIC: step_anthropic_native(S, st, out, R); break;
      case AIGW_STREAM_AWS_ANTHROPIC: step_aws_anthropic(S, st, out, R); break;
      case AIGW_STREAM_OPENAI_COMPLETIONS: step_openai(S, st, out, R, true); break;
      case AIGW_STREAM_MESSAGES_OPENAI: step_messages_openai(S, st, out, R); break;
      case AIGW_STREAM_MESSAGES_OPENAI_BUFFERED: step_messages_openai_buffered(S, st, out, R); break;
      case AIGW_STREAM_MESSAGES_AWS_ANTHROPIC: step_messages_aws_anthropic(S, st, out, R); break;
      default: R.status = AIGW_DECLINED; R.reason = AIGW_R_SCHEMA; break;
    }
  }
  R.carry_len = S.end - S.beg;
  P.results[i] = R;
}

// /v1/responses steps: the shared step kernel leaves them DECLINED (a kind it does not know); this kernel runs after it and writes
// their results.  It reads the call's bytes in place: there is no carry.
__global__ void __launch_bounds__(64) stream_responses_kernel(const __grid_constant__ StreamParams P) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P.n) return;
  const StreamStep st = P.steps[i];
  StreamSlot& S = P.slots[st.slot];
  if (S.kind != AIGW_STREAM_OPENAI_RESPONSES) return;
  aigw_chunk_result R; memset(&R, 0, sizeof R);
  R.out_off = st.out_off;
  if (S.flags & SF_DEAD) { R.status = (uint8_t)S.dead_status; R.reason = (uint8_t)S.dead_reason; }
  else step_openai_responses(S, st, P.in + st.in_off, P.out + st.out_off, R);
  P.results[i] = R;   // carry_len 0
}

__global__ void __launch_bounds__(128) stream_pack_kernel(const __grid_constant__ StreamParams P) {
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= P.n) return;
  aigw_chunk_result& R = P.results[warp];
  const uint32_t len = R.out_len + R.model_len;
  if (len == 0) { if (lane == 0) R.out_off = 0; return; }
  unsigned long long o = 0;
  if (lane == 0) o = atomicAdd(P.packed_used, (unsigned long long)((len + 15u) & ~15u));
  o = __shfl_sync(0xffffffffu, o, 0);
  if (o + len > P.packed_cap) { if (lane == 0) { R.status = AIGW_DECLINED; R.reason = AIGW_R_ARENA_FULL; R.out_len = 0; R.model_len = 0; R.out_off = 0; } return; }
  const uint8_t* src = P.out + P.steps[warp].out_off; uint8_t* dst = P.packed + o;
  for (uint32_t i = lane; i < len; i += 32) dst[i] = src[i];
  if (lane == 0) R.out_off = o;
}

}  // namespace

cudaError_t launch_stream_init(StreamSlot* slots, const uint32_t* slot_ids, uint32_t n, const uint8_t* tmpl, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  stream_init_kernel<<<(n * 32 + 127) / 128, 128, 0, st>>>(slots, slot_ids, n, tmpl);
  return cudaGetLastError();
}

cudaError_t launch_stream_steps(const StreamParams& P, cudaStream_t st) {
  static DeviceOnce once;
  {
    const cudaError_t e0 = device_once(once, nullptr, [&](int*) {
      SchemaBlob a = build_schema(); cudaError_t e = cudaMemcpyToSymbol(g_chunk_schema, &a, sizeof a); if (e != cudaSuccess) return e;
      a = build_completion_schema(); e = cudaMemcpyToSymbol(g_cmpl_schema, &a, sizeof a); if (e != cudaSuccess) return e;
      { RespSchemaBlob r = build_resp_schema(); e = cudaMemcpyToSymbol(g_o2a_resp_schema, &r, sizeof r); if (e != cudaSuccess) return e; }
      { RspSchemaBlob r = build_responses_schema(); e = cudaMemcpyToSymbol(g_rsp_schema, &r, sizeof r); if (e != cudaSuccess) return e; }
      BedrockSchema b = build_schema_bedrock(); e = cudaMemcpyToSymbol(g_conv_schema, &b, sizeof b); if (e != cudaSuccess) return e;
      AnSchema c = build_an_schema(); e = cudaMemcpyToSymbol(g_an_schema, &c, sizeof c); if (e != cudaSuccess) return e;
      uint32_t tab[256];
      for (uint32_t i = 0; i < 256; i++) { uint32_t v = i; for (int k = 0; k < 8; k++) v = (v & 1u) ? 0xEDB88320u ^ (v >> 1) : v >> 1; tab[i] = v; }
      return cudaMemcpyToSymbol(g_crc_tab, tab, sizeof tab);
    });
    if (e0 != cudaSuccess) return e0;
  }
  if (P.n == 0) return cudaSuccess;
  stream_append_kernel<<<(P.n * 32 + 127) / 128, 128, 0, st>>>(P);
  stream_step_kernel<<<(P.n + 63) / 64, 64, 0, st>>>(P);
  stream_responses_kernel<<<(P.n + 63) / 64, 64, 0, st>>>(P);
  stream_pack_kernel<<<(P.n * 32 + 127) / 128, 128, 0, st>>>(P);
  return cudaGetLastError();
}
#else   // the CPU-side parser harness (tools/stream_host_check.cpp) compiles only the per-thread step functions above
}  // namespace
#endif  // AIGW_HOST_HARNESS

}  // namespace aigw
