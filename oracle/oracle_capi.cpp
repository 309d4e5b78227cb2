// ORACLE — TEST INFRASTRUCTURE ONLY (see ojson.hpp header).
// C entry points so tests/, smoke() and bench.py's cpu_baseline / --impl reference legs can
// drive the restatement through ctypes.  Built by oracle/Makefile into oracle/liboracle.so.
#include <malloc.h>

#include <atomic>
#include <chrono>
#include <thread>

#include "bedrock_response.hpp"
#include "bedrock_stream.hpp"
#include "anthropic_stream.hpp"
#include "anthropic_native.hpp"
#include "aws_anthropic_stream.hpp"
#include "gemini.hpp"
#include "gemini_stream.hpp"
namespace oracle { TranslateResult gemini_request_body(const ChatReq& r, const std::string& model_override) { return gemini::request_body(r, model_override); } }
#include "bpe.hpp"
#include "cel.hpp"
#include "sha256.hpp"
#include "embeddings.hpp"
#include "mutate.hpp"
#include "response_error.hpp"
#include "messages.hpp"
#include "messages_translated.hpp"
#include "stream.hpp"
#include "completions.hpp"
#include "messages_openai_response.hpp"
#include "messages_aws_anthropic_stream.hpp"
#include "translate.hpp"

using namespace oracle;

// The batch helpers run one worker per host thread.  glibc's defaults return freed memory to the kernel and map large blocks
// eagerly, which serialises 128 workers on the process's mm lock (the rate then varies widely from run to run);
// keeping freed memory in the arenas makes the CPU baseline both faster and repeatable — closer to Go's per-P allocator caches.
__attribute__((constructor)) static void oracle_tune_allocator() {
  if (getenv("ORACLE_NO_MALLOPT")) return;
  mallopt(M_MMAP_THRESHOLD, 1 << 30); mallopt(M_TRIM_THRESHOLD, 1 << 30);
}

extern "C" {

struct oracle_result {
  int32_t status;      // oracle::Status
  int32_t body_kind;   // oracle::BodyKind
  int32_t stream;
  int32_t has_mutated;
  uint64_t body_len, path_len, model_len, err_len, mutated_len;
  char* body; char* path; char* model; char* err; char* mutated;
};

static char* dup(const std::string& s) { char* p = (char*)malloc(s.size() + 1); memcpy(p, s.data(), s.size()); p[s.size()] = 0; return p; }

void oracle_chat_translate(int schema, const char* body, uint64_t len, const char* model_override, const char* prefix,
                           int cost_configured, int force, oracle_result* out) {
  TranslateResult r = chat_translate(schema, std::string_view(body, len), model_override ? model_override : "", prefix ? prefix : "", cost_configured != 0, force != 0);
  memset(out, 0, sizeof *out);
  out->status = r.err.status; out->body_kind = r.body_kind; out->stream = r.stream; out->has_mutated = r.has_mutated;
  std::string path; for (auto& h : r.headers) if (h.name == ":path") path = h.value;
  out->body = dup(r.body); out->body_len = r.body.size();
  out->path = dup(path); out->path_len = path.size();
  out->model = dup(r.model); out->model_len = r.model.size();
  out->err = dup(r.err.msg); out->err_len = r.err.msg.size();
  out->mutated = dup(r.mutated_body); out->mutated_len = r.mutated_body.size();
}
void oracle_embeddings_translate(int schema, const char* body, uint64_t len, const char* model_override, const char* prefix, int force, oracle_result* out) {
  TranslateResult r = embeddings_translate(schema, std::string_view(body, len), model_override ? model_override : "", prefix ? prefix : "", force != 0);
  memset(out, 0, sizeof *out);
  out->status = r.err.status; out->body_kind = r.body_kind; out->stream = 0; out->has_mutated = 0;
  std::string path; for (auto& h : r.headers) if (h.name == ":path") path = h.value;
  out->body = dup(r.body); out->body_len = r.body.size();
  out->path = dup(path); out->path_len = path.size();
  out->model = dup(r.model); out->model_len = r.model.size();
  out->err = dup(r.err.msg); out->err_len = r.err.msg.size();
  out->mutated = dup(""); out->mutated_len = 0;
}
void oracle_messages_translate(int schema, const char* body, uint64_t len, const char* model_override, const char* api_version, int force, oracle_result* out) {
  // base 0 / 1 (OpenAI / AWS Bedrock): the full re-map (messages_translated.hpp); api_version then carries the OpenAI path prefix
  const int mbase = schema & 15;
  TranslateResult r = (mbase == SCHEMA_MSG_OPENAI || mbase == SCHEMA_MSG_AWS_BEDROCK)
                          ? messages_translate_full(schema, std::string_view(body, len), model_override ? model_override : "", api_version ? api_version : "")
                          : messages_translate(schema, std::string_view(body, len), model_override ? model_override : "", api_version ? api_version : "", force != 0);
  memset(out, 0, sizeof *out);
  out->status = r.err.status; out->body_kind = r.body_kind; out->stream = r.stream ? 1 : 0; out->has_mutated = 0;
  std::string path; for (auto& h : r.headers) if (h.name == ":path") path = h.value;
  out->body = dup(r.body); out->body_len = r.body.size();
  out->path = dup(path); out->path_len = path.size();
  out->model = dup(r.model); out->model_len = r.model.size();
  out->err = dup(r.err.msg); out->err_len = r.err.msg.size();
  out->mutated = dup(""); out->mutated_len = 0;
}
void oracle_result_free(oracle_result* r) { free(r->body); free(r->path); free(r->model); free(r->err); free(r->mutated); memset(r, 0, sizeof *r); }

// Batch form used for CPU-baseline timing: translate n bodies with `threads` workers, return
// total output bytes and per-body status/len (no output retention).  Seconds of wall time returned.
double oracle_chat_translate_batch(int schema, const uint8_t* bodies, const uint64_t* offsets, uint32_t n, int cost_configured,
                                   int threads, int32_t* status, uint32_t* out_len, uint64_t* total_out) {
  std::atomic<uint32_t> next{0}; std::atomic<uint64_t> tot{0};
  auto t0 = std::chrono::steady_clock::now();
  auto work = [&] {
    for (;;) {
      uint32_t i = next.fetch_add(64);
      if (i >= n) break;
      uint32_t e = std::min(n, i + 64); uint64_t loc = 0;
      for (; i < e; i++) {
        TranslateResult r = chat_translate(schema, std::string_view((const char*)bodies + offsets[i], offsets[i + 1] - offsets[i]), "", "", cost_configured != 0, false);
        if (status) status[i] = r.err.status;
        if (out_len) out_len[i] = (uint32_t)r.body.size();
        loc += r.body.size();
      }
      tot += loc;
    }
  };
  if (threads <= 1) work();
  else { std::vector<std::thread> th; for (int t = 0; t < threads; t++) th.emplace_back(work); for (auto& t : th) t.join(); }
  if (total_out) *total_out = tot.load();
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

// ---- S1: streaming usage scan
struct oracle_usage { uint32_t input, output, total, cached, cache_creation, reasoning, mask; };
static void put(oracle_usage* o, const TokenUsage& u) { o->input = u.input; o->output = u.output; o->total = u.total; o->cached = u.cached; o->cache_creation = u.cache_creation; o->reasoning = u.reasoning; o->mask = u.mask; }

void* oracle_sse_open() { return new SSEOpenAIState(); }
void oracle_sse_close(void* h) { delete (SSEOpenAIState*)h; }
// feeds one chunk; `call` = usage returned by this ResponseBody call
void oracle_sse_feed(void* h, const char* chunk, uint64_t len, oracle_usage* call) {
  auto* st = (SSEOpenAIState*)h; TokenUsage u = sse_openai_feed(*st, std::string_view(chunk, len)); put(call, u);
}
uint64_t oracle_sse_model(void* h, char* buf, uint64_t cap) {
  auto* st = (SSEOpenAIState*)h; uint64_t n = std::min<uint64_t>(cap, st->streaming_model.size()); memcpy(buf, st->streaming_model.data(), n); return st->streaming_model.size();
}
uint64_t oracle_sse_buffered(void* h) { return ((SSEOpenAIState*)h)->buffered.size(); }

// Whole-stream helper for batch timing/parity: stream s = chunks [chunk_off[s], chunk_off[s+1]) of the
// chunk table (byte offsets chunk_byte_off[c]..chunk_byte_off[c+1]); result = Override-accumulated usage.
double oracle_sse_batch(const uint8_t* bytes, const uint64_t* chunk_byte_off, const uint32_t* chunk_off, uint32_t n_streams, int threads, oracle_usage* out) {
  std::atomic<uint32_t> next{0};
  auto t0 = std::chrono::steady_clock::now();
  auto work = [&] {
    for (;;) {
      uint32_t s = next.fetch_add(16); if (s >= n_streams) break;
      uint32_t e = std::min(n_streams, s + 16);
      for (; s < e; s++) {
        SSEOpenAIState st; TokenUsage acc;
        for (uint32_t c = chunk_off[s]; c < chunk_off[s + 1]; c++) {
          TokenUsage u = sse_openai_feed(st, std::string_view((const char*)bytes + chunk_byte_off[c], chunk_byte_off[c + 1] - chunk_byte_off[c]));
          acc.override_with(u);
        }
        put(&out[s], acc);
      }
    }
  };
  if (threads <= 1) work();
  else { std::vector<std::thread> th; for (int t = 0; t < threads; t++) th.emplace_back(work); for (auto& t : th) t.join(); }
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

int oracle_response_openai(const char* body, uint64_t len, const char* request_model, oracle_usage* out, char* model_buf, uint64_t cap, uint64_t* model_len) {
  TokenUsage tu; std::string rm;
  bool ok = response_openai(std::string_view(body, len), request_model ? request_model : "", tu, rm);
  put(out, tu); uint64_t n = std::min<uint64_t>(cap, rm.size()); memcpy(model_buf, rm.data(), n); *model_len = rm.size();
  return ok ? 0 : 1;
}
int oracle_response_embeddings(const char* body, uint64_t len, oracle_usage* out, char* model_buf, uint64_t cap, uint64_t* model_len) {
  TokenUsage tu; std::string rm;
  bool ok = response_embeddings(std::string_view(body, len), tu, rm);
  put(out, tu); uint64_t n = std::min<uint64_t>(cap, rm.size()); memcpy(model_buf, rm.data(), n); *model_len = rm.size();
  return ok ? 0 : 1;
}
// ---- /v1/completions: stream usage scan (one ResponseBody call per feed) and the buffered branch
void* oracle_completions_sse_open() { return new SSECompletionsState(); }
void oracle_completions_sse_close(void* h) { delete (SSECompletionsState*)h; }
void oracle_completions_sse_feed(void* h, const char* chunk, uint64_t len, oracle_usage* call) {
  auto* st = (SSECompletionsState*)h; TokenUsage u = sse_completions_feed(*st, std::string_view(chunk, len)); put(call, u);
}
uint64_t oracle_completions_sse_model(void* h, char* buf, uint64_t cap) {
  auto* st = (SSECompletionsState*)h; uint64_t n = std::min<uint64_t>(cap, st->streaming_model.size()); memcpy(buf, st->streaming_model.data(), n); return st->streaming_model.size();
}
uint64_t oracle_completions_sse_buffered(void* h) { return ((SSECompletionsState*)h)->buffered.size(); }
int oracle_response_completions(const char* body, uint64_t len, oracle_usage* out, char* model_buf, uint64_t cap, uint64_t* model_len) {
  TokenUsage tu; std::string rm;
  bool ok = response_completions(std::string_view(body, len), tu, rm);
  put(out, tu); uint64_t n = std::min<uint64_t>(cap, rm.size()); memcpy(model_buf, rm.data(), n); *model_len = rm.size();
  return ok ? 0 : 1;
}
// ---- T5 response direction, OpenAI backend: OpenAI SSE -> Anthropic SSE (one ResponseBody call per feed) and the buffered form
struct o2a_handle { OpenAIToAnthropicStream st; std::string model; };
void* oracle_messages_openai_stream_open(const char* request_model) { auto* h = new o2a_handle(); h->st.request_model = request_model ? request_model : ""; return h; }
void oracle_messages_openai_stream_close(void* h) { delete (o2a_handle*)h; }
// returns malloc'd output (free with oracle_free)
char* oracle_messages_openai_stream_feed(void* hv, const char* chunk, uint64_t len, int eos, uint64_t* out_len, oracle_usage* usage, int* status) {
  auto* h = (o2a_handle*)hv; std::string o; TokenUsage u;
  const Status s = messages_openai_stream_feed(h->st, std::string_view(chunk, len), eos != 0, o, u, h->model);
  put(usage, u); *status = (int)s; *out_len = o.size();
  char* r = (char*)malloc(o.size() + 1); memcpy(r, o.data(), o.size()); r[o.size()] = 0; return r;
}
uint64_t oracle_messages_openai_stream_model(void* hv, char* buf, uint64_t cap) { auto* h = (o2a_handle*)hv; uint64_t n = std::min<uint64_t>(cap, h->model.size()); memcpy(buf, h->model.data(), n); return h->model.size(); }
uint64_t oracle_messages_openai_stream_buffered(void* hv) { return ((o2a_handle*)hv)->st.buffer.size(); }
char* oracle_messages_openai_response(const char* body, uint64_t len, const char* request_model, uint64_t* out_len, oracle_usage* usage, char* model_buf, uint64_t cap, uint64_t* model_len, int* ok) {
  std::string o, rm; TokenUsage u;
  *ok = messages_openai_response(std::string_view(body, len), request_model ? request_model : "", o, u, rm) ? 1 : 0;
  put(usage, u); uint64_t n = std::min<uint64_t>(cap, rm.size()); memcpy(model_buf, rm.data(), n); *model_len = rm.size(); *out_len = o.size();
  char* r = (char*)malloc(o.size() + 1); memcpy(r, o.data(), o.size()); r[o.size()] = 0; return r;
}
// ---- T5: /v1/messages on Anthropic behind AWS Bedrock, stream (eventstream-wrapped chunks -> Anthropic SSE)
struct maa_handle { MessagesAwsAnthropicStream st; std::string model; };
void* oracle_messages_aws_anthropic_open(const char* request_model) { auto* h = new maa_handle(); h->st.nat.request_model = request_model ? request_model : ""; return h; }
void oracle_messages_aws_anthropic_close(void* h) { delete (maa_handle*)h; }
char* oracle_messages_aws_anthropic_feed(void* hv, const char* chunk, uint64_t len, int eos, uint64_t* out_len, oracle_usage* usage, int* status) {
  auto* h = (maa_handle*)hv; std::string o; TokenUsage u;
  const Status s = messages_aws_anthropic_stream_feed(h->st, std::string_view(chunk, len), eos != 0, o, u, h->model);
  put(usage, u); *status = (int)s; *out_len = o.size();
  char* r = (char*)malloc(o.size() + 1); memcpy(r, o.data(), o.size()); r[o.size()] = 0; return r;
}
uint64_t oracle_messages_aws_anthropic_model(void* hv, char* buf, uint64_t cap) { auto* h = (maa_handle*)hv; uint64_t n = std::min<uint64_t>(cap, h->model.size()); memcpy(buf, h->model.data(), n); return h->model.size(); }
uint64_t oracle_messages_aws_anthropic_buffered(void* hv) { return ((maa_handle*)hv)->st.buffered.size(); }
uint64_t oracle_eval_cost(int type, const oracle_usage* u) { TokenUsage t; t.input = u->input; t.output = u->output; t.total = u->total; t.cached = u->cached; t.cache_creation = u->cache_creation; t.reasoning = u->reasoning; t.mask = u->mask; return eval_cost(type, t); }

// ---- S2: Bedrock eventstream → OpenAI SSE.  Replays ResponseBody over the given chunking; returns malloc'd output.
char* oracle_bedrock_stream(const uint8_t* bytes, const uint64_t* chunk_off, uint32_t n_chunks, const char* request_model, const char* response_id,
                            int64_t created, uint64_t* out_len, oracle_usage* usage) {
  BedrockStreamState st; BedrockStreamCfg cfg; cfg.request_model = request_model ? request_model : ""; cfg.response_id = response_id ? response_id : ""; cfg.created = created;
  std::string out; TokenUsage acc;
  for (uint32_t c = 0; c < n_chunks; c++) {
    TokenUsage u;
    bedrock_stream_feed(st, cfg, std::string_view((const char*)bytes + chunk_off[c], chunk_off[c + 1] - chunk_off[c]), c + 1 == n_chunks, out, u);
    acc.override_with(u);
  }
  if (n_chunks == 0) out += "data: [DONE]\n";
  put(usage, acc); *out_len = out.size();
  return dup(out);
}
double oracle_bedrock_stream_batch(const uint8_t* bytes, const uint64_t* stream_off, uint32_t n_streams, const char* request_model, const char* response_id, int64_t created,
                                   int threads, uint64_t* total_out) {
  std::atomic<uint32_t> next{0}; std::atomic<uint64_t> tot{0};
  auto t0 = std::chrono::steady_clock::now();
  auto work = [&] {
    for (;;) {
      uint32_t s = next.fetch_add(16); if (s >= n_streams) break;
      uint32_t e = std::min(n_streams, s + 16);
      for (; s < e; s++) {
        BedrockStreamState st; BedrockStreamCfg cfg; cfg.request_model = request_model; cfg.response_id = response_id; cfg.created = created;
        std::string out; TokenUsage u;
        bedrock_stream_feed(st, cfg, std::string_view((const char*)bytes + stream_off[s], stream_off[s + 1] - stream_off[s]), true, out, u);
        tot += out.size();
      }
    }
  };
  if (threads <= 1) work(); else { std::vector<std::thread> th; for (int t = 0; t < threads; t++) th.emplace_back(work); for (auto& t : th) t.join(); }
  if (total_out) *total_out = tot.load();
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}
// ---- R1 (Bedrock): buffered Converse response → OpenAI ChatCompletionResponse.  Returns oracle::Status; *out is malloc'd.
int oracle_bedrock_response(const char* body, uint64_t len, const char* request_model, const char* response_id, int64_t created, char** out, uint64_t* out_len, oracle_usage* usage) {
  BedrockStreamCfg cfg; cfg.request_model = request_model ? request_model : ""; cfg.response_id = response_id ? response_id : ""; cfg.created = created;
  std::string o; TokenUsage u; const Status st = bedrock_response(std::string_view(body, len), cfg, o, u);
  put(usage, u); *out = dup(o); *out_len = o.size();
  return (int)st;
}
int oracle_bedrock_response_anthropic(const char* body, uint64_t len, const char* request_model, const char* response_id, char** out, uint64_t* out_len, oracle_usage* usage) {
  BedrockStreamCfg cfg; cfg.request_model = request_model ? request_model : ""; cfg.response_id = response_id ? response_id : ""; cfg.created = 0;
  std::string o; TokenUsage u; const Status st = bedrock_response(std::string_view(body, len), cfg, o, u, true);
  put(usage, u); *out = dup(o); *out_len = o.size();
  return (int)st;
}
double oracle_bedrock_response_batch(const uint8_t* bodies, const uint64_t* offsets, uint32_t n, int threads, uint64_t* total_out) {
  std::atomic<uint32_t> next{0}; std::atomic<uint64_t> tot{0};
  auto t0 = std::chrono::steady_clock::now();
  auto work = [&] {
    BedrockStreamCfg cfg; cfg.request_model = "m"; cfg.response_id = "r"; cfg.created = 7;
    for (;;) {
      uint32_t i = next.fetch_add(64); if (i >= n) break;
      uint32_t e = std::min(n, i + 64); uint64_t loc = 0;
      for (; i < e; i++) { std::string o; TokenUsage u; bedrock_response(std::string_view((const char*)bodies + offsets[i], offsets[i + 1] - offsets[i]), cfg, o, u); loc += o.size(); }
      tot += loc;
    }
  };
  if (threads <= 1) work(); else { std::vector<std::thread> th; for (int t = 0; t < threads; t++) th.emplace_back(work); for (auto& t : th) t.join(); }
  if (total_out) *total_out = tot.load();
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}
// stateful form of the Bedrock stream oracle: one ResponseBody call per feed
struct BedrockHandle { BedrockStreamState st; BedrockStreamCfg cfg; };
void* oracle_bedrock_open(const char* request_model, const char* response_id, int64_t created) { auto* h = new BedrockHandle(); h->cfg.request_model = request_model ? request_model : ""; h->cfg.response_id = response_id ? response_id : ""; h->cfg.created = created; return h; }
void oracle_bedrock_close(void* h) { delete (BedrockHandle*)h; }
void oracle_bedrock_feed(void* hv, const char* chunk, uint64_t len, int eos, char** out, uint64_t* out_len, oracle_usage* usage) {
  auto* h = (BedrockHandle*)hv; std::string o; TokenUsage u;
  bedrock_stream_feed(h->st, h->cfg, std::string_view(chunk, len), eos != 0, o, u);
  put(usage, u); *out = dup(o); *out_len = o.size();
}
// ---- S3 / R1 (Anthropic): SSE events → OpenAI SSE, per ResponseBody call; buffered Message → ChatCompletionResponse
struct AnthropicHandle { AnthropicStreamState st; AnthropicStreamCfg cfg; };
void* oracle_anthropic_open(const char* request_model, int64_t created) { auto* h = new AnthropicHandle(); h->cfg.request_model = request_model ? request_model : ""; h->cfg.created = created; return h; }
void oracle_anthropic_close(void* h) { delete (AnthropicHandle*)h; }
// returns oracle::Status of this call; *out (malloc'd) = the body mutation of this call; usage = the TokenUsage the call returns
int oracle_anthropic_feed(void* hv, const char* chunk, uint64_t len, int eos, char** out, uint64_t* out_len, oracle_usage* usage) {
  auto* h = (AnthropicHandle*)hv; std::string o; TokenUsage u;
  const Status s = anthropic_stream_feed(h->st, h->cfg, std::string_view(chunk, len), eos != 0, o, u);
  if (s != OK) o.clear();
  put(usage, u); *out = dup(o); *out_len = o.size();
  return (int)s;
}
int oracle_anthropic_response(const char* body, uint64_t len, const char* request_model, int64_t created, char** out, uint64_t* out_len, oracle_usage* usage, char* model_buf, uint64_t cap, uint64_t* model_len) {
  AnthropicStreamCfg cfg; cfg.request_model = request_model ? request_model : ""; cfg.created = created;
  std::string o, rm; TokenUsage u; const Status s = anthropic_response(std::string_view(body, len), cfg, o, u, rm);
  put(usage, u); *out = dup(o); *out_len = o.size();
  uint64_t n = std::min<uint64_t>(cap, rm.size()); memcpy(model_buf, rm.data(), n); *model_len = rm.size();
  return (int)s;
}
// ---- Translator.ResponseError
int oracle_response_error(int kind, const char* body, uint64_t len, const char* status_code, const char* aws_error_type, int json_content_type, char** out, uint64_t* out_len) {
  std::string o; const Status s = response_error(kind, std::string_view(body, len), status_code ? status_code : "", aws_error_type ? aws_error_type : "", json_content_type != 0, o);
  *out = dup(o); *out_len = o.size();
  return (int)s;
}
// ---- K4: byte-level BPE token count (self-oracle)
void* oracle_bpe_load(const uint16_t* byte_to_id, const uint32_t* merges, uint32_t n) { auto* v = new BpeVocab(); bpe_load(*v, byte_to_id, merges, n); return v; }
void oracle_bpe_free(void* v) { delete (BpeVocab*)v; }
// counts[i] = tokens of text i; returns the seconds the count took with `threads` workers
double oracle_bpe_count_batch(void* vv, const char* text, const uint64_t* off, const uint32_t* len, uint64_t n, int threads, uint32_t* counts) {
  const BpeVocab& V = *(const BpeVocab*)vv;
  if (threads < 1) threads = 1;
  const auto t0 = std::chrono::steady_clock::now();
  std::atomic<uint64_t> next{0};
  auto work = [&]() { for (;;) { const uint64_t b = next.fetch_add(256); if (b >= n) break; const uint64_t e = std::min<uint64_t>(n, b + 256); for (uint64_t i = b; i < e; i++) counts[i] = bpe_count(V, std::string_view(text + off[i], len[i])); } };
  std::vector<std::thread> th; for (int t = 1; t < threads; t++) th.emplace_back(work);
  work(); for (auto& x : th) x.join();
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}
// BASELINE config 3 on the CPU: per request EmbeddingsEndpointSpec.ParseBody (decode of the whole body) + the BPE count of every string input.
// tokens[i] = sum over request i's inputs, 0xFFFFFFFF when ParseBody fails or the input is not a list of strings; returns the seconds taken.
double oracle_embeddings_count_batch(void* vv, const char* bodies, const uint64_t* off, const uint32_t* len, uint64_t n, int threads, uint32_t* tokens, uint32_t* n_inputs) {
  const BpeVocab& V = *(const BpeVocab*)vv;
  if (threads < 1) threads = 1;
  const auto t0 = std::chrono::steady_clock::now();
  std::atomic<uint64_t> next{0};
  auto work = [&]() {
    for (;;) {
      const uint64_t i = next.fetch_add(1); if (i >= n) break;
      tokens[i] = 0xffffffffu; if (n_inputs) n_inputs[i] = 0;
      Value root; std::string perr;
      if (!oj::parse(std::string_view(bodies + off[i], len[i]), root, perr)) continue;
      EmbReq r; if (parse_embedding_request(root, r)) continue;
      uint32_t sum = 0;
      if (r.kind == EmbReq::STR) { sum = bpe_count(V, r.str); if (n_inputs) n_inputs[i] = 1; }
      else if (r.kind == EmbReq::STRS) { for (auto& t : r.strs) sum += bpe_count(V, t); if (n_inputs) n_inputs[i] = (uint32_t)r.strs.size(); }
      else if (r.kind != EmbReq::NONE) continue;
      tokens[i] = sum;
    }
  };
  std::vector<std::thread> th; for (int t = 1; t < threads; t++) th.emplace_back(work);
  work(); for (auto& x : th) x.join();
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}
// ---- S3 behind AWS (eventstream-wrapped Anthropic events)
struct AwsAnthropicHandle { AwsAnthropicStreamState st; AnthropicStreamCfg cfg; };
void* oracle_aws_anthropic_open(const char* request_model, int64_t created) { auto* h = new AwsAnthropicHandle(); h->cfg.request_model = request_model ? request_model : ""; h->cfg.created = created; return h; }
void oracle_aws_anthropic_close(void* h) { delete (AwsAnthropicHandle*)h; }
int oracle_aws_anthropic_feed(void* hv, const char* chunk, uint64_t len, int eos, char** out, uint64_t* out_len, oracle_usage* usage) {
  auto* h = (AwsAnthropicHandle*)hv; std::string o; TokenUsage u;
  const Status s = aws_anthropic_stream_feed(h->st, h->cfg, std::string_view(chunk, len), eos != 0, o, u);
  if (s != OK) o.clear();
  put(usage, u); *out = dup(o); *out_len = o.size();
  return (int)s;
}
// ---- native /v1/messages responses (usage scan, nothing rewritten)
void* oracle_native_anthropic_open(const char* request_model) { auto* h = new NativeAnthropicStream(); h->request_model = request_model ? request_model : ""; return h; }
void oracle_native_anthropic_close(void* h) { delete (NativeAnthropicStream*)h; }
int oracle_native_anthropic_feed(void* hv, const char* chunk, uint64_t len, oracle_usage* usage, char* model_buf, uint64_t cap, uint64_t* model_len) {
  auto* h = (NativeAnthropicStream*)hv; TokenUsage u; std::string m;
  const Status s = native_anthropic_feed(*h, std::string_view(chunk, len), u, m);
  put(usage, u); uint64_t n = std::min<uint64_t>(cap, m.size()); memcpy(model_buf, m.data(), n); *model_len = m.size();
  return (int)s;
}
int oracle_native_anthropic_response(const char* body, uint64_t len, const char* request_model, oracle_usage* usage, char* model_buf, uint64_t cap, uint64_t* model_len) {
  TokenUsage u; std::string m;
  const Status s = native_anthropic_response(std::string_view(body, len), request_model ? request_model : "", u, m);
  put(usage, u); uint64_t n = std::min<uint64_t>(cap, m.size()); memcpy(model_buf, m.data(), n); *model_len = m.size();
  return (int)s;
}
// ---- S4 / R1 (Gemini)
struct GeminiHandle { GeminiStreamState st; GeminiCfg cfg; };
void* oracle_gemini_open(const char* request_model) { auto* h = new GeminiHandle(); h->cfg.request_model = request_model ? request_model : ""; return h; }
void oracle_gemini_close(void* h) { delete (GeminiHandle*)h; }
int oracle_gemini_feed(void* hv, const char* chunk, uint64_t len, int eos, char** out, uint64_t* out_len, oracle_usage* usage, uint64_t* buffered) {
  auto* h = (GeminiHandle*)hv; std::string o; TokenUsage u;
  const Status s = gemini_stream_feed(h->st, h->cfg, std::string_view(chunk, len), eos != 0, o, u);
  if (s != OK) o.clear();
  put(usage, u); *out = dup(o); *out_len = o.size(); if (buffered) *buffered = h->st.buffered.size();
  return (int)s;
}
int oracle_gemini_response(const char* body, uint64_t len, const char* request_model, char** out, uint64_t* out_len, oracle_usage* usage, char* model_buf, uint64_t cap, uint64_t* model_len) {
  GeminiCfg cfg; cfg.request_model = request_model ? request_model : "";
  std::string o, rm; TokenUsage u; const Status s = gemini_response(std::string_view(body, len), cfg, o, u, rm);
  put(usage, u); *out = dup(o); *out_len = o.size();
  uint64_t n = std::min<uint64_t>(cap, rm.size()); memcpy(model_buf, rm.data(), n); *model_len = rm.size();
  return (int)s;
}
// ---- B1: body mutation.  removes: n_rm NUL-terminated strings; sets: n_set (path, value) pairs.  Returns 0, or 1 = not restated.
int oracle_body_mutate(const char* body, uint64_t len, const char* const* removes, uint32_t n_rm, const char* const* set_paths, const char* const* set_values, uint32_t n_set,
                       char** out, uint64_t* out_len) {
  std::vector<std::string> rm; for (uint32_t i = 0; i < n_rm; i++) rm.emplace_back(removes[i]);
  std::vector<BodySet> st; for (uint32_t i = 0; i < n_set; i++) st.push_back({set_paths[i], set_values[i]});
  std::string o; const int rc = body_mutate(std::string_view(body, len), rm, st, o);
  *out = dup(o); *out_len = o.size();
  return rc;
}
double oracle_body_mutate_batch(const uint8_t* bodies, const uint64_t* offsets, uint32_t n, const char* const* removes, uint32_t n_rm, const char* const* set_paths,
                                const char* const* set_values, uint32_t n_set, int threads, uint64_t* total_out) {
  std::vector<std::string> rm; for (uint32_t i = 0; i < n_rm; i++) rm.emplace_back(removes[i]);
  std::vector<BodySet> st; for (uint32_t i = 0; i < n_set; i++) st.push_back({set_paths[i], set_values[i]});
  std::atomic<uint32_t> next{0}; std::atomic<uint64_t> tot{0};
  auto t0 = std::chrono::steady_clock::now();
  auto work = [&] {
    for (;;) {
      uint32_t i = next.fetch_add(64); if (i >= n) break;
      uint32_t e = std::min(n, i + 64); uint64_t loc = 0;
      for (; i < e; i++) { std::string o; body_mutate(std::string_view((const char*)bodies + offsets[i], offsets[i + 1] - offsets[i]), rm, st, o); loc += o.size(); }
      tot += loc;
    }
  };
  if (threads <= 1) work(); else { std::vector<std::thread> th; for (int t = 0; t < threads; t++) th.emplace_back(work); for (auto& t : th) t.join(); }
  if (total_out) *total_out = tot.load();
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}
// ---- SigV4 payload hash
void oracle_sha256(const uint8_t* p, uint64_t n, uint8_t* out32) { sha256(p, (size_t)n, out32); }
double oracle_sha256_batch(const uint8_t* bytes, const uint64_t* offsets, const uint32_t* lens, uint32_t n, int threads, uint8_t* digests) {
  std::atomic<uint32_t> next{0};
  auto t0 = std::chrono::steady_clock::now();
  auto work = [&] { for (;;) { uint32_t i = next.fetch_add(64); if (i >= n) break; uint32_t e = std::min(n, i + 64); for (; i < e; i++) sha256(bytes + offsets[i], lens[i], digests + 32ull * i); } };
  if (threads <= 1) work(); else { std::vector<std::thread> th; for (int t = 0; t < threads; t++) th.emplace_back(work); for (auto& t : th) t.join(); }
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}
// ---- CEL cost expressions.  compile: 0 ok / 1 unsupported or compile error / 2 rejected by the sanity evaluation
void* oracle_cel_compile(const char* expr, int* rc) { auto* p = new cel::Program(); std::string err; *rc = cel::compile(expr, *p, err); if (*rc) { delete p; return nullptr; } return p; }
void oracle_cel_free(void* p) { delete (cel::Program*)p; }
// evaluate: returns 0 and the cost, or the error class (1 integer overflow, 2 unsigned overflow, 3 divide by zero, 4 modulus by zero, 5 negative result)
int oracle_cel_eval(void* p, const char* model, const char* backend, const char* route, const uint32_t tok[6], uint64_t* out) {
  cel::Vars v; v.model = model; v.backend = backend; v.route = route; for (int k = 0; k < 6; k++) v.tok[k] = tok[k];
  *out = 0; return cel::evaluate(*(cel::Program*)p, v, *out);
}
void oracle_free(void* p) { free(p); }
uint32_t oracle_crc32(const uint8_t* p, uint64_t n) { return crc32_ieee(p, n); }

// float formatting probe for tests
uint64_t oracle_fmt_f64(double v, char* buf, uint64_t cap) { std::string s; oj::enc_f64(s, v); uint64_t n = std::min<uint64_t>(cap, s.size()); memcpy(buf, s.data(), n); return s.size(); }
}
