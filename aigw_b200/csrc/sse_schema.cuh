// Schema table of openai.ChatCompletionResponseChunk for the typed JSON walker (tjson.cuh); shared by the whole-stream usage
// scan (sse_kernel.cu) and the per-chunk stream steps (stream_kernel.cu).  Each translation unit keeps its own device copy.
#pragma once
#include <cstring>

#include "tjson.cuh"

namespace aigw {
using namespace tj;

// ------------------------------------------------------------------ schema: ChatCompletionResponseChunk
// (internal/apischema/openai/openai.go:1497-1565 chunk/choice/delta, :2064-2083 Usage, :1464-1495 details,
//  :1323-1361 logprobs, :1424-1443 annotations, :1875-1879 StreamReasoningContent, :1789-1807 created)
enum Cap : uint8_t { C_PROMPT = 0, C_COMPLETION = 1, C_TOTAL = 2, C_REASONING = 3, C_CACHED = 4, C_CACHE_CREATION = 5,
                     C_OBJ_USAGE = 0, C_OBJ_CTD = 1, C_OBJ_PTD = 2, C_SPAN_MODEL = 0, NOCAP = 0xff };
enum N : uint8_t { N_ANY = 0, N_STR, N_INT, N_FLOAT, N_ROOT, N_CHOICES, N_CHOICE, N_DELTA, N_TOOLCALLS, N_TOOLCALL, N_FUNC, N_ANNOTS, N_ANNOT, N_URLCIT,
                   N_REASON, N_B64, N_LOGPROBS, N_TOKLPS, N_TOKLP, N_INTS, N_TOPLPS, N_TOPLP, N_USAGE, N_CTD, N_PTD, N_CREATED, N_MODEL,
                   N_PROMPT, N_COMPLETION, N_TOTAL, N_REASONING_TOK, N_CACHED, N_CACHE_CREATION,
                   N_CM_CHOICES, N_CM_CHOICE, N_CM_LOGPROBS, N_STRS, N_FLOATS, N_CM_TOPS, N_MAPF, N_COUNT };

struct FieldDef { uint8_t owner; const char* key; uint8_t node; };
static const FieldDef kFields[] = {
  {N_ROOT, "id", N_STR}, {N_ROOT, "choices", N_CHOICES}, {N_ROOT, "created", N_CREATED}, {N_ROOT, "model", N_MODEL}, {N_ROOT, "service_tier", N_STR},
  {N_ROOT, "system_fingerprint", N_STR}, {N_ROOT, "object", N_STR}, {N_ROOT, "usage", N_USAGE}, {N_ROOT, "obfuscation", N_STR},
  {N_CHOICE, "index", N_INT}, {N_CHOICE, "delta", N_DELTA}, {N_CHOICE, "logprobs", N_LOGPROBS}, {N_CHOICE, "finish_reason", N_STR},
  {N_DELTA, "content", N_STR}, {N_DELTA, "role", N_STR}, {N_DELTA, "tool_calls", N_TOOLCALLS}, {N_DELTA, "annotations", N_ANNOTS}, {N_DELTA, "reasoning_content", N_REASON},
  {N_TOOLCALL, "index", N_INT}, {N_TOOLCALL, "id", N_STR}, {N_TOOLCALL, "function", N_FUNC}, {N_TOOLCALL, "type", N_STR},
  {N_FUNC, "arguments", N_STR}, {N_FUNC, "name", N_STR},
  {N_ANNOT, "type", N_STR}, {N_ANNOT, "url_citation", N_URLCIT},
  {N_URLCIT, "end_index", N_INT}, {N_URLCIT, "start_index", N_INT}, {N_URLCIT, "url", N_STR}, {N_URLCIT, "title", N_STR},
  {N_REASON, "text", N_STR}, {N_REASON, "signature", N_STR}, {N_REASON, "redactedContent", N_B64},
  {N_LOGPROBS, "content", N_TOKLPS}, {N_LOGPROBS, "refusal", N_TOKLPS},
  {N_TOKLP, "token", N_STR}, {N_TOKLP, "bytes", N_INTS}, {N_TOKLP, "logprob", N_FLOAT}, {N_TOKLP, "top_logprobs", N_TOPLPS},
  {N_TOPLP, "token", N_STR}, {N_TOPLP, "bytes", N_INTS}, {N_TOPLP, "logprob", N_FLOAT},
  {N_USAGE, "prompt_tokens", N_PROMPT}, {N_USAGE, "completion_tokens", N_COMPLETION}, {N_USAGE, "total_tokens", N_TOTAL},
  {N_USAGE, "completion_tokens_details", N_CTD}, {N_USAGE, "prompt_tokens_details", N_PTD},
  {N_CTD, "text_tokens", N_INT}, {N_CTD, "accepted_prediction_tokens", N_INT}, {N_CTD, "audio_tokens", N_INT}, {N_CTD, "reasoning_tokens", N_REASONING_TOK}, {N_CTD, "rejected_prediction_tokens", N_INT},
  {N_PTD, "text_tokens", N_INT}, {N_PTD, "audio_tokens", N_INT}, {N_PTD, "cached_tokens", N_CACHED}, {N_PTD, "cache_creation_input_tokens", N_CACHE_CREATION},
};
static constexpr int kNumFields = sizeof(kFields) / sizeof(kFields[0]);

struct alignas(16) SchemaBlob {
  Node nodes[N_COUNT];
  Field fields[64];
  char keys[768];
};
static_assert(kNumFields <= 64, "field table too small");

static inline SchemaBlob build_schema() {
  SchemaBlob b; memset(&b, 0, sizeof b);
  auto set = [&](int n, uint8_t kind, uint8_t cap = NOCAP, uint8_t elem = 0) { b.nodes[n].kind = kind; b.nodes[n].cap = cap; b.nodes[n].elem = elem; };
  set(N_ANY, K_ANY); set(N_STR, K_STR); set(N_INT, K_INT); set(N_FLOAT, K_FLOAT);
  set(N_ROOT, K_OBJ); set(N_CHOICES, K_ARR, NOCAP, N_CHOICE); set(N_CHOICE, K_OBJ); set(N_DELTA, K_OBJ);
  set(N_TOOLCALLS, K_ARR, NOCAP, N_TOOLCALL); set(N_TOOLCALL, K_OBJ); set(N_FUNC, K_OBJ);
  set(N_ANNOTS, K_ARR, NOCAP, N_ANNOT); set(N_ANNOT, K_OBJ); set(N_URLCIT, K_OBJ); set(N_REASON, K_OBJ); set(N_B64, K_B64);
  set(N_LOGPROBS, K_OBJ); set(N_TOKLPS, K_ARR, NOCAP, N_TOKLP); set(N_TOKLP, K_OBJ); set(N_INTS, K_ARR, NOCAP, N_INT);
  set(N_TOPLPS, K_ARR, NOCAP, N_TOPLP); set(N_TOPLP, K_OBJ);
  set(N_USAGE, K_OBJ, C_OBJ_USAGE); set(N_CTD, K_OBJ, C_OBJ_CTD); set(N_PTD, K_OBJ, C_OBJ_PTD);
  set(N_CREATED, K_CREATED); set(N_MODEL, K_STR, C_SPAN_MODEL);
  set(N_PROMPT, K_INT, C_PROMPT); set(N_COMPLETION, K_INT, C_COMPLETION); set(N_TOTAL, K_INT, C_TOTAL);
  set(N_REASONING_TOK, K_INT, C_REASONING); set(N_CACHED, K_INT, C_CACHED); set(N_CACHE_CREATION, K_INT, C_CACHE_CREATION);
  int ko = 0;
  for (int f = 0; f < kNumFields; f++) {
    const FieldDef& d = kFields[f];
    Node& o = b.nodes[d.owner];
    if (o.nf == 0) o.f0 = (uint8_t)f;   // fields of one owner are contiguous in kFields
    o.nf++;
    int kl = (int)strlen(d.key);
    b.fields[f].koff = (uint16_t)ko; b.fields[f].klen = (uint8_t)kl; b.fields[f].node = d.node;
    memcpy(b.keys + ko, d.key, kl); ko += kl;
  }
  return b;
}

// ------------------------------------------------------------------ schema: CompletionResponse (legacy /v1/completions; the stream
// chunks and the buffered body share the shape: internal/apischema/openai/openai.go:2000-2055; Usage :2064-2081)
static const FieldDef kCmplFields[] = {
  {N_ROOT, "id", N_STR}, {N_ROOT, "object", N_STR}, {N_ROOT, "created", N_CREATED}, {N_ROOT, "model", N_MODEL}, {N_ROOT, "system_fingerprint", N_STR},
  {N_ROOT, "choices", N_CM_CHOICES}, {N_ROOT, "usage", N_USAGE},
  {N_CM_CHOICE, "text", N_STR}, {N_CM_CHOICE, "index", N_INT}, {N_CM_CHOICE, "logprobs", N_CM_LOGPROBS}, {N_CM_CHOICE, "finish_reason", N_STR},
  {N_CM_LOGPROBS, "tokens", N_STRS}, {N_CM_LOGPROBS, "token_logprobs", N_FLOATS}, {N_CM_LOGPROBS, "top_logprobs", N_CM_TOPS}, {N_CM_LOGPROBS, "text_offset", N_INTS},
  {N_USAGE, "prompt_tokens", N_PROMPT}, {N_USAGE, "completion_tokens", N_COMPLETION}, {N_USAGE, "total_tokens", N_TOTAL},
  {N_USAGE, "completion_tokens_details", N_CTD}, {N_USAGE, "prompt_tokens_details", N_PTD},
  {N_CTD, "text_tokens", N_INT}, {N_CTD, "accepted_prediction_tokens", N_INT}, {N_CTD, "audio_tokens", N_INT}, {N_CTD, "reasoning_tokens", N_REASONING_TOK}, {N_CTD, "rejected_prediction_tokens", N_INT},
  {N_PTD, "text_tokens", N_INT}, {N_PTD, "audio_tokens", N_INT}, {N_PTD, "cached_tokens", N_CACHED}, {N_PTD, "cache_creation_input_tokens", N_CACHE_CREATION},
};
static constexpr int kNumCmplFields = sizeof(kCmplFields) / sizeof(kCmplFields[0]);
static_assert(kNumCmplFields <= 64, "field table too small");

static inline SchemaBlob build_completion_schema() {
  SchemaBlob b; memset(&b, 0, sizeof b);
  auto set = [&](int n, uint8_t kind, uint8_t cap = NOCAP, uint8_t elem = 0) { b.nodes[n].kind = kind; b.nodes[n].cap = cap; b.nodes[n].elem = elem; };
  set(N_ANY, K_ANY); set(N_STR, K_STR); set(N_INT, K_INT); set(N_FLOAT, K_FLOAT);
  set(N_ROOT, K_OBJ); set(N_CM_CHOICES, K_ARR, NOCAP, N_CM_CHOICE); set(N_CM_CHOICE, K_OBJ); set(N_CM_LOGPROBS, K_OBJ);
  set(N_STRS, K_ARR, NOCAP, N_STR); set(N_FLOATS, K_ARR, NOCAP, N_FLOAT); set(N_INTS, K_ARR, NOCAP, N_INT);
  set(N_CM_TOPS, K_ARR, NOCAP, N_MAPF); set(N_MAPF, K_MAP, NOCAP, N_FLOAT);   // []map[string]float64
  set(N_USAGE, K_OBJ, C_OBJ_USAGE); set(N_CTD, K_OBJ, C_OBJ_CTD); set(N_PTD, K_OBJ, C_OBJ_PTD);
  set(N_CREATED, K_CREATED); set(N_MODEL, K_STR, C_SPAN_MODEL);
  set(N_PROMPT, K_INT, C_PROMPT); set(N_COMPLETION, K_INT, C_COMPLETION); set(N_TOTAL, K_INT, C_TOTAL);
  set(N_REASONING_TOK, K_INT, C_REASONING); set(N_CACHED, K_INT, C_CACHED); set(N_CACHE_CREATION, K_INT, C_CACHE_CREATION);
  int ko = 0;
  for (int f = 0; f < kNumCmplFields; f++) {
    const FieldDef& d = kCmplFields[f];
    Node& o = b.nodes[d.owner];
    if (o.nf == 0) o.f0 = (uint8_t)f;   // fields of one owner are contiguous in kCmplFields
    o.nf++;
    int kl = (int)strlen(d.key);
    b.fields[f].koff = (uint16_t)ko; b.fields[f].klen = (uint8_t)kl; b.fields[f].node = d.node;
    memcpy(b.keys + ko, d.key, kl); ko += kl;
  }
  return b;
}

// ------------------------------------------------------------------ schema: openai.Response (/v1/responses; walked by walk<CAP, true>)
// Response :5845-6039, ResponseUsage :6663-6694, the output-item union :6147 (message :4013-4138 with the content and annotation
// unions :4047-4266, function_call :4784, reasoning :4977), tools :2694 (function :2780), tool_choice :5654, instructions :6062,
// text.format :2439-2522, reasoning :2525; the stream events response.created / response.completed :7729,7839.
// Every tag the reference knows is listed: a tag this subset does not restate maps to X_DECL (DECLINE); any other tag fails.
// The captured members come first in their object (the walker tracks repeats among the first 32 members only).
enum XN : uint8_t { X_ANY = 0, X_STR, X_INT, X_FLOAT, X_BOOL, X_DECL, X_EVENT, X_ROOT, X_CREATED, X_PCREATED, X_F32, X_MODEL,
                    X_ERROR, X_INCOMPLETE, X_INSTR, X_INSTR_ARR, X_STRMAP, X_ANYMAP, X_OUTPUT, X_ITEM, X_MSG, X_CONTENT, X_PARTS, X_PART,
                    X_OTEXT, X_REFUSAL, X_ANNOTS, X_ANNOT, X_FCIT, X_UCIT, X_CCIT, X_FPATH, X_LPS, X_LP, X_INTS, X_TOPS, X_TOP,
                    X_FCALL, X_RITEM, X_TEXTPARTS, X_TEXTPART, X_TC, X_TC_U, X_TC_FUNC, X_TOOLS, X_TOOL, X_FTOOL, X_CONV, X_PROMPT,
                    X_REASONING, X_TEXT, X_FORMAT, X_FMT_TYPE, X_FMT_SCHEMA, X_USAGE, X_ITD, X_OTD,
                    X_IN, X_OUT, X_TOTAL, X_CACHED, X_CREATION, X_REASONING_TOK, X_COUNT };
enum : uint8_t { C_OBJ_RESPONSE = 3 };   // obj_seen bit: the event's `response` was a non-null object
static const FieldDef kRspFields[] = {
  {X_EVENT, "response", X_ROOT}, {X_EVENT, "type", X_STR}, {X_EVENT, "sequence_number", X_INT},
  {X_ROOT, "model", X_MODEL}, {X_ROOT, "usage", X_USAGE}, {X_ROOT, "id", X_STR}, {X_ROOT, "created_at", X_CREATED}, {X_ROOT, "completed_at", X_PCREATED},
  {X_ROOT, "error", X_ERROR}, {X_ROOT, "incomplete_details", X_INCOMPLETE}, {X_ROOT, "instructions", X_INSTR}, {X_ROOT, "metadata", X_STRMAP},
  {X_ROOT, "object", X_STR}, {X_ROOT, "output", X_OUTPUT}, {X_ROOT, "parallel_tool_calls", X_BOOL}, {X_ROOT, "temperature", X_FLOAT},
  {X_ROOT, "tool_choice", X_TC}, {X_ROOT, "tools", X_TOOLS}, {X_ROOT, "top_p", X_FLOAT}, {X_ROOT, "background", X_BOOL}, {X_ROOT, "conversation", X_CONV},
  {X_ROOT, "max_output_tokens", X_INT}, {X_ROOT, "max_tool_calls", X_INT}, {X_ROOT, "previous_response_id", X_STR}, {X_ROOT, "prompt", X_PROMPT},
  {X_ROOT, "prompt_cache_key", X_STR}, {X_ROOT, "prompt_cache_retention", X_STR}, {X_ROOT, "reasoning", X_REASONING}, {X_ROOT, "safety_identifier", X_STR},
  {X_ROOT, "service_tier", X_STR}, {X_ROOT, "status", X_STR}, {X_ROOT, "text", X_TEXT}, {X_ROOT, "top_logprobs", X_INT}, {X_ROOT, "truncation", X_STR},
  {X_ROOT, "user", X_STR}, {X_ROOT, "presence_penalty", X_F32}, {X_ROOT, "frequency_penalty", X_F32}, {X_ROOT, "store", X_BOOL},
  {X_ERROR, "code", X_STR}, {X_ERROR, "message", X_STR},
  {X_INCOMPLETE, "reason", X_STR},
  {X_ITEM, "message", X_MSG}, {X_ITEM, "file_search_call", X_DECL}, {X_ITEM, "function_call", X_FCALL}, {X_ITEM, "function_call_output", X_DECL},
  {X_ITEM, "web_search_call", X_DECL}, {X_ITEM, "computer_call", X_DECL}, {X_ITEM, "reasoning", X_RITEM}, {X_ITEM, "compaction", X_DECL},
  {X_ITEM, "image_generation_call", X_DECL}, {X_ITEM, "code_interpreter_call", X_DECL}, {X_ITEM, "local_shell_call", X_DECL}, {X_ITEM, "shell_call", X_DECL},
  {X_ITEM, "shell_call_output", X_DECL}, {X_ITEM, "apply_patch_call", X_DECL}, {X_ITEM, "apply_patch_call_output", X_DECL}, {X_ITEM, "mcp_call", X_DECL},
  {X_ITEM, "mcp_list_tools", X_DECL}, {X_ITEM, "mcp_approval_request", X_DECL}, {X_ITEM, "custom_tool_call", X_DECL},
  {X_MSG, "id", X_STR}, {X_MSG, "content", X_CONTENT}, {X_MSG, "status", X_STR}, {X_MSG, "role", X_STR}, {X_MSG, "type", X_STR},
  {X_PART, "output_text", X_OTEXT}, {X_PART, "refusal", X_REFUSAL},
  {X_OTEXT, "annotations", X_ANNOTS}, {X_OTEXT, "text", X_STR}, {X_OTEXT, "logprobs", X_LPS}, {X_OTEXT, "type", X_STR},
  {X_REFUSAL, "refusal", X_STR}, {X_REFUSAL, "type", X_STR},
  {X_ANNOT, "file_citation", X_FCIT}, {X_ANNOT, "url_citation", X_UCIT}, {X_ANNOT, "container_file_citation", X_CCIT}, {X_ANNOT, "file_path", X_FPATH},
  {X_FCIT, "file_id", X_STR}, {X_FCIT, "filename", X_STR}, {X_FCIT, "index", X_INT}, {X_FCIT, "type", X_STR},
  {X_UCIT, "end_index", X_INT}, {X_UCIT, "start_index", X_INT}, {X_UCIT, "title", X_STR}, {X_UCIT, "url", X_STR}, {X_UCIT, "type", X_STR},
  {X_CCIT, "container_id", X_STR}, {X_CCIT, "end_index", X_INT}, {X_CCIT, "file_id", X_STR}, {X_CCIT, "filename", X_STR}, {X_CCIT, "start_index", X_INT}, {X_CCIT, "type", X_STR},
  {X_FPATH, "file_id", X_STR}, {X_FPATH, "index", X_INT}, {X_FPATH, "type", X_STR},
  {X_LP, "token", X_STR}, {X_LP, "bytes", X_INTS}, {X_LP, "logprob", X_FLOAT}, {X_LP, "top_logprobs", X_TOPS},
  {X_TOP, "token", X_STR}, {X_TOP, "bytes", X_INTS}, {X_TOP, "logprob", X_FLOAT},
  {X_FCALL, "arguments", X_STR}, {X_FCALL, "call_id", X_STR}, {X_FCALL, "name", X_STR}, {X_FCALL, "id", X_STR}, {X_FCALL, "status", X_STR}, {X_FCALL, "type", X_STR},
  {X_RITEM, "id", X_STR}, {X_RITEM, "summary", X_TEXTPARTS}, {X_RITEM, "encrypted_content", X_STR}, {X_RITEM, "content", X_TEXTPARTS}, {X_RITEM, "status", X_STR}, {X_RITEM, "type", X_STR},
  {X_TEXTPART, "text", X_STR}, {X_TEXTPART, "type", X_STR},
  {X_TC_U, "allowed_tools", X_DECL}, {X_TC_U, "file_search", X_DECL}, {X_TC_U, "web_search_preview", X_DECL}, {X_TC_U, "computer_use_preview", X_DECL},
  {X_TC_U, "web_search_preview_2025_03_11", X_DECL}, {X_TC_U, "image_generation", X_DECL}, {X_TC_U, "code_interpreter", X_DECL}, {X_TC_U, "function", X_TC_FUNC},
  {X_TC_U, "mcp", X_DECL}, {X_TC_U, "custom", X_DECL}, {X_TC_U, "apply_patch", X_DECL}, {X_TC_U, "shell", X_DECL},
  {X_TC_FUNC, "name", X_STR}, {X_TC_FUNC, "type", X_STR},
  {X_TOOL, "function", X_FTOOL}, {X_TOOL, "file_search", X_DECL}, {X_TOOL, "computer_use_preview", X_DECL}, {X_TOOL, "web_search", X_DECL},
  {X_TOOL, "web_search_2025_08_26", X_DECL}, {X_TOOL, "mcp", X_DECL}, {X_TOOL, "code_interpreter", X_DECL}, {X_TOOL, "image_generation", X_DECL},
  {X_TOOL, "custom", X_DECL}, {X_TOOL, "local_shell", X_DECL}, {X_TOOL, "shell", X_DECL}, {X_TOOL, "web_search_preview", X_DECL},
  {X_TOOL, "web_search_preview_2025_03_11", X_DECL}, {X_TOOL, "apply_patch", X_DECL},
  {X_FTOOL, "strict", X_BOOL}, {X_FTOOL, "parameters", X_ANYMAP}, {X_FTOOL, "name", X_STR}, {X_FTOOL, "description", X_STR}, {X_FTOOL, "type", X_STR},
  {X_CONV, "id", X_STR},
  {X_PROMPT, "id", X_STR}, {X_PROMPT, "variables", X_DECL}, {X_PROMPT, "version", X_STR},
  {X_REASONING, "effort", X_STR}, {X_REASONING, "generate_summary", X_STR}, {X_REASONING, "summary", X_STR},
  {X_TEXT, "format", X_FORMAT}, {X_TEXT, "verbosity", X_STR},
  {X_FORMAT, "text", X_FMT_TYPE}, {X_FORMAT, "json_schema", X_FMT_SCHEMA}, {X_FORMAT, "json_object", X_FMT_TYPE},
  {X_FMT_TYPE, "type", X_STR},
  {X_FMT_SCHEMA, "name", X_STR}, {X_FMT_SCHEMA, "schema", X_ANYMAP}, {X_FMT_SCHEMA, "strict", X_BOOL}, {X_FMT_SCHEMA, "description", X_STR}, {X_FMT_SCHEMA, "type", X_STR},
  {X_USAGE, "input_tokens", X_IN}, {X_USAGE, "input_tokens_details", X_ITD}, {X_USAGE, "output_tokens", X_OUT}, {X_USAGE, "output_tokens_details", X_OTD},
  {X_USAGE, "total_tokens", X_TOTAL},
  {X_ITD, "cached_tokens", X_CACHED}, {X_ITD, "cache_creation_input_tokens", X_CREATION},
  {X_OTD, "reasoning_tokens", X_REASONING_TOK},
};
static constexpr int kNumRspFields = sizeof(kRspFields) / sizeof(kRspFields[0]);
struct alignas(16) RspSchemaBlob { Node nodes[X_COUNT]; Field fields[192]; char keys[2560]; };
static_assert(kNumRspFields <= 192, "responses field table too small");

static inline RspSchemaBlob build_responses_schema() {
  RspSchemaBlob b; memset(&b, 0, sizeof b);
  auto set = [&](int n, uint8_t kind, uint8_t cap = NOCAP, uint8_t elem = 0) { b.nodes[n].kind = kind; b.nodes[n].cap = cap; b.nodes[n].elem = elem; };
  set(X_ANY, K_ANY); set(X_STR, K_STR); set(X_INT, K_INT); set(X_FLOAT, K_FLOAT); set(X_BOOL, K_BOOL); set(X_DECL, K_DECLINE);
  set(X_EVENT, K_OBJ); set(X_ROOT, K_OBJ, C_OBJ_RESPONSE); set(X_CREATED, K_CREATED); set(X_PCREATED, K_PCREATED); set(X_F32, K_F32); set(X_MODEL, K_STR, C_SPAN_MODEL);
  set(X_ERROR, K_OBJ); set(X_INCOMPLETE, K_OBJ);
  set(X_INSTR, K_STROBJ, NOCAP, X_INSTR_ARR); set(X_INSTR_ARR, K_ARR, NOCAP, X_DECL);   // a string, null or []; input items are not restated
  set(X_STRMAP, K_MAP, NOCAP, X_STR); set(X_ANYMAP, K_MAP, NOCAP, X_ANY);
  set(X_OUTPUT, K_ARR, NOCAP, X_ITEM); set(X_ITEM, K_UNION); set(X_MSG, K_OBJ);
  set(X_CONTENT, K_STRARR, NOCAP, X_PARTS); set(X_PARTS, K_ARR, NOCAP, X_PART); set(X_PART, K_UNION); set(X_OTEXT, K_OBJ); set(X_REFUSAL, K_OBJ);
  set(X_ANNOTS, K_ARR, NOCAP, X_ANNOT); set(X_ANNOT, K_UNION); set(X_FCIT, K_OBJ); set(X_UCIT, K_OBJ); set(X_CCIT, K_OBJ); set(X_FPATH, K_OBJ);
  set(X_LPS, K_ARR, NOCAP, X_LP); set(X_LP, K_OBJ); set(X_INTS, K_ARR, NOCAP, X_INT); set(X_TOPS, K_ARR, NOCAP, X_TOP); set(X_TOP, K_OBJ);
  set(X_FCALL, K_OBJ); set(X_RITEM, K_OBJ); set(X_TEXTPARTS, K_ARR, NOCAP, X_TEXTPART); set(X_TEXTPART, K_OBJ);
  set(X_TC, K_STROBJ, NOCAP, X_TC_U); set(X_TC_U, K_UNION); set(X_TC_FUNC, K_OBJ);   // "a string, else gjson type"
  set(X_TOOLS, K_ARR, NOCAP, X_TOOL); set(X_TOOL, K_UNION); set(X_FTOOL, K_OBJ);
  set(X_CONV, K_OBJ); set(X_PROMPT, K_OBJ); set(X_REASONING, K_OBJ); set(X_TEXT, K_OBJ); set(X_FORMAT, K_UNION); set(X_FMT_TYPE, K_OBJ); set(X_FMT_SCHEMA, K_OBJ);
  set(X_USAGE, K_OBJ, C_OBJ_USAGE); set(X_ITD, K_OBJ); set(X_OTD, K_OBJ);
  set(X_IN, K_INT, C_PROMPT); set(X_OUT, K_INT, C_COMPLETION); set(X_TOTAL, K_INT, C_TOTAL);
  set(X_CACHED, K_INT, C_CACHED); set(X_CREATION, K_INT, C_CACHE_CREATION); set(X_REASONING_TOK, K_INT, C_REASONING);
  int ko = 0;
  for (int f = 0; f < kNumRspFields; f++) {
    const FieldDef& d = kRspFields[f];
    Node& o = b.nodes[d.owner];
    if (o.nf == 0) o.f0 = (uint8_t)f;   // fields (and union tags) of one owner are contiguous in kRspFields
    o.nf++;
    int kl = (int)strlen(d.key);
    b.fields[f].koff = (uint16_t)ko; b.fields[f].klen = (uint8_t)kl; b.fields[f].node = d.node;
    memcpy(b.keys + ko, d.key, kl); ko += kl;
  }
  return b;
}

// ------------------------------------------------------------------ schema: cohere.RerankV2Response (walked by walk<CAP, true>)
// internal/apischema/cohere/rerank_v2.go.  Every float64 member is K_F64; meta.tokens' two counts are captured as uint32(float64).
enum QN : uint8_t { Q_ANY = 0, Q_STR, Q_INT, Q_F64, Q_BOOL, Q_ROOT, Q_RESULTS, Q_RESULT, Q_META, Q_APIVER, Q_BILLED, Q_TOKENS, Q_STRS,
                    Q_IN, Q_OUT, Q_COUNT };
static const FieldDef kRerankFields[] = {
  {Q_ROOT, "results", Q_RESULTS}, {Q_ROOT, "id", Q_STR}, {Q_ROOT, "meta", Q_META},
  {Q_RESULT, "index", Q_INT}, {Q_RESULT, "relevance_score", Q_F64},
  {Q_META, "api_version", Q_APIVER}, {Q_META, "billed_units", Q_BILLED}, {Q_META, "tokens", Q_TOKENS}, {Q_META, "cached_tokens", Q_F64}, {Q_META, "warnings", Q_STRS},
  {Q_APIVER, "version", Q_STR}, {Q_APIVER, "is_deprecated", Q_BOOL}, {Q_APIVER, "is_experimental", Q_BOOL},
  {Q_BILLED, "images", Q_F64}, {Q_BILLED, "input_tokens", Q_F64}, {Q_BILLED, "output_tokens", Q_F64}, {Q_BILLED, "search_units", Q_F64}, {Q_BILLED, "classifications", Q_F64},
  {Q_TOKENS, "input_tokens", Q_IN}, {Q_TOKENS, "output_tokens", Q_OUT},
};
static constexpr int kNumRerankFields = sizeof(kRerankFields) / sizeof(kRerankFields[0]);
static_assert(kNumRerankFields <= 64 && Q_COUNT <= N_COUNT, "the rerank schema uses a SchemaBlob");

static inline SchemaBlob build_rerank_schema() {
  SchemaBlob b; memset(&b, 0, sizeof b);
  auto set = [&](int n, uint8_t kind, uint8_t cap = NOCAP, uint8_t elem = 0) { b.nodes[n].kind = kind; b.nodes[n].cap = cap; b.nodes[n].elem = elem; };
  set(Q_ANY, K_ANY); set(Q_STR, K_STR); set(Q_INT, K_INT); set(Q_F64, K_F64); set(Q_BOOL, K_BOOL);
  set(Q_ROOT, K_OBJ); set(Q_RESULTS, K_ARR, NOCAP, Q_RESULT); set(Q_RESULT, K_OBJ); set(Q_META, K_OBJ); set(Q_APIVER, K_OBJ); set(Q_BILLED, K_OBJ);
  set(Q_TOKENS, K_OBJ, C_OBJ_USAGE); set(Q_STRS, K_ARR, NOCAP, Q_STR);
  set(Q_IN, K_F64, C_PROMPT); set(Q_OUT, K_F64, C_COMPLETION);
  int ko = 0;
  for (int f = 0; f < kNumRerankFields; f++) {
    const FieldDef& d = kRerankFields[f];
    Node& o = b.nodes[d.owner];
    if (o.nf == 0) o.f0 = (uint8_t)f;   // fields of one owner are contiguous in kRerankFields
    o.nf++;
    int kl = (int)strlen(d.key);
    b.fields[f].koff = (uint16_t)ko; b.fields[f].klen = (uint8_t)kl; b.fields[f].node = d.node;
    memcpy(b.keys + ko, d.key, kl); ko += kl;
  }
  return b;
}

// ------------------------------------------------------------------ R1: non-stream ChatCompletionResponse usage
// json.NewDecoder(body).Decode(&openai.ChatCompletionResponse{}) then usage / model
// (internal/translator/openai_openai.go:146-174; struct internal/apischema/openai/openai.go:1269-1306,1365-1422).
enum RN : uint8_t { R_ANY = 0, R_STR, R_INT, R_FLOAT, R_ROOT, R_CHOICES, R_CHOICE, R_MSG, R_TOOLCALLS, R_TOOLCALL, R_FUNC, R_CACHE, R_ANNOTS, R_ANNOT, R_URLCIT,
                  R_AUDIO, R_REASON_U, R_REASON_O, R_REASON_BLOCK, R_REASON_TEXT, R_B64, R_THINKS, R_THINK, R_LOGPROBS, R_TOKLPS, R_TOKLP, R_INTS, R_TOPLPS, R_TOPLP,
                  R_USAGE, R_CTD, R_PTD, R_CREATED, R_MODEL, R_PROMPT, R_COMPLETION, R_TOTAL, R_REASONING_TOK, R_CACHED, R_CACHE_CREATION,
                  R_EM_DATA, R_EM_ITEM, R_EM_VEC, R_EM_FLOATS, R_EM_USAGE, R_COUNT };
static const FieldDef kRespFields[] = {
  {R_ROOT, "id", R_STR}, {R_ROOT, "choices", R_CHOICES}, {R_ROOT, "created", R_CREATED}, {R_ROOT, "model", R_MODEL}, {R_ROOT, "service_tier", R_STR},
  {R_ROOT, "system_fingerprint", R_STR}, {R_ROOT, "object", R_STR}, {R_ROOT, "usage", R_USAGE}, {R_ROOT, "obfuscation", R_STR},
  {R_CHOICE, "finish_reason", R_STR}, {R_CHOICE, "index", R_INT}, {R_CHOICE, "logprobs", R_LOGPROBS}, {R_CHOICE, "message", R_MSG},
  {R_MSG, "content", R_STR}, {R_MSG, "role", R_STR}, {R_MSG, "tool_calls", R_TOOLCALLS}, {R_MSG, "annotations", R_ANNOTS}, {R_MSG, "audio", R_AUDIO},
  {R_MSG, "reasoning_content", R_REASON_U}, {R_MSG, "thinking_blocks", R_THINKS}, {R_MSG, "safety_ratings", R_ANY}, {R_MSG, "grounding_metadata", R_ANY},
  {R_TOOLCALL, "id", R_STR}, {R_TOOLCALL, "function", R_FUNC}, {R_TOOLCALL, "type", R_STR}, {R_TOOLCALL, "cache_control", R_CACHE},
  {R_FUNC, "arguments", R_STR}, {R_FUNC, "name", R_STR},
  {R_CACHE, "type", R_STR}, {R_CACHE, "ttl", R_STR},
  {R_ANNOT, "type", R_STR}, {R_ANNOT, "url_citation", R_URLCIT},
  {R_URLCIT, "end_index", R_INT}, {R_URLCIT, "start_index", R_INT}, {R_URLCIT, "url", R_STR}, {R_URLCIT, "title", R_STR},
  {R_AUDIO, "data", R_STR}, {R_AUDIO, "expires_at", R_INT}, {R_AUDIO, "id", R_STR}, {R_AUDIO, "transcript", R_STR},
  {R_REASON_O, "reasoningContent", R_REASON_BLOCK},
  {R_REASON_BLOCK, "reasoningText", R_REASON_TEXT}, {R_REASON_BLOCK, "redactedContent", R_B64},
  {R_REASON_TEXT, "text", R_STR}, {R_REASON_TEXT, "signature", R_STR},
  {R_THINK, "type", R_STR}, {R_THINK, "thinking", R_STR}, {R_THINK, "signature", R_STR}, {R_THINK, "data", R_STR},
  {R_LOGPROBS, "content", R_TOKLPS}, {R_LOGPROBS, "refusal", R_TOKLPS},
  {R_TOKLP, "token", R_STR}, {R_TOKLP, "bytes", R_INTS}, {R_TOKLP, "logprob", R_FLOAT}, {R_TOKLP, "top_logprobs", R_TOPLPS},
  {R_TOPLP, "token", R_STR}, {R_TOPLP, "bytes", R_INTS}, {R_TOPLP, "logprob", R_FLOAT},
  {R_USAGE, "prompt_tokens", R_PROMPT}, {R_USAGE, "completion_tokens", R_COMPLETION}, {R_USAGE, "total_tokens", R_TOTAL},
  {R_USAGE, "completion_tokens_details", R_CTD}, {R_USAGE, "prompt_tokens_details", R_PTD},
  {R_CTD, "text_tokens", R_INT}, {R_CTD, "accepted_prediction_tokens", R_INT}, {R_CTD, "audio_tokens", R_INT}, {R_CTD, "reasoning_tokens", R_REASONING_TOK}, {R_CTD, "rejected_prediction_tokens", R_INT},
  {R_PTD, "text_tokens", R_INT}, {R_PTD, "audio_tokens", R_INT}, {R_PTD, "cached_tokens", R_CACHED}, {R_PTD, "cache_creation_input_tokens", R_CACHE_CREATION},
};
static constexpr int kNumRespFields = sizeof(kRespFields) / sizeof(kRespFields[0]);
struct alignas(16) RespSchemaBlob { Node nodes[R_COUNT]; Field fields[80]; char keys[1024]; };
static_assert(kNumRespFields <= 80, "response field table too small");

static inline RespSchemaBlob build_resp_schema() {
  RespSchemaBlob b; memset(&b, 0, sizeof b);
  auto set = [&](int n, uint8_t kind, uint8_t cap = NOCAP, uint8_t elem = 0) { b.nodes[n].kind = kind; b.nodes[n].cap = cap; b.nodes[n].elem = elem; };
  set(R_ANY, K_ANY); set(R_STR, K_STR); set(R_INT, K_INT); set(R_FLOAT, K_FLOAT);
  set(R_ROOT, K_OBJ); set(R_CHOICES, K_ARR, NOCAP, R_CHOICE); set(R_CHOICE, K_OBJ); set(R_MSG, K_OBJ);
  set(R_TOOLCALLS, K_ARR, NOCAP, R_TOOLCALL); set(R_TOOLCALL, K_OBJ); set(R_FUNC, K_OBJ); set(R_CACHE, K_OBJ);
  set(R_ANNOTS, K_ARR, NOCAP, R_ANNOT); set(R_ANNOT, K_OBJ); set(R_URLCIT, K_OBJ); set(R_AUDIO, K_OBJ);
  set(R_REASON_U, K_STROBJ, NOCAP, R_REASON_O); set(R_REASON_O, K_OBJ); set(R_REASON_BLOCK, K_OBJ); set(R_REASON_TEXT, K_OBJ); set(R_B64, K_B64);
  set(R_THINKS, K_ARR, NOCAP, R_THINK); set(R_THINK, K_OBJ);
  set(R_LOGPROBS, K_OBJ); set(R_TOKLPS, K_ARR, NOCAP, R_TOKLP); set(R_TOKLP, K_OBJ); set(R_INTS, K_ARR, NOCAP, R_INT); set(R_TOPLPS, K_ARR, NOCAP, R_TOPLP); set(R_TOPLP, K_OBJ);
  set(R_USAGE, K_OBJ, C_OBJ_USAGE); set(R_CTD, K_OBJ, C_OBJ_CTD); set(R_PTD, K_OBJ, C_OBJ_PTD);
  set(R_CREATED, K_CREATED); set(R_MODEL, K_STR, C_SPAN_MODEL);
  set(R_PROMPT, K_INT, C_PROMPT); set(R_COMPLETION, K_INT, C_COMPLETION); set(R_TOTAL, K_INT, C_TOTAL);
  set(R_REASONING_TOK, K_INT, C_REASONING); set(R_CACHED, K_INT, C_CACHED); set(R_CACHE_CREATION, K_INT, C_CACHE_CREATION);
  int ko = 0;
  for (int f = 0; f < kNumRespFields; f++) {
    const FieldDef& d = kRespFields[f];
    Node& o = b.nodes[d.owner];
    if (o.nf == 0) o.f0 = (uint8_t)f;
    o.nf++;
    int kl = (int)strlen(d.key);
    b.fields[f].koff = (uint16_t)ko; b.fields[f].klen = (uint8_t)kl; b.fields[f].node = d.node;
    memcpy(b.keys + ko, d.key, kl); ko += kl;
  }
  return b;
}


}  // namespace aigw
