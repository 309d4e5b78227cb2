// /v1/responses requests above the translate pass's 64 KiB ceiling (and below it) to the OpenAI backend:
// ResponsesEndpointSpec.ParseBody's verdict over the restated subset of openai.ResponseRequest, the ":path" and the sjson model
// override, with the semantics group 10 of the translate pass gives them (rq_tag, rq_variant, rq_struct, rq_value, plan_responses,
// openai_request_result in chat_walk_impl.cuh).  sm_90a only.
//
// responses_large_kernel: one CTA of 256 threads per request, the stages of large_request.cuh (scan, depth, grammar, emit) around
// this file's walk and plan:
//   walk      thread 0 checks every restated member in body order over the jump table: the same checks in the same order with the
//             same reasons, so the first problem decides as in the translate pass.  Key and tag ids come from lookup_id on the raw
//             bytes against the translate pass's own table (make_rq_id_tables); a key or tag with a backslash declines before its
//             id is needed.  map[string]any members (tool parameters, text.format.schema) and unknown members are only
//             grammar-checked, as there.
//   plan      ":path" from the configuration, then the body unchanged, the original bytes (force_body_mutation), or with the
//             model override spliced: the first "model" value replaced, or the member appended before the root's '}' (sjson
//             rebuilds the root, so the bytes outside its braces go)
#include "responses_large_kernel.cuh"

#include "canon_number.cuh"
#include "large_request.cuh"
// after large_request.cuh: it defines FULL as a macro
#include "chat_internal.cuh"

namespace aigw {

static __device__ IdTables g_rl_ids = make_rq_id_tables();   // the translate pass's group-10 key and tag ids

struct RlScratch {};

// ---------------------------------------------------------------- the walk (thread 0)
// A restatement, not a reuse: the translate pass's Walker reads a 16-bit token word with the ids of its index stage and is
// compiled once per schema group.  This one reads 24-bit positions and looks the ids up as it goes.  A change to group 10's checks
// has to be made in both; test_responses_large_gpu.py compares the two on the translate pass's corpora.
struct RqWalk {
  using Scratch = RlScratch;
  static constexpr bool kFlatArrays = false;
  LDoc d;
  Scratch A;
  uint32_t* stk;
  int reason = 0, pending = 0;   // pending: never set (no translator of this schema answers 422 / 500)

  static __device__ __forceinline__ RlScratch scratch(uint2*) { return RlScratch{}; }
  __device__ void decline(int r) { if (!reason) reason = r; }
  __device__ bool bad() const { return reason != 0; }
  __device__ bool is_str(uint32_t v) const { return d.ty(v) == '"'; }
  __device__ bool is_obj(uint32_t v) const { return d.ty(v) == '{'; }
  __device__ bool is_arr(uint32_t v) const { return d.ty(v) == '['; }
  __device__ bool is_bool(uint32_t v) const { const uint32_t c = d.ty(v); return c == 't' || c == 'f'; }
  __device__ bool is_num(uint32_t v) const { const uint32_t c = d.ty(v); return c == '-' || c - '0' < 10u; }
  __device__ bool is_null(uint32_t v) const { return d.ty(v) == 'n'; }
  // the id of string token i (a key: key = true) as the translate pass's index stage gives it to a string without a backslash;
  // every caller has declined a string with one before it asks
  __device__ uint32_t id(uint32_t i, bool key) const {
    const uint32_t n = d.str_len(i);
    if (n < 1u || n > (uint32_t)kMaxIdLen || d.str_has_backslash(i)) return 0;
    return lookup_id<true>(&g_rl_ids, d.s + d.str_off(i), n, key);
  }

  __device__ bool check_scalar_type(uint32_t v, int kind /*0 str,1 bool,2 int,3 float*/) {
    bool ok;
    if (kind == 0) ok = is_str(v);
    else if (kind == 1) ok = is_bool(v);
    else {
      ok = is_num(v);
      if (ok && kind == 2) {
        const uint32_t e = d.scalar_end(v), o = d.tok(v);
        ok = canon_number(d.s + o, e - o, true) != 0;
        if (!ok) {   // a fraction or an exponent in an integer field is the decoder's type error: ParseBody's 400
          bool frac = false; for (uint32_t i = o; i < e; i++) { const uint32_t c = d.s[i]; if (c == '.' || c == 'e' || c == 'E') frac = true; }
          decline(frac ? AIGW_R_E400_TYPE : AIGW_R_NUMBER); return false;
        }
      }
    }
    if (!ok) decline(AIGW_R_E400_TYPE);
    return ok;
  }

  enum RqKind { RQ_TOP, RQ_CONV, RQ_SOPT, RQ_REASONING, RQ_TEXT, RQ_FMT_PLAIN, RQ_FMT_SCHEMA, RQ_TC_FUNC, RQ_TOOL_FUNC, RQ_EASY, RQ_OUTMSG,
                RQ_FCALL, RQ_FCOUT, RQ_RITEM, RQ_TEXTPART, RQ_ITEMREF, RQ_IN_IMAGE, RQ_IN_FILE, RQ_OUT_TEXT, RQ_OUT_REFUSAL };
  enum RqType { RT_SKIP, RT_STR, RT_BOOL, RT_INT, RT_F64, RT_F32, RT_MAPANY, RT_MAPSTR, RT_ARRSTR, RT_ARRDECL, RT_STRDECL, RT_DECL,
                RT_INPUT, RT_CONV, RT_TC, RT_TOOLS, RT_FORMAT, RT_EASYCONTENT, RT_OUTCONTENT, RT_ARRTEXT, RT_OBJ = 32 /* + RqKind */ };
  // the decoder's view of member `id` in a struct of kind `k`: RT_SKIP for a key the struct does not have
  __device__ static uint32_t rq_type(int k, uint32_t id) {
    switch (k) {
      case RQ_TOP:
        switch (id) {
          case RQK_background: case RQK_parallel_tool_calls: case RQK_store: case RQK_stream: return RT_BOOL;
          case RQK_max_output_tokens: case RQK_max_tool_calls: case RQK_top_logprobs: return RT_INT;
          case RQK_temperature: case RQK_top_p: return RT_F64;
          case RQK_presence_penalty: case RQK_frequency_penalty: return RT_F32;
          case RQK_instructions: case RQK_previous_response_id: case RQK_prompt_cache_key: case RQK_safety_identifier: case RQK_user:
          case RQK_prompt_cache_retention: case RQK_service_tier: case RQK_truncation: case RQK_model: return RT_STR;
          case RQK_include: return RT_ARRSTR;
          case RQK_metadata: return RT_MAPSTR;
          case RQK_conversation: return RT_CONV;
          case RQK_stream_options: return RT_OBJ + RQ_SOPT;
          case RQK_reasoning: return RT_OBJ + RQ_REASONING;
          case RQK_text: return RT_OBJ + RQ_TEXT;
          case RQK_tool_choice: return RT_TC;
          case RQK_tools: return RT_TOOLS;
          case RQK_input: return RT_INPUT;
          case RQK_DECL: return RT_DECL;
          default: return RT_SKIP;
        }
      case RQ_CONV: return id == RQK_id ? RT_STR : RT_SKIP;
      case RQ_SOPT: return id == RQK_include_obfuscation ? RT_BOOL : RT_SKIP;
      case RQ_REASONING: return (id == RQK_effort || id == RQK_generate_summary || id == RQK_summary) ? RT_STR : RT_SKIP;
      case RQ_TEXT: return id == RQK_verbosity ? RT_STR : id == RQK_format ? RT_FORMAT : RT_SKIP;
      case RQ_FMT_PLAIN: return id == RQK_type ? RT_STR : RT_SKIP;
      case RQ_FMT_SCHEMA: return (id == RQK_name || id == RQK_description || id == RQK_type) ? RT_STR : id == RQK_schema ? RT_MAPANY : id == RQK_strict ? RT_BOOL : RT_SKIP;
      case RQ_TC_FUNC: return (id == RQK_name || id == RQK_type) ? RT_STR : RT_SKIP;
      case RQ_TOOL_FUNC: return (id == RQK_name || id == RQK_description || id == RQK_type) ? RT_STR : id == RQK_parameters ? RT_MAPANY : id == RQK_strict ? RT_BOOL : RT_SKIP;
      case RQ_EASY: return (id == RQK_role || id == RQK_type) ? RT_STR : id == RQK_content ? RT_EASYCONTENT : RT_SKIP;
      case RQ_OUTMSG: return (id == RQK_id || id == RQK_status || id == RQK_role || id == RQK_type) ? RT_STR : id == RQK_content ? RT_OUTCONTENT : RT_SKIP;
      case RQ_FCALL: return (id == RQK_arguments || id == RQK_call_id || id == RQK_name || id == RQK_id || id == RQK_status || id == RQK_type) ? RT_STR : RT_SKIP;
      case RQ_FCOUT: return (id == RQK_call_id || id == RQK_id || id == RQK_status || id == RQK_type) ? RT_STR : id == RQK_output ? RT_STRDECL : RT_SKIP;
      case RQ_RITEM: return (id == RQK_id || id == RQK_encrypted_content || id == RQK_status || id == RQK_type) ? RT_STR : (id == RQK_summary || id == RQK_content) ? RT_ARRTEXT : RT_SKIP;
      case RQ_TEXTPART: return (id == RQK_text || id == RQK_type) ? RT_STR : RT_SKIP;
      case RQ_ITEMREF: return (id == RQK_id || id == RQK_type) ? RT_STR : RT_SKIP;
      case RQ_IN_IMAGE: return (id == RQK_detail || id == RQK_file_id || id == RQK_image_url || id == RQK_type) ? RT_STR : RT_SKIP;
      case RQ_IN_FILE: return (id == RQK_file_id || id == RQK_file_data || id == RQK_file_url || id == RQK_filename || id == RQK_type) ? RT_STR : RT_SKIP;
      case RQ_OUT_TEXT: return (id == RQK_text || id == RQK_type) ? RT_STR : (id == RQK_annotations || id == RQK_logprobs) ? RT_ARRDECL : RT_SKIP;
      case RQ_OUT_REFUSAL: return (id == RQK_refusal || id == RQK_type) ? RT_STR : RT_SKIP;
      default: return RT_SKIP;
    }
  }
  // gjson.GetBytes(obj, "type").String() for a union: the tag id of the first top-level "type" string (0 for a string the table
  // does not hold), -1 when it is missing, null or "", -2 after a decline.  Also whether "role" and "content" exist, and the first
  // role's value id.
  __device__ int rq_tag(uint32_t obj, bool& role_content, uint32_t& role) {
    int tag = -1; bool have_tag = false, has_role = false, has_content = false; role = 0;
    for (uint32_t m = obj + 1; d.ty(m) != '}'; m = d.after(m + 3)) {
      if (d.str_has_backslash(m)) { decline(AIGW_R_ESCAPE); return -2; }
      const uint32_t id_ = id(m, true), v = m + 3;
      if (id_ == RQK_type && !have_tag) {
        have_tag = true;
        if (is_str(v)) { if (d.str_has_backslash(v)) { decline(AIGW_R_ESCAPE); return -2; } tag = d.str_len(v) ? (int)id(v, false) : -1; }
        else if (!is_null(v)) { decline(AIGW_R_CONTENT); return -2; }
      } else if (id_ == RQK_role && !has_role) { has_role = true; if (is_str(v)) { if (d.str_has_backslash(v)) { decline(AIGW_R_ESCAPE); return -2; } role = id(v, false); } }
      else if (id_ == RQK_content) has_content = true;
    }
    role_content = has_role && has_content;
    return tag;
  }
  // a tagged union element: the struct kind its tag selects, or -1 (declined)
  __device__ int rq_variant(uint32_t v, uint32_t t) {
    if (!is_obj(v)) { decline(AIGW_R_CONTENT); return -1; }
    bool rc; uint32_t role; const int tag = rq_tag(v, rc, role);
    if (tag == -2) return -1;
    int k = -1;
    if (t == RT_INPUT) {
      if (tag == -1) k = rc ? RQ_EASY : -1;
      else if (tag == RQV_message) k = role == RQV_assistant ? RQ_OUTMSG : RQ_EASY;
      else if (tag == RQV_function_call) k = RQ_FCALL;
      else if (tag == RQV_function_call_output) k = RQ_FCOUT;
      else if (tag == RQV_reasoning) k = RQ_RITEM;
      else if (tag == RQV_item_reference) k = RQ_ITEMREF;
    } else if (t == RT_EASYCONTENT) k = tag == RQV_input_text ? RQ_TEXTPART : tag == RQV_input_image ? RQ_IN_IMAGE : tag == RQV_input_file ? RQ_IN_FILE : -1;
    else if (t == RT_OUTCONTENT) k = tag == RQV_output_text ? RQ_OUT_TEXT : tag == RQV_refusal ? RQ_OUT_REFUSAL : -1;
    else if (t == RT_TOOLS || t == RT_TC) k = tag == RQV_function ? (t == RT_TOOLS ? RQ_TOOL_FUNC : RQ_TC_FUNC) : -1;
    else if (t == RT_FORMAT) k = (tag == RQV_text || tag == RQV_json_object) ? RQ_FMT_PLAIN : tag == RQV_json_schema ? RQ_FMT_SCHEMA : -1;
    if (k < 0) decline(AIGW_R_CONTENT);
    return k;
  }
  // one struct of kind k, members in body order; L is its nesting level (the request 0; items, tools, text 1; content parts,
  // summaries, text.format 2), so that every level is its own function and the walk has no recursion
  template <int L>
  __device__ bool rq_struct(uint32_t obj, int k) {
    uint64_t seen = 0;
    for (uint32_t m = obj + 1; d.ty(m) != '}'; m = d.after(m + 3)) {
      if (d.str_has_backslash(m)) { decline(AIGW_R_ESCAPE); return false; }
      const uint32_t id_ = id(m, true);
      const uint32_t t = id_ ? rq_type(k, id_) : (uint32_t)RT_SKIP;
      if (t == RT_SKIP) continue;
      if (t == RT_DECL) { decline(AIGW_R_UNSUPPORTED_FIELD); return false; }
      if (seen & (1ull << id_)) { decline(AIGW_R_DUP_KEY); return false; }
      seen |= 1ull << id_;
      if (k == RQ_TOP && id_ == RQK_model && is_str(m + 3) && d.str_has_backslash(m + 3)) { decline(AIGW_R_ESCAPE); return false; }
      if (!rq_value<L>(m + 3, t)) return false;
    }
    return true;
  }
  template <int L>
  __device__ bool rq_value(uint32_t v, uint32_t t) {
    if (is_null(v)) {   // a no-op for plain members; a union's UnmarshalJSON gets "null": the string forms decode it, these three fail
      if (t == RT_FORMAT || t == RT_OUTCONTENT || t == RT_STRDECL) { decline(AIGW_R_CONTENT); return false; }
      return true;
    }
    switch (t) {
      case RT_STR: case RT_BOOL: case RT_INT: case RT_F64: return check_scalar_type(v, t == RT_STR ? 0 : t == RT_BOOL ? 1 : t == RT_INT ? 2 : 3);
      case RT_F32: {
        if (!is_num(v)) { decline(AIGW_R_E400_TYPE); return false; }
        const uint32_t o = d.tok(v), e = d.scalar_end(v), i = o + (d.s[o] == '-' ? 1u : 0u);
        uint32_t ie = i; while (ie < e && is_digit(d.s[ie])) ie++;
        bool ex = false; for (uint32_t q = ie; q < e; q++) ex |= (d.s[q] | 0x20u) == 'e';
        if (ex || ie - i > 38u) { decline(AIGW_R_NUMBER); return false; }   // the float32 range is not restated
        return true;
      }
      case RT_MAPANY: if (!is_obj(v)) { decline(AIGW_R_E400_TYPE); return false; } return true;
      case RT_MAPSTR:
        if (!is_obj(v)) { decline(AIGW_R_E400_TYPE); return false; }
        for (uint32_t m = v + 1; d.ty(m) != '}'; m = d.after(m + 3)) {
          if (d.str_has_backslash(m)) { decline(AIGW_R_ESCAPE); return false; }
          if (!is_null(m + 3) && !check_scalar_type(m + 3, 0)) return false;
        }
        return true;
      case RT_ARRSTR: case RT_ARRDECL:
        if (!is_arr(v)) { decline(AIGW_R_E400_TYPE); return false; }
        for (uint32_t e = v + 1; d.ty(e) != ']'; e = d.after(e)) {
          if (t == RT_ARRDECL) { decline(AIGW_R_UNSUPPORTED_FIELD); return false; }   // annotations / logprobs on an assistant message
          if (!is_null(e) && !check_scalar_type(e, 0)) return false;
        }
        return true;
      case RT_STRDECL: if (!is_str(v)) { decline(AIGW_R_CONTENT); return false; } return true;   // function_call_output.output: the item list is not restated
      case RT_CONV:   // a string, else {id}
        if (is_str(v)) return true;
        if (!is_obj(v)) { decline(AIGW_R_E400_TYPE); return false; }
        if constexpr (L < 2) return rq_struct<L + 1>(v, RQ_CONV); else { decline(AIGW_R_DEPTH); return false; }
      case RT_TC:     // any string, else the tag
        if (is_str(v)) return true;
        [[fallthrough]];
      case RT_FORMAT: {
        const int k = rq_variant(v, t);
        if (k < 0) return false;
        if constexpr (L < 2) return rq_struct<L + 1>(v, k); else { decline(AIGW_R_DEPTH); return false; }
      }
      case RT_INPUT: case RT_EASYCONTENT: case RT_OUTCONTENT:   // a string, or a list of tagged elements
        if (is_str(v)) return true;
        [[fallthrough]];
      case RT_TOOLS: case RT_ARRTEXT:
        if (!is_arr(v)) { decline(AIGW_R_E400_TYPE); return false; }
        for (uint32_t e = v + 1; d.ty(e) != ']'; e = d.after(e)) {
          int k = RQ_TEXTPART;
          if (t == RT_ARRTEXT) { if (is_null(e)) continue; if (!is_obj(e)) { decline(AIGW_R_E400_TYPE); return false; } }   // plain structs: null is a no-op
          else if ((k = rq_variant(e, t)) < 0) return false;
          if constexpr (L < 2) { if (!rq_struct<L + 1>(e, k)) return false; } else { decline(AIGW_R_DEPTH); return false; }
        }
        return true;
      default:
        if (t >= RT_OBJ) {
          if (!is_obj(v)) { decline(AIGW_R_E400_TYPE); return false; }
          if constexpr (L < 2) return rq_struct<L + 1>(v, (int)(t - RT_OBJ)); else { decline(AIGW_R_DEPTH); return false; }
        }
        return true;
    }
  }

  // model: the "model" value when it is a string (ParseBody's model), else kNone; model_raw: its value token, null included (the
  // override's splice point), kNone when absent; stream: the "stream" value, kNone when absent
  struct Top { uint32_t model, stream, model_raw; };
  // plan_responses up to openai_request_result: the root, every restated member, then the model and stream members
  __device__ bool scan_top(Top& t) {
    t.model = t.stream = t.model_raw = kNone;
    if (!is_obj(0)) { decline(is_null(0) ? AIGW_R_ROOT : AIGW_R_E400_TYPE); return false; }
    if (!rq_struct<0>(0, RQ_TOP)) return false;
    for (uint32_t m = 1; d.ty(m) != '}'; m = d.after(m + 3)) {
      const uint32_t id_ = id(m, true);
      if (id_ == RQK_model) t.model_raw = m + 3; else if (id_ == RQK_stream) t.stream = m + 3;
    }
    if (t.model_raw != kNone && is_str(t.model_raw)) {
      if (d.str_has_backslash(t.model_raw)) { decline(AIGW_R_ESCAPE); return false; }
      t.model = t.model_raw;
    }
    return true;
  }
  __device__ void check(const Top&) {}   // every check ran in scan_top
};

// openai_request_result after the model span and the stream flag (large_request.cuh)
__device__ int cl_plan(const ChatLargeParams& P, RqWalk& W, const RqWalk::Top& t, bool, ClRec& R) { return cl_openai_plan(P, W, t, R); }

__global__ void __launch_bounds__(kClThreads, 2) responses_large_kernel(const __grid_constant__ ChatLargeParams P) {
  __shared__ ClShared S;
  cl_request_loop<RqWalk>(P, S);
}

uint64_t responses_large_slice_bytes(uint32_t max_len) {
  const uint64_t tc = chat_large_tok_cap(max_len);
  return (tc * 4u * 2u + 8u + (tc + 1u) * 8u + 255u) & ~255ull;   // words, jump table, escape counts
}

int responses_large_grid(int sm_count, uint32_t max_len) {
  uint64_t g = kClWorkspace / responses_large_slice_bytes(max_len);
  if (g > (uint64_t)sm_count * 2u) g = (uint64_t)sm_count * 2u;
  return g < 1 ? 1 : (int)g;
}

cudaError_t launch_responses_large(const ChatLargeParams& P, int grid, cudaStream_t st) {
  responses_large_kernel<<<P.n < (uint32_t)grid ? (P.n ? P.n : 1u) : (uint32_t)grid, kClThreads, 0, st>>>(P);
  return cudaGetLastError();
}

}  // namespace aigw
