// /v1/completions requests above the translate pass's 64 KiB ceiling (and below it) to the OpenAI backend:
// CompletionsEndpointSpec.ParseBody's verdict over openai.CompletionRequest, the ":path" and the sjson model override, with the
// semantics group 11 of the translate pass gives them (cp_int64, cp_f64, cp_prompt, plan_completions, openai_request_result in
// chat_walk_impl.cuh).  sm_90a only.
//
// completions_large_kernel: one CTA of 256 threads per request, the stages of large_request.cuh (scan, depth, flat arrays,
// grammar, emit) around this file's walk and plan:
//   flat      every thread: the flat arrays of scalars (token-id prompts above all) get their jump and a flag, so the grammar check
//             steps over each in one move and the walk takes an all-int64 array of `prompt` without visiting its elements
//   walk      thread 0 checks every member in body order: the same checks in the same order with the same reasons and the same
//             duplicate rule, so the first problem decides as in the translate pass.  Key ids come from lookup_id on the raw
//             bytes against the translate pass's own table (make_cp_id_tables); a key with a backslash declines before its id is
//             needed.  Unknown members are only grammar-checked, as there.
//   plan      ":path" from the configuration, then the body unchanged, the original bytes (force_body_mutation), or with the
//             model override spliced (cl_openai_plan, shared with responses_large_kernel)
#include "completions_large_kernel.cuh"

#include "large_request.cuh"
// after large_request.cuh: it defines FULL as a macro
#include "chat_internal.cuh"

namespace aigw {

static __device__ IdTables g_cpl_ids = make_cp_id_tables();   // the translate pass's group-11 key ids

// the walk's part of the slice: the flat-array stage's flag byte per token (read at '[' tokens only)
struct CplScratch { uint8_t* flag; };

// ---------------------------------------------------------------- the walk (thread 0)
// A restatement, not a reuse: the translate pass's Walker reads a 16-bit token word with the ids of its index stage and is
// compiled once per schema group.  This one reads 24-bit positions and looks the ids up as it goes.  A change to group 11's checks
// has to be made in both; test_completions_large_gpu.py compares the two on the translate pass's corpora.
struct CpWalk {
  using Scratch = CplScratch;
  static constexpr bool kFlatArrays = true;
  LDoc d;
  Scratch A;
  uint32_t* stk;
  int reason = 0, pending = 0;   // pending: never set (no translator of this schema answers 422 / 500)

  static __device__ __forceinline__ CplScratch scratch(uint2* rest) { return CplScratch{(uint8_t*)rest}; }
  __device__ void decline(int r) { if (!reason) reason = r; }
  __device__ bool bad() const { return reason != 0; }
  __device__ bool is_str(uint32_t v) const { return d.ty(v) == '"'; }
  __device__ bool is_obj(uint32_t v) const { return d.ty(v) == '{'; }
  __device__ bool is_arr(uint32_t v) const { return d.ty(v) == '['; }
  __device__ bool is_bool(uint32_t v) const { const uint32_t c = d.ty(v); return c == 't' || c == 'f'; }
  __device__ bool is_num(uint32_t v) const { const uint32_t c = d.ty(v); return c == '-' || c - '0' < 10u; }
  __device__ bool is_null(uint32_t v) const { return d.ty(v) == 'n'; }
  // the id of key token i as the translate pass's index stage gives it to a key without a backslash; every caller has declined
  // a key with one before it asks
  __device__ uint32_t id(uint32_t i) const {
    const uint32_t n = d.str_len(i);
    if (n < 1u || n > (uint32_t)kMaxIdLen || d.str_has_backslash(i)) return 0;
    return lookup_id<true>(&g_cpl_ids, d.s + d.str_off(i), n, true);
  }
  // kind 0 string, 1 bool: the only kinds group 11 asks for
  __device__ bool check_scalar_type(uint32_t v, int kind) {
    const bool ok = kind == 0 ? is_str(v) : is_bool(v);
    if (!ok) decline(AIGW_R_E400_TYPE);
    return ok;
  }

  // Go int / int64 member: the decoder's exact range.  A fraction or an exponent and a value outside int64 are its type errors.
  // The grammar check has run, so the digits have no leading zero.
  __device__ bool cp_int64(uint32_t v) {
    if (!is_num(v)) { decline(AIGW_R_E400_TYPE); return false; }
    const uint32_t o = d.tok(v), e = d.scalar_end(v), i = o + (d.s[o] == '-' ? 1u : 0u);
    for (uint32_t q = i; q < e; q++) if (!is_digit(d.s[q])) { decline(AIGW_R_E400_TYPE); return false; }
    if (e - i < 19u) return true;
    if (e - i > 19u) { decline(AIGW_R_E400_TYPE); return false; }
    const char* lim = "9223372036854775808";   // -2^63; the positive bound is one less
    int c = 0;
    for (uint32_t q = 0; q < 19u && !c; q++) c = (int)d.s[i + q] - (int)lim[q];
    if (c > 0 || (c == 0 && i == o)) { decline(AIGW_R_E400_TYPE); return false; }
    return true;
  }
  // float64 member: up to 308 integer digits and no exponent is below the float64 overflow; beyond it the body declines
  __device__ bool cp_f64(uint32_t v) {
    if (!is_num(v)) { decline(AIGW_R_E400_TYPE); return false; }
    const uint32_t o = d.tok(v), e = d.scalar_end(v), i = o + (d.s[o] == '-' ? 1u : 0u);
    uint32_t ie = i; while (ie < e && is_digit(d.s[ie])) ie++;
    bool ex = false; for (uint32_t q = ie; q < e; q++) ex |= (d.s[q] | 0x20u) == 'e';
    if (ex || ie - i > 308u) { decline(AIGW_R_NUMBER); return false; }
    return true;
  }
  // PromptUnion: a string; [] ([]string{}); else the first element picks the form: '"' []string, '[' [][]int64, '-' or a digit
  // []int64, in which null elements (and null inner arrays) decode; any other first element is a 400, and so is a later element
  // of the wrong kind.  A null prompt declines.  An array the flat stage flagged CL_ALL_INT64 holds only nulls and int64
  // literals, so the per-element loop over it would pass: it is skipped.  The first-element dispatch stays as it is.
  __device__ bool cp_prompt(uint32_t v) {
    if (is_str(v)) return true;
    if (!is_arr(v)) { decline(is_null(v) ? AIGW_R_CONTENT : AIGW_R_E400_TYPE); return false; }
    const uint32_t f = v + 1;
    if (d.ty(f) == ']') return true;
    if (is_str(f)) {
      for (uint32_t q = f; d.ty(q) != ']'; q = d.after(q)) if (!is_str(q) && !is_null(q)) { decline(AIGW_R_E400_TYPE); return false; }
      return true;
    }
    if (is_arr(f)) {
      for (uint32_t q = f; d.ty(q) != ']'; q = d.after(q)) {
        if (is_null(q)) continue;
        if (!is_arr(q)) { decline(AIGW_R_E400_TYPE); return false; }
        if (A.flag[q] & CL_ALL_INT64) continue;
        for (uint32_t x = q + 1; d.ty(x) != ']'; x = d.after(x)) if (!is_null(x) && !cp_int64(x)) return false;
      }
      return true;
    }
    if (is_num(f)) {
      if (A.flag[v] & CL_ALL_INT64) return true;
      for (uint32_t q = f; d.ty(q) != ']'; q = d.after(q)) if (!is_null(q) && !cp_int64(q)) return false;
      return true;
    }
    decline(AIGW_R_E400_TYPE); return false;
  }

  // model: the "model" value when it is a string (ParseBody's model), else kNone; model_raw: its value token, null included (the
  // override's splice point), kNone when absent; stream: the "stream" value, kNone when absent
  struct Top { uint32_t model, stream, model_raw; };
  // plan_completions up to openai_request_result: the root, then every member in body order
  __device__ bool scan_top(Top& t) {
    t.model = t.stream = t.model_raw = kNone;
    if (!is_obj(0)) { decline(is_null(0) ? AIGW_R_ROOT : AIGW_R_E400_TYPE); return false; }
    uint32_t seen = 0;
    for (uint32_t m = 1; d.ty(m) != '}'; m = d.after(m + 3)) {
      if (d.str_has_backslash(m)) { decline(AIGW_R_ESCAPE); return false; }
      const uint32_t id_ = id(m);
      if (id_ == CPK_NONE || id_ == CPK_include_usage) continue;   // unknown to CompletionRequest: skipped whatever its value
      if (seen & (1u << id_)) { decline(AIGW_R_DUP_KEY); return false; }
      seen |= 1u << id_;
      const uint32_t v = m + 3;
      if (id_ == CPK_model) t.model_raw = v;
      else if (id_ == CPK_stream) t.stream = v;
      if (id_ == CPK_stop) {           // any: every JSON value decodes, but a number in it becomes a float64 (cp_f64's rule)
        const uint32_t e = d.next(v);
        for (uint32_t q = v; q < e; q++) if (is_num(q) && !cp_f64(q)) return false;
        continue;
      }
      if (id_ == CPK_prompt) { if (!cp_prompt(v)) return false; continue; }
      if (is_null(v)) continue;       // a no-op for every other member
      switch (id_) {
        case CPK_model: case CPK_suffix: case CPK_user:
          if (!check_scalar_type(v, 0)) return false;
          if (id_ == CPK_model && d.str_has_backslash(v)) { decline(AIGW_R_ESCAPE); return false; }
          break;
        case CPK_echo: case CPK_stream: if (!check_scalar_type(v, 1)) return false; break;
        case CPK_best_of: case CPK_logprobs: case CPK_max_tokens: case CPK_n: case CPK_seed: if (!cp_int64(v)) return false; break;
        case CPK_frequency_penalty: case CPK_presence_penalty: case CPK_temperature: case CPK_top_p: if (!cp_f64(v)) return false; break;
        case CPK_logit_bias:   // map[string]int
          if (!is_obj(v)) { decline(AIGW_R_E400_TYPE); return false; }
          for (uint32_t k = v + 1; d.ty(k) != '}'; k = d.after(k + 3)) {
            if (d.str_has_backslash(k)) { decline(AIGW_R_ESCAPE); return false; }
            if (!is_null(k + 3) && !cp_int64(k + 3)) return false;
          }
          break;
        case CPK_stream_options: {   // *StreamOptions: include_usage bool, other keys skipped
          if (!is_obj(v)) { decline(AIGW_R_E400_TYPE); return false; }
          bool iu = false;
          for (uint32_t k = v + 1; d.ty(k) != '}'; k = d.after(k + 3)) {
            if (d.str_has_backslash(k)) { decline(AIGW_R_ESCAPE); return false; }
            if (id(k) != CPK_include_usage) continue;
            if (iu) { decline(AIGW_R_DUP_KEY); return false; }
            iu = true;
            if (!is_null(k + 3) && !check_scalar_type(k + 3, 1)) return false;
          }
          break;
        }
        default: break;
      }
    }
    if (t.model_raw != kNone && is_str(t.model_raw)) t.model = t.model_raw;   // its backslash declined above
    return true;
  }
  __device__ void check(const Top&) {}   // every check ran in scan_top
};

// openai_request_result after the model span and the stream flag (large_request.cuh)
__device__ int cl_plan(const ChatLargeParams& P, CpWalk& W, const CpWalk::Top& t, bool, ClRec& R) { return cl_openai_plan(P, W, t, R); }

__global__ void __launch_bounds__(kClThreads, 2) completions_large_kernel(const __grid_constant__ ChatLargeParams P) {
  __shared__ ClShared S;
  cl_request_loop<CpWalk>(P, S);
}

uint64_t completions_large_slice_bytes(uint32_t max_len) {
  const uint64_t tc = chat_large_tok_cap(max_len);
  return (tc * 4u * 2u + 8u + (tc + 1u) * 8u + tc + 255u) & ~255ull;   // words, jump table, escape counts, flat-array flags
}

int completions_large_grid(int sm_count, uint32_t max_len) {
  uint64_t g = kClWorkspace / completions_large_slice_bytes(max_len);
  if (g > (uint64_t)sm_count * 2u) g = (uint64_t)sm_count * 2u;
  return g < 1 ? 1 : (int)g;
}

cudaError_t launch_completions_large(const ChatLargeParams& P, int grid, cudaStream_t st) {
  completions_large_kernel<<<P.n < (uint32_t)grid ? (P.n ? P.n : 1u) : (uint32_t)grid, kClThreads, 0, st>>>(P);
  return cudaGetLastError();
}

}  // namespace aigw
