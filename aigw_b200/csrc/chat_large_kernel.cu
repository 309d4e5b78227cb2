// /v1/chat/completions requests above the translate pass's 64 KiB ceiling (and below it) to the OpenAI and Azure OpenAI
// passthroughs: ChatCompletionsEndpointSpec.ParseBody's verdict, the ":path" and at most two sjson edits, with the semantics group
// 1 of the translate pass gives them (scan_top, passthrough_accepts, plan_passthrough / plan_azure in chat_walk_impl.cuh).
// sm_90a only.
//
// chat_large_kernel: one CTA of 256 threads per request, the stages of large_request.cuh (scan, depth, grammar, emit) around this
// file's walk and plan:
//   walk      thread 0 runs scan_top and the dry Bedrock plan (ClWalkT<ClNoOut>, chat_bedrock_walk.cuh) over the jump table:
//             the same checks in the same order, so the first problem decides as in the translate pass (ParseBody's 400s, then a
//             pending 422 / 500 as AIGW_R_CONTENT).  A tool call's "arguments" string is unescaped into the CTA's slice,
//             tokenized and checked there.
//   plan      the record as at most 12 copy ops: ":path" from literals (and the Azure deployment from the body), then the body
//             with edit A (stream_options.include_usage) and edit B (the model override) spliced in body order
#include "chat_large_kernel.cuh"

#include <string.h>

#include "chat_bedrock_walk.cuh"

namespace aigw {

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
