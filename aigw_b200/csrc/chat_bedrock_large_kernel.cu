// /v1/chat/completions requests above the translate pass's 64 KiB ceiling (and below it) to AWS Bedrock Converse: ParseBody's
// verdict, the ":path" /model/{PathEscape(model or override)}/converse[-stream] and the Converse body, with the semantics group 0 of
// the translate pass gives them (scan_top and plan_bedrock in chat_walk_impl.cuh).  sm_90a only.
//
// chat_bedrock_large_kernel: one CTA of 256 threads per request, the scan and depth pass of large_request.cuh, then the record
// phase of chat_large_record_impl.cuh with this planner: the emitting Bedrock plan (ClWalkT<ClOut>, chat_bedrock_walk.cuh) makes
// the checks of the dry plan chat_large_kernel runs, in the same order, and records the Converse body; tool "parameters" are body
// spans in key order.  "system" follows "messages" in the record: a second pass over the messages records it.
#include "chat_bedrock_large_kernel.cuh"

#include "chat_large_record_impl.cuh"

namespace aigw {
namespace {

// plan_bedrock after ParseBody's top-level checks: ":path" /model/{PathEscape(model or override)}/converse[-stream], then the
// Converse body
struct BlPlan : ClChatTop {
  static __device__ __forceinline__ void plan(const ChatLargeParams& P, ClShared& S, RecWalk& W, const RecWalk::Top& t, bool stream) {
    if (!W.bad()) {
      W.lit(L_PATH_MODEL);
      rec_path_model<true>(P, S, W, t);
      W.lit(L_PATH_CONVERSE);
      if (stream) W.lit(L_PATH_STREAM);
      if (W.o.olen > 0xffffu) W.decline(AIGW_R_TOO_LARGE);   // path_len is 16 bits
    }
    S.path_len = (uint32_t)W.o.olen;
    if (!W.bad()) W.plan(t);
  }
};

__global__ void __launch_bounds__(kClThreads, 2) chat_bedrock_large_kernel(const __grid_constant__ ChatLargeParams P) {
  __shared__ ClShared S;
  cl_request_loop<ClRecordRequest<BlPlan>>(P, S);
}

}  // namespace

cudaError_t launch_chat_bedrock_large(const ChatLargeParams& P, int grid, cudaStream_t st) {
  chat_bedrock_large_kernel<<<P.n < (uint32_t)grid ? (P.n ? P.n : 1u) : (uint32_t)grid, kClThreads, 0, st>>>(P);
  return cudaGetLastError();
}

}  // namespace aigw
