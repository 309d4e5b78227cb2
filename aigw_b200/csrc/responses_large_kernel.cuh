// /v1/responses requests of any size below 16 MiB to the OpenAI backend: ResponsesEndpointSpec.ParseBody's verdict, the ":path" and
// at most one sjson edit (the model override), as group 10 of the translate pass (plan_responses in chat_walk_impl.cuh) gives them,
// one CTA streaming one request (responses_large_kernel.cu).  The call's parameters are chat_large_kernel's (ChatLargeParams,
// chat_large_lits with the "/…/responses" path); azure and cost_configured are not read.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "chat_large_kernel.cuh"

namespace aigw {

// A slice holds the tokens, the jump table and the escape counts of the call's longest request (chat_large_tok_cap tokens): about
// 8 bytes per byte of it.  No walk scratch.
uint64_t responses_large_slice_bytes(uint32_t max_len);
int responses_large_grid(int sm_count, uint32_t max_len);
cudaError_t launch_responses_large(const ChatLargeParams& P, int grid, cudaStream_t st);

}  // namespace aigw
