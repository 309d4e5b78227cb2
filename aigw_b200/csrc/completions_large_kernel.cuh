// /v1/completions requests of any size below 16 MiB to the OpenAI backend: CompletionsEndpointSpec.ParseBody's verdict, the
// ":path" and at most one sjson edit (the model override), as group 11 of the translate pass (plan_completions in
// chat_walk_impl.cuh) gives them, one CTA streaming one request (completions_large_kernel.cu).  The call's parameters are
// chat_large_kernel's (ChatLargeParams, chat_large_lits with the "/…/completions" path); azure and cost_configured are not read.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "chat_large_kernel.cuh"

namespace aigw {

// A slice holds the tokens, the jump table, the escape counts and the flat-array flags of the call's longest request
// (chat_large_tok_cap tokens): about 8.5 bytes per byte of it.
uint64_t completions_large_slice_bytes(uint32_t max_len);
int completions_large_grid(int sm_count, uint32_t max_len);
cudaError_t launch_completions_large(const ChatLargeParams& P, int grid, cudaStream_t st);

}  // namespace aigw
