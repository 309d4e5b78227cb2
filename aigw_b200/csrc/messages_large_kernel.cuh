// /v1/messages requests of any size below 16 MiB to the backends that need a full re-map of the request (OpenAI chat completions,
// AWS Bedrock Converse): the verdict and the request plan_messages_full (chat_walk_impl.cuh) gives them in group 9 of the translate
// pass, one CTA streaming one request (messages_large_kernel.cu).  Runs on ChatLargeParams (chat_large_kernel.cuh) with max_len
// set, in the slice of chat_record_large_slice_bytes / chat_record_large_grid.
#pragma once
#include "chat_large_record.cuh"

namespace aigw {

cudaError_t launch_messages_large(const ChatLargeParams& P, int grid, cudaStream_t st);

}  // namespace aigw
