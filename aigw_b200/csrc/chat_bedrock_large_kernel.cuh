// /v1/chat/completions requests of any size below 16 MiB to AWS Bedrock Converse: ParseBody's verdict and the Converse request
// plan_bedrock (chat_walk_impl.cuh) gives them in group 0 of the translate pass, one CTA streaming one request
// (chat_bedrock_large_kernel.cu).  Runs on ChatLargeParams (chat_large_kernel.cuh) with max_len set.
#pragma once
#include "chat_large_record.cuh"

namespace aigw {

// the slice and grid of chat_record_large_slice_bytes / chat_record_large_grid (chat_large_record.cuh)
cudaError_t launch_chat_bedrock_large(const ChatLargeParams& P, int grid, cudaStream_t st);

}  // namespace aigw
