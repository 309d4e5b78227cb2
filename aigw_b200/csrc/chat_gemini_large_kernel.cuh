// /v1/chat/completions requests of any size below 16 MiB to Gemini on GCP Vertex AI (generateContent / streamGenerateContent):
// ParseBody's verdict and the request plan_gemini (chat_walk_impl.cuh) gives them in group 3 of the translate pass, one CTA
// streaming one request (chat_gemini_large_kernel.cu).  Runs on ChatLargeParams (chat_large_kernel.cuh) with max_len set, in the
// slice of chat_record_large_slice_bytes / chat_record_large_grid.
#pragma once
#include "chat_large_record.cuh"

namespace aigw {

cudaError_t launch_chat_gemini_large(const ChatLargeParams& P, int grid, cudaStream_t st);

}  // namespace aigw
