// aigw_b200 — OpenAI SSE usage scan (S1) for sm_90a.
//
// Replaces openAIToOpenAITranslatorV1ChatCompletion.ResponseBody (stream) →
// extractUsageFromBufferEvent (internal/translator/openai_openai.go:131-145,179-215) plus the
// per-call metrics.TokenUsage.Override merge (internal/metrics/metrics.go:258-283,
// call site internal/extproc/processor_impl.go:514).
//
// Observation used: every Set… of a usage line overwrites and Override is latest-set-wins, so
// the merged usage after the last chunk depends only on the ORDER of complete '\n'-terminated
// lines, not on where the chunk boundaries fall; the only chunking artefact is the unterminated
// tail, which the reference never parses.  The kernel therefore walks a stream's bytes tile by
// tile with the partial last line carried over, exactly the carry the reference keeps in
// `o.buffered`.
//
// Mapping: one warp per stream; a tile of the stream is staged in shared memory with 16-byte
// loads; newline positions come from ballots; every complete line is handed to ONE lane, which
// runs a table-driven, byte-sequential typed JSON walk (json.Unmarshal into
// ChatCompletionResponseChunk, internal/apischema/openai/openai.go:1497-1565,2064-2083,1789-1807):
// 32 lines in flight per warp.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/aigw_b200.h"

namespace aigw {

struct SseParams {
  const uint8_t* bytes;
  const uint64_t* chunk_off;     // n_chunks+1
  const uint32_t* chunk_first;   // n_streams+1
  uint32_t n_streams;
  aigw_sse_result* results;
  unsigned int* next;
};

cudaError_t launch_sse_usage(const SseParams& P, int sm_count, cudaStream_t st);
cudaError_t launch_response_usage(const uint8_t* bodies, const uint64_t* offsets, const uint32_t* lens, uint32_t n, aigw_sse_result* results, cudaStream_t st, int embeddings = 0 /* 0 chat completion, 1 embeddings, 2 legacy completions, 3 /v1/responses, 4 Cohere /v2/rerank */);
cudaError_t launch_usage_costs(const aigw_sse_result* results, uint32_t n, const int32_t* cost_types, uint32_t n_costs, unsigned long long* out, cudaStream_t st);

}  // namespace aigw
