// aigw_b200 — Bedrock ConverseStream (AWS eventstream) → OpenAI SSE back-translation (S2) for sm_90a.
//
// Replaces openAIToAWSBedrockTranslatorV1ChatCompletion.ResponseBody for streamed responses
// (internal/translator/openai_awsbedrock.go:695-732), extractAmazonEventStreamEvents (:829-852),
// convertEvent (:858-1006), the stop-reason mapping (:601-621) and the usage arithmetic of
// metrics.ExtractTokenUsageFromExplicitCaching (internal/metrics/metrics.go:292-307).
//
// Observation used: the concatenated SSE text of a stream depends only on the ORDER of complete,
// CRC-valid frames, never on where the HTTP chunk boundaries fall (the reference buffers partial
// frames in `bufferedBody`), so a stream is processed from its concatenated bytes.
//
// Two kernels, both one warp per stream:
//   frames kernel  stages the stream tile by tile in shared memory; lane 0 walks the frame chain
//                  (length prelude + prelude CRC); then ONE LANE PER FRAME checks the message CRC,
//                  reads the headers, runs the typed JSON walk of the payload
//                  (awsbedrock.ConverseStreamEvent, internal/apischema/awsbedrock/awsbedrock.go:423-503)
//                  and sizes its output chunk; the stream state the reference threads through the
//                  events (role, tool-call index) is resolved with ballots; a 48-byte record per
//                  output chunk goes to the workspace, the stream's output range is bump-allocated.
//   emit kernel    one lane per record writes its `data: {...}\n\n` chunk into a shared-memory tile
//                  whose alignment matches the destination; the warp flushes with 16-byte stores.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/aigw_b200.h"

namespace aigw {

struct alignas(16) BedrockRec {   // one output chunk
  uint32_t kf;          // kind | flags << 8
  uint32_t out_len;
  uint32_t tool_index;
  uint32_t role_off, role_len;   // span in the stream's bytes (0 length: omitted)
  uint32_t a[6];        // kind-specific spans (offset,len pairs, relative to the stream start) or counters
  uint32_t pad;
};
static_assert(sizeof(BedrockRec) == 48, "record layout");

struct BedrockStreamParams {
  const uint8_t* bytes;
  const uint64_t* stream_off;    // n_streams+1 (absolute offsets into `bytes`)
  uint64_t off_base;             // stream_off[0]: workspace slots are relative to it
  uint64_t out_bias;             // added to the reported out_off (sub-batches of one host call share an arena)
  uint32_t n_streams;
  uint8_t* out; uint64_t out_capacity;
  aigw_stream_result* results;
  unsigned long long* out_used;
  unsigned int* next;            // two work counters (frames kernel, emit kernel)
  BedrockRec* recs;              // slot of stream s starts at (stream_off[s]-off_base)/32 + 2*s
  uint32_t* rec_count;           // n_streams (0xffffffff: stream declined)
  uint64_t* out_pos;             // n_streams: offset of the stream's text inside `out`
  long long created;
  uint32_t id_len, model_len;
  char id[128], model[128];      // response id / request model, already checked to need no JSON escaping
};

size_t bedrock_work_bytes(uint64_t total_bytes, uint32_t n_streams);
void bedrock_work_layout(BedrockStreamParams& P, uint8_t* work, uint32_t n_streams);
cudaError_t launch_bedrock_stream(const BedrockStreamParams& P, int sm_count, cudaStream_t st);

}  // namespace aigw
