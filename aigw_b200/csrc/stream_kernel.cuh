// aigw_b200 — stateful per-chunk response streams (SURVEY §8b: aigw_stream_open / chunk / close), sm_90a.
//
// The reference calls Translator.ResponseBody(headers, body, endOfStream) once per upstream chunk and carries only the
// undecoded tail between calls (internal/translator/translator.go:41-76; openai_openai.go:131-145,179-193 partial line;
// openai_awsbedrock.go:695-732,829-852 partial frame; anthropic_helper.go:826-857 partial event).  Here that state lives on the
// device: one fixed-size slot per open stream holds the parser state and the carry bytes, and ONE call processes a batch of
// (stream, chunk) pairs:
//   append kernel  (warp per step)    compacts the slot's carry and appends the new chunk bytes, coalesced
//   step kernel    (thread per step)  decodes every complete unit (line / eventstream frame / SSE event) of the slot's
//                                     buffer with the table-driven typed JSON walker, advances the stream state and writes the
//                                     call's body mutation into its reserved output range
//   pack kernel    (warp per step)    moves the mutations into one dense arena (bump allocation) for a single D2H copy
// Thread-per-step is deliberate: a chunk call carries 80 B – a few KB and one to five units; the batch supplies the
// parallelism (100 k streams per call in BASELINE config 4).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/aigw_b200.h"

namespace aigw {

static constexpr uint32_t kStreamSlotBytes = 16384, kStreamHdrBytes = 768, kStreamCarryCap = kStreamSlotBytes - kStreamHdrBytes;
enum StreamFlags : uint32_t { SF_SENT_FIRST = 1, SF_DEAD = 2, SF_TOOL_ACTIVE = 4, SF_HAVE_CREATED = 8 };

struct alignas(16) StreamSlot {
  uint32_t kind, beg, end, flags;            // [beg, end): undecoded bytes in buf (the append kernel moves them to the front)
  int32_t tool_index; uint32_t stop_reason, id_len, model_len;
  uint32_t rmodel_len, role_len, dead_status, dead_reason;
  aigw_usage usage;                          // accumulated (Anthropic); unused by the other kinds
  long long created; int32_t active_index; uint32_t _r0;
  char id[160];                              // response id: cfg (Bedrock) or message.id (Anthropic), raw JSON string bytes
  char model[160];                           // request model (cfg)
  char rmodel[160];                          // OpenAI: last response model seen (streamingResponseModel)
  char role[64];                             // Bedrock: role of the latest messageStart
  uint8_t _pad[kStreamHdrBytes - 640];
  uint8_t buf[kStreamCarryCap];
};
static_assert(sizeof(StreamSlot) == kStreamSlotBytes, "slot layout");

struct StreamStep { uint32_t slot, len, eos, out_cap; uint64_t in_off, out_off; };   // 32 bytes

struct StreamParams {
  StreamSlot* slots;
  const uint8_t* in;             // the call's chunk bytes (device)
  uint8_t* out;                  // reserved output ranges (device)
  uint8_t* packed;               // dense arena
  unsigned long long* packed_used;
  uint64_t packed_cap;
  const StreamStep* steps;
  aigw_chunk_result* results;
  uint32_t n;
};

cudaError_t launch_stream_steps(const StreamParams& P, cudaStream_t st);
// slots [first, first+n) := header template `tmpl` (kStreamHdrBytes bytes on the device)
cudaError_t launch_stream_init(StreamSlot* slots, const uint32_t* slot_ids, uint32_t n, const uint8_t* tmpl, cudaStream_t st);

}  // namespace aigw
