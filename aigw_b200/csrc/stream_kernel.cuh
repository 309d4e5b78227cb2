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

// Output range of one call: the body the step writes, then the response model.  B = carry + chunk bytes the step decodes,
// ml = the stream's request model length (≤ 160).  A unit is the smallest piece of input that yields output (a line, an SSE
// event, an eventstream frame, a Gemini part); 16·B pays 16 bytes of output per input byte, so a kind needs more only where
// one unit writes more than 16 bytes per byte it consumed:
//   kind                        smallest unit with output                  most output of that unit             16·unit   extra per unit
//   AWS Bedrock                 51 B: 16 B frame + 35 B metadata payload   ≤ 192 + id + model + role ≤ 576       816      0
//   GCP Anthropic               30 B: "event: message_stop\ndata: {}\n\n"    ≤ 160 + id + model ≤ 480             480       0
//   AWS Anthropic               60 B: frame of base64 {"type":"message_stop"}   the same ≤ 480                  960       0
//   GCP Gemini                  4 B: "{}" + a 2-byte delimiter             66 + model (choices [])               64        2 + ml
//   Gemini buffered             the whole body                              fixed text ≤ 500 + model             -         0
//   /v1/messages, OpenAI        48 B: a data line with one text delta      ≤ 200 + its text                     768       0
//   /v1/messages, OpenAI, buf.  3 B: one tool call "{}," in the body        49: {"type":"tool_use",…,"input":{}}  48        1
//   /v1/messages, AWS Anthropic frame ≥ 16 B + its event JSON           the event JSON + ≤ 40                 -         0
// (id, role and the text of a unit come from the input and are paid by 16·B except where they repeat in every unit: the Bedrock
// id / model / role and the Anthropic message id, at most 160, 160, 64 and 160 bytes, are in the table.)  Once per call: 1024 for
// one-time text (message_start, the end-of-stream chunk, [DONE], a last Gemini part without a delimiter) and the model.
// The usage-only kinds (OpenAI, completions, native Anthropic, /v1/responses) write only the model: their bound stays 16·B + 1024.
inline uint32_t stream_out_cap(uint32_t kind, uint64_t bytes, uint32_t model_len) {
  uint64_t oc = 16ull * bytes + 1024u;
  switch (kind) {
    case AIGW_STREAM_OPENAI: case AIGW_STREAM_OPENAI_COMPLETIONS: case AIGW_STREAM_ANTHROPIC: case AIGW_STREAM_OPENAI_RESPONSES: break;
    case AIGW_STREAM_GCP_GEMINI: oc += model_len + (bytes / 4 + 1) * (2ull + model_len); break;
    case AIGW_STREAM_MESSAGES_OPENAI_BUFFERED: oc += model_len + bytes / 3 + 1; break;
    default: oc += model_len; break;
  }
  return (uint32_t)(oc > 0x7fffffffull ? 0x7fffffffull : oc);
}

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
