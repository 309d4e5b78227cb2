// /v1/chat/completions requests of any size below 16 MiB to the OpenAI and Azure OpenAI passthroughs: ParseBody's verdict, the
// ":path" and at most two sjson edits, as group 1 of the translate pass (scan_top, passthrough_accepts, plan_passthrough /
// plan_azure in chat_walk_impl.cuh) gives them, one CTA streaming one request (chat_large_kernel.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/aigw_b200.h"

namespace aigw {

// literals of the records; the last three are the call's configuration text (OpenAI path, override, api-version)
enum ChatLargeLit : uint32_t {
  CL_TRUE, CL_COMMA, CL_QUOTE, CL_IU_MEMBER, CL_IU_OBJ, CL_SO_APPEND, CL_MODEL_MEMBER, CL_AZ_PREFIX, CL_AZ_SUFFIX,
  CL_OPENAI_PATH, CL_OVERRIDE, CL_VERSION, CL_COUNT
};

struct ChatLargeParams {
  const uint8_t* bodies;      // requests back to back, each start 16-byte aligned
  const uint64_t* offsets;    // n
  const uint32_t* lens;       // n
  uint32_t n;
  aigw_doc_result* results;   // n
  uint8_t* ws;                // chat_large_grid() slices of chat_large_slice_bytes(max_len) bytes, one per CTA
  uint64_t slice;
  uint32_t tok_cap;
  unsigned int* next;         // work counter (zeroed by the caller)
  uint8_t* out;               // output arena, 16-byte aligned
  uint64_t out_capacity;
  unsigned long long* out_used;
  uint32_t call_reason;       // non-zero: every request is DECLINED with this reason (wrong schema)
  uint32_t azure;             // AIGW_SCHEMA_AZURE_OPENAI, else AIGW_SCHEMA_OPENAI
  uint32_t cost_configured;
  uint32_t force_mutation;
  uint32_t override_len;      // 0: no model override
  uint32_t override_ok;       // the override needs no JSON escaping
  uint16_t lit_off[CL_COUNT];
  uint16_t lit_len[CL_COUNT];
  char lits[512];
  uint32_t max_len;           // the call's longest request (the record kernels of chat_large_record.cuh: the slice's layout)
  uint32_t gcp;               // chat_anthropic_large_kernel: AIGW_SCHEMA_GCP_ANTHROPIC, else AIGW_SCHEMA_AWS_ANTHROPIC
  uint32_t bedrock;           // messages_large_kernel: AIGW_SCHEMA_MSG_AWS_BEDROCK, else AIGW_SCHEMA_MSG_OPENAI
};

static constexpr uint32_t kChatLargeMaxDepth = 48;
// one tool call's "arguments" string is unescaped into the CTA's slice and checked there: at most kChatArgMax bytes each, and at
// most kChatArgTotal bytes per request (the serial bound of the walk); above either the request declines with AIGW_R_SCRATCH
static constexpr uint32_t kChatArgMax = 64u * 1024u;
static constexpr uint32_t kChatArgTotal = 256u * 1024u;
// the work of the key-order check over tool parameters and arguments objects, per request: member visits plus the key bytes
// compared (AIGW_R_SCRATCH above).  The check is quadratic in an object's members; this keeps a hostile body's cost to a few
// hundred milliseconds of one thread (DESIGN §4.9)
static constexpr uint32_t kChatAnyWork = 1u << 18;
// a request may hold len / 2 + 1024 scan tokens (AIGW_R_TOKENS above).  Real requests are mostly string bytes and stay far below
// it; a body made of one-byte scalars or empty strings reaches one token per byte and declines.  Every slice is sized for the
// call's longest request
__host__ __device__ inline uint32_t chat_large_tok_cap(uint32_t len) { return len / 2u + 1024u; }
uint64_t chat_large_slice_bytes(uint32_t max_len);
int chat_large_grid(int sm_count, uint32_t max_len);
// fills lits / lit_off / lit_len from the constant literals and the configuration text
void chat_large_lits(ChatLargeParams& P, const char* openai_path, uint32_t path_len, const char* override_model, uint32_t override_len,
                     const char* version, uint32_t version_len);
cudaError_t launch_chat_large(const ChatLargeParams& P, int grid, cudaStream_t st);

}  // namespace aigw
