// /v1/embeddings requests of any size below 16 MiB: EmbeddingsEndpointSpec.ParseBody and the OpenAI / Azure passthrough, the GCP
// Vertex AI predict request and the Amazon Titan InvokeModel request, as plan_embeddings (chat_walk_impl.cuh) gives them to the
// AIGW_SCHEMA_EMB_* schemas, one CTA streaming one request (emb_large_kernel.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/aigw_b200.h"

namespace aigw {

// literals of the records; the last three are the call's configuration text (OpenAI path, override, api-version)
enum EmbLit : uint32_t {
  EL_INSTANCES, EL_CONTENT, EL_NEXT, EL_TASK, EL_TITLE, EL_LAST, EL_PARAMS, EL_AUTOTRUNC, EL_DIMS, EL_END, EL_GOOGLE_PATH, EL_PREDICT,
  EL_AZ_PATH1, EL_AZ_PATH2, EL_TITAN_OPEN, EL_TITAN_DIMS, EL_PATH_MODEL, EL_INVOKE, EL_NULL, EL_EMPTY_STR, EL_COMMA, EL_MODEL_MEMBER,
  EL_QUOTE, EL_LBRACE, EL_RBRACE, EL_LBRACK, EL_OPENAI_PATH, EL_OVERRIDE, EL_VERSION, EL_COUNT
};

struct EmbLargeParams {
  const uint8_t* bodies;      // requests back to back, each start 16-byte aligned
  const uint64_t* offsets;    // n
  const uint32_t* lens;       // n
  uint32_t n;
  aigw_doc_result* results;   // n
  uint8_t* ws;                // emb_large_grid() slices of emb_large_slice_bytes(max_len) bytes, one per CTA
  uint64_t slice;
  uint32_t tok_cap, esc_cap, op_cap;
  unsigned int* next;         // work counter (zeroed by the caller)
  uint8_t* out;               // output arena, 16-byte aligned
  uint64_t out_capacity;
  unsigned long long* out_used;
  uint32_t call_reason;       // non-zero: every request is DECLINED with this reason (wrong schema)
  uint32_t base;              // AIGW_SCHEMA_OPENAI / _AWS_BEDROCK (Titan) / _AZURE_OPENAI / _GCP_VERTEX
  uint32_t force_mutation;
  uint32_t override_len;      // 0: no model override
  uint32_t override_ok;       // the override needs no JSON escaping
  uint16_t lit_off[EL_COUNT];
  uint16_t lit_len[EL_COUNT];
  char override_model[128];   // raw, for the Titan path escape
  char lits[768];
};

static constexpr uint32_t kEmbMaxDepth = 48;
static constexpr uint32_t kEmbScratch = 65536 + 64;   // the Titan ":path" after PathEscape (at most 65535 bytes)
// a request may hold len / 2 + 1024 scan tokens (a token-id array costs two per id), len / 4 + 1024 re-spelled escapes (\/ \b \f
// and \u; each takes at least two body bytes, \u six) and 2 * (len / 2 + 1024) copy ops (an input element gives at most six:
// a null element with a task type and a title); every slice is sized for the call's longest request
__host__ __device__ inline uint32_t emb_tok_cap(uint32_t len) { return len / 2u + 1024u; }
__host__ __device__ inline uint32_t emb_esc_cap(uint32_t len) { return len / 4u + 1024u; }
__host__ __device__ inline uint32_t emb_op_cap(uint32_t len) { return 2u * emb_tok_cap(len); }
// the longest record (path and body) a request of len bytes may produce: 16 bytes per body byte and 64 KiB, and never less than
// the longest record the translate pass writes (0xffff chunks of 16 bytes), so that no body it accepts is declined here
static constexpr uint64_t kEmbTranslatePassRecordMax = 0xffffull * 16u;
__host__ __device__ inline uint64_t emb_out_ceiling(uint32_t len) { const uint64_t c = 16ull * len + 65536u; return c > kEmbTranslatePassRecordMax ? c : kEmbTranslatePassRecordMax; }
uint64_t emb_large_slice_bytes(uint32_t max_len);
int emb_large_grid(int sm_count, uint32_t max_len);
// fills lits / lit_off / lit_len from the constant literals and the configuration text
void emb_large_lits(EmbLargeParams& P, const char* openai_path, uint32_t path_len, const char* override_model, uint32_t override_len,
                    const char* version, uint32_t version_len);
cudaError_t launch_emb_large(const EmbLargeParams& P, int grid, cudaStream_t st);

}  // namespace aigw
