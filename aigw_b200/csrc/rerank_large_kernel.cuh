// Cohere /v2/rerank requests of any size below 16 MiB: RerankEndpointSpec.ParseBody + cohereToCohereTranslatorV2Rerank.RequestBody
// as AIGW_SCHEMA_RERANK_COHERE restates them in the translate pass, one CTA streaming one request (rerank_large_kernel.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/aigw_b200.h"

namespace aigw {

// What the emit kernel writes after ":path": body[keep_b, cut_b) + literal + body[cut_e, keep_e).  lit: 0 none, 1 the override
// as a JSON string (the model value replaced), 2 / 3 the member ,"model":"…" / "model":"…" appended before the root's '}'.
struct RerankSplice { uint32_t keep_b, cut_b, cut_e, keep_e, lit; };

struct RerankLargeParams {
  const uint8_t* bodies;      // requests back to back, each start 16-byte aligned
  const uint64_t* offsets;    // n
  const uint32_t* lens;       // n
  uint32_t n;
  aigw_doc_result* results;   // n
  RerankSplice* splice;       // n
  uint32_t* tok_ws;           // rerank_scan_grid() slices of tok_cap token words (position | type << 24)
  uint8_t* dep_ws;            // the same slices of tok_cap bytes: bracket depth after each token
  uint32_t tok_cap;
  unsigned int* next_scan;    // work counters (zeroed by the caller)
  unsigned int* next_emit;
  uint8_t* out;               // output arena, 16-byte aligned
  uint64_t out_capacity;
  unsigned long long* out_used;
  uint32_t call_reason;       // non-zero: every request is DECLINED with this reason (wrong schema, :path too long)
  uint32_t force_mutation;
  uint32_t override_len;      // 0: no model override
  uint32_t override_ok;       // the override needs no JSON escaping
  uint32_t path_len;
  char override_model[128];
  char path[128];
};

static constexpr uint32_t kRerankMaxDepth = 48;
// a request may hold len / 4 + 1024 scan tokens (never more than the call's slice, tok_cap = max_len / 4 + 1024)
__host__ __device__ inline uint32_t rerank_tok_cap(uint32_t len) { return len / 4u + 1024u; }
int rerank_scan_grid(int sm_count, uint32_t tok_cap);
cudaError_t launch_rerank_large(const RerankLargeParams& P, int sm_count, cudaStream_t st);   // scan, then emit, on st

}  // namespace aigw
