// K2 launcher: picks the walk kernel of the schema's group (chat_walk_g*.cu, one translation unit per group).
#include "chat_internal.cuh"

#include <cstdlib>

namespace aigw {

#define AIGW_WALK_DECL(g) cudaError_t launch_chat_walk_g##g(const ChatParams&, uint32_t, uint32_t, uint8_t*, const WorkLayout&, cudaStream_t, int);
AIGW_WALK_DECL(0) AIGW_WALK_DECL(1) AIGW_WALK_DECL(2) AIGW_WALK_DECL(3) AIGW_WALK_DECL(4) AIGW_WALK_DECL(5) AIGW_WALK_DECL(6) AIGW_WALK_DECL(7) AIGW_WALK_DECL(8) AIGW_WALK_DECL(9) AIGW_WALK_DECL(10) AIGW_WALK_DECL(11) AIGW_WALK_DECL(12)
#undef AIGW_WALK_DECL
#define AIGW_SMALL_DECL(g) cudaError_t launch_chat_small_g##g(const ChatParams&, uint32_t, uint32_t, const uint64_t*, cudaStream_t);
AIGW_SMALL_DECL(0) AIGW_SMALL_DECL(1) AIGW_SMALL_DECL(2) AIGW_SMALL_DECL(3) AIGW_SMALL_DECL(4) AIGW_SMALL_DECL(5) AIGW_SMALL_DECL(6) AIGW_SMALL_DECL(7) AIGW_SMALL_DECL(8) AIGW_SMALL_DECL(9) AIGW_SMALL_DECL(10) AIGW_SMALL_DECL(11) AIGW_SMALL_DECL(12)
#undef AIGW_SMALL_DECL

// resident walk blocks per SM.  The launch bound keeps room for AIGW_WALK_BLOCKS (the register budget: the Bedrock walk uses 116
// registers), but fewer warps run faster.  On an H100 80GB HBM3 at a 700 W power limit (SM 1980 MHz, no throttle reason), profiled
// walk time per 1 M 4 KB bodies (bench.py config 2, AIGW_WALK_CTAS, one session): 3.36-3.37 ms at 3 blocks over 3 runs, 3.38 ms at
// 2 blocks, 3.54 ms at 4 blocks.
constexpr int kWalkBlocksPerSm = 3;

cudaError_t launch_chat_walk(const ChatParams& P, uint32_t doc0, uint32_t ndocs, uint8_t* work, const WorkLayout& layout, cudaStream_t st, int sm_count) {
  static const int env_ctas = getenv("AIGW_WALK_CTAS") ? atoi(getenv("AIGW_WALK_CTAS")) : 0;   // experiment: another number of resident blocks per SM
  const int sms = sm_count * (env_ctas > 0 && env_ctas <= AIGW_WALK_BLOCKS ? env_ctas : kWalkBlocksPerSm);
  const uint32_t s = P.schema;
  if (s & (uint32_t)AIGW_SCHEMA_RERANK) return launch_chat_walk_g12(P, doc0, ndocs, work, layout, st, sms);   // declines every base but Cohere
  if (s & (uint32_t)AIGW_SCHEMA_COMPLETIONS) return launch_chat_walk_g11(P, doc0, ndocs, work, layout, st, sms);   // declines every base but OpenAI
  if (s & (uint32_t)AIGW_SCHEMA_RESPONSES) return launch_chat_walk_g10(P, doc0, ndocs, work, layout, st, sms);   // declines every base but OpenAI
  if (s & (uint32_t)AIGW_SCHEMA_MESSAGES)   // the full re-maps (OpenAI / Bedrock targets) have their own kernel
    return ((s & 15u) == (uint32_t)AIGW_SCHEMA_OPENAI || (s & 15u) == (uint32_t)AIGW_SCHEMA_AWS_BEDROCK) ? launch_chat_walk_g9(P, doc0, ndocs, work, layout, st, sms) : launch_chat_walk_g7(P, doc0, ndocs, work, layout, st, sms);
  if ((s & 56u) == (uint32_t)AIGW_SCHEMA_RESP_ERROR) return launch_chat_walk_g8(P, doc0, ndocs, work, layout, st, sms);
  if ((s & 48u) == (uint32_t)AIGW_SCHEMA_RESP_AWS_BEDROCK)
    return ((s & 15u) == (uint32_t)AIGW_SCHEMA_GCP_ANTHROPIC || (s & 15u) == (uint32_t)AIGW_SCHEMA_ANTHROPIC) ? launch_chat_walk_g5(P, doc0, ndocs, work, layout, st, sms) : launch_chat_walk_g4(P, doc0, ndocs, work, layout, st, sms);
  if (s & (uint32_t)AIGW_SCHEMA_EMBEDDINGS) return launch_chat_walk_g6(P, doc0, ndocs, work, layout, st, sms);
  switch (s) {
    case AIGW_SCHEMA_AWS_BEDROCK: return launch_chat_walk_g0(P, doc0, ndocs, work, layout, st, sms);
    case AIGW_SCHEMA_GCP_ANTHROPIC: case AIGW_SCHEMA_AWS_ANTHROPIC: return launch_chat_walk_g2(P, doc0, ndocs, work, layout, st, sms);
    case AIGW_SCHEMA_GCP_VERTEX: return launch_chat_walk_g3(P, doc0, ndocs, work, layout, st, sms);
    default: return launch_chat_walk_g1(P, doc0, ndocs, work, layout, st, sms);   // OpenAI / Azure; a schema without a planner declines every document with AIGW_R_SCHEMA
  }
}

// fused small-batch kernel (one CTA per document, bodies of at most 5120 bytes): chat_walk_impl.cuh
cudaError_t launch_chat_small(const ChatParams& P, uint32_t doc0, uint32_t ndocs, const uint64_t* out_slot, cudaStream_t st) {
  const uint32_t s = P.schema;
  if (s & (uint32_t)AIGW_SCHEMA_RERANK) return launch_chat_small_g12(P, doc0, ndocs, out_slot, st);
  if (s & (uint32_t)AIGW_SCHEMA_COMPLETIONS) return launch_chat_small_g11(P, doc0, ndocs, out_slot, st);
  if (s & (uint32_t)AIGW_SCHEMA_RESPONSES) return launch_chat_small_g10(P, doc0, ndocs, out_slot, st);
  if (s & (uint32_t)AIGW_SCHEMA_MESSAGES)
    return ((s & 15u) == (uint32_t)AIGW_SCHEMA_OPENAI || (s & 15u) == (uint32_t)AIGW_SCHEMA_AWS_BEDROCK) ? launch_chat_small_g9(P, doc0, ndocs, out_slot, st) : launch_chat_small_g7(P, doc0, ndocs, out_slot, st);
  if ((s & 56u) == (uint32_t)AIGW_SCHEMA_RESP_ERROR) return launch_chat_small_g8(P, doc0, ndocs, out_slot, st);
  if ((s & 48u) == (uint32_t)AIGW_SCHEMA_RESP_AWS_BEDROCK)
    return ((s & 15u) == (uint32_t)AIGW_SCHEMA_GCP_ANTHROPIC || (s & 15u) == (uint32_t)AIGW_SCHEMA_ANTHROPIC) ? launch_chat_small_g5(P, doc0, ndocs, out_slot, st) : launch_chat_small_g4(P, doc0, ndocs, out_slot, st);
  if (s & (uint32_t)AIGW_SCHEMA_EMBEDDINGS) return launch_chat_small_g6(P, doc0, ndocs, out_slot, st);
  switch (s) {
    case AIGW_SCHEMA_AWS_BEDROCK: return launch_chat_small_g0(P, doc0, ndocs, out_slot, st);
    case AIGW_SCHEMA_GCP_ANTHROPIC: case AIGW_SCHEMA_AWS_ANTHROPIC: return launch_chat_small_g2(P, doc0, ndocs, out_slot, st);
    case AIGW_SCHEMA_GCP_VERTEX: return launch_chat_small_g3(P, doc0, ndocs, out_slot, st);
    default: return launch_chat_small_g1(P, doc0, ndocs, out_slot, st);
  }
}

}  // namespace aigw
