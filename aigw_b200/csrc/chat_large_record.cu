// The slice and grid of the large-request chat kernels that rebuild the body (chat_large_record.cuh).
#include "chat_large_record.cuh"

#include "large_request.cuh"

namespace aigw {

uint64_t chat_record_large_slice_bytes(uint32_t max_len) {
  const uint64_t tc = chat_large_tok_cap(max_len);
  const uint64_t toks = tc * 4u * 2u + 8u + (tc + 1u) * 8u;                                       // words, jump table, escape counts
  const uint64_t args = (uint64_t)(kChatArgMax + 2u) * (8u + 4u + 4u) + kChatArgMax + 16u + 16u;   // the "arguments" text in hand
  const uint64_t ops = (uint64_t)rec_op_cap(max_len) * 16u;
  const uint64_t scr = (uint64_t)rec_rs_cap(max_len) + kRecArgOut;
  return (toks + args + ops + scr + 255u) & ~255ull;
}

int chat_record_large_grid(int sm_count, uint32_t max_len) {
  uint64_t g = kClWorkspace / chat_record_large_slice_bytes(max_len);
  if (g > (uint64_t)sm_count * 2u) g = (uint64_t)sm_count * 2u;
  return g < 1 ? 1 : (int)g;
}

}  // namespace aigw
