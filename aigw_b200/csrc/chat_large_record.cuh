// The CTA slice of the large-request chat kernels that rebuild the body (chat_bedrock_large_kernel.cu,
// chat_anthropic_large_kernel.cu): their record is an unbounded list of copy ops (chat_large_record_impl.cuh).  Both run on
// ChatLargeParams (chat_large_kernel.cuh) with max_len set.
#pragma once
#include "chat_large_kernel.cuh"

namespace aigw {

// The CTA's slice: chat_large_kernel's (token words, jump table, escape counts, the "arguments" text in hand), then
//   ops        rec_op_cap(max_len) copy ops of 16 bytes: a body span, a literal or a scratch span, with its output end
//   scratch    rec_rs_cap(max_len) bytes of re-spelled strings and the configuration text of the ":path" and body, then
//              kRecArgOut bytes of re-serialised tool-call arguments
// A request may plan len / 2 + 4096 ops (AIGW_R_OPS above).  A body span is merged with the span before it when they touch, so
// realistic requests stay far below it; a string that alternates re-spelled escapes with single plain bytes ("\/a" repeated: a
// scratch op and a body op per three bytes) passes it at about 25 KB.
__host__ __device__ inline uint32_t rec_op_cap(uint32_t len) { return len / 2u + 4096u; }
// a re-spelled string is at most three times its bytes (a backslash-b becomes a six-byte u-escape), the escaped model of the
// ":path" three times the model's bytes (or of the override's 128), the api-version its 64 bytes: the scratch never runs out for a
// body below max_len
__host__ __device__ inline uint32_t rec_rs_cap(uint32_t len) { return 3u * len + 1024u; }
// the arguments of a request re-serialise to at most their unescaped bytes (kChatArgTotal in all): compact, the same strings, a
// canonical number is a prefix of the number it was
static constexpr uint32_t kRecArgOut = kChatArgTotal + 1024u;
// a record (":path" and body) above this declines with AIGW_R_OUT_SPACE and body_len 0
static constexpr uint32_t kRecOutCeiling = 0xfffffff0u;

uint64_t chat_record_large_slice_bytes(uint32_t max_len);
int chat_record_large_grid(int sm_count, uint32_t max_len);

}  // namespace aigw
