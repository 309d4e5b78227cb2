// aigw_b200 — route/backend body mutation (B1) for sm_90a.
//
// Replaces BodyMutator.Mutate (internal/bodymutator/body_mutator.go:77-119) as applied by applyBodyMutation
// (internal/extproc/util.go:107-131) to the translated request body, or to the original one when the translator left it
// unchanged: sjson.DeleteBytes of every `remove` key, then sjson.SetRawBytes / SetBytes of every `set` key, all top-level
// (internal/filterapi/filterconfig.go:258-277).
//
// The sequential edits commute into one pass because every path is a distinct top-level key (the host folds the
// configured lists into per-key actions): a member is kept, deleted, or has its value replaced; keys that are set but
// absent (or removed first) are appended before the root's closing brace in configuration order.  sjson's comma rule for
// deletes (the comma in front goes, or the one behind for the first member) leaves exactly `alive members joined by ","`
// whenever the object has no whitespace between members; bodies that do have such whitespace and need a delete are
// declined, the one place where the byte result would depend on which comma sjson happened to take.
//
// Mapping: one warp per body.  The body is staged in shared memory; per 1 KiB round each lane classifies 32 bytes
// (string interior through the quote/backslash carry chain, braces, commas, whitespace), a warp prefix sum of the brace
// deltas gives every lane its starting depth, and the depth-1 commas plus the root braces become the member separators.
// One lane per member parses `"key" : value` and matches the key table; lane 0 folds the member actions into a short list
// of copy pieces (maximal input runs, replacement values, appended members); the warp copies the pieces to the output
// arena (bump allocated, 16-byte aligned like the translate records).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/aigw_b200.h"

namespace aigw {

constexpr int kMutMaxKeys = 16;
constexpr int kMutTextCap = 3072;

struct MutateKey { uint16_t name_off, name_len;   // bare key bytes (for matching)
                   uint16_t memb_off, memb_len;   // `"key":value` text to append
                   uint16_t val_off, val_len;     // raw replacement value
                   uint8_t remove, set; uint16_t pad; };

struct MutateParams {
  const uint8_t* bodies; const uint64_t* offsets; const uint32_t* lens; uint32_t n;
  uint8_t* out; uint64_t out_capacity; uint64_t out_bias;
  aigw_mut_result* results;
  unsigned long long* out_used;
  unsigned int* next;
  uint32_t n_keys;
  MutateKey keys[kMutMaxKeys];
  char text[kMutTextCap];
};

cudaError_t launch_body_mutate(const MutateParams& P, uint32_t max_len, int sm_count, cudaStream_t st);

}  // namespace aigw
