// Fused small-batch kernel (index + walk + emit, one CTA per document) for schema group 11; see chat_walk_impl.cuh.
#define AIGW_WALK_GROUP 11
#define AIGW_WALK_SMALL 1
#include "chat_walk_impl.cuh"
