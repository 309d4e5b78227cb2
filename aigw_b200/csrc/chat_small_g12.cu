// Fused small-batch kernel (index + walk + emit, one CTA per document) for schema group 12; see chat_walk_impl.cuh.
#define AIGW_WALK_GROUP 12
#define AIGW_WALK_SMALL 1
#include "chat_walk_impl.cuh"
