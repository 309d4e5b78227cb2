// K2 (validate + schema walk) for schema group 12; see chat_walk_impl.cuh for the groups and the reason for one kernel per group.
#define AIGW_WALK_GROUP 12
#include "chat_walk_impl.cuh"
