// What engine.cu lends the engine group (group.cu) inside libb200rank.so; none of it is exported.
#pragma once
#include <cstdint>

#include "../../include/b200_rank.h"

#define B200_INTERNAL __attribute__((visibility("hidden")))

// The refusals b200_rank_topk can give a query before it touches the device -- the argument checks, the plan's refusal
// for the whole batch, the host CSR arrays and host object_rows -- with the same codes and messages (B200_OK: none).
// `k_out` gets the columns of the output arrays.
B200_INTERNAL int b200_check_query(const b200_rank_engine* engine, const b200_rank_query* query, int32_t* k_out);

// Sets the message b200_rank_last_error() returns on the calling thread; returns `code`.
B200_INTERNAL int b200_set_error(int code, const char* message);
