// Internals shared by the single-call front ends: batcher.cpp's queue, dispatchers and latency probe serve every engine call
// of the gm_match_batch shape.  gm_batcher_* dispatch to gm_match_batch; retain_batcher.cpp's gm_retain_batcher_* to
// gm_retain_match_batch.  Not part of the public ABI (include/gpumqtt.h).
#pragma once
#include "../../include/gpumqtt.h"

namespace gm {

using BatchCall = int32_t (*)(gm_engine* e, const char* blob, const uint32_t* offsets, uint64_t n, gm_span* out_spans, uint32_t* out_ids, uint64_t cap_ids,
                              uint64_t* needed, int32_t* status);

// what a batcher dispatches to: the engine call, its name (error messages) and whether gm_submit_publish may feed it (a
// PUBLISH topic is a topic name, not a filter)
struct BatcherTarget { BatchCall call; const char* name; bool raw_packets; };

int32_t batcher_create(gm_engine* e, const gm_batcher_config* cfg, const BatcherTarget& target, gm_batcher** out);
int32_t batcher_probe(gm_engine* e, const BatcherTarget& target, const char* blob, const uint32_t* offsets, uint64_t n, uint32_t burst, uint32_t rounds,
                      uint32_t max_wait_us, gm_latency* out);

}  // namespace gm
