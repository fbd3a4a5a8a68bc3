// SUBSCRIBE side of the single-call front end.  RetainStorage::get is called once per subscription, from many session tasks
// (rmqtt/src/session.rs:1336-1357); a reconnect storm resubscribes thousands of sessions at once.  The retained batcher is
// batcher.cpp's queue and dispatchers over gm_retain_match_batch: one filter per gm_submit, the handles of the retained
// messages it matches in the callback.  (Kept out of batcher.cpp so that the PUBLISH front end references only gm_match_batch.)
#include "batcher_internal.h"

namespace {
const gm::BatcherTarget kRetained{gm_retain_match_batch, "gm_retain_match_batch", false};
}

extern "C" {

int32_t gm_retain_batcher_create(gm_engine* e, const gm_batcher_config* cfg, gm_batcher** out) { return gm::batcher_create(e, cfg, kRetained, out); }

int32_t gm_retain_batcher_probe(gm_engine* e, const char* blob, const uint32_t* offsets, uint64_t n, uint32_t burst, uint32_t rounds, uint32_t max_wait_us,
                                gm_latency* out) {
    return gm::batcher_probe(e, kRetained, blob, offsets, n, burst, rounds, max_wait_us, out);
}

}  // extern "C"
