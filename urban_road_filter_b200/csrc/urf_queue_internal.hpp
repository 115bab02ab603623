// urf_queue_internal.hpp — the two pieces of urf_queue_next_batch that urf_mq_next_batch needs separately, and the idle
// rule of the mq's settings (host code, C++ linkage, not part of include/urf.h). urf_mq first asks every device queue how far its run of finished scans reaches,
// cuts the global order at the first scan that is not done, and only then has each queue lend exactly its share.
#pragma once

#include <cstdint>

#include "../../include/urf.h"

namespace urf_internal {

// Gives back the slots lent by earlier urf_queue_next* calls, waits up to timeout_ms (< 0: forever, 0: no wait) until the
// oldest live scan is done, and returns how many consecutive scans from the oldest on are done (at most max_results).
// URF_ERR_TIMEOUT / URF_ERR_CLOSED as for urf_queue_next; with timeout_ms == 0 a queue whose oldest scan is not done
// returns 0 instead of URF_ERR_TIMEOUT.
int queue_done_run(urf_queue* q, int max_results, int timeout_ms);

// Lends the next `count` scans, which queue_done_run has seen done, in submission order: scan j goes to index dst[j] of
// tags / rcs / outs / label_views (each may be NULL except outs). Returns the number lent.
int queue_lend_run(urf_queue* q, int count, const int* dst, uint64_t* tags, int32_t* rcs, urf_result* outs, const void** label_views);

// Runs fn(ctx, arg) on the context of every device of the mq, in device order, while nothing is in flight (everything
// submitted has been collected): URF_ERR_INVALID otherwise. Stops at the first error and returns it. Stand-in devices
// (urf_mq_create_with) have no context and are skipped.
int mq_apply_idle(urf_mq* mq, int (*fn)(urf_ctx*, const void*), const void* arg);

}  // namespace urf_internal
