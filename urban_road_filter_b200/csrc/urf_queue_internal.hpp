// urf_queue_internal.hpp — what urf_queue.cpp and urf_mq.cpp share (host code, C++ linkage, not part of include/urf.h):
// the timed wait, the scan kinds and the submit behind the submits of both, the two halves of a
// delivery call, which urf_mq needs separately, the copy of a lent scan's labels and order, and the idle rule of the mq's
// settings. urf_mq first asks every device queue how far its run of finished scans reaches, cuts
// the global order at the first scan that is not done, and only then has each queue lend exactly its share.
#pragma once

#include <chrono>
#include <condition_variable>
#include <cstdint>
#include <mutex>

#include "../../include/urf.h"

namespace urf_internal {

// cv.wait(lk, pred) for up to timeout_ms (< 0: forever): false when the time ran out with pred still false.
template <class Pred>
bool wait_for(std::condition_variable& cv, std::unique_lock<std::mutex>& lk, int timeout_ms, Pred pred) {
  if (timeout_ms < 0) { cv.wait(lk, pred); return true; }
  return cv.wait_for(lk, std::chrono::milliseconds(timeout_ms), pred);
}

// What a queue's scans are, and which submits it takes: float4 points (urf_*_submit*), PointCloud2 records of one format
// (urf_*_submit_cloud2*) or of the formats of a table (urf_*_submit_format*).
enum class ScanKind { Float4, Records, Formats };

// URF_OK when q takes scans of `kind` and fmt is the index of one of its formats (0 for the float4 and record kinds);
// URF_ERR_INVALID otherwise.
int queue_check_kind(const urf_queue* q, ScanKind kind, int fmt);

// The submit behind urf_queue_submit* and urf_mq_submit*: queue_check_kind, then data holds n records of the queue's
// format `fmt`; by_reference as urf_queue_submit_ref, otherwise copied into the slot.
int queue_submit(urf_queue* q, ScanKind kind, int fmt, const void* data, int n, uint64_t tag, int timeout_ms, bool by_reference);

// Gives back the slots lent by earlier delivery calls, waits up to timeout_ms (< 0: forever, 0: no wait) until the
// oldest live scan is done, and returns how many consecutive scans from the oldest on are done (at most max_results).
// URF_ERR_TIMEOUT / URF_ERR_CLOSED as for urf_queue_next; with timeout_ms == 0 a queue whose oldest scan is not done
// returns 0 instead of URF_ERR_TIMEOUT.
int queue_done_run(urf_queue* q, int max_results, int timeout_ms);

// Lends the next `count` scans, which queue_done_run has just seen done, in submission order: scan j goes to index dst[j]
// of tags / rcs / outs / label_views (each may be NULL except outs). Returns the number lent.
int queue_lend_run(urf_queue* q, int count, const int* dst, uint64_t* tags, int32_t* rcs, urf_result* outs, const void** label_views);

// The copy-out of urf_queue_next / urf_mq_next for the oldest scan the last delivery call lent: puts the caller's buffers
// (out's members on entry; order and ring_start only with URF_QUEUE_ORDER) back into *out and copies the n_in labels into
// `label` (int32, widened from an int8 slot), and with URF_QUEUE_ORDER the n_order entries of the emission order into
// `order` and n_rings + 1 entries into `ring_start`. NULL buffers are skipped; nothing is copied for a failed scan.
void queue_copy_lent(const urf_queue* q, int32_t* label, int32_t* order, int32_t* ring_start, urf_result* out);

// Makes p (already validated) the set of the queue's next parameter generation: `gen`, or with gen == 0 the queue's last
// plus one. Every scan accepted from now on carries it. Returns the generation, or URF_ERR_CLOSED after urf_queue_close.
// urf_mq passes its own numbers, so that a device queue's results report the mq's generations.
int queue_update_params(urf_queue* q, const urf_params* p, int32_t gen);

// Runs fn(ctx, arg) on the context of every device of the mq, in device order, while nothing is in flight (everything
// submitted has been collected): URF_ERR_INVALID otherwise. Stops at the first error and returns it. Stand-in devices
// (urf_mq_create_with) have no context and are skipped.
int mq_apply_idle(urf_mq* mq, int (*fn)(urf_ctx*, const void*), const void* arg);

}  // namespace urf_internal
