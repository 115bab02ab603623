// urf_queue.cpp — streaming ingest in front of urf_process_batch (include/urf.h, SURVEY.md §8 f4). Host code only.
//
// Replaces the reference's depth-1 subscriber (`nh->subscribe(params::topicName, 1, &Detector::filtered, this)`,
// lidar_segmentation.cpp:53): scans that arrive while a scan is being processed are staged instead of dropped, and the
// worker hands everything that is pending to one batched call.
//
// Slot life cycle (all transitions under one mutex):
//   FREE -> FILLING (producer copies the scan, lock released) -> PENDING -> RUNNING (worker) -> DONE -> FREE (consumer)
//   PENDING -> FREE when URF_QUEUE_DROP_OLDEST needs room (the scan is counted as dropped, never delivered).
// Results are delivered in submission order: every accepted scan gets a sequence number when it becomes PENDING and the
// consumer waits for the smallest live one. urf_queue_next_batch hands out the whole run of DONE slots that follows it.
//
// Label slots are int32, or int8 with URF_QUEUE_LABEL8: the worker then asks the batch body for one-byte labels (float4
// queues go through urf_enqueue_cloud2_batch with 16-byte records, as the synchronous path went through
// urf_process_cloud2_batch).
//
// On a real context the worker keeps two batches in flight (urf_enqueue_batch / urf_finish_batch): it enqueues what is
// pending, enqueues the next pending run too if there is one, and only then waits for the oldest batch, so the copies of
// one batch overlap the kernels of the other and the device does not wait for the host's round trip between batches.
#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <cstddef>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <mutex>
#include <thread>
#include <vector>

#include "../../include/urf.h"
#include "urf_queue_internal.hpp"

namespace {
enum SlotState { FREE = 0, FILLING, PENDING, RUNNING, DONE, VIEWED };   // VIEWED: delivered, its labels lent to the consumer
struct Slot {
  SlotState state = FREE;
  uint64_t seq = 0, tag = 0;
  int n = 0, rc = URF_OK;
  float* in = nullptr;       // max_points * bytes_per_point bytes (pinned for the real queue)
  const float* ext = nullptr;   // urf_queue_submit_ref: the caller's buffer is used in place (no copy)
  int32_t* label = nullptr;  // max_points; NULL in a real URF_QUEUE_LABEL8 queue
  int8_t* label8 = nullptr;  // max_points, URF_QUEUE_LABEL8 only
  urf_result res{};
};
}  // namespace

struct urf_queue {
  urf_ctx* ctx = nullptr;                  // real queue: batches go through urf_enqueue*_batch / urf_finish_batch
  urf_queue_process_fn fn = nullptr;       // stand-in, synchronous (urf_queue_create_with)
  urf_queue_process_fn enq = nullptr;      // stand-in, asynchronous pair (urf_queue_create_with_async)
  urf_queue_finish_fn fin = nullptr;
  void* user = nullptr;
  bool pinned = false;
  int max_points = 0, max_batch = 1, policy = URF_QUEUE_BLOCK;
  bool label8 = false;         // URF_QUEUE_LABEL8: int8 label slots
  // record format of the scans: step == 0: (x, y, z, intensity) float4 points; step > 0: raw PointCloud2 records of `step`
  // bytes (urf_queue_create_cloud2), handed to urf_process_cloud2_batch and unpacked on the device
  int step = 0, ox = 0, oy = 4, oz = 8, oi = -1;
  size_t bytes_per_point = 16;
  std::vector<Slot> slots;
  std::mutex mu;
  std::condition_variable cv_free, cv_pending, cv_done;
  uint64_t next_seq = 1;       // sequence number of the next accepted scan
  std::vector<int> lent;       // slots lent out by urf_queue_next_view / _next_batch, given back on the consumer's next call
  std::vector<std::pair<uint64_t, int>> live;   // consumer scratch (under mu): live slots in submission order
  bool closed = false;
  urf_queue_stats st{};
  std::thread worker;
};

namespace {

template <class Pred>
bool wait_for(std::condition_variable& cv, std::unique_lock<std::mutex>& lk, int timeout_ms, Pred pred) {
  if (timeout_ms < 0) { cv.wait(lk, pred); return true; }
  return cv.wait_for(lk, std::chrono::milliseconds(timeout_ms), pred);
}

// One batch of the worker: the slots it took and the arguments of its batch call (which must outlive an asynchronous
// batch until its finish).
struct Run {
  std::vector<int> idx;
  std::vector<const float*> ptrs;
  std::vector<int> ns;
  std::vector<urf_result> outs;
  std::vector<int8_t*> l8;
};

// Takes every pending scan, oldest first, up to max_batch, into r (the slots become RUNNING: from here on they count as
// started and DROP_OLDEST no longer drops them). wait: first block until a scan is pending or the queue is closed.
// Returns the number taken; *closed tells whether the queue was closed.
int take_run(urf_queue* q, Run& r, bool wait, bool* closed) {
  r.idx.clear();
  {
    std::unique_lock<std::mutex> lk(q->mu);
    if (wait)
      q->cv_pending.wait(lk, [&] {
        if (q->closed) return true;
        for (const Slot& s : q->slots) if (s.state == PENDING) return true;
        return false;
      });
    for (;;) {
      int best = -1;
      for (int i = 0; i < (int)q->slots.size(); i++) {
        const Slot& s = q->slots[i];
        if (s.state == PENDING && (best < 0 || s.seq < q->slots[best].seq)) best = i;
      }
      if (best < 0 || (int)r.idx.size() >= q->max_batch) break;
      q->slots[best].state = RUNNING;
      r.idx.push_back(best);
    }
    *closed = q->closed;
    if (r.idx.empty()) return 0;
    q->st.batches++;
    if ((int)r.idx.size() > q->st.largest_batch) q->st.largest_batch = (int)r.idx.size();
  }
  const int B = (int)r.idx.size();
  r.ptrs.resize(B); r.ns.resize(B); r.l8.resize(B); r.outs.assign(B, urf_result{});
  for (int j = 0; j < B; j++) {                           // RUNNING slots belong to the worker: read outside the lock
    const Slot& s = q->slots[r.idx[j]];
    r.ptrs[j] = s.ext ? s.ext : s.in; r.ns[j] = s.n;
    r.outs[j].label = s.label;                            // NULL in a real int8 queue: no int32 label copy is issued
    r.l8[j] = s.label8;
  }
  return B;
}

// Publishes a finished (or failed) run: its slots become DONE with status rc.
void complete_run(urf_queue* q, const Run& r, int rc) {
  if (!q->ctx && q->label8 && rc == URF_OK)               // a stand-in writes int32 labels: the queue narrows them into the slot
    for (int i : r.idx) {
      const Slot& s = q->slots[i];
      for (int k = 0; k < s.n; k++) s.label8[k] = (int8_t)s.label[k];
    }
  {
    std::lock_guard<std::mutex> lk(q->mu);
    for (size_t j = 0; j < r.idx.size(); j++) {
      Slot& s = q->slots[r.idx[j]];
      s.res = r.outs[j]; s.rc = rc; s.state = DONE;
      q->st.processed++;
    }
  }
  q->cv_done.notify_all();
}

int enqueue_run(urf_queue* q, Run& r) {
  const int B = (int)r.idx.size();
  if (q->enq) return q->enq(q->user, r.ptrs.data(), r.ns.data(), B, r.outs.data());
  if (q->step == 0 && !q->label8) return urf_enqueue_batch(q->ctx, r.ptrs.data(), r.ns.data(), B, r.outs.data(), nullptr);
  // float4 scans with int8 labels are 16-byte records (x, y, z, intensity at 0, 4, 8, 12) to the record body
  const bool f4 = q->step == 0;
  return urf_enqueue_cloud2_batch(q->ctx, reinterpret_cast<const void* const*>(r.ptrs.data()), r.ns.data(), B, f4 ? 16 : q->step,
                                  f4 ? 0 : q->ox, f4 ? 4 : q->oy, f4 ? 8 : q->oz, f4 ? 12 : q->oi, r.outs.data(),
                                  q->label8 ? r.l8.data() : nullptr);
}

void note_in_flight(urf_queue* q, int k) {
  std::lock_guard<std::mutex> lk(q->mu);
  if (k > q->st.most_in_flight) q->st.most_in_flight = k;
}

// Synchronous stand-in (urf_queue_create_with): one batch call at a time.
void worker_loop_sync(urf_queue* q) {
  Run r;
  for (;;) {
    bool closed = false;
    if (!take_run(q, r, true, &closed)) { if (closed) return; continue; }
    note_in_flight(q, 1);
    complete_run(q, r, q->fn(q->user, r.ptrs.data(), r.ns.data(), (int)r.idx.size(), r.outs.data()));
  }
}

// Two batches in flight: enqueue what is pending, enqueue the next pending run while a batch slot is free, then finish the
// oldest batch. The queue drains what was accepted before a close before the worker returns.
void worker_loop_async(urf_queue* q) {
  std::deque<Run> flight;                                 // enqueued, oldest first (at most two)
  for (;;) {
    while (flight.size() < 2) {
      Run r;
      bool closed = false;
      if (!take_run(q, r, flight.empty(), &closed)) {
        if (flight.empty() && closed) return;
        break;
      }
      const int rc = enqueue_run(q, r);
      if (rc != URF_OK) { complete_run(q, r, rc); continue; }   // nothing of a refused batch is in flight
      flight.push_back(std::move(r));                     // the vectors' storage, which the batch points at, moves along
      note_in_flight(q, (int)flight.size());
    }
    if (flight.empty()) continue;
    const int rc = q->fin ? q->fin(q->user) : urf_finish_batch(q->ctx);
    complete_run(q, flight.front(), rc);
    flight.pop_front();
  }
}

void worker_loop(urf_queue* q) {
  if (q->fn) worker_loop_sync(q);
  else worker_loop_async(q);
}

void free_slot(const urf_queue* q, Slot& s) {
  for (void* p : {(void*)s.in, (void*)s.label, (void*)s.label8}) {
    if (q->pinned) urf_pinned_free(p); else std::free(p);
  }
  s.in = nullptr; s.label = nullptr; s.label8 = nullptr;
}

// Exactly one of ctx (real queue, pinned slots), fn (synchronous stand-in) and enq + fin (asynchronous stand-in) is set.
int create_common(urf_queue** out, urf_ctx* ctx, urf_queue_process_fn fn, urf_queue_process_fn enq, urf_queue_finish_fn fin, void* user,
                  int max_points, int slots, int max_batch, int policy, int step = 0, int ox = 0, int oy = 4, int oz = 8, int oi = -1) {
  const bool label8 = (policy & URF_QUEUE_LABEL8) != 0;
  policy &= ~URF_QUEUE_LABEL8;
  if (!out || (!ctx && !fn && !(enq && fin)) || max_points < 1 || slots < 1 || max_batch < 1 ||
      (policy != URF_QUEUE_BLOCK && policy != URF_QUEUE_DROP_OLDEST))
    return URF_ERR_INVALID;
  const bool pinned = ctx != nullptr;
  urf_queue* q = new urf_queue;
  q->ctx = ctx; q->fn = fn; q->enq = enq; q->fin = fin; q->user = user;
  q->pinned = pinned; q->max_points = max_points; q->max_batch = max_batch; q->policy = policy;
  q->label8 = label8;
  q->step = step; q->ox = ox; q->oy = oy; q->oz = oz; q->oi = oi;
  q->bytes_per_point = step > 0 ? (size_t)step : 16;
  q->slots.resize(slots);
  // int8 slots hold max_points bytes of labels; a stand-in batch function still writes int32 labels, which need a buffer
  const bool want32 = !label8 || !ctx, want8 = label8;
  auto alloc = [pinned](size_t bytes) { return pinned ? urf_pinned_alloc(bytes) : std::malloc(bytes); };
  for (Slot& s : q->slots) {
    const size_t in_bytes = q->bytes_per_point * (size_t)max_points;
    s.in = static_cast<float*>(alloc(in_bytes));
    if (want32) s.label = static_cast<int32_t*>(alloc(sizeof(int32_t) * (size_t)max_points));
    if (want8) s.label8 = static_cast<int8_t*>(alloc((size_t)max_points));
    if (!s.in || (want32 && !s.label) || (want8 && !s.label8)) {
      for (Slot& t : q->slots) free_slot(q, t);
      delete q;
      return URF_ERR_NOMEM;
    }
  }
  q->worker = std::thread(worker_loop, q);
  *out = q;
  return URF_OK;
}

}  // namespace

extern "C" {

int urf_queue_create(urf_queue** out, urf_ctx* ctx, int max_points, int slots, int max_batch, int policy) {
  if (!ctx) return URF_ERR_INVALID;
  return create_common(out, ctx, nullptr, nullptr, nullptr, nullptr, max_points, slots, max_batch, policy);
}

int urf_queue_create_cloud2(urf_queue** out, urf_ctx* ctx, int max_points, int slots, int max_batch, int policy, int point_step, int off_x,
                            int off_y, int off_z, int off_intensity) {
  if (!ctx || point_step < 12 || point_step > URF_MAX_POINT_STEP) return URF_ERR_INVALID;
  for (int o : {off_x, off_y, off_z}) if (o < 0 || o + 4 > point_step) return URF_ERR_INVALID;
  if (off_intensity >= 0 && off_intensity + 4 > point_step) return URF_ERR_INVALID;
  return create_common(out, ctx, nullptr, nullptr, nullptr, nullptr, max_points, slots, max_batch, policy, point_step, off_x, off_y, off_z,
                       off_intensity);
}

int urf_queue_create_with(urf_queue** out, urf_queue_process_fn fn, void* user, int max_points, int slots, int max_batch, int policy) {
  if (!fn) return URF_ERR_INVALID;
  return create_common(out, nullptr, fn, nullptr, nullptr, user, max_points, slots, max_batch, policy);
}

int urf_queue_create_with_async(urf_queue** out, urf_queue_process_fn enqueue, urf_queue_finish_fn finish, void* user, int max_points,
                                int slots, int max_batch, int policy) {
  if (!enqueue || !finish) return URF_ERR_INVALID;
  return create_common(out, nullptr, nullptr, enqueue, finish, user, max_points, slots, max_batch, policy);
}

namespace {
int submit_common(urf_queue* q, const void* data, int n, uint64_t tag, int timeout_ms, bool by_reference) {
  if (!q || n < 0 || (n > 0 && !data)) return URF_ERR_INVALID;
  if (n > q->max_points) return URF_ERR_CAPACITY;
  int slot = -1;
  {
    std::unique_lock<std::mutex> lk(q->mu);
    auto find = [&] {
      if (q->closed) return true;
      for (int i = 0; i < (int)q->slots.size(); i++) if (q->slots[i].state == FREE) { slot = i; return true; }
      if (q->policy == URF_QUEUE_DROP_OLDEST) {           // lidar_segmentation.cpp:53: the subscriber keeps only the newest scan
        int best = -1;
        for (int i = 0; i < (int)q->slots.size(); i++) {
          const Slot& s = q->slots[i];
          if (s.state == PENDING && (best < 0 || s.seq < q->slots[best].seq)) best = i;
        }
        if (best >= 0) { q->st.dropped++; slot = best; return true; }
      }
      return false;
    };
    if (!wait_for(q->cv_free, lk, timeout_ms, find)) return URF_ERR_TIMEOUT;
    if (q->closed) return URF_ERR_CLOSED;
    q->slots[slot].state = FILLING;                       // a dropped scan's sequence number simply never reaches DONE
  }
  Slot& s = q->slots[slot];
  bool closed_late = false;
  if (by_reference) s.ext = static_cast<const float*>(data);
  else { s.ext = nullptr; if (n > 0) std::memcpy(s.in, data, q->bytes_per_point * (size_t)n); }
  {
    std::lock_guard<std::mutex> lk(q->mu);
    if (q->closed) {                                      // closed while copying: the worker may already be gone
      s.state = FREE;
      closed_late = true;
    } else {
      s.n = n; s.tag = tag; s.rc = URF_OK;
      s.seq = q->next_seq++;
      s.state = PENDING;
      q->st.submitted++;
    }
  }
  if (closed_late) {
    // a consumer whose last look at the slots still saw this one FILLING must get to see the drained state: close()'s
    // own notify may have come before that look
    q->cv_done.notify_all();
    q->cv_free.notify_one();
    return URF_ERR_CLOSED;
  }
  q->cv_pending.notify_one();
  q->cv_done.notify_all();                                // a consumer waiting on a dropped sequence number re-evaluates
  return URF_OK;
}
}  // namespace

int urf_queue_submit(urf_queue* q, const float* xyzi, int n, uint64_t tag, int timeout_ms) {
  if (q && q->step != 0) return URF_ERR_INVALID;           // a record queue takes urf_queue_submit_cloud2
  return submit_common(q, xyzi, n, tag, timeout_ms, false);
}

int urf_queue_submit_ref(urf_queue* q, const float* xyzi, int n, uint64_t tag, int timeout_ms) {
  if (q && q->step != 0) return URF_ERR_INVALID;
  return submit_common(q, xyzi, n, tag, timeout_ms, true);
}

int urf_queue_submit_cloud2(urf_queue* q, const void* data, int n_points, uint64_t tag, int timeout_ms) {
  if (q && q->step == 0) return URF_ERR_INVALID;
  return submit_common(q, data, n_points, tag, timeout_ms, false);
}

namespace {
int next_common(urf_queue* q, uint64_t* tag, urf_result* out, const int32_t** label_view, int timeout_ms);
}

int urf_queue_next(urf_queue* q, uint64_t* tag, urf_result* out, int timeout_ms) { return next_common(q, tag, out, nullptr, timeout_ms); }

int urf_queue_next_view(urf_queue* q, uint64_t* tag, urf_result* out, const int32_t** label_view, int timeout_ms) {
  if (!label_view || (q && q->label8)) return URF_ERR_INVALID;         // int8 slots have no int32 view: urf_queue_next_batch
  return next_common(q, tag, out, label_view, timeout_ms);
}

namespace {
// Gives the slots lent by the previous urf_queue_next_view / _next_batch call back to the producers (mu held).
void release_lent(urf_queue* q) {
  if (q->lent.empty()) return;
  for (int i : q->lent) q->slots[i].state = FREE;
  q->lent.clear();
  q->cv_free.notify_all();
}

// The oldest live scan (smallest sequence number among PENDING / RUNNING / DONE slots): 1 and *slot when it is DONE,
// 2 when the queue is closed and drained, 0 otherwise (mu held).
int front_state(const urf_queue* q, int* slot) {
  int best = -1;
  bool filling = false;
  for (int i = 0; i < (int)q->slots.size(); i++) {
    const Slot& s = q->slots[i];
    if (s.state == FILLING) filling = true;
    if ((s.state == PENDING || s.state == RUNNING || s.state == DONE) && (best < 0 || s.seq < q->slots[best].seq)) best = i;
  }
  if (best >= 0 && q->slots[best].state == DONE) { *slot = best; return 1; }
  if (best < 0 && !filling && q->closed) return 2;
  return 0;
}

// Waits up to timeout_ms until the oldest live scan is done: URF_OK, URF_ERR_TIMEOUT or URF_ERR_CLOSED (mu held).
int wait_front(urf_queue* q, std::unique_lock<std::mutex>& lk, int timeout_ms, int* slot) {
  int state = 0;
  if (!wait_for(q->cv_done, lk, timeout_ms, [&] { return (state = front_state(q, slot)) != 0; })) return URF_ERR_TIMEOUT;
  return state == 2 ? (int)URF_ERR_CLOSED : (int)URF_OK;
}

// The run of DONE slots at the front, in submission order, at most max_results of them, into q->live (mu held).
// A dropped scan's slot was reused and carries a new sequence number, so it is skipped like in urf_queue_next.
int done_run(urf_queue* q, int max_results) {
  q->live.clear();
  for (int i = 0; i < (int)q->slots.size(); i++) {
    const SlotState st = q->slots[i].state;
    if (st == PENDING || st == RUNNING || st == DONE) q->live.emplace_back(q->slots[i].seq, i);
  }
  std::sort(q->live.begin(), q->live.end());
  int k = 0;
  while (k < (int)q->live.size() && k < max_results && q->slots[q->live[k].second].state == DONE) k++;
  q->live.resize(k);
  return k;
}

// Marks the k slots of q->live as lent (invisible to producers and the worker until release_lent) (mu held).
void lend(urf_queue* q, int k) {
  for (int j = 0; j < k; j++) { q->slots[q->live[j].second].state = VIEWED; q->lent.push_back(q->live[j].second); }
  q->st.delivered += (uint64_t)k;
}

// The fields of a finished scan the consumer gets: counts and flags, and only the n_vert vertices that exist.
void copy_result(urf_result* dst, const urf_result& src) {
  std::memcpy(dst, &src, offsetof(urf_result, label));
  dst->label = nullptr; dst->ring = nullptr; dst->order = nullptr; dst->ring_start = nullptr;
  const int nv = std::min(std::max(src.n_vert, 0), URF_MAX_VERTS);
  std::memcpy(dst->vert, src.vert, sizeof(src.vert[0]) * (size_t)nv);
}

// Hands out the slots lent by lend(): slot[j] goes to index dst ? dst[j] : j. Runs outside the lock (the slots are ours).
void hand_out(const urf_queue* q, const int* slot, int k, const int* dst, uint64_t* tags, int32_t* rcs, urf_result* outs,
              const void** label_views) {
  for (int j = 0; j < k; j++) {
    const Slot& s = q->slots[slot[j]];
    const int o = dst ? dst[j] : j;
    if (tags) tags[o] = s.tag;
    if (rcs) rcs[o] = s.rc;
    copy_result(&outs[o], s.res);
    if (label_views) label_views[o] = s.rc != URF_OK ? nullptr : q->label8 ? (const void*)s.label8 : (const void*)s.label;
  }
}

// label_view != NULL: no copy — *label_view points at the labels inside the queue's staging slot, which stays reserved
// (not reusable by producers) until this consumer's next urf_queue_next* call on the queue.
int next_common(urf_queue* q, uint64_t* tag, urf_result* out, const int32_t** label_view, int timeout_ms) {
  if (!q || !out) return URF_ERR_INVALID;
  std::unique_lock<std::mutex> lk(q->mu);
  release_lent(q);                                        // the slots lent out by the previous call come back now
  int slot = -1;
  const int wrc = wait_front(q, lk, timeout_ms, &slot);
  if (wrc != URF_OK) return wrc;
  Slot& s = q->slots[slot];
  int32_t* user_label = out->label;
  const int rc = s.rc;
  *out = s.res;
  out->label = user_label; out->ring = nullptr; out->order = nullptr; out->ring_start = nullptr;
  if (tag) *tag = s.tag;
  q->st.delivered++;
  if (label_view) {                                       // lend the slot: DONE slots are invisible to producers and the worker
    *label_view = rc == URF_OK ? s.label : nullptr;
    s.state = VIEWED;
    q->lent.push_back(slot);
    return rc;
  }
  const int n = s.n;
  s.state = VIEWED;                                       // ours: invisible to producers, the worker and other consumers
  lk.unlock();                                            // the copy runs outside the lock
  if (user_label && rc == URF_OK && n > 0) {
    if (q->label8) for (int i = 0; i < n; i++) user_label[i] = s.label8[i];      // int8 slot: widened for the caller
    else std::memcpy(user_label, s.label, sizeof(int32_t) * (size_t)n);
  }
  lk.lock();
  s.state = FREE;
  lk.unlock();
  q->cv_free.notify_one();
  return rc;
}
}  // namespace

int urf_queue_next_batch(urf_queue* q, int max_results, uint64_t* tags, int32_t* rcs, urf_result* outs, const void** label_views,
                         int timeout_ms) {
  if (!q || !outs || max_results < 1) return URF_ERR_INVALID;
  std::vector<int> idx;
  {
    std::unique_lock<std::mutex> lk(q->mu);               // the only lock round of the call
    release_lent(q);
    int front = -1;
    const int wrc = wait_front(q, lk, timeout_ms, &front);
    if (wrc != URF_OK) return wrc;
    const int k = done_run(q, max_results);               // >= 1: the front is done
    for (int j = 0; j < k; j++) idx.push_back(q->live[j].second);
    lend(q, k);
  }
  hand_out(q, idx.data(), (int)idx.size(), nullptr, tags, rcs, outs, label_views);
  return (int)idx.size();
}

void urf_queue_release_view(urf_queue* q) {
  if (!q) return;
  std::lock_guard<std::mutex> lk(q->mu);
  release_lent(q);
}

int urf_queue_get_stats(urf_queue* q, urf_queue_stats* st) {
  if (!q || !st) return URF_ERR_INVALID;
  std::lock_guard<std::mutex> lk(q->mu);
  *st = q->st;
  st->pending = 0;
  for (const Slot& s : q->slots) if (s.state == PENDING || s.state == RUNNING || s.state == FILLING) st->pending++;
  return URF_OK;
}

void urf_queue_close(urf_queue* q) {
  if (!q) return;
  {
    std::lock_guard<std::mutex> lk(q->mu);
    q->closed = true;
  }
  q->cv_pending.notify_all();
  q->cv_free.notify_all();
  q->cv_done.notify_all();
}

void urf_queue_destroy(urf_queue* q) {
  if (!q) return;
  urf_queue_close(q);
  if (q->worker.joinable()) q->worker.join();             // the worker drains what is pending before it returns
  for (Slot& s : q->slots) free_slot(q, s);
  delete q;
}

}  // extern "C"

namespace urf_internal {

int queue_done_run(urf_queue* q, int max_results, int timeout_ms) {
  std::unique_lock<std::mutex> lk(q->mu);
  release_lent(q);
  int front = -1;
  const int wrc = wait_front(q, lk, timeout_ms, &front);
  if (wrc == URF_ERR_TIMEOUT && timeout_ms == 0) return 0;
  if (wrc != URF_OK) return wrc;
  return done_run(q, max_results);
}

int queue_lend_run(urf_queue* q, int count, const int* dst, uint64_t* tags, int32_t* rcs, urf_result* outs, const void** label_views) {
  std::vector<int> idx;
  {
    std::lock_guard<std::mutex> lk(q->mu);
    // a run that was done stays done (only this consumer takes scans out), so this is the run queue_done_run counted
    const int k = done_run(q, count);
    for (int j = 0; j < k; j++) idx.push_back(q->live[j].second);
    lend(q, k);
  }
  hand_out(q, idx.data(), (int)idx.size(), dst, tags, rcs, outs, label_views);
  return (int)idx.size();
}

}  // namespace urf_internal
