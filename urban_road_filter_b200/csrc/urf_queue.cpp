// urf_queue.cpp — streaming ingest in front of urf_process_batch (include/urf.h, SURVEY.md §8 f4). Host code only.
//
// Replaces the reference's depth-1 subscriber (`nh->subscribe(params::topicName, 1, &Detector::filtered, this)`,
// lidar_segmentation.cpp:53): scans that arrive while a scan is being processed are staged instead of dropped, and the
// worker takes everything that is pending (up to max_batch scans) as one batch.
//
// Slot life cycle (all transitions under one mutex):
//   FREE -> FILLING (producer copies the scan, lock released) -> PENDING -> RUNNING (worker) -> DONE -> FREE (consumer)
//   PENDING -> FREE when URF_QUEUE_DROP_OLDEST needs room (the scan is counted as dropped, never delivered).
// Results are delivered in submission order: every accepted scan gets a sequence number when it becomes PENDING and the
// consumer waits for the smallest live one. Every delivery call (urf_queue_next / _next_view / _next_batch, and the mq's)
// takes the run of DONE slots that starts there through take_done_run and hands it out through hand_out.
//
// Label slots are int32, or int8 with URF_QUEUE_LABEL8: the worker then asks the batch body for one-byte labels (float4
// queues go through urf_enqueue_cloud2_batch with 16-byte records, as the synchronous path went through
// urf_process_cloud2_batch). With URF_QUEUE_ORDER a slot also holds the scan's emission order and ring_start: the worker
// points the batch call's outs at them, the batch body fills them as it does for any caller, and delivery lends them with
// the labels.
//
// Scan kinds: float4 points, records of one format (urf_queue_create_cloud2), or records of the formats of a table, each
// submit naming its scan's format (urf_queue_create_formats). A slot holds max_points records of the largest format, remembers
// its scan's format, and a formats queue's run goes to urf_enqueue_cloud2_batch_mixed with each scan's format.
//
// The worker is one loop with a depth. On a real context it keeps two batches in flight (urf_enqueue_batch /
// urf_finish_batch): it enqueues what is pending, enqueues the next pending run too if there is one, and only then waits
// for the oldest batch, so the copies of one batch overlap the kernels of the other and the device does not wait for the
// host's round trip between batches. A synchronous stand-in (urf_queue_create_with) is the same loop at depth 1.
//
// Parameter generations (urf_queue_update_params): a scan is stamped with the queue's generation when it becomes PENDING,
// under the same lock that gives it its sequence number. Generations therefore never decrease along the sequence numbers,
// a run taken oldest-first ends at the first scan of another generation, and the worker applies a run's set to the context
// just before it enqueues the run. `sets` holds the set of each generation a pending scan or the next submit may carry.
#include <algorithm>
#include <cstddef>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <map>
#include <mutex>
#include <thread>
#include <vector>

#include "../../include/urf.h"
#include "urf_params.hpp"
#include "urf_queue_internal.hpp"

using urf_internal::ScanKind;

namespace {
enum SlotState { FREE = 0, FILLING, PENDING, RUNNING, DONE, VIEWED };   // VIEWED: delivered, its labels lent to the consumer
struct Slot {
  SlotState state = FREE;
  uint64_t seq = 0, tag = 0;
  int32_t gen = 0;           // parameter generation in force when the scan became PENDING
  int n = 0, rc = URF_OK;
  int fmt = 0;               // the scan's index into the queue's formats (0 but in a formats queue)
  float* in = nullptr;       // max_points * bytes_per_point bytes (pinned for the real queue)
  const float* ext = nullptr;   // urf_queue_submit_ref / _cloud2_ref: the caller's buffer is used in place (no copy)
  int32_t* label = nullptr;  // max_points; NULL in a real URF_QUEUE_LABEL8 queue
  int8_t* label8 = nullptr;  // max_points, URF_QUEUE_LABEL8 only
  int32_t* order = nullptr;       // max_points, URF_QUEUE_ORDER only: the emission order
  int32_t* ring_start = nullptr;  // URF_MAX_CHANNELS + 1, URF_QUEUE_ORDER only
  urf_result res{};
};
}  // namespace

struct urf_queue {
  urf_ctx* ctx = nullptr;                  // real queue: batches go through urf_enqueue*_batch / urf_finish_batch
  urf_queue_process_fn enq = nullptr;      // stand-in: with fin the asynchronous pair (urf_queue_create_with_async), alone
  urf_queue_finish_fn fin = nullptr;       // the synchronous batch function (urf_queue_create_with), which does it all
  void* user = nullptr;
  urf_queue_params_fn params_fn = nullptr;   // stand-in: called where a real queue's worker calls urf_set_params_next
  bool pinned = false;
  int max_points = 0, max_batch = 1, policy = URF_QUEUE_BLOCK;
  int depth = 2;               // batches the worker keeps in flight: 2, or 1 around a synchronous stand-in
  bool label8 = false;         // URF_QUEUE_LABEL8: int8 label slots
  bool order = false;          // URF_QUEUE_ORDER: every slot also holds the scan's emission order and ring offsets
  // what the scans are: (x, y, z, intensity) float4 points, raw PointCloud2 records of one format (urf_queue_create_cloud2),
  // or records of the formats of a table, each submit naming its own (urf_queue_create_formats); records are handed to the
  // batch body as they are and unpacked on the device
  ScanKind kind = ScanKind::Float4;
  std::vector<urf_cloud2_format> formats;   // float4: {16, 0, 4, 8, 12}; records: the one format; formats: the table
  size_t bytes_per_point = 16;              // the largest point_step of `formats`
  urf_cloud2_user rec{};       // record stand-in (urf_queue_create_cloud2_with): `user` points here, rec.user is the creator's
  urf_formats_user fu{};       // formats stand-in (urf_queue_create_formats_with): the same, with the table and the run's indices
  std::vector<Slot> slots;
  std::mutex mu;
  std::condition_variable cv_free, cv_pending, cv_done;
  uint64_t next_seq = 1;       // sequence number of the next accepted scan
  int32_t gen = 0;             // generation stamped on the next accepted scan
  std::map<int32_t, urf_params> sets;   // generation -> set, from the oldest one a PENDING scan carries up to `gen`
  // Consumer side. The header allows one consumer at a time, so only that thread changes `lent`, and it may read it
  // outside the lock: after a delivery call `lent` is exactly the run that call took, in submission order.
  std::vector<int> lent;       // slots lent out by the last delivery call, given back on the consumer's next call
  std::vector<std::pair<uint64_t, int>> live;   // scratch (under mu): live slots in submission order
  bool closed = false;
  urf_queue_stats st{};
  std::thread worker;
};

namespace {

using urf_internal::wait_for;

// One batch of the worker: the slots it took and the arguments of its batch call (which must outlive an asynchronous
// batch until its finish).
struct Run {
  int32_t gen = 0;             // the generation of every scan of the run
  bool apply = false;          // gen differs from the last one the worker applied: `set` goes to the ctx (or hook) first
  urf_params set{};
  urf_queue_params_fn params_fn = nullptr;
  std::vector<int> idx;
  std::vector<const float*> ptrs;
  std::vector<int> ns;
  std::vector<int32_t> fidx;             // per scan: its index into the queue's formats
  std::vector<urf_cloud2_format> fmts;   // per scan: its format (a formats queue's mixed batch)
  std::vector<urf_result> outs;
  std::vector<int8_t*> l8;
  int rc = URF_OK;             // synchronous stand-in: what the batch function returned, reported by finish_run
};

// Drops the sets no PENDING scan carries, except the current generation's (mu held). A RUNNING scan's set, if its run
// still has to apply it, was copied into the run.
void prune_sets(urf_queue* q) {
  int32_t keep = q->gen;
  for (const Slot& s : q->slots) if (s.state == PENDING) keep = std::min(keep, s.gen);
  q->sets.erase(q->sets.begin(), q->sets.lower_bound(keep));
}

// Takes every pending scan of the oldest pending scan's generation, oldest first, up to max_batch, into r (the slots become
// RUNNING: from here on they count as started and DROP_OLDEST no longer drops them). `applied`: the generation the worker
// last applied; a run of another one carries its set. wait: first block until a scan is pending or the queue is closed.
// Returns the number taken; *closed tells whether the queue was closed.
int take_run(urf_queue* q, Run& r, int32_t applied, bool wait, bool* closed) {
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
      if (r.idx.empty()) r.gen = q->slots[best].gen;
      else if (q->slots[best].gen != r.gen) break;        // a batch never mixes generations
      q->slots[best].state = RUNNING;
      r.idx.push_back(best);
    }
    *closed = q->closed;
    if (r.idx.empty()) return 0;
    // generation 0 has no stored set (it is what the ctx had): generations only grow, so a run of it never follows another
    const auto it = q->sets.find(r.gen);
    r.apply = r.gen != applied && it != q->sets.end();
    if (r.apply) r.set = it->second;
    r.params_fn = q->params_fn;
    prune_sets(q);
    q->st.batches++;
    if ((int)r.idx.size() > q->st.largest_batch) q->st.largest_batch = (int)r.idx.size();
  }
  const int B = (int)r.idx.size();
  r.ptrs.resize(B); r.ns.resize(B); r.fidx.resize(B); r.fmts.resize(B); r.l8.resize(B); r.outs.assign(B, urf_result{});
  for (int j = 0; j < B; j++) {                           // RUNNING slots belong to the worker: read outside the lock
    const Slot& s = q->slots[r.idx[j]];
    r.ptrs[j] = s.ext ? s.ext : s.in; r.ns[j] = s.n;
    r.fidx[j] = s.fmt; r.fmts[j] = q->formats[s.fmt];
    r.outs[j].label = s.label;                            // NULL in a real int8 queue: no int32 label copy is issued
    r.outs[j].order = s.order; r.outs[j].ring_start = s.ring_start;   // NULL without URF_QUEUE_ORDER: no ring sort, no copy
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
      s.res = r.outs[j]; s.res.params_gen = r.gen;        // the queue's numbering, not the context's
      s.rc = rc; s.state = DONE;
      q->st.processed++;
    }
  }
  q->cv_done.notify_all();
}

// Applies run r's set, if it carries one, to the context (its batches already enqueued keep theirs) or the stand-in's hook,
// and records the generation in *applied. A failure fails the run like a refused enqueue.
int apply_run(urf_queue* q, const Run& r, int32_t* applied) {
  if (!r.apply) return URF_OK;
  int rc = URF_OK;
  if (q->ctx) {
    rc = urf_set_params_next(q->ctx, &r.set);
    if (rc > 0) rc = URF_OK;                              // the context's own generation number
  } else if (r.params_fn) {
    rc = r.params_fn(q->user, &r.set, r.gen);
  }
  if (rc == URF_OK) *applied = r.gen;
  return rc;
}

// Starts run r. A synchronous stand-in does all its work here, and that counts as accepted: finish_run reports how it went.
int enqueue_run(urf_queue* q, Run& r) {
  const int B = (int)r.idx.size();
  if (q->enq) {
    q->fu.fmt = r.fidx.data();                            // a formats stand-in's indices, for the call (it is synchronous)
    const int rc = q->enq(q->user, r.ptrs.data(), r.ns.data(), B, r.outs.data());
    q->fu.fmt = nullptr;
    if (q->fin) return rc;
    r.rc = rc;
    return URF_OK;
  }
  if (q->kind == ScanKind::Float4 && !q->label8) return urf_enqueue_batch(q->ctx, r.ptrs.data(), r.ns.data(), B, r.outs.data(), nullptr);
  const auto data = reinterpret_cast<const void* const*>(r.ptrs.data());
  int8_t* const* l8 = q->label8 ? r.l8.data() : nullptr;
  if (q->kind == ScanKind::Formats) return urf_enqueue_cloud2_batch_mixed(q->ctx, data, r.ns.data(), r.fmts.data(), B, r.outs.data(), l8);
  // float4 scans with int8 labels are 16-byte records (x, y, z, intensity at 0, 4, 8, 12) to the record body
  const urf_cloud2_format& f = q->formats[0];
  return urf_enqueue_cloud2_batch(q->ctx, data, r.ns.data(), B, f.point_step, f.off_x, f.off_y, f.off_z, f.off_intensity, r.outs.data(), l8);
}

// Waits for the oldest run in flight, r.
int finish_run(urf_queue* q, const Run& r) { return q->ctx ? urf_finish_batch(q->ctx) : q->fin ? q->fin(q->user) : r.rc; }

// q->depth batches in flight: enqueue what is pending, enqueue the next pending run while a batch slot is free, then finish
// the oldest batch. At depth 1 no second run is taken before the first is published. The queue drains what was accepted
// before a close before the worker returns.
void worker_loop(urf_queue* q) {
  std::deque<Run> flight;                                 // enqueued, oldest first (at most q->depth)
  int32_t applied = 0;                                    // generation of the parameters the last enqueued run used
  for (;;) {
    while ((int)flight.size() < q->depth) {
      Run r;
      bool closed = false;
      if (!take_run(q, r, applied, flight.empty(), &closed)) {
        if (flight.empty() && closed) return;
        break;
      }
      int rc = apply_run(q, r, &applied);
      if (rc == URF_OK) rc = enqueue_run(q, r);
      if (rc != URF_OK) { complete_run(q, r, rc); continue; }   // nothing of a refused batch is in flight
      flight.push_back(std::move(r));                     // the vectors' storage, which the batch points at, moves along
      std::lock_guard<std::mutex> lk(q->mu);
      q->st.most_in_flight = std::max(q->st.most_in_flight, (int32_t)flight.size());
    }
    if (flight.empty()) continue;
    complete_run(q, flight.front(), finish_run(q, flight.front()));
    flight.pop_front();
  }
}

void free_slot(const urf_queue* q, Slot& s) {
  for (void* p : {(void*)s.in, (void*)s.label, (void*)s.label8, (void*)s.order, (void*)s.ring_start}) {
    if (q->pinned) urf_pinned_free(p); else std::free(p);
  }
  s.in = nullptr; s.label = nullptr; s.label8 = nullptr; s.order = nullptr; s.ring_start = nullptr;
}

// Either ctx (real queue, pinned slots) or enq (stand-in; synchronous, and the worker's depth 1, without fin) is set.
// kind Records / Formats: the record formats (one, or the table), which the caller has checked.
int create_common(urf_queue** out, urf_ctx* ctx, urf_queue_process_fn enq, urf_queue_finish_fn fin, void* user,
                  int max_points, int slots, int max_batch, int policy, ScanKind kind = ScanKind::Float4,
                  const urf_cloud2_format* formats = nullptr, int n_formats = 0) {
  const bool label8 = (policy & URF_QUEUE_LABEL8) != 0, order = (policy & URF_QUEUE_ORDER) != 0;
  policy &= ~(URF_QUEUE_LABEL8 | URF_QUEUE_ORDER);
  if (!out || (!ctx && !enq) || max_points < 1 || slots < 1 || max_batch < 1 ||
      (policy != URF_QUEUE_BLOCK && policy != URF_QUEUE_DROP_OLDEST))
    return URF_ERR_INVALID;
  const bool pinned = ctx != nullptr;
  urf_queue* q = new urf_queue;
  q->ctx = ctx; q->enq = enq; q->fin = fin; q->user = user;
  q->pinned = pinned; q->max_points = max_points; q->max_batch = max_batch; q->policy = policy;
  q->label8 = label8; q->order = order; q->depth = ctx || fin ? 2 : 1;
  q->kind = kind;
  if (kind == ScanKind::Float4) q->formats.assign(1, urf_cloud2_format{16, 0, 4, 8, 12});
  else q->formats.assign(formats, formats + n_formats);
  q->bytes_per_point = 0;
  for (const urf_cloud2_format& f : q->formats) q->bytes_per_point = std::max(q->bytes_per_point, (size_t)f.point_step);
  if (!ctx && kind == ScanKind::Records) {
    const urf_cloud2_format& f = q->formats[0];
    q->rec = urf_cloud2_user{user, f.point_step, f.off_x, f.off_y, f.off_z, f.off_intensity};
    q->user = &q->rec;
  }
  if (!ctx && kind == ScanKind::Formats) { q->fu = urf_formats_user{user, q->formats.data(), (int32_t)q->formats.size(), nullptr}; q->user = &q->fu; }
  q->slots.resize(slots); q->lent.reserve(slots); q->live.reserve(slots);
  // int8 slots hold max_points bytes of labels; a stand-in batch function still writes int32 labels, which need a buffer
  const bool want32 = !label8 || !ctx, want8 = label8;
  auto alloc = [pinned](size_t bytes) { return pinned ? urf_pinned_alloc(bytes) : std::malloc(bytes); };
  for (Slot& s : q->slots) {
    const size_t in_bytes = q->bytes_per_point * (size_t)max_points;
    s.in = static_cast<float*>(alloc(in_bytes));
    if (want32) s.label = static_cast<int32_t*>(alloc(sizeof(int32_t) * (size_t)max_points));
    if (want8) s.label8 = static_cast<int8_t*>(alloc((size_t)max_points));
    if (order) {
      s.order = static_cast<int32_t*>(alloc(sizeof(int32_t) * (size_t)max_points));
      s.ring_start = static_cast<int32_t*>(alloc(sizeof(int32_t) * (URF_MAX_CHANNELS + 1)));
    }
    if (!s.in || (want32 && !s.label) || (want8 && !s.label8) || (order && (!s.order || !s.ring_start))) {
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
  return create_common(out, ctx, nullptr, nullptr, nullptr, max_points, slots, max_batch, policy);
}

int urf_queue_create_cloud2(urf_queue** out, urf_ctx* ctx, int max_points, int slots, int max_batch, int policy, int point_step, int off_x,
                            int off_y, int off_z, int off_intensity) {
  const urf_cloud2_format f{point_step, off_x, off_y, off_z, off_intensity};
  if (!ctx || urf::check_cloud2_format(f) != URF_OK) return URF_ERR_INVALID;
  return create_common(out, ctx, nullptr, nullptr, nullptr, max_points, slots, max_batch, policy, ScanKind::Records, &f, 1);
}

int urf_queue_create_cloud2_with(urf_queue** out, urf_queue_process_fn fn, void* user, int max_points, int slots, int max_batch,
                                 int policy, int point_step, int off_x, int off_y, int off_z, int off_intensity) {
  const urf_cloud2_format f{point_step, off_x, off_y, off_z, off_intensity};
  if (!fn || urf::check_cloud2_format(f) != URF_OK) return URF_ERR_INVALID;
  return create_common(out, nullptr, fn, nullptr, user, max_points, slots, max_batch, policy, ScanKind::Records, &f, 1);
}

int urf_queue_create_formats(urf_queue** out, urf_ctx* ctx, int max_points, int slots, int max_batch, int policy,
                             const urf_cloud2_format* formats, int n_formats) {
  if (!ctx || urf::check_format_table(formats, n_formats) != URF_OK) return URF_ERR_INVALID;
  return create_common(out, ctx, nullptr, nullptr, nullptr, max_points, slots, max_batch, policy, ScanKind::Formats, formats, n_formats);
}

int urf_queue_create_formats_with(urf_queue** out, urf_queue_process_fn fn, void* user, int max_points, int slots, int max_batch,
                                  int policy, const urf_cloud2_format* formats, int n_formats) {
  if (!fn || urf::check_format_table(formats, n_formats) != URF_OK) return URF_ERR_INVALID;
  return create_common(out, nullptr, fn, nullptr, user, max_points, slots, max_batch, policy, ScanKind::Formats, formats, n_formats);
}

int urf_queue_create_with(urf_queue** out, urf_queue_process_fn fn, void* user, int max_points, int slots, int max_batch, int policy) {
  if (!fn) return URF_ERR_INVALID;
  return create_common(out, nullptr, fn, nullptr, user, max_points, slots, max_batch, policy);
}

int urf_queue_create_with_async(urf_queue** out, urf_queue_process_fn enqueue, urf_queue_finish_fn finish, void* user, int max_points,
                                int slots, int max_batch, int policy) {
  if (!enqueue || !finish) return URF_ERR_INVALID;
  return create_common(out, nullptr, enqueue, finish, user, max_points, slots, max_batch, policy);
}


int urf_queue_submit(urf_queue* q, const float* xyzi, int n, uint64_t tag, int timeout_ms) {
  return urf_internal::queue_submit(q, ScanKind::Float4, 0, xyzi, n, tag, timeout_ms, false);
}

int urf_queue_submit_ref(urf_queue* q, const float* xyzi, int n, uint64_t tag, int timeout_ms) {
  return urf_internal::queue_submit(q, ScanKind::Float4, 0, xyzi, n, tag, timeout_ms, true);
}

int urf_queue_submit_cloud2(urf_queue* q, const void* data, int n_points, uint64_t tag, int timeout_ms) {
  return urf_internal::queue_submit(q, ScanKind::Records, 0, data, n_points, tag, timeout_ms, false);
}

int urf_queue_submit_cloud2_ref(urf_queue* q, const void* data, int n_points, uint64_t tag, int timeout_ms) {
  return urf_internal::queue_submit(q, ScanKind::Records, 0, data, n_points, tag, timeout_ms, true);
}

int urf_queue_submit_format(urf_queue* q, int fmt, const void* data, int n_points, uint64_t tag, int timeout_ms) {
  return urf_internal::queue_submit(q, ScanKind::Formats, fmt, data, n_points, tag, timeout_ms, false);
}

int urf_queue_submit_format_ref(urf_queue* q, int fmt, const void* data, int n_points, uint64_t tag, int timeout_ms) {
  return urf_internal::queue_submit(q, ScanKind::Formats, fmt, data, n_points, tag, timeout_ms, true);
}

int urf_queue_update_params(urf_queue* q, const urf_params* p) {
  if (!q || !p || urf::validate_params(p) != URF_OK) return URF_ERR_INVALID;
  return urf_internal::queue_update_params(q, p, 0);
}

int urf_queue_set_params_hook(urf_queue* q, urf_queue_params_fn fn) {
  if (!q || q->ctx) return URF_ERR_INVALID;
  std::lock_guard<std::mutex> lk(q->mu);
  q->params_fn = fn;
  return URF_OK;
}

namespace {
// Gives the slots lent by the previous urf_queue_next_view / _next_batch call back to the producers (mu held).
void release_lent(urf_queue* q) {
  if (q->lent.empty()) return;
  for (int i : q->lent) q->slots[i].state = FREE;
  q->lent.clear();
  q->cv_free.notify_all();
}

// The run of DONE slots that starts with the oldest live scan (smallest sequence number among PENDING / RUNNING / DONE
// slots), in submission order, at most max_results of them, into q->live: its length, 0 while the oldest live scan is not
// done, URF_ERR_CLOSED when the queue is closed and drained (mu held). A dropped scan's slot was reused and carries a new
// sequence number, so it is skipped.
int done_run(urf_queue* q, int max_results) {
  q->live.clear();
  bool filling = false;
  for (int i = 0; i < (int)q->slots.size(); i++) {
    const SlotState st = q->slots[i].state;
    if (st == FILLING) filling = true;
    if (st == PENDING || st == RUNNING || st == DONE) q->live.emplace_back(q->slots[i].seq, i);
  }
  if (q->live.empty()) return q->closed && !filling ? (int)URF_ERR_CLOSED : 0;
  std::sort(q->live.begin(), q->live.end());
  int k = 0;
  while (k < (int)q->live.size() && k < max_results && q->slots[q->live[k].second].state == DONE) k++;
  q->live.resize(k);
  return k;
}

// The first half of every delivery call (mu held): the slots lent by the previous call come back, then waits up to
// timeout_ms for done_run to find a run (>= 1) or the drained queue (URF_ERR_CLOSED); URF_ERR_TIMEOUT otherwise.
int wait_done_run(urf_queue* q, std::unique_lock<std::mutex>& lk, int max_results, int timeout_ms) {
  release_lent(q);
  int k = 0;
  if (!wait_for(q->cv_done, lk, timeout_ms, [&] { return (k = done_run(q, max_results)) != 0; })) return URF_ERR_TIMEOUT;
  return k;
}

// The second half (mu held): the first k slots of q->live become lent: VIEWED slots are invisible to producers and the
// worker until release_lent, so the consumer reads them outside the lock.
int lend(urf_queue* q, int k) {
  for (int j = 0; j < k; j++) { q->slots[q->live[j].second].state = VIEWED; q->lent.push_back(q->live[j].second); }
  q->st.delivered += (uint64_t)k;
  return k;
}

// Both halves in the one lock round of a urf_queue_next* call: the number of slots now in q->lent, or the error code.
int take_done_run(urf_queue* q, int max_results, int timeout_ms) {
  std::unique_lock<std::mutex> lk(q->mu);
  const int k = wait_done_run(q, lk, max_results, timeout_ms);
  return k < 0 ? k : lend(q, k);
}

// The fields of a finished scan the consumer gets: counts and flags, and only the n_vert vertices that exist.
void copy_result(urf_result* dst, const urf_result& src) {
  std::memcpy(dst, &src, offsetof(urf_result, label));
  dst->label = nullptr; dst->ring = nullptr; dst->order = nullptr; dst->ring_start = nullptr;
  const int nv = std::min(std::max(src.n_vert, 0), URF_MAX_VERTS);
  std::memcpy(dst->vert, src.vert, sizeof(src.vert[0]) * (size_t)nv);
}

// Hands out the slots of q->lent: the j-th goes to index dst ? dst[j] : j; with URF_QUEUE_ORDER the order and ring_start
// of a scan that did not fail point into its slot. Runs outside the lock (the slots are ours).
void hand_out(const urf_queue* q, const int* dst, uint64_t* tags, int32_t* rcs, urf_result* outs, const void** label_views) {
  for (int j = 0; j < (int)q->lent.size(); j++) {
    const Slot& s = q->slots[q->lent[j]];
    const int o = dst ? dst[j] : j;
    if (tags) tags[o] = s.tag;
    if (rcs) rcs[o] = s.rc;
    copy_result(&outs[o], s.res);
    if (q->order && s.rc == URF_OK) { outs[o].order = s.order; outs[o].ring_start = s.ring_start; }
    if (label_views) label_views[o] = s.rc != URF_OK ? nullptr : q->label8 ? (const void*)s.label8 : (const void*)s.label;
  }
}
}  // namespace

int urf_queue_next_batch(urf_queue* q, int max_results, uint64_t* tags, int32_t* rcs, urf_result* outs, const void** label_views,
                         int timeout_ms) {
  if (!q || !outs || max_results < 1) return URF_ERR_INVALID;
  const int k = take_done_run(q, max_results, timeout_ms);
  if (k > 0) hand_out(q, nullptr, tags, rcs, outs, label_views);
  return k;
}

// No copy: *label_view points at the labels inside the queue's staging slot, which stays reserved (not reusable by
// producers) until this consumer's next urf_queue_next* call on the queue.
int urf_queue_next_view(urf_queue* q, uint64_t* tag, urf_result* out, const int32_t** label_view, int timeout_ms) {
  if (!q || !out || !label_view || q->label8) return URF_ERR_INVALID;  // int8 slots have no int32 view: urf_queue_next_batch
  int32_t rc = URF_OK;
  const void* view = nullptr;
  const int k = urf_queue_next_batch(q, 1, tag, &rc, out, &view, timeout_ms);
  if (k < 0) return k;
  *label_view = static_cast<const int32_t*>(view);
  return rc;
}

int urf_queue_next(urf_queue* q, uint64_t* tag, urf_result* out, int timeout_ms) {
  if (!q || !out) return URF_ERR_INVALID;
  int32_t* const label = out->label, * const order = out->order, * const ring_start = out->ring_start;   // the caller's
  int32_t rc = URF_OK;
  const int k = urf_queue_next_batch(q, 1, tag, &rc, out, nullptr, timeout_ms);
  if (k < 0) return k;
  urf_internal::queue_copy_lent(q, label, order, ring_start, out);   // outside the lock
  urf_queue_release_view(q);                              // nothing stays lent: the slot goes back to the producers at once
  return rc;
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

int queue_check_kind(const urf_queue* q, ScanKind kind, int fmt) {
  if (!q || kind != q->kind || fmt < 0 || fmt >= (int)q->formats.size()) return URF_ERR_INVALID;
  return URF_OK;
}

int queue_done_run(urf_queue* q, int max_results, int timeout_ms) {
  std::unique_lock<std::mutex> lk(q->mu);
  const int k = wait_done_run(q, lk, max_results, timeout_ms);
  return k == URF_ERR_TIMEOUT && timeout_ms == 0 ? 0 : k;
}

int queue_lend_run(urf_queue* q, int count, const int* dst, uint64_t* tags, int32_t* rcs, urf_result* outs, const void** label_views) {
  {
    std::lock_guard<std::mutex> lk(q->mu);
    // only this consumer takes scans out and rebuilds q->live, so the run queue_done_run left there is still done
    lend(q, std::min(count, (int)q->live.size()));
  }
  hand_out(q, dst, tags, rcs, outs, label_views);
  return (int)q->lent.size();
}

int queue_submit(urf_queue* q, ScanKind kind, int fmt, const void* data, int n, uint64_t tag, int timeout_ms, bool by_reference) {
  if (queue_check_kind(q, kind, fmt) != URF_OK || n < 0 || (n > 0 && !data)) return URF_ERR_INVALID;
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
  else { s.ext = nullptr; if (n > 0) std::memcpy(s.in, data, (size_t)q->formats[fmt].point_step * (size_t)n); }
  {
    std::lock_guard<std::mutex> lk(q->mu);
    if (q->closed) {                                      // closed while copying: the worker may already be gone
      s.state = FREE;
      closed_late = true;
    } else {
      s.n = n; s.fmt = fmt; s.tag = tag; s.rc = URF_OK;
      s.seq = q->next_seq++; s.gen = q->gen;
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

int queue_update_params(urf_queue* q, const urf_params* p, int32_t gen) {
  std::lock_guard<std::mutex> lk(q->mu);
  if (q->closed) return URF_ERR_CLOSED;
  q->gen = gen > 0 ? gen : q->gen + 1;
  q->sets[q->gen] = *p;
  prune_sets(q);
  return q->gen;
}

void queue_copy_lent(const urf_queue* q, int32_t* label, int32_t* order, int32_t* ring_start, urf_result* out) {
  const Slot& s = q->slots[q->lent.front()];
  out->label = label;
  if (q->order) { out->order = order; out->ring_start = ring_start; }
  if (s.rc != URF_OK) return;
  if (label && s.n > 0) {
    if (q->label8) for (int i = 0; i < s.n; i++) label[i] = s.label8[i];   // int8 slot: widened for the caller
    else std::memcpy(label, s.label, sizeof(int32_t) * (size_t)s.n);
  }
  if (!q->order) return;
  if (order && s.res.n_order > 0) std::memcpy(order, s.order, sizeof(int32_t) * (size_t)std::min(s.res.n_order, s.n));
  if (ring_start) std::memcpy(ring_start, s.ring_start, sizeof(int32_t) * (size_t)(std::min(std::max(s.res.n_rings, 0), URF_MAX_CHANNELS) + 1));
}

}  // namespace urf_internal
