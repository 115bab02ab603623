// urf_mq.cpp — ONE ingest stream over SEVERAL GPUs (include/urf.h urf_mq, BASELINE config 4: a continuous scan stream
// sharded across the GPUs of one box). Host code only.
//
// The reference is a single subscriber with queue depth 1 (`nh->subscribe(params::topicName, 1, &Detector::filtered, this)`,
// lidar_segmentation.cpp:53); the demo graph feeds four LiDAR topics (config/demo1.rviz:91,121,151,181). urf_mq keeps one
// submit/next interface in front of N devices: every device owns a context and a streaming queue (urf_queue: pinned
// staging slots for float4 scans or, in a record mq, for the PointCloud2 records of one sensor format (of the formats of a
// table, each scan naming its own, in a formats mq) + one worker thread
// that takes whatever is pending as one batch and keeps two batches in flight); a scan goes to the device with the fewest
// scans in flight (ties: round-robin), and results come back in the order the submissions completed.
// Scans are independent units, so there is nothing to exchange between devices (no collective on this path).
//
// Ordering: urf_queue delivers each device's scans in the order their submit calls completed, so the global order only
// has to remember WHICH device holds the next scan: a FIFO of device indices, appended after a device accepted a scan
// (under that device's submit mutex, so that the k-th entry naming a device is the k-th scan its queue accepted).
//
// Delivery (take_front_run, behind urf_mq_next / _next_view / _next_batch) cuts the front of that FIFO at the first scan
// that is not done yet: every device queue involved reports how many of its oldest scans are done, and then lends exactly
// the ones before the cut.
//
// Parameter updates (urf_mq_update_params) take every device's submit mutex, in device order, and then give each device
// queue the mq's next generation. No scan can then be between its queue's acceptance and its entry in `order`, so the
// update falls at one point of the global order on every device at once.
#include <algorithm>
#include <cstring>
#include <deque>
#include <mutex>
#include <vector>

#include "../../include/urf.h"
#include "urf_params.hpp"
#include "urf_queue_internal.hpp"

struct urf_mq {
  struct Dev {
    int device = -1;
    urf_ctx* ctx = nullptr;          // owned (NULL with the test hook)
    urf_queue* q = nullptr;
    uint64_t submitted = 0, delivered = 0;
    int inflight = 0;                // accepted or being copied, not yet delivered
    std::mutex submit_mu;            // held from the device queue's submit to the append to `order`: one device's entries
                                     // enter `order` in the order its queue accepted them (copies to DIFFERENT devices overlap)
  };
  std::deque<Dev> dev;               // deque: Dev holds a mutex and must not move
  std::mutex mu;
  std::condition_variable cv;        // a device index was appended / the mq was closed
  std::deque<int> order;             // device of the next scans to deliver, oldest first
  int rr = 0;                        // round-robin cursor for ties
  int submitting = 0;                // submit calls between device choice and order append
  bool closed = false;
  bool label8 = false;               // int8 label slots on every device (urf_mq_create_label8)
  int32_t gen = 0;                   // last parameter generation; changed only with every device's submit_mu held
  // Scratch of take_front_run. The header allows ONE consumer thread, so it needs no lock.
  std::vector<int> ds;               // devices of the first scans in the global order (a snapshot of `order`'s front)
  std::vector<int> want, done, used; // per device: its entries in ds / how many of them are done (-1: not asked yet) /
                                     // how many the last call lent, which are still lent when the next call begins
  std::vector<std::vector<int>> dst; // per device: output positions of its share, in its queue's order
};

namespace {

int pick_device(urf_mq* m) {         // fewest scans in flight; ties go round-robin so an idle box is loaded evenly
  const int n = (int)m->dev.size();
  int best = -1;
  for (int j = 0; j < n; j++) {
    const int d = (m->rr + j) % n;
    if (best < 0 || m->dev[d].inflight < m->dev[best].inflight) best = d;
  }
  m->rr = (best + 1) % n;
  return best;
}

// kind: what the submit call hands in (float4 points, records, or records of table format fmt); every device queue has the
// mq's kind and format table, so the first one answers whether the mq takes it, before a device is chosen.
int submit_common(urf_mq* m, urf_internal::ScanKind kind, int fmt, const void* data, int n, uint64_t tag, int timeout_ms, bool by_reference) {
  if (!m || urf_internal::queue_check_kind(m->dev[0].q, kind, fmt) != URF_OK) return URF_ERR_INVALID;
  int d;
  {
    std::lock_guard<std::mutex> lk(m->mu);
    if (m->closed) return URF_ERR_CLOSED;
    d = pick_device(m);
    m->dev[d].inflight++;
    m->submitting++;
  }
  // outside the mq lock: the copy into the device's pinned slot (or the wait for a free slot) runs in parallel for
  // producers that were dealt different devices
  std::lock_guard<std::mutex> dev_lk(m->dev[d].submit_mu);
  const int rc = urf_internal::queue_submit(m->dev[d].q, kind, fmt, data, n, tag, timeout_ms, by_reference);
  {
    std::lock_guard<std::mutex> lk(m->mu);
    m->submitting--;
    if (rc == URF_OK) { m->order.push_back(d); m->dev[d].submitted++; }
    else m->dev[d].inflight--;
  }
  m->cv.notify_all();
  return rc;
}

// fn == NULL: a context (with `params`, if given) and a pinned queue on each of `devices`; otherwise stand-in devices
// around fn, which gets users[j] for device j. Every device queue gets `policy` and the scan kind: float4, the one record
// format formats[0] (Records), or the format table (Formats). The first device that cannot be made ends the attempt.
int create(urf_mq** out, const int* devices, urf_queue_process_fn fn, void* const* users, int n_devices, int max_points,
           int slots_per_device, int max_batch, const urf_params* params, int policy,
           urf_internal::ScanKind kind = urf_internal::ScanKind::Float4, const urf_cloud2_format* formats = nullptr, int n_formats = 0) {
  using urf_internal::ScanKind;
  // BLOCK with the slot options only: the mq has no drop policy
  if (!out || (!devices && !fn) || n_devices < 1 || max_points < 1 || slots_per_device < 1 || max_batch < 1 ||
      (policy & ~(URF_QUEUE_LABEL8 | URF_QUEUE_ORDER)) != URF_QUEUE_BLOCK ||
      (kind != ScanKind::Float4 && urf::check_format_table(formats, n_formats) != URF_OK))
    return URF_ERR_INVALID;
  *out = nullptr;
  urf_mq* m = new urf_mq;
  m->label8 = (policy & URF_QUEUE_LABEL8) != 0;
  for (int j = 0; j < n_devices; j++) m->dev.emplace_back();
  m->want.resize(n_devices); m->done.resize(n_devices); m->used.resize(n_devices); m->dst.resize(n_devices);
  for (int j = 0; j < n_devices; j++) {
    urf_mq::Dev& d = m->dev[j];
    d.device = fn ? j : devices[j];
    int rc = URF_OK;
    void* const user = users ? users[j] : nullptr;
    const urf_cloud2_format* f = formats;
    if (fn && kind == ScanKind::Records)
      rc = urf_queue_create_cloud2_with(&d.q, fn, user, max_points, slots_per_device, max_batch, policy, f->point_step, f->off_x,
                                        f->off_y, f->off_z, f->off_intensity);
    else if (fn && kind == ScanKind::Formats)
      rc = urf_queue_create_formats_with(&d.q, fn, user, max_points, slots_per_device, max_batch, policy, formats, n_formats);
    else if (fn) rc = urf_queue_create_with(&d.q, fn, user, max_points, slots_per_device, max_batch, policy);
    else {
      rc = urf_create(&d.ctx, d.device, max_points, max_batch);
      if (rc == URF_OK && params) rc = urf_set_params(d.ctx, params);
      if (rc == URF_OK && kind == ScanKind::Records)
        rc = urf_queue_create_cloud2(&d.q, d.ctx, max_points, slots_per_device, max_batch, policy, f->point_step, f->off_x, f->off_y,
                                     f->off_z, f->off_intensity);
      else if (rc == URF_OK && kind == ScanKind::Formats)
        rc = urf_queue_create_formats(&d.q, d.ctx, max_points, slots_per_device, max_batch, policy, formats, n_formats);
      else if (rc == URF_OK) rc = urf_queue_create(&d.q, d.ctx, max_points, slots_per_device, max_batch, policy);
    }
    if (rc != URF_OK) { urf_mq_destroy(m); return rc; }
  }
  *out = m;
  return URF_OK;
}

// The one delivery routine: lends the run of finished scans at the front of the global order, at most max_results of
// them, and returns its length (>= 1), or URF_ERR_TIMEOUT (the oldest scan's entry stays at the front) / URF_ERR_CLOSED.
// Outputs as urf_mq_next_batch.
int take_front_run(urf_mq* m, int max_results, uint64_t* tags, int32_t* rcs, urf_result* outs, const void** label_views, int timeout_ms) {
  const int D = (int)m->dev.size();
  // slots lent by the previous call belong to device queues: they go back before this call waits for producers, who may
  // need them, and before a queue lends new ones
  for (int d = 0; d < D; d++)
    if (m->used[d]) { urf_queue_release_view(m->dev[d].q); m->used[d] = 0; }
  {
    std::unique_lock<std::mutex> lk(m->mu);
    if (!urf_internal::wait_for(m->cv, lk, timeout_ms, [&] { return !m->order.empty() || (m->closed && m->submitting == 0); }))
      return URF_ERR_TIMEOUT;
    if (m->order.empty()) return URF_ERR_CLOSED;          // closed and drained
    m->ds.assign(m->order.begin(), m->order.begin() + std::min<size_t>((size_t)max_results, m->order.size()));
  }
  // Only this consumer takes entries out of `order` and scans out of the queues, so the snapshot's front stays valid and
  // a scan seen done stays done. The k-th entry naming device d is the k-th oldest scan in d's queue.
  const std::vector<int>& ds = m->ds;
  std::vector<int>& want = m->want, & done = m->done, & used = m->used;
  for (int d = 0; d < D; d++) { want[d] = 0; done[d] = -1; m->dst[d].clear(); }
  for (int d : ds) want[d]++;
  const int r = urf_internal::queue_done_run(m->dev[ds[0]].q, want[ds[0]], timeout_ms);   // waits for the oldest scan
  if (r < 0) return r;
  done[ds[0]] = r;
  int k = 0;
  for (; k < (int)ds.size(); k++) {                       // the run ends at the first scan that is not done on its device
    const int d = ds[k];
    if (done[d] < 0) done[d] = std::max(0, urf_internal::queue_done_run(m->dev[d].q, want[d], 0));
    if (used[d] == done[d]) break;
    used[d]++;
    m->dst[d].push_back(k);
  }
  for (int d = 0; d < D; d++)
    if (used[d]) urf_internal::queue_lend_run(m->dev[d].q, used[d], m->dst[d].data(), tags, rcs, outs, label_views);
  {
    std::lock_guard<std::mutex> lk(m->mu);
    m->order.erase(m->order.begin(), m->order.begin() + k);
    for (int d = 0; d < D; d++) { m->dev[d].inflight -= used[d]; m->dev[d].delivered += (uint64_t)used[d]; }
  }
  return k;
}

}  // namespace

namespace urf_internal {
int mq_apply_idle(urf_mq* m, int (*fn)(urf_ctx*, const void*), const void* arg) {
  // like the reference's paramsCallback between two scan callbacks (single spin thread, src/main.cpp:54): the caller
  // reconfigures between scans — everything submitted must have been collected
  {
    std::lock_guard<std::mutex> lk(m->mu);
    if (!m->order.empty() || m->submitting) return URF_ERR_INVALID;
  }
  for (urf_mq::Dev& d : m->dev)
    if (d.ctx) { const int rc = fn(d.ctx, arg); if (rc != URF_OK) return rc; }
  return URF_OK;
}
}  // namespace urf_internal

extern "C" {

int urf_mq_create(urf_mq** out, const int* devices, int n_devices, int max_points, int slots_per_device, int max_batch,
                  const urf_params* params) {
  return create(out, devices, nullptr, nullptr, n_devices, max_points, slots_per_device, max_batch, params, URF_QUEUE_BLOCK);
}

int urf_mq_create_label8(urf_mq** out, const int* devices, int n_devices, int max_points, int slots_per_device, int max_batch,
                         const urf_params* params) {
  return create(out, devices, nullptr, nullptr, n_devices, max_points, slots_per_device, max_batch, params, URF_QUEUE_BLOCK | URF_QUEUE_LABEL8);
}

int urf_mq_create_with(urf_mq** out, urf_queue_process_fn fn, void* const* users, int n_devices, int max_points, int slots_per_device,
                       int max_batch) {
  return create(out, nullptr, fn, users, n_devices, max_points, slots_per_device, max_batch, nullptr, URF_QUEUE_BLOCK);
}

int urf_mq_create_with_label8(urf_mq** out, urf_queue_process_fn fn, void* const* users, int n_devices, int max_points,
                              int slots_per_device, int max_batch) {
  return create(out, nullptr, fn, users, n_devices, max_points, slots_per_device, max_batch, nullptr, URF_QUEUE_BLOCK | URF_QUEUE_LABEL8);
}

int urf_mq_create_policy(urf_mq** out, const int* devices, int n_devices, int max_points, int slots_per_device, int max_batch,
                         const urf_params* params, int policy) {
  return create(out, devices, nullptr, nullptr, n_devices, max_points, slots_per_device, max_batch, params, policy);
}

int urf_mq_create_with_policy(urf_mq** out, urf_queue_process_fn fn, void* const* users, int n_devices, int max_points,
                              int slots_per_device, int max_batch, int policy) {
  return create(out, nullptr, fn, users, n_devices, max_points, slots_per_device, max_batch, nullptr, policy);
}

int urf_mq_create_cloud2(urf_mq** out, const int* devices, int n_devices, int max_points, int slots_per_device, int max_batch,
                         const urf_params* params, int policy, int point_step, int off_x, int off_y, int off_z, int off_intensity) {
  const urf_cloud2_format f{point_step, off_x, off_y, off_z, off_intensity};
  return create(out, devices, nullptr, nullptr, n_devices, max_points, slots_per_device, max_batch, params, policy,
                urf_internal::ScanKind::Records, &f, 1);
}

int urf_mq_create_cloud2_with(urf_mq** out, urf_queue_process_fn fn, void* const* users, int n_devices, int max_points,
                              int slots_per_device, int max_batch, int policy, int point_step, int off_x, int off_y, int off_z,
                              int off_intensity) {
  const urf_cloud2_format f{point_step, off_x, off_y, off_z, off_intensity};
  return create(out, nullptr, fn, users, n_devices, max_points, slots_per_device, max_batch, nullptr, policy,
                urf_internal::ScanKind::Records, &f, 1);
}

int urf_mq_create_formats(urf_mq** out, const int* devices, int n_devices, int max_points, int slots_per_device, int max_batch,
                          const urf_params* params, int policy, const urf_cloud2_format* formats, int n_formats) {
  return create(out, devices, nullptr, nullptr, n_devices, max_points, slots_per_device, max_batch, params, policy,
                urf_internal::ScanKind::Formats, formats, n_formats);
}

int urf_mq_create_formats_with(urf_mq** out, urf_queue_process_fn fn, void* const* users, int n_devices, int max_points,
                               int slots_per_device, int max_batch, int policy, const urf_cloud2_format* formats, int n_formats) {
  return create(out, nullptr, fn, users, n_devices, max_points, slots_per_device, max_batch, nullptr, policy,
                urf_internal::ScanKind::Formats, formats, n_formats);
}

int urf_mq_set_params(urf_mq* m, const urf_params* p) {
  if (!m || !p) return URF_ERR_INVALID;
  return urf_internal::mq_apply_idle(m, [](urf_ctx* c, const void* q) { return urf_set_params(c, static_cast<const urf_params*>(q)); }, p);
}

int urf_mq_update_params(urf_mq* m, const urf_params* p) {
  if (!m || !p || urf::validate_params(p) != URF_OK) return URF_ERR_INVALID;
  std::vector<std::unique_lock<std::mutex>> held;         // device order: two updates cannot each hold what the other waits for
  held.reserve(m->dev.size());
  for (urf_mq::Dev& d : m->dev) held.emplace_back(d.submit_mu);
  {
    std::lock_guard<std::mutex> lk(m->mu);
    if (m->closed) return URF_ERR_CLOSED;
  }
  const int32_t g = ++m->gen;
  for (urf_mq::Dev& d : m->dev) {
    const int rc = urf_internal::queue_update_params(d.q, p, g);
    if (rc < 0) return rc;                                // closed meanwhile: no scan is accepted any more anyway
  }
  return g;
}

int urf_mq_set_params_hook(urf_mq* m, urf_queue_params_fn fn) {
  if (!m) return URF_ERR_INVALID;
  for (urf_mq::Dev& d : m->dev) if (d.ctx) return URF_ERR_INVALID;
  for (urf_mq::Dev& d : m->dev) urf_queue_set_params_hook(d.q, fn);
  return URF_OK;
}

using urf_internal::ScanKind;
int urf_mq_submit(urf_mq* m, const float* xyzi, int n, uint64_t tag, int timeout_ms) {
  return submit_common(m, ScanKind::Float4, 0, xyzi, n, tag, timeout_ms, false);
}
int urf_mq_submit_ref(urf_mq* m, const float* xyzi, int n, uint64_t tag, int timeout_ms) {
  return submit_common(m, ScanKind::Float4, 0, xyzi, n, tag, timeout_ms, true);
}
int urf_mq_submit_cloud2(urf_mq* m, const void* data, int n_points, uint64_t tag, int timeout_ms) {
  return submit_common(m, ScanKind::Records, 0, data, n_points, tag, timeout_ms, false);
}
int urf_mq_submit_cloud2_ref(urf_mq* m, const void* data, int n_points, uint64_t tag, int timeout_ms) {
  return submit_common(m, ScanKind::Records, 0, data, n_points, tag, timeout_ms, true);
}
int urf_mq_submit_format(urf_mq* m, int fmt, const void* data, int n_points, uint64_t tag, int timeout_ms) {
  return submit_common(m, ScanKind::Formats, fmt, data, n_points, tag, timeout_ms, false);
}
int urf_mq_submit_format_ref(urf_mq* m, int fmt, const void* data, int n_points, uint64_t tag, int timeout_ms) {
  return submit_common(m, ScanKind::Formats, fmt, data, n_points, tag, timeout_ms, true);
}

int urf_mq_next_batch(urf_mq* m, int max_results, uint64_t* tags, int32_t* rcs, urf_result* outs, const void** label_views,
                      int timeout_ms) {
  if (!m || !outs || max_results < 1) return URF_ERR_INVALID;
  return take_front_run(m, max_results, tags, rcs, outs, label_views, timeout_ms);
}

int urf_mq_next_view(urf_mq* m, uint64_t* tag, urf_result* out, const int32_t** label_view, int timeout_ms) {
  if (!m || !out || !label_view || m->label8) return URF_ERR_INVALID;
  int32_t rc = URF_OK;
  const void* view = nullptr;
  const int k = take_front_run(m, 1, tag, &rc, out, &view, timeout_ms);
  if (k < 0) return k;
  *label_view = static_cast<const int32_t*>(view);
  return rc;
}

int urf_mq_next(urf_mq* m, uint64_t* tag, urf_result* out, int timeout_ms) {
  if (!m || !out) return URF_ERR_INVALID;
  int32_t* const label = out->label, * const order = out->order, * const ring_start = out->ring_start;   // the caller's
  int32_t rc = URF_OK;
  const int k = take_front_run(m, 1, tag, &rc, out, nullptr, timeout_ms);
  if (k < 0) return k;
  const int d = m->ds[0];
  urf_internal::queue_copy_lent(m->dev[d].q, label, order, ring_start, out);
  urf_queue_release_view(m->dev[d].q);                    // nothing stays lent: the slot goes back to the producers at once
  m->used[d] = 0;
  return rc;
}

int urf_mq_get_stats(urf_mq* m, urf_mq_stats* st) {
  if (!m || !st) return URF_ERR_INVALID;
  std::memset(st, 0, sizeof(*st));
  std::lock_guard<std::mutex> lk(m->mu);
  st->n_devices = (int32_t)m->dev.size();
  for (size_t j = 0; j < m->dev.size() && j < URF_MQ_MAX_DEVICES; j++) {
    st->submitted[j] = m->dev[j].submitted; st->delivered[j] = m->dev[j].delivered;
    urf_queue_stats qs{};
    if (m->dev[j].q && urf_queue_get_stats(m->dev[j].q, &qs) == URF_OK) { st->batches[j] = qs.batches; st->largest_batch[j] = qs.largest_batch; }
  }
  st->pending = (int32_t)m->order.size();
  return URF_OK;
}

void urf_mq_close(urf_mq* m) {
  if (!m) return;
  {
    std::lock_guard<std::mutex> lk(m->mu);
    m->closed = true;
  }
  for (urf_mq::Dev& d : m->dev) if (d.q) urf_queue_close(d.q);
  m->cv.notify_all();
}

void urf_mq_destroy(urf_mq* m) {
  if (!m) return;
  urf_mq_close(m);
  for (urf_mq::Dev& d : m->dev) {
    if (d.q) urf_queue_destroy(d.q);
    if (d.ctx) urf_destroy(d.ctx);
  }
  delete m;
}

}  // extern "C"
