// tests/kat/queue_order_stress.cpp — ThreadSanitizer stress of the emission order through a running urf_queue
// (URF_QUEUE_ORDER; built with -fsanitize=thread, no CUDA): the queue runs the two-batches-in-flight worker around a stand-in
// device (urf_queue_create_with_async) whose parameter hook stands for urf_set_params_next. Several producers submit, one
// thread updates the parameters at random moments, one consumer takes batches of results with urf_queue_next_batch. The
// device writes, for every scan, labels, an order and ring offsets that are functions of the scan's producer, number and
// size and of the generation its batch ran with. Exits 0 when
//   - every delivered scan's labels, order[:n_order] and ring_start[:n_rings + 1] views hold exactly that payload for its
//     tag and params_gen, and order / ring_start are non-NULL;
//   - one producer's scans come back in its order, each accepted scan exactly once (or dropped, with DROP_OLDEST);
// and TSAN reported nothing (TSAN makes the exit code non-zero on a report).
// usage: queue_order_stress <producers> <scans per producer> <slots> <max_batch> <policy (URF_QUEUE_* bits; ORDER is added)>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <deque>
#include <mutex>
#include <random>
#include <thread>
#include <vector>
#include "../../include/urf.h"

// stand-ins for the CUDA side of liburf_b200.so (never reached: the queue is created around the stand-in device)
extern "C" void* urf_pinned_alloc(size_t) { return nullptr; }
extern "C" void urf_pinned_free(void*) {}
extern "C" int urf_create(urf_ctx**, int, int, int) { return URF_ERR_NO_DEVICE; }
extern "C" void urf_destroy(urf_ctx*) {}
extern "C" int urf_set_params(urf_ctx*, const urf_params*) { return URF_ERR_NO_DEVICE; }

namespace {
constexpr int N = 24;                                  // largest scan

// the payload of scan k of producer p with n points, run with generation g: a rotation of the first n_order indices
// and n_rings rings of equal size (the last one takes the rest)
struct Payload {
  int n_order, n_rings, shift;
  int order(int i) const { return (i + shift) % N % (n_order > 0 ? n_order : 1); }
  int ring_start(int r) const { return r == n_rings ? n_order : r * (n_order / n_rings); }
};
Payload payload(int p, long k, int n, int32_t g) {
  Payload y;
  y.n_order = n - (int)(k % 3) > 0 ? n - (int)(k % 3) : 0;
  y.n_rings = 1 + (int)((k + p + g) % 7);
  y.shift = (int)((k * 7 + p + g) % N);
  return y;
}
int label_of(long k, int i) { return (int)(k % 100 + i) + 7; }

urf_params set_of(int32_t g) {
  urf_params p{};
  p.interval = 0.18; p.beamZone = 30; p.channels = 64;
  p.curb_points = 1 + g % 4096;
  return p;
}

struct Batch {
  const float* const* xyzi;
  const int* n;
  int batch;
  urf_result* outs;
  int32_t gen;
  bool done = false;
};

struct Device {
  std::mutex mu;
  std::condition_variable cv;
  std::deque<Batch> q;
  bool stop = false;
  int32_t gen = 0;                                     // generation of the set the device holds
  long null_order = 0;
  std::thread th;

  void run() {
    std::unique_lock<std::mutex> lk(mu);
    for (;;) {
      Batch* b = nullptr;
      cv.wait(lk, [&] {
        for (Batch& x : q) if (!x.done) { b = &x; return true; }
        return stop;
      });
      if (!b) return;
      lk.unlock();
      long nulls = 0;
      for (int j = 0; j < b->batch; j++) {
        urf_result& o = b->outs[j];
        const float* s = b->xyzi[j];
        const int n = b->n[j], p = (int)s[1];
        const long k = (long)s[2];
        for (int i = 0; i < n; i++) o.label[i] = label_of(k, i);
        o.status = URF_OK; o.n_in = n;
        if (!o.order || !o.ring_start) { nulls++; continue; }
        const Payload y = payload(p, k, n, b->gen);
        o.n_order = y.n_order; o.n_rings = y.n_rings;
        for (int i = 0; i < y.n_order; i++) o.order[i] = y.order(i);
        for (int r = 0; r <= y.n_rings; r++) o.ring_start[r] = y.ring_start(r);
      }
      lk.lock();
      null_order += nulls;
      b->done = true;
      cv.notify_all();
    }
  }
};

int hook(void* user, const urf_params*, int32_t gen) {
  Device* d = static_cast<Device*>(user);
  std::lock_guard<std::mutex> lk(d->mu);
  d->gen = gen;
  return URF_OK;
}

int enqueue(void* user, const float* const* xyzi, const int* n, int batch, urf_result* outs) {
  Device* d = static_cast<Device*>(user);
  std::lock_guard<std::mutex> lk(d->mu);
  d->q.push_back(Batch{xyzi, n, batch, outs, d->gen});
  d->cv.notify_all();
  return URF_OK;
}

int finish(void* user) {
  Device* d = static_cast<Device*>(user);
  std::unique_lock<std::mutex> lk(d->mu);
  if (d->q.empty()) return URF_ERR_INVALID;
  d->cv.wait(lk, [&] { return d->q.front().done; });
  d->q.pop_front();
  return URF_OK;
}
}  // namespace

int main(int argc, char** argv) {
  const int P = argc > 1 ? atoi(argv[1]) : 4, K = argc > 2 ? atoi(argv[2]) : 2000, slots = argc > 3 ? atoi(argv[3]) : 6,
            mb = argc > 4 ? atoi(argv[4]) : 4, policy = (argc > 5 ? atoi(argv[5]) : URF_QUEUE_BLOCK) | URF_QUEUE_ORDER;
  const bool label8 = (policy & URF_QUEUE_LABEL8) != 0;
  Device dev;
  dev.th = std::thread(&Device::run, &dev);
  urf_queue* q = nullptr;
  if (urf_queue_create_with_async(&q, enqueue, finish, &dev, N, slots, mb, policy) != URF_OK) return 2;
  if (urf_queue_set_params_hook(q, hook) != URF_OK) return 2;
  std::atomic<bool> producing{true};
  std::atomic<int32_t> updates{0};
  std::thread updater([&] {
    std::mt19937 rng(777);
    while (producing.load()) {
      std::this_thread::sleep_for(std::chrono::microseconds(rng() % 400));
      const urf_params p = set_of(updates.load() + 1);
      if (urf_queue_update_params(q, &p) != updates.load() + 1) { fprintf(stderr, "update failed\n"); exit(3); }
      updates++;
    }
  });
  std::atomic<long> accepted{0};
  std::vector<std::thread> prod;
  for (int p = 0; p < P; p++) prod.emplace_back([&, p] {
    std::vector<float> pts(4 * N);
    for (int k = 0; k < K; k++) {
      const int n = 1 + (k + p) % N;
      for (int i = 0; i < n; i++) { pts[4 * i] = (float)i; pts[4 * i + 1] = (float)p; pts[4 * i + 2] = (float)k; }
      const int rc = urf_queue_submit(q, pts.data(), n, ((uint64_t)p << 32) | (uint64_t)k, -1);
      if (rc != URF_OK) { fprintf(stderr, "submit rc=%d\n", rc); exit(3); }
      accepted++;
    }
  });
  long delivered = 0, bad = 0, checked = 0;
  std::vector<long> last(P, -1);
  std::thread cons([&] {
    std::vector<uint64_t> tags(8);
    std::vector<int32_t> rcs(8);
    std::vector<urf_result> outs(8);
    std::vector<const void*> views(8);
    std::mt19937 rng(99);
    for (;;) {
      const int k = urf_queue_next_batch(q, 1 + (int)(rng() % 8), tags.data(), rcs.data(), outs.data(), views.data(), -1);
      if (k == URF_ERR_CLOSED) break;
      if (k < 1) { bad++; continue; }
      for (int j = 0; j < k; j++) {
        const int p = (int)(tags[j] >> 32); const long s = (long)(tags[j] & 0xffffffffu);
        if (s <= last[p]) bad++;
        last[p] = s;
        delivered++;
        const urf_result& o = outs[j];
        const int n = 1 + (int)((s + p) % N);
        if (rcs[j] != URF_OK || o.n_in != n || !views[j] || !o.order || !o.ring_start) { bad++; continue; }
        for (int i = 0; i < n; i++) {
          const int v = label8 ? static_cast<const int8_t*>(views[j])[i] : static_cast<const int32_t*>(views[j])[i];
          if (v != (label8 ? (int)(int8_t)label_of(s, i) : label_of(s, i))) { bad++; break; }
        }
        const Payload y = payload(p, s, n, o.params_gen);
        if (o.n_order != y.n_order || o.n_rings != y.n_rings) { bad++; continue; }
        for (int i = 0; i < y.n_order; i++) if (o.order[i] != y.order(i)) { bad++; break; }
        for (int r = 0; r <= y.n_rings; r++) if (o.ring_start[r] != y.ring_start(r)) { bad++; break; }
        checked++;
      }
    }
  });
  for (auto& t : prod) t.join();
  producing.store(false);
  updater.join();
  urf_queue_close(q);
  cons.join();
  urf_queue_stats st{};
  urf_queue_get_stats(q, &st);
  urf_queue_destroy(q);
  {
    std::lock_guard<std::mutex> lk(dev.mu);
    dev.stop = true;
  }
  dev.cv.notify_all();
  dev.th.join();
  const bool drop = (policy & URF_QUEUE_DROP_OLDEST) != 0;
  const bool ok = bad == 0 && dev.null_order == 0 && checked == delivered && st.submitted == (uint64_t)accepted.load() &&
                  st.processed + st.dropped == st.submitted && st.delivered == (uint64_t)delivered &&
                  (drop || st.dropped == 0) && updates.load() > 1;
  printf("producers=%d scans=%ld delivered=%ld checked=%ld dropped=%llu batches=%llu updates=%d null_order=%ld bad=%ld %s\n", P,
         accepted.load(), delivered, checked, (unsigned long long)st.dropped, (unsigned long long)st.batches, updates.load(),
         dev.null_order, bad, ok ? "OK" : "FAIL");
  return ok ? 0 : 1;
}
