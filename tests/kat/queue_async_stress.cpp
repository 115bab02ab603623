// tests/kat/queue_async_stress.cpp — ThreadSanitizer stress of the two-batches-in-flight worker of urf_queue.cpp (built with
// -fsanitize=thread, no CUDA): the queue is created with urf_queue_create_with_async around a stand-in device — enqueue
// hands the batch to a device thread that computes it while the worker, producers and consumer go on; finish waits for the
// oldest batch. Some batches fail at enqueue and some at finish. Exits 0 when every accepted scan was delivered exactly
// once, with its payload or with the error of its batch, in per-producer order, the worker never had more than two batches
// enqueued and did have two at some point, and TSAN reported nothing (TSAN makes the exit code non-zero on a report).
// usage: queue_async_stress <producers> <scans per producer> <slots> <max_batch> <policy (URF_QUEUE_* bits)>
#include <atomic>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <deque>
#include <mutex>
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
constexpr int kFailEnqueue = 13, kFailFinish = 17;     // every 13th enqueue is refused, every 17th batch fails at finish

struct Batch {
  const float* const* xyzi;
  const int* n;
  int batch;
  urf_result* outs;
  bool done = false;
};

struct Device {
  std::mutex mu;
  std::condition_variable cv;
  std::deque<Batch> q;                                 // enqueued, oldest first
  bool stop = false;
  long enqueued = 0, finished = 0;
  int most_in_flight = 0;
  bool over = false;                                   // more than two batches enqueued at once
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
      lk.unlock();                                     // the batch's buffers belong to the device until it is done
      for (int j = 0; j < b->batch; j++) {
        for (int i = 0; i < b->n[j]; i++) b->outs[j].label[i] = (int)b->xyzi[j][4 * i] + 7;
        b->outs[j].status = URF_OK; b->outs[j].n_in = b->n[j];
      }
      lk.lock();
      b->done = true;                                  // deque elements stay put while others are appended behind them
      cv.notify_all();
    }
  }
};

int enqueue(void* user, const float* const* xyzi, const int* n, int batch, urf_result* outs) {
  Device* d = static_cast<Device*>(user);
  std::lock_guard<std::mutex> lk(d->mu);
  if (++d->enqueued % kFailEnqueue == 0) return URF_ERR_CUDA;
  d->q.push_back(Batch{xyzi, n, batch, outs});
  if ((int)d->q.size() > 2) d->over = true;
  if ((int)d->q.size() > d->most_in_flight) d->most_in_flight = (int)d->q.size();
  d->cv.notify_all();
  return URF_OK;
}

int finish(void* user) {
  Device* d = static_cast<Device*>(user);
  std::unique_lock<std::mutex> lk(d->mu);
  if (d->q.empty()) return URF_ERR_INVALID;
  d->cv.wait(lk, [&] { return d->q.front().done; });
  d->q.pop_front();
  return ++d->finished % kFailFinish == 0 ? URF_ERR_CUDA : URF_OK;
}
}  // namespace

int main(int argc, char** argv) {
  const int P = argc > 1 ? atoi(argv[1]) : 4, K = argc > 2 ? atoi(argv[2]) : 2000, slots = argc > 3 ? atoi(argv[3]) : 6,
            mb = argc > 4 ? atoi(argv[4]) : 4, policy = argc > 5 ? atoi(argv[5]) : URF_QUEUE_BLOCK;
  const bool label8 = (policy & URF_QUEUE_LABEL8) != 0;
  const int N = 24;
  Device dev;
  dev.th = std::thread(&Device::run, &dev);
  urf_queue* q = nullptr;
  if (urf_queue_create_with_async(&q, enqueue, finish, &dev, N, slots, mb, policy) != URF_OK) return 2;
  std::atomic<long> accepted{0};
  std::vector<std::thread> prod;
  for (int p = 0; p < P; p++) prod.emplace_back([&, p] {
    std::vector<float> pts(4 * N);
    for (int k = 0; k < K; k++) {
      const int n = 1 + (k + p) % N;
      for (int i = 0; i < n; i++) pts[4 * i] = (float)(k % 100 + i);
      const int rc = urf_queue_submit(q, pts.data(), n, ((uint64_t)p << 32) | (uint64_t)k, -1);
      if (rc != URF_OK) { fprintf(stderr, "submit rc=%d\n", rc); exit(3); }
      accepted++;
    }
  });
  long delivered = 0, failed = 0, bad = 0;
  std::vector<long> last(P, -1);
  std::thread cons([&] {
    std::vector<uint64_t> tags(8);
    std::vector<int32_t> rcs(8);
    std::vector<urf_result> outs(8);
    std::vector<const void*> views(8);
    for (;;) {                                         // batched delivery: views of the lent slots, int8 or int32
      const int k = urf_queue_next_batch(q, 8, tags.data(), rcs.data(), outs.data(), views.data(), -1);
      if (k == URF_ERR_CLOSED) break;
      if (k < 1) { bad++; continue; }
      for (int j = 0; j < k; j++) {
        const int p = (int)(tags[j] >> 32); const long s = (long)(tags[j] & 0xffffffffu);
        if (s <= last[p]) bad++;                       // per-producer order (drops may leave gaps)
        last[p] = s;
        delivered++;
        if (rcs[j] != URF_OK) { failed++; if (rcs[j] != URF_ERR_CUDA || views[j]) bad++; continue; }
        const int n = 1 + (int)((s + p) % N);
        if (outs[j].n_in != n || !views[j]) { bad++; continue; }
        for (int i = 0; i < n; i++) {
          const int want = (int)(s % 100 + i) + 7;
          const int got = label8 ? static_cast<const int8_t*>(views[j])[i] : static_cast<const int32_t*>(views[j])[i];
          if (got != (label8 ? (int)(int8_t)want : want)) { bad++; break; }
        }
      }
    }
  });
  for (auto& t : prod) t.join();
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
  const bool ok = bad == 0 && st.submitted == (uint64_t)accepted.load() && st.processed + st.dropped == st.submitted &&
                  st.delivered == (uint64_t)delivered && st.delivered == st.processed && (drop || st.dropped == 0) && failed > 0 &&
                  !dev.over && dev.most_in_flight == 2 && dev.q.empty();
  printf("producers=%d scans=%ld delivered=%ld failed=%ld dropped=%llu batches=%llu largest_batch=%d most_in_flight=%d bad=%ld %s\n", P,
         accepted.load(), delivered, failed, (unsigned long long)st.dropped, (unsigned long long)st.batches, st.largest_batch,
         dev.most_in_flight, bad, ok ? "OK" : "FAIL");
  return ok ? 0 : 1;
}
