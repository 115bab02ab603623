// tests/kat/queue_params_stress.cpp — ThreadSanitizer stress of parameter updates on a running urf_queue (built with
// -fsanitize=thread, no CUDA): the queue runs the two-batches-in-flight worker around a stand-in device
// (urf_queue_create_with_async) whose parameter hook (urf_queue_set_params_hook) stands for urf_set_params_next. Several
// producers submit, one thread updates the parameters at random moments, one consumer takes batches of results. The device
// computes every batch with the set it was given last and writes that set's generation into each scan's flags; every 11th
// hook call fails, which fails its run. Exits 0 when
//   - no batch mixes generations: every delivered scan's params_gen equals the generation of the set its batch ran with,
//     and the hook was always handed the set stored for that generation;
//   - every scan carries the generation in force when it was accepted: at least the last update that returned before its
//     submit call began, at most the last update that had begun when its submit call returned;
//   - delivered generations never go backwards for one producer's scans;
// every accepted scan was delivered exactly once with its payload (or its run's error), and TSAN reported nothing (TSAN makes
// the exit code non-zero on a report).
// usage: queue_params_stress <producers> <scans per producer> <slots> <max_batch> <policy (URF_QUEUE_* bits)>
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
constexpr int kFailHook = 11;

// the set of generation g (a valid one: the update validates it): the fields the hook checks are functions of g
urf_params set_of(int32_t g) {
  urf_params p{};
  p.interval = 0.18; p.beamZone = 30; p.channels = 64;
  p.dmin_param = 10 + g;
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
  long hooks = 0, bad_sets = 0, hook_fails = 0;
  bool over = false;
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
      for (int j = 0; j < b->batch; j++) {
        for (int i = 0; i < b->n[j]; i++) b->outs[j].label[i] = (int)b->xyzi[j][4 * i] + 7;
        b->outs[j].status = URF_OK; b->outs[j].n_in = b->n[j]; b->outs[j].flags = b->gen;
      }
      lk.lock();
      b->done = true;
      cv.notify_all();
    }
  }
};

int hook(void* user, const urf_params* p, int32_t gen) {
  Device* d = static_cast<Device*>(user);
  std::lock_guard<std::mutex> lk(d->mu);
  const urf_params want = set_of(gen);
  if (p->dmin_param != want.dmin_param || p->curb_points != want.curb_points) d->bad_sets++;
  if (++d->hooks % kFailHook == 0) { d->hook_fails++; return URF_ERR_CUDA; }
  d->gen = gen;
  return URF_OK;
}

int enqueue(void* user, const float* const* xyzi, const int* n, int batch, urf_result* outs) {
  Device* d = static_cast<Device*>(user);
  std::lock_guard<std::mutex> lk(d->mu);
  d->q.push_back(Batch{xyzi, n, batch, outs, d->gen});
  if ((int)d->q.size() > 2) d->over = true;
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

struct Bounds { int32_t lo = 0, hi = 0; };
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
  if (urf_queue_set_params_hook(q, hook) != URF_OK) return 2;
  std::atomic<int32_t> begun{0}, returned{0};          // last update that has begun / returned
  std::atomic<bool> producing{true};
  long bad = 0;
  std::thread updater([&] {
    std::mt19937 rng(12345);
    while (producing.load()) {
      std::this_thread::sleep_for(std::chrono::microseconds(rng() % 400));
      const int32_t g = begun.load() + 1;
      begun.store(g);
      const urf_params p = set_of(g);
      const int rc = urf_queue_update_params(q, &p);
      if (rc != g) { fprintf(stderr, "update rc=%d want %d\n", rc, g); exit(3); }
      returned.store(g);
    }
  });
  std::vector<std::vector<Bounds>> bounds(P, std::vector<Bounds>(K));
  std::vector<std::vector<char>> accepted_k(P, std::vector<char>(K, 0));
  std::atomic<long> accepted{0};
  std::vector<std::thread> prod;
  for (int p = 0; p < P; p++) prod.emplace_back([&, p] {
    std::vector<float> pts(4 * N);
    for (int k = 0; k < K; k++) {
      const int n = 1 + (k + p) % N;
      for (int i = 0; i < n; i++) pts[4 * i] = (float)(k % 100 + i);
      const int32_t lo = returned.load();
      const int rc = urf_queue_submit(q, pts.data(), n, ((uint64_t)p << 32) | (uint64_t)k, -1);
      bounds[p][k] = Bounds{lo, begun.load()};
      if (rc != URF_OK) { fprintf(stderr, "submit rc=%d\n", rc); exit(3); }
      accepted_k[p][k] = 1;
      accepted++;
    }
  });
  struct Got { int p; long k; int32_t gen; };
  std::vector<Got> got;
  long delivered = 0, failed = 0;
  std::vector<int32_t> last_gen(P, -1);
  std::vector<long> last(P, -1);
  std::thread cons([&] {
    std::vector<uint64_t> tags(8);
    std::vector<int32_t> rcs(8);
    std::vector<urf_result> outs(8);
    std::vector<const void*> views(8);
    for (;;) {
      const int k = urf_queue_next_batch(q, 8, tags.data(), rcs.data(), outs.data(), views.data(), -1);
      if (k == URF_ERR_CLOSED) break;
      if (k < 1) { bad++; continue; }
      for (int j = 0; j < k; j++) {
        const int p = (int)(tags[j] >> 32); const long s = (long)(tags[j] & 0xffffffffu);
        const int32_t g = outs[j].params_gen;
        if (s <= last[p] || g < last_gen[p]) bad++;   // per-producer order, and generations never go backwards
        last[p] = s; last_gen[p] = g;
        got.push_back(Got{p, s, g});
        delivered++;
        if (rcs[j] != URF_OK) { failed++; if (rcs[j] != URF_ERR_CUDA || views[j]) bad++; continue; }
        if (outs[j].flags != g) bad++;                 // the batch ran with another generation's set
        const int n = 1 + (int)((s + p) % N);
        if (outs[j].n_in != n || !views[j]) { bad++; continue; }
        for (int i = 0; i < n; i++) {
          const int want = (int)(s % 100 + i) + 7;
          const int v = label8 ? static_cast<const int8_t*>(views[j])[i] : static_cast<const int32_t*>(views[j])[i];
          if (v != (label8 ? (int)(int8_t)want : want)) { bad++; break; }
        }
      }
    }
  });
  for (auto& t : prod) t.join();
  producing.store(false);
  updater.join();
  urf_queue_close(q);
  cons.join();
  long out_of_bounds = 0;
  for (const Got& g : got) {
    const Bounds& b = bounds[g.p][g.k];
    if (!accepted_k[g.p][g.k] || g.gen < b.lo || g.gen > b.hi) out_of_bounds++;
  }
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
  const bool ok = bad == 0 && out_of_bounds == 0 && dev.bad_sets == 0 && !dev.over && dev.q.empty() &&
                  st.submitted == (uint64_t)accepted.load() && st.processed + st.dropped == st.submitted &&
                  st.delivered == (uint64_t)delivered && st.delivered == st.processed && (drop || st.dropped == 0) &&
                  returned.load() > 1 && dev.hooks > 1 && (dev.hook_fails == 0 || failed > 0);
  printf("producers=%d scans=%ld delivered=%ld failed=%ld dropped=%llu batches=%llu updates=%d hooks=%ld hook_fails=%ld "
         "out_of_bounds=%ld bad_sets=%ld bad=%ld %s\n", P, accepted.load(), delivered, failed, (unsigned long long)st.dropped,
         (unsigned long long)st.batches, returned.load(), dev.hooks, dev.hook_fails, out_of_bounds, dev.bad_sets, bad,
         ok ? "OK" : "FAIL");
  return ok ? 0 : 1;
}
