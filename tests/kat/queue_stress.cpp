// tests/kat/queue_stress.cpp — ThreadSanitizer stress of urf_queue.cpp (built with -fsanitize=thread, no CUDA):
// P producers and one consumer around a stand-in batch function; both policies; exits 0 when every accepted scan was
// delivered exactly once with the right payload and per-producer order, and TSAN reported nothing (TSAN makes the exit
// code non-zero on a report).
// usage: queue_stress <producers> <scans per producer> <slots> <max_batch> <policy>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>
#include "../../include/urf.h"

// stand-ins for the CUDA side of liburf_b200.so (never reached: the queue is created with urf_queue_create_with)
extern "C" void* urf_pinned_alloc(size_t) { return nullptr; }
extern "C" void urf_pinned_free(void*) {}
extern "C" int urf_create(urf_ctx**, int, int, int) { return URF_ERR_NO_DEVICE; }
extern "C" void urf_destroy(urf_ctx*) {}
extern "C" int urf_set_params(urf_ctx*, const urf_params*) { return URF_ERR_NO_DEVICE; }

static std::atomic<int> g_batches{0};
static int fake(void*, const float* const* xyzi, const int* n, int batch, urf_result* outs) {
  g_batches++;
  for (int j = 0; j < batch; j++) {
    for (int i = 0; i < n[j]; i++) outs[j].label[i] = (int)xyzi[j][4 * i] + 7;
    outs[j].status = URF_OK; outs[j].n_in = n[j];
  }
  if ((g_batches.load() & 7) == 0) std::this_thread::yield();
  return URF_OK;
}

// close while producers are inside submit (some blocked on a full queue, some copying): every producer must come back
// (URF_OK or URF_ERR_CLOSED), and a consumer blocked in urf_queue_next(-1) must see the drained state — the lost-wakeup
// case of a producer that finds the queue closed after its copy.
static int close_during_submit(int rounds) {
  for (int r = 0; r < rounds; r++) {
    urf_queue* q = nullptr;
    const int N = 4096;
    if (urf_queue_create_with(&q, fake, nullptr, N, 2, 1, URF_QUEUE_BLOCK) != URF_OK) return 2;
    std::atomic<int> ok{0}, closed{0}, other{0};
    std::vector<std::thread> prod;
    for (int p = 0; p < 6; p++) prod.emplace_back([&] {
      std::vector<float> pts(4 * N, 1.0f);
      for (int k = 0; k < 50; k++) {
        const int rc = urf_queue_submit(q, pts.data(), N, (uint64_t)k, -1);
        if (rc == URF_OK) ok++; else if (rc == URF_ERR_CLOSED) { closed++; break; } else other++;
      }
    });
    std::atomic<int> got{0};
    std::thread cons([&] {
      std::vector<int32_t> lab(N);
      for (;;) {
        urf_result res{}; res.label = lab.data();
        const int rc = urf_queue_next(q, nullptr, &res, -1);
        if (rc == URF_ERR_CLOSED) break;
        got++;
      }
    });
    std::this_thread::sleep_for(std::chrono::microseconds(200 + 137 * r));
    urf_queue_close(q);
    for (auto& t : prod) t.join();
    cons.join();                                            // hangs here if the wakeup is lost
    urf_queue_stats st{};
    urf_queue_get_stats(q, &st);
    urf_queue_destroy(q);
    if (other.load() || (uint64_t)got.load() != st.delivered || st.submitted != (uint64_t)ok.load() || st.delivered != st.submitted) {
      printf("close_during_submit round %d: ok=%d closed=%d other=%d got=%d submitted=%llu FAIL\n", r, ok.load(), closed.load(), other.load(),
             got.load(), (unsigned long long)st.submitted);
      return 1;
    }
  }
  printf("close_during_submit rounds=%d OK\n", rounds);
  return 0;
}

// urf_mq around stand-in devices: D devices, P producers (copying and by-reference submits), one consumer; every scan is
// delivered exactly once with its own payload, per-producer order holds, and the load is spread over the devices.
static int mq_stress(int D, int P, int K) {
  const int N = 24;
  urf_mq* m = nullptr;
  if (urf_mq_create_with(&m, fake, nullptr, D, N, 3, 2) != URF_OK) return 2;
  std::vector<std::vector<float>> keep((size_t)P * K);      // by-reference scans stay alive until delivered
  std::vector<std::thread> prod;
  for (int p = 0; p < P; p++) prod.emplace_back([&, p] {
    for (int k = 0; k < K; k++) {
      const int n = 1 + (k + p) % N;
      std::vector<float>& pts = keep[(size_t)p * K + k];
      pts.assign(4 * N, 0.f);
      for (int i = 0; i < n; i++) pts[4 * i] = (float)(k % 1000 + i);
      const uint64_t tag = ((uint64_t)p << 32) | (uint64_t)k;
      const int rc = (k & 1) ? urf_mq_submit_ref(m, pts.data(), n, tag, -1) : urf_mq_submit(m, pts.data(), n, tag, -1);
      if (rc != URF_OK) { fprintf(stderr, "mq submit rc=%d\n", rc); exit(3); }
    }
  });
  long delivered = 0, bad = 0;
  std::vector<long> last(P, -1);
  std::thread cons([&] {
    std::vector<int32_t> lab(N);
    for (;;) {
      urf_result r{}; r.label = lab.data();
      uint64_t tag = 0;
      const int32_t* view = nullptr;                         // every other result is read in place (no label copy)
      const bool use_view = (delivered & 1) != 0;
      const int rc = use_view ? urf_mq_next_view(m, &tag, &r, &view, -1) : urf_mq_next(m, &tag, &r, -1);
      if (rc == URF_ERR_CLOSED) break;
      if (rc != URF_OK) { bad++; continue; }
      const int32_t* got = use_view ? view : lab.data();
      const int p = (int)(tag >> 32); const long k = (long)(tag & 0xffffffffu);
      if (k <= last[p]) bad++;
      last[p] = k;
      const int n = 1 + (int)((k + p) % N);
      if (r.n_in != n || !got) bad++;
      else for (int i = 0; i < n; i++) if (got[i] != (int)(k % 1000 + i) + 7) { bad++; break; }
      delivered++;
    }
  });
  for (auto& t : prod) t.join();
  urf_mq_close(m);
  cons.join();
  urf_mq_stats st{};
  urf_mq_get_stats(m, &st);
  urf_mq_destroy(m);
  uint64_t sub = 0, del = 0, mn = ~0ull;
  for (int d = 0; d < D; d++) { sub += st.submitted[d]; del += st.delivered[d]; mn = st.submitted[d] < mn ? st.submitted[d] : mn; }
  const bool ok = bad == 0 && delivered == (long)P * K && sub == (uint64_t)P * K && del == sub && st.n_devices == D && mn > 0;
  printf("mq devices=%d producers=%d scans=%ld delivered=%ld least_loaded_device=%llu bad=%ld %s\n", D, P, (long)P * K, delivered,
         (unsigned long long)mn, bad, ok ? "OK" : "FAIL");
  return ok ? 0 : 1;
}

int main(int argc, char** argv) {
  if (argc > 1 && !strcmp(argv[1], "close")) return close_during_submit(argc > 2 ? atoi(argv[2]) : 40);
  if (argc > 1 && !strcmp(argv[1], "mq")) return mq_stress(argc > 2 ? atoi(argv[2]) : 4, argc > 3 ? atoi(argv[3]) : 3, argc > 4 ? atoi(argv[4]) : 1500);
  const int P = argc > 1 ? atoi(argv[1]) : 4, K = argc > 2 ? atoi(argv[2]) : 2000, slots = argc > 3 ? atoi(argv[3]) : 6,
            mb = argc > 4 ? atoi(argv[4]) : 4, policy = argc > 5 ? atoi(argv[5]) : URF_QUEUE_BLOCK;
  const int N = 24;
  urf_queue* q = nullptr;
  if (urf_queue_create_with(&q, fake, nullptr, N, slots, mb, policy) != URF_OK) return 2;
  std::atomic<long> accepted{0};
  std::vector<std::thread> prod;
  for (int p = 0; p < P; p++) prod.emplace_back([&, p] {
    std::vector<float> pts(4 * N);
    for (int k = 0; k < K; k++) {
      const int n = 1 + (k + p) % N;
      for (int i = 0; i < n; i++) pts[4 * i] = (float)(k % 1000 + i);
      const int rc = urf_queue_submit(q, pts.data(), n, ((uint64_t)p << 32) | (uint64_t)k, -1);
      if (rc != URF_OK) { fprintf(stderr, "submit rc=%d\n", rc); exit(3); }
      accepted++;
    }
  });
  long delivered = 0, bad = 0;
  std::vector<long> last(P, -1);
  std::thread cons([&] {
    std::vector<int32_t> lab(N);
    for (;;) {
      urf_result r{}; r.label = lab.data();
      uint64_t tag = 0;
      const int rc = urf_queue_next(q, &tag, &r, -1);
      if (rc == URF_ERR_CLOSED) break;
      if (rc != URF_OK) { bad++; continue; }
      const int p = (int)(tag >> 32); const long k = (long)(tag & 0xffffffffu);
      if (k <= last[p]) bad++;                               // per-producer order (drops may leave gaps)
      last[p] = k;
      const int n = 1 + (int)((k + p) % N);
      if (r.n_in != n) bad++;
      for (int i = 0; i < n; i++) if (lab[i] != (int)(k % 1000 + i) + 7) { bad++; break; }
      delivered++;
    }
  });
  for (auto& t : prod) t.join();
  urf_queue_close(q);
  cons.join();
  urf_queue_stats st{};
  urf_queue_get_stats(q, &st);
  urf_queue_destroy(q);
  const bool ok = bad == 0 && st.submitted == (uint64_t)accepted.load() && st.processed + st.dropped == st.submitted &&
                  st.delivered == (uint64_t)delivered && st.delivered == st.processed && (policy == URF_QUEUE_DROP_OLDEST || st.dropped == 0);
  printf("producers=%d scans=%ld delivered=%ld dropped=%llu batches=%llu largest_batch=%d bad=%ld %s\n", P, accepted.load(), delivered,
         (unsigned long long)st.dropped, (unsigned long long)st.batches, st.largest_batch, bad, ok ? "OK" : "FAIL");
  return ok ? 0 : 1;
}
