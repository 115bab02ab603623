// tests/kat/queue_batch_stress.cpp — ThreadSanitizer stress of batched delivery (urf_queue_next_batch, urf_mq_next_batch)
// and int8 label slots (URF_QUEUE_LABEL8), built with -fsanitize=thread from urf_queue.cpp + urf_mq.cpp, no CUDA. P
// producers and one consumer around a stand-in batch function; exits 0 when every accepted scan was delivered exactly once
// with the right labels and per-producer order, and TSAN reported nothing (a report makes the exit code non-zero).
// usage: queue_batch_stress queue <producers> <scans per producer> <slots> <max_batch> <policy> <max_results> <label8>
//        queue_batch_stress mq <devices> <producers> <scans per producer> <max_results> <label8>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>
#include "../../include/urf.h"

// stand-ins for the CUDA side of liburf_b200.so (never reached: the queues are created with the test hooks)
extern "C" void* urf_pinned_alloc(size_t) { return nullptr; }
extern "C" void urf_pinned_free(void*) {}
extern "C" int urf_create(urf_ctx**, int, int, int) { return URF_ERR_NO_DEVICE; }
extern "C" void urf_destroy(urf_ctx*) {}
extern "C" int urf_set_params(urf_ctx*, const urf_params*) { return URF_ERR_NO_DEVICE; }

// label[i] = x[i] + 7 (x < 100, so it fits an int8 slot); one vertex per scan carrying its first x. `user` = delay in us
// (uneven stand-in devices); every 13th batch fails when g_fail is set.
static std::atomic<int> g_batches{0};
static bool g_fail = false;
static int fake(void* user, const float* const* xyzi, const int* n, int batch, urf_result* outs) {
  const int b = g_batches++;
  const long us = (long)(intptr_t)user;
  if (us) std::this_thread::sleep_for(std::chrono::microseconds(us));
  if (g_fail && b % 13 == 5) return URF_ERR_CUDA;
  for (int j = 0; j < batch; j++) {
    for (int i = 0; i < n[j]; i++) outs[j].label[i] = (int)xyzi[j][4 * i] + 7;
    outs[j].status = URF_OK; outs[j].n_in = n[j]; outs[j].n_vert = 1;
    outs[j].vert[0][0] = n[j] ? xyzi[j][0] : -1.f;
  }
  if ((b & 7) == 0) std::this_thread::yield();
  return URF_OK;
}

static int n_of(int p, long k, int N) { return 1 + (int)((k + p) % N); }
static float x_of(long k, int i) { return (float)((k + i) % 90); }

// Checks one delivered scan; `last` holds per-producer order. Returns false on a wrong payload.
static bool check(uint64_t tag, int32_t rc, const urf_result& r, const void* view, bool label8, int N, std::vector<long>& last, long& failed) {
  const int p = (int)(tag >> 32);
  const long k = (long)(tag & 0xffffffffu);
  if (k <= last[p]) return false;
  last[p] = k;
  if (rc != URF_OK) { failed++; return view == nullptr; }
  const int n = n_of(p, k, N);
  if (r.n_in != n || !view || r.n_vert != 1 || r.vert[0][0] != x_of(k, 0) || r.label || r.ring || r.order || r.ring_start) return false;
  for (int i = 0; i < n; i++) {
    const int want = (int)x_of(k, i) + 7;
    const int got = label8 ? static_cast<const int8_t*>(view)[i] : static_cast<const int32_t*>(view)[i];
    if (got != want) return false;
  }
  return true;
}

static void produce(int p, int K, int N, bool by_ref_ok, std::vector<std::vector<float>>* keep,
                    int (*sub)(void*, const float*, int, uint64_t, bool), void* target) {
  std::vector<float> pts(4 * N);
  for (int k = 0; k < K; k++) {
    const int n = n_of(p, k, N);
    const bool ref = by_ref_ok && (k & 1);
    float* dst = ref ? (*keep)[(size_t)p * K + k].data() : pts.data();
    for (int i = 0; i < n; i++) dst[4 * i] = x_of(k, i);
    const int rc = sub(target, dst, n, ((uint64_t)p << 32) | (uint64_t)k, ref);
    if (rc != URF_OK) { fprintf(stderr, "submit rc=%d\n", rc); exit(3); }
  }
}

static int queue_stress(int P, int K, int slots, int mb, int policy, int maxr, bool label8) {
  const int N = 24;
  g_fail = true;
  urf_queue* q = nullptr;
  if (urf_queue_create_with(&q, fake, nullptr, N, slots, mb, policy | (label8 ? URF_QUEUE_LABEL8 : 0)) != URF_OK) return 2;
  std::vector<std::thread> prod;
  auto sub = [](void* t, const float* x, int n, uint64_t tag, bool) { return urf_queue_submit(static_cast<urf_queue*>(t), x, n, tag, -1); };
  for (int p = 0; p < P; p++) prod.emplace_back(produce, p, K, N, false, nullptr, +sub, (void*)q);
  long delivered = 0, bad = 0, failed = 0, calls = 0, largest = 0;
  std::vector<long> last(P, -1);
  std::thread cons([&] {
    std::vector<uint64_t> tags(maxr);
    std::vector<int32_t> rcs(maxr);
    std::vector<urf_result> outs(maxr);
    std::vector<const void*> views(maxr);
    std::vector<int32_t> lab(N);
    for (;;) {
      const int mode = (int)(calls++ % 7);                    // mostly batches, now and then a single next / next_view in between
      if (mode == 3) {
        urf_result r{}; r.label = lab.data();
        uint64_t tag = 0;
        const int rc = urf_queue_next(q, &tag, &r, -1);
        if (rc == URF_ERR_CLOSED) break;
        r.label = nullptr;
        if (!check(tag, rc, r, rc == URF_OK ? lab.data() : nullptr, false, N, last, failed)) bad++;
        delivered++;
        continue;
      }
      if (mode == 5 && !label8) {
        urf_result r{};
        uint64_t tag = 0;
        const int32_t* view = nullptr;
        const int rc = urf_queue_next_view(q, &tag, &r, &view, -1);
        if (rc == URF_ERR_CLOSED) break;
        if (!check(tag, rc, r, view, false, N, last, failed)) bad++;
        delivered++;
        continue;
      }
      const int want = 1 + (int)(calls % maxr);
      const int k = urf_queue_next_batch(q, want, tags.data(), rcs.data(), outs.data(), views.data(), -1);
      if (k == URF_ERR_CLOSED) break;
      if (k < 1 || k > want) { bad++; break; }
      largest = std::max(largest, (long)k);
      for (int j = 0; j < k; j++) if (!check(tags[j], rcs[j], outs[j], views[j], label8, N, last, failed)) bad++;
      delivered += k;
    }
  });
  for (auto& t : prod) t.join();
  urf_queue_close(q);
  cons.join();
  urf_queue_stats st{};
  urf_queue_get_stats(q, &st);
  urf_queue_destroy(q);
  const bool ok = bad == 0 && st.delivered == (uint64_t)delivered && st.delivered == st.processed && st.processed + st.dropped == st.submitted &&
                  st.submitted == (uint64_t)P * K && (policy == URF_QUEUE_DROP_OLDEST || st.dropped == 0);
  printf("queue producers=%d scans=%d delivered=%ld failed=%ld dropped=%llu largest_run=%ld label8=%d bad=%ld %s\n", P, P * K, delivered, failed,
         (unsigned long long)st.dropped, largest, (int)label8, bad, ok ? "OK" : "FAIL");
  return ok ? 0 : 1;
}

// urf_mq_next_batch over stand-in devices of uneven speed: one call spans several devices, the global order holds.
static int mq_stress(int D, int P, int K, int maxr, bool label8) {
  const int N = 24;
  std::vector<void*> users(D);
  for (int d = 0; d < D; d++) users[d] = (void*)(intptr_t)((d * 37) % 5 * 40);  // 0..160 us per batch, device-dependent
  urf_mq* m = nullptr;
  const int rc0 = label8 ? urf_mq_create_with_label8(&m, fake, users.data(), D, N, 3, 2) : urf_mq_create_with(&m, fake, users.data(), D, N, 3, 2);
  if (rc0 != URF_OK) return 2;
  std::vector<std::vector<float>> keep((size_t)P * K, std::vector<float>(4 * N));   // by-reference scans stay alive until the end
  std::vector<std::thread> prod;
  auto sub = [](void* t, const float* x, int n, uint64_t tag, bool ref) {
    urf_mq* mq = static_cast<urf_mq*>(t);
    return ref ? urf_mq_submit_ref(mq, x, n, tag, -1) : urf_mq_submit(mq, x, n, tag, -1);
  };
  for (int p = 0; p < P; p++) prod.emplace_back(produce, p, K, N, true, &keep, +sub, (void*)m);
  long delivered = 0, bad = 0, failed = 0, calls = 0, largest = 0;
  std::vector<long> last(P, -1);
  std::thread cons([&] {
    std::vector<uint64_t> tags(maxr);
    std::vector<int32_t> rcs(maxr);
    std::vector<urf_result> outs(maxr);
    std::vector<const void*> views(maxr);
    std::vector<int32_t> lab(N);
    for (;;) {
      if (calls++ % 5 == 4) {                                 // a single next in between
        urf_result r{}; r.label = lab.data();
        uint64_t tag = 0;
        const int rc = urf_mq_next(m, &tag, &r, -1);
        if (rc == URF_ERR_CLOSED) break;
        r.label = nullptr;
        if (!check(tag, rc, r, rc == URF_OK ? lab.data() : nullptr, false, N, last, failed)) bad++;
        delivered++;
        continue;
      }
      const int want = 1 + (int)(calls % maxr);
      const int k = urf_mq_next_batch(m, want, tags.data(), rcs.data(), outs.data(), views.data(), -1);
      if (k == URF_ERR_CLOSED) break;
      if (k < 1 || k > want) { bad++; break; }
      largest = std::max(largest, (long)k);
      for (int j = 0; j < k; j++) if (!check(tags[j], rcs[j], outs[j], views[j], label8, N, last, failed)) bad++;
      delivered += k;
    }
  });
  for (auto& t : prod) t.join();
  urf_mq_close(m);
  cons.join();
  urf_mq_stats st{};
  urf_mq_get_stats(m, &st);
  urf_mq_destroy(m);
  uint64_t sub_n = 0, del = 0;
  for (int d = 0; d < D; d++) { sub_n += st.submitted[d]; del += st.delivered[d]; }
  const bool ok = bad == 0 && delivered == (long)P * K && sub_n == (uint64_t)P * K && del == sub_n && st.pending == 0;
  printf("mq devices=%d producers=%d scans=%d delivered=%ld failed=%ld largest_run=%ld label8=%d bad=%ld %s\n", D, P, P * K, delivered, failed,
         largest, (int)label8, bad, ok ? "OK" : "FAIL");
  return ok ? 0 : 1;
}

int main(int argc, char** argv) {
  auto arg = [&](int i, int dflt) { return argc > i ? atoi(argv[i]) : dflt; };
  if (argc > 1 && !strcmp(argv[1], "mq")) return mq_stress(arg(2, 4), arg(3, 2), arg(4, 800), arg(5, 8), arg(6, 1) != 0);
  if (argc > 1 && !strcmp(argv[1], "queue"))
    return queue_stress(arg(2, 4), arg(3, 1500), arg(4, 6), arg(5, 4), arg(6, URF_QUEUE_BLOCK), arg(7, 6), arg(8, 1) != 0);
  fprintf(stderr, "usage: see the header of tests/kat/queue_batch_stress.cpp\n");
  return 2;
}
