// tests/kat/queue_formats_stress.cpp — ThreadSanitizer stress of a formats mq (urf_mq_create_formats_with: PointCloud2
// records of several formats over stand-in devices; built with -fsanitize=thread from urf_queue.cpp + urf_mq.cpp, no CUDA).
// Several producers submit records, scan k of producer p in format (k + p) % 4 of a four-format table (48-, 32-, packed 22-
// and 16-byte records), alternating urf_mq_submit_format from one scratch buffer that they overwrite as soon as the call
// returns and urf_mq_submit_format_ref from buffers that stay untouched until the end; one thread updates the parameters at
// random moments; one consumer takes batches with urf_mq_next_batch. Every stand-in device reads each scan's format index
// from its urf_formats_user, decodes the records at that format's offsets, and writes labels (and with URF_QUEUE_ORDER an
// order and ring offsets) that are functions of the scan's producer, number and size and of the generation its batch ran
// with. Exits 0 when
//   - every stand-in call got the mq's format table, each scan its submitted format index, and every record it decoded held
//     the scan it belongs to;
//   - every delivered scan's labels (and order[:n_order], ring_start[:n_rings + 1]) hold exactly that payload for its tag
//     and params_gen;
//   - one producer's scans come back in its order, each accepted scan exactly once;
//   - some batch mixed formats, unless no batch held more than one scan;
// and TSAN reported nothing (TSAN makes the exit code non-zero on a report).
// usage: queue_formats_stress <producers> <scans per producer> <devices> <slots per device> <policy (LABEL8 / ORDER bits)>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <thread>
#include <vector>
#include "../../include/urf.h"

// stand-ins for the CUDA side of liburf_b200.so (never reached: the mq is created around stand-in devices)
extern "C" void* urf_pinned_alloc(size_t) { return nullptr; }
extern "C" void urf_pinned_free(void*) {}
extern "C" int urf_create(urf_ctx**, int, int, int) { return URF_ERR_NO_DEVICE; }
extern "C" void urf_destroy(urf_ctx*) {}
extern "C" int urf_set_params(urf_ctx*, const urf_params*) { return URF_ERR_NO_DEVICE; }

namespace {
constexpr int N = 24;                                  // largest scan
constexpr int F = 4;
const urf_cloud2_format kTable[F] = {{48, 0, 4, 8, 16}, {32, 0, 4, 8, 16}, {22, 0, 4, 8, 12}, {16, 0, 4, 8, 12}};

int n_of(int p, long k) { return 1 + (int)((k + p) % N); }
int fmt_of(int p, long k) { return (int)((k + p) % F); }
int label_of(long k, int i) { return (int)(k % 100 + i) + 7; }
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

// Record i of scan k of producer p in format f: x = i, y = p, z = k, intensity = -i, and the other bytes a function of all.
void fill(unsigned char* rec, int p, long k, int n, const urf_cloud2_format& f) {
  for (int i = 0; i < n; i++) {
    unsigned char* r = rec + (size_t)i * f.point_step;
    for (int b = 0; b < f.point_step; b++) r[b] = (unsigned char)(b + i + p + k);
    const float v[4] = {(float)i, (float)p, (float)k, -(float)i};
    const int off[4] = {f.off_x, f.off_y, f.off_z, f.off_intensity};
    for (int c = 0; c < 4; c++) std::memcpy(r + off[c], &v[c], sizeof(float));
  }
}

struct Device {                                        // touched only by its queue's worker thread (batch function and hook)
  int32_t gen = 0;
  long bad_table = 0, bad_records = 0, mixed = 0;
  int largest = 0;
};

int hook(void* user, const urf_params*, int32_t gen) {
  static_cast<Device*>(static_cast<urf_formats_user*>(user)->user)->gen = gen;
  return URF_OK;
}

int process(void* user, const float* const* xyzi, const int* n, int batch, urf_result* outs) {
  const urf_formats_user* u = static_cast<const urf_formats_user*>(user);
  Device* d = static_cast<Device*>(u->user);
  if (u->n_formats != F || std::memcmp(u->formats, kTable, sizeof(kTable)) != 0 || !u->fmt) { d->bad_table++; return URF_OK; }
  d->largest = std::max(d->largest, batch);
  bool mixed = false;
  for (int j = 0; j < batch; j++) {
    const int fi = u->fmt[j];
    mixed |= fi != u->fmt[0];
    if (fi < 0 || fi >= F) { d->bad_table++; continue; }
    const urf_cloud2_format& f = kTable[fi];
    const unsigned char* rec = reinterpret_cast<const unsigned char*>(xyzi[j]);
    float y, z;
    std::memcpy(&y, rec + f.off_y, sizeof(float));
    std::memcpy(&z, rec + f.off_z, sizeof(float));
    const int p = (int)y;
    const long k = (long)z;
    std::vector<unsigned char> want((size_t)n[j] * f.point_step);
    fill(want.data(), p, k, n[j], f);
    if (n[j] != n_of(p, k) || fi != fmt_of(p, k) || std::memcmp(want.data(), rec, want.size()) != 0) d->bad_records++;
    urf_result& o = outs[j];
    for (int i = 0; i < n[j]; i++) o.label[i] = label_of(k, i);
    o.status = URF_OK; o.n_in = n[j];
    if (!o.order || !o.ring_start) continue;
    const Payload py = payload(p, k, n[j], d->gen);
    o.n_order = py.n_order; o.n_rings = py.n_rings;
    for (int i = 0; i < py.n_order; i++) o.order[i] = py.order(i);
    for (int r = 0; r <= py.n_rings; r++) o.ring_start[r] = py.ring_start(r);
  }
  d->mixed += mixed;
  return URF_OK;
}
}  // namespace

int main(int argc, char** argv) {
  const int P = argc > 1 ? atoi(argv[1]) : 4, K = argc > 2 ? atoi(argv[2]) : 2000, D = argc > 3 ? atoi(argv[3]) : 3,
            slots = argc > 4 ? atoi(argv[4]) : 4, policy = argc > 5 ? atoi(argv[5]) : URF_QUEUE_ORDER;
  const bool label8 = (policy & URF_QUEUE_LABEL8) != 0, order = (policy & URF_QUEUE_ORDER) != 0;
  std::vector<Device> devs(D);
  std::vector<void*> users(D);
  for (int d = 0; d < D; d++) users[d] = &devs[d];
  urf_mq* mq = nullptr;
  if (urf_mq_create_formats_with(&mq, process, users.data(), D, N, slots, 3, policy, kTable, F) != URF_OK) return 2;
  if (urf_mq_set_params_hook(mq, hook) != URF_OK) return 2;
  std::atomic<bool> producing{true};
  std::atomic<int32_t> updates{0};
  std::thread updater([&] {
    std::mt19937 rng(4242);
    while (producing.load()) {
      std::this_thread::sleep_for(std::chrono::microseconds(rng() % 500));
      urf_params p{};
      p.interval = 0.18; p.beamZone = 30; p.channels = 64;
      p.curb_points = 1 + updates.load() % 4096;
      if (urf_mq_update_params(mq, &p) != updates.load() + 1) { fprintf(stderr, "update failed\n"); exit(3); }
      updates++;
    }
  });
  std::atomic<long> accepted{0}, by_ref{0};
  std::vector<std::vector<unsigned char>> kept(P);     // by-reference records: untouched until every result is in
  std::vector<std::thread> prod;
  for (int p = 0; p < P; p++) prod.emplace_back([&, p] {
    std::vector<unsigned char>& mine = kept[p];
    mine.resize((size_t)K * N * URF_MAX_POINT_STEP);
    std::vector<unsigned char> scratch((size_t)N * URF_MAX_POINT_STEP);
    for (int k = 0; k < K; k++) {
      const int n = n_of(p, k), f = fmt_of(p, k);
      const uint64_t tag = ((uint64_t)p << 32) | (uint64_t)k;
      int rc;
      if ((k / F + p) % 2) {
        unsigned char* rec = mine.data() + (size_t)k * N * URF_MAX_POINT_STEP;
        fill(rec, p, k, n, kTable[f]);
        rc = urf_mq_submit_format_ref(mq, f, rec, n, tag, -1);
        by_ref++;
      } else {
        fill(scratch.data(), p, k, n, kTable[f]);
        rc = urf_mq_submit_format(mq, f, scratch.data(), n, tag, -1);
        std::memset(scratch.data(), 0xab, scratch.size());   // the mq copied the records: overwriting them changes nothing
      }
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
    std::mt19937 rng(17);
    for (;;) {
      const int k = urf_mq_next_batch(mq, 1 + (int)(rng() % 8), tags.data(), rcs.data(), outs.data(), views.data(), -1);
      if (k == URF_ERR_CLOSED) break;
      if (k < 1) { bad++; continue; }
      for (int j = 0; j < k; j++) {
        const int p = (int)(tags[j] >> 32); const long s = (long)(tags[j] & 0xffffffffu);
        if (s <= last[p]) bad++;
        last[p] = s;
        delivered++;
        const urf_result& o = outs[j];
        const int n = n_of(p, s);
        if (rcs[j] != URF_OK || o.n_in != n || !views[j] || (order != (o.order != nullptr))) { bad++; continue; }
        for (int i = 0; i < n; i++) {
          const int v = label8 ? static_cast<const int8_t*>(views[j])[i] : static_cast<const int32_t*>(views[j])[i];
          if (v != (label8 ? (int)(int8_t)label_of(s, i) : label_of(s, i))) { bad++; break; }
        }
        if (order) {
          const Payload y = payload(p, s, n, o.params_gen);
          if (o.n_order != y.n_order || o.n_rings != y.n_rings) { bad++; continue; }
          for (int i = 0; i < y.n_order; i++) if (o.order[i] != y.order(i)) { bad++; break; }
          for (int r = 0; r <= y.n_rings; r++) if (o.ring_start[r] != y.ring_start(r)) { bad++; break; }
        }
        checked++;
      }
    }
  });
  for (auto& t : prod) t.join();
  producing.store(false);
  updater.join();
  urf_mq_close(mq);
  cons.join();
  urf_mq_stats st{};
  urf_mq_get_stats(mq, &st);
  urf_mq_destroy(mq);
  uint64_t submitted = 0, got = 0;
  long bad_table = 0, bad_records = 0, mixed = 0;
  int largest = 0;
  for (int d = 0; d < D; d++) {
    submitted += st.submitted[d]; got += st.delivered[d];
    bad_table += devs[d].bad_table; bad_records += devs[d].bad_records; mixed += devs[d].mixed;
    largest = std::max(largest, devs[d].largest);
  }
  const bool ok = bad == 0 && bad_table == 0 && bad_records == 0 && checked == delivered && delivered == accepted.load() &&
                  submitted == (uint64_t)accepted.load() && got == (uint64_t)delivered && updates.load() > 1 && by_ref.load() > 0 &&
                  (mixed > 0 || largest <= 1);
  printf("producers=%d devices=%d scans=%ld by_reference=%ld delivered=%ld checked=%ld updates=%d largest_batch=%d mixed_batches=%ld "
         "bad_table=%ld bad_records=%ld bad=%ld %s\n", P, D, accepted.load(), by_ref.load(), delivered, checked, updates.load(), largest,
         mixed, bad_table, bad_records, bad, ok ? "OK" : "FAIL");
  return ok ? 0 : 1;
}
