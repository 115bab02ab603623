// tools/mq_bench.cpp — throughput of the multi-GPU ingest (include/urf.h urf_mq) from ONE process: K distinct scans (raw
// float4 records read from a file written by scripts/bench_mq.py) are streamed `rounds` times through N devices by P
// producer threads and one consumer, once with copying submits (memcpy into the device queue's pinned slot) and once by
// reference (scans already in pinned memory, no host copy). Prints one JSON line per mode: scans/s and the host-side
// limiter it points at. Host tool: links liburf_b200.so, no CUDA code of its own.
//   usage: mq_bench <scans.bin> <points per scan> <n_scans_in_file> <n_devices> <producers> <total scans> <slots> <max_batch>
//          [full_roi channels interval [modes max_results [order]]]
// modes: comma-separated subset of 0 (copying submit), 1 (by reference), 2 (by reference, labels viewed in place with
// urf_mq_next_view), 3 (by reference, int8 label slots, results taken with urf_mq_next_batch, up to max_results per call);
// default 0,1,2. order: 1 creates the device queues with URF_QUEUE_ORDER (every batch runs the ring sort and copies the
// emission order back; mode 3 reads n_order of every view); default 0.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>
#include "../include/urf.h"

int main(int argc, char** argv) {
  if (argc < 9) { fprintf(stderr, "usage: see the header of tools/mq_bench.cpp\n"); return 2; }
  const char* path = argv[1];
  const int n = atoi(argv[2]), K = atoi(argv[3]), D = atoi(argv[4]), P = atoi(argv[5]), total = atoi(argv[6]), slots = atoi(argv[7]),
            mb = atoi(argv[8]);
  const int full_roi = argc > 9 ? atoi(argv[9]) : 1, channels = argc > 10 ? atoi(argv[10]) : 64;
  const double interval = argc > 11 ? atof(argv[11]) : 0.18;
  std::vector<int> modes = {0, 1, 2};
  if (argc > 12) { modes.clear(); for (const char* c = argv[12]; *c; c++) if (*c >= '0' && *c <= '3') modes.push_back(*c - '0'); }
  const int max_results = argc > 13 ? atoi(argv[13]) : 64;
  const bool order = argc > 14 && atoi(argv[14]) != 0;
  const size_t bytes = (size_t)n * 16;
  std::vector<float*> pinned(K);
  FILE* f = fopen(path, "rb");
  if (!f) { perror(path); return 2; }
  for (int k = 0; k < K; k++) {
    pinned[k] = static_cast<float*>(urf_pinned_alloc(bytes));
    if (!pinned[k] || fread(pinned[k], 1, bytes, f) != bytes) { fprintf(stderr, "cannot read scan %d\n", k); return 2; }
  }
  fclose(f);
  std::vector<std::vector<float>> pageable(K);                    // the copying mode reads from ordinary (pageable) memory, like a driver
  for (int k = 0; k < K; k++) pageable[k].assign(pinned[k], pinned[k] + (size_t)n * 4);
  urf_params prm;
  urf_default_params(&prm);
  prm.channels = channels; prm.interval = interval;
  if (full_roi) { prm.min_x = prm.min_y = prm.min_z = -200; prm.max_x = prm.max_y = prm.max_z = 200; }
  std::vector<int> devs(D);
  for (int d = 0; d < D; d++) devs[d] = d;
  for (int mode : modes) {                                        // 0: copying submit, 1: by reference (pinned), 2: 1 + labels viewed in place,
                                                                  // 3: 1 + int8 slots delivered in runs (urf_mq_next_batch)
    urf_mq* mq = nullptr;
    const int policy = URF_QUEUE_BLOCK | (mode == 3 ? URF_QUEUE_LABEL8 : 0) | (order ? URF_QUEUE_ORDER : 0);
    int rc = urf_mq_create_policy(&mq, devs.data(), D, n, slots, mb, &prm, policy);
    if (rc != URF_OK) { fprintf(stderr, "urf_mq_create: %s (%s)\n", urf_strerror(rc), urf_last_cuda_error(nullptr)); return 1; }
    std::vector<int32_t> lab(n);
    std::atomic<long> road{0}, ordered{0};
    auto run = [&](int count, bool timed) {
      std::vector<std::thread> prod;
      const auto t0 = std::chrono::steady_clock::now();
      for (int p = 0; p < P; p++) prod.emplace_back([&, p] {
        for (int i = p; i < count; i += P) {
          const int k = i % K;
          const int r = mode ? urf_mq_submit_ref(mq, pinned[k], n, (uint64_t)i, -1) : urf_mq_submit(mq, pageable[k].data(), n, (uint64_t)i, -1);
          if (r != URF_OK) { fprintf(stderr, "submit: %s\n", urf_strerror(r)); exit(1); }
        }
      });
      std::thread cons([&] {
        if (mode == 3) {
          std::vector<uint64_t> tags(max_results);
          std::vector<int32_t> rcs(max_results);
          std::vector<urf_result> outs(max_results);
          std::vector<const void*> views(max_results);
          for (int i = 0; i < count;) {
            const int k = urf_mq_next_batch(mq, std::min(max_results, count - i), tags.data(), rcs.data(), outs.data(), views.data(), -1);
            if (k < 1) { fprintf(stderr, "next_batch: %s\n", urf_strerror(k)); exit(1); }
            for (int j = 0; j < k; j++) {
              if (rcs[j] != URF_OK) { fprintf(stderr, "next_batch: %s\n", urf_strerror(rcs[j])); exit(1); }
              if (timed) road += outs[j].n_road;
              if (timed && outs[j].order && outs[j].ring_start && outs[j].n_order > 0)
                ordered += outs[j].order[outs[j].n_order - 1] >= 0 ? outs[j].n_order : 0;
            }
            i += k;
          }
          return;
        }
        for (int i = 0; i < count; i++) {
          urf_result res; memset(&res, 0, sizeof(res)); res.label = lab.data();
          uint64_t tag;
          const int32_t* view = nullptr;
          const int r = mode == 2 ? urf_mq_next_view(mq, &tag, &res, &view, -1) : urf_mq_next(mq, &tag, &res, -1);
          if (r != URF_OK) { fprintf(stderr, "next: %s\n", urf_strerror(r)); exit(1); }
          if (timed) road += res.n_road;
        }
      });
      for (auto& t : prod) t.join();
      cons.join();
      return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    };
    run(std::min(total, 4 * D * mb), false);                      // warm-up
    const double s = run(total, true);
    urf_mq_stats st;
    urf_mq_get_stats(mq, &st);
    int largest = 0; unsigned long long mn = ~0ull, mx = 0;
    for (int d = 0; d < D; d++) { largest = st.largest_batch[d] > largest ? st.largest_batch[d] : largest; mn = st.submitted[d] < mn ? st.submitted[d] : mn; mx = st.submitted[d] > mx ? st.submitted[d] : mx; }
    printf("{\"mq_bench\": \"%s\", \"devices\": %d, \"producers\": %d, \"points_per_scan\": %d, \"scans\": %d, \"seconds\": %.4f, \"scans_per_sec\": %.1f, "
           "\"mpoints_per_sec\": %.1f, \"h2d_gb_per_sec\": %.2f, \"largest_batch\": %d, \"per_device_min_max\": [%llu, %llu], \"road_points\": %ld, "
           "\"order\": %d, \"ordered_points\": %ld}\n",
           mode == 3 ? "by_reference_pinned_label8_next_batch" : mode == 2 ? "by_reference_pinned_labels_viewed_in_place" : mode ? "by_reference_pinned" : "copying_submit", D, P, n, total, s, total / s, total / s * n / 1e6, total / s * bytes / 1e9, largest, mn, mx,
           road.load(), (int)order, ordered.load());
    fflush(stdout);
    urf_mq_destroy(mq);
  }
  for (float* p : pinned) urf_pinned_free(p);
  return 0;
}
