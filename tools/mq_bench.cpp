// tools/mq_bench.cpp — throughput of the multi-GPU ingest (include/urf.h urf_mq) from ONE process: K distinct scans (raw
// float4 records read from a file written by scripts/bench_mq.py) are streamed `rounds` times through N devices by P
// producer threads and one consumer, once with copying submits (memcpy into the device queue's pinned slot) and once by
// reference (scans already in pinned memory, no host copy). Prints one JSON line per mode: scans/s and the host-side
// limiter it points at. Host tool: links liburf_b200.so, no CUDA code of its own.
//   usage: mq_bench <scans.bin> <points per scan> <n_scans_in_file> <n_devices> <producers> <total scans> <slots> <max_batch>
//          [full_roi channels interval [modes max_results [order [point_step off_x off_y off_z off_intensity]]]]
// modes: comma-separated subset of 0 (copying submit), 1 (by reference), 2 (by reference, labels viewed in place with
// urf_mq_next_view), 3 (by reference, int8 label slots, results taken with urf_mq_next_batch, up to max_results per call);
// default 0,1,2. order: 1 creates the device queues with URF_QUEUE_ORDER (every batch runs the ring sort and copies the
// emission order back; mode 3 reads n_order of every view); default 0.
// point_step > 0: the file holds PointCloud2 records of that many bytes per point (x / y / z / intensity FLOAT32 at the
// offsets given, off_intensity -1: none) instead of float4 points, and only the record modes run, both delivered as mode 3:
//   4: a record mq (urf_mq_create_cloud2), scans submitted as they are with urf_mq_submit_cloud2_ref;
//   5: a float4 mq; each producer first repacks the scan's records into (x, y, z, intensity) points, inside the timed
//      region, into the next of its own D * slots + 1 pinned buffers, and submits that with urf_mq_submit_ref. A scan of a
//      producer cannot be undelivered D * slots + 1 submits later (the mq holds D * slots scans), so a buffer is never
//      rewritten before its scan's copy has run.
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
  if (argc > 12) { modes.clear(); for (const char* c = argv[12]; *c; c++) if (*c >= '0' && *c <= '5') modes.push_back(*c - '0'); }
  const int max_results = argc > 13 ? atoi(argv[13]) : 64;
  const bool order = argc > 14 && atoi(argv[14]) != 0;
  const int step = argc > 15 ? atoi(argv[15]) : 0, ox = argc > 16 ? atoi(argv[16]) : 0, oy = argc > 17 ? atoi(argv[17]) : 4,
            oz = argc > 18 ? atoi(argv[18]) : 8, oi = argc > 19 ? atoi(argv[19]) : -1;
  for (int m : modes)
    if ((m >= 4) != (step > 0)) { fprintf(stderr, "modes 4 and 5 need a record file (point_step > 0), modes 0-3 a float4 file\n"); return 2; }
  const size_t bytes = (size_t)n * (step > 0 ? step : 16);       // one scan in the file
  std::vector<float*> pinned(K);
  FILE* f = fopen(path, "rb");
  if (!f) { perror(path); return 2; }
  for (int k = 0; k < K; k++) {
    pinned[k] = static_cast<float*>(urf_pinned_alloc(bytes));
    if (!pinned[k] || fread(pinned[k], 1, bytes, f) != bytes) { fprintf(stderr, "cannot read scan %d\n", k); return 2; }
  }
  fclose(f);
  std::vector<std::vector<float>> pageable(K);                    // the copying mode reads from ordinary (pageable) memory, like a driver
  if (step == 0) for (int k = 0; k < K; k++) pageable[k].assign(pinned[k], pinned[k] + (size_t)n * 4);
  const int ring = D * slots + 1;                                 // mode 5: repack buffers per producer
  std::vector<std::vector<float*>> repacked(P);
  if (std::find(modes.begin(), modes.end(), 5) != modes.end())
    for (auto& bufs : repacked)
      for (int r = 0; r < ring; r++) {
        bufs.push_back(static_cast<float*>(urf_pinned_alloc((size_t)n * 16)));
        if (!bufs.back()) { fprintf(stderr, "cannot allocate repack buffers\n"); return 2; }
      }
  auto repack = [&](const unsigned char* rec, float* dst) {       // what a producer without record submits does per scan
    for (int i = 0; i < n; i++, rec += step, dst += 4) {
      std::memcpy(dst, rec + ox, 4); std::memcpy(dst + 1, rec + oy, 4); std::memcpy(dst + 2, rec + oz, 4);
      if (oi >= 0) std::memcpy(dst + 3, rec + oi, 4); else dst[3] = 0.f;
    }
  };
  urf_params prm;
  urf_default_params(&prm);
  prm.channels = channels; prm.interval = interval;
  if (full_roi) { prm.min_x = prm.min_y = prm.min_z = -200; prm.max_x = prm.max_y = prm.max_z = 200; }
  std::vector<int> devs(D);
  for (int d = 0; d < D; d++) devs[d] = d;
  for (int mode : modes) {                                        // 0: copying submit, 1: by reference (pinned), 2: 1 + labels viewed in place,
                                                                  // 3: 1 + int8 slots delivered in runs (urf_mq_next_batch),
                                                                  // 4: records by reference, 5: records repacked, both as 3
    urf_mq* mq = nullptr;
    const int policy = URF_QUEUE_BLOCK | (mode >= 3 ? URF_QUEUE_LABEL8 : 0) | (order ? URF_QUEUE_ORDER : 0);
    int rc = mode == 4 ? urf_mq_create_cloud2(&mq, devs.data(), D, n, slots, mb, &prm, policy, step, ox, oy, oz, oi)
                       : urf_mq_create_policy(&mq, devs.data(), D, n, slots, mb, &prm, policy);
    if (rc != URF_OK) { fprintf(stderr, "urf_mq_create: %s (%s)\n", urf_strerror(rc), urf_last_cuda_error(nullptr)); return 1; }
    std::vector<int32_t> lab(n);
    std::atomic<long> road{0}, ordered{0};
    auto run = [&](int count, bool timed) {
      std::vector<std::thread> prod;
      const auto t0 = std::chrono::steady_clock::now();
      for (int p = 0; p < P; p++) prod.emplace_back([&, p] {
        int next_buf = 0;
        for (int i = p; i < count; i += P) {
          const int k = i % K;
          int r;
          if (mode == 4) r = urf_mq_submit_cloud2_ref(mq, pinned[k], n, (uint64_t)i, -1);
          else if (mode == 5) {
            float* buf = repacked[p][next_buf];
            next_buf = (next_buf + 1) % ring;
            repack(reinterpret_cast<const unsigned char*>(pinned[k]), buf);
            r = urf_mq_submit_ref(mq, buf, n, (uint64_t)i, -1);
          } else r = mode ? urf_mq_submit_ref(mq, pinned[k], n, (uint64_t)i, -1) : urf_mq_submit(mq, pageable[k].data(), n, (uint64_t)i, -1);
          if (r != URF_OK) { fprintf(stderr, "submit: %s\n", urf_strerror(r)); exit(1); }
        }
      });
      std::thread cons([&] {
        if (mode >= 3) {
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
    const int h2d_bytes = mode == 4 ? step : 16;                  // input bytes per point that cross PCIe
    static const char* const names[] = {"copying_submit", "by_reference_pinned", "by_reference_pinned_labels_viewed_in_place",
                                        "by_reference_pinned_label8_next_batch", "records_by_reference_label8_next_batch",
                                        "records_repacked_to_float4_by_reference_label8_next_batch"};
    printf("{\"mq_bench\": \"%s\", \"devices\": %d, \"producers\": %d, \"points_per_scan\": %d, \"scans\": %d, \"seconds\": %.4f, \"scans_per_sec\": %.1f, "
           "\"mpoints_per_sec\": %.1f, \"h2d_gb_per_sec\": %.2f, \"largest_batch\": %d, \"per_device_min_max\": [%llu, %llu], \"road_points\": %ld, "
           "\"order\": %d, \"ordered_points\": %ld, \"h2d_bytes_per_point\": %d}\n",
           names[mode], D, P, n, total, s, total / s, total / s * n / 1e6, total / s * n * h2d_bytes / 1e9, largest, mn, mx,
           road.load(), (int)order, ordered.load(), h2d_bytes);
    fflush(stdout);
    urf_mq_destroy(mq);
  }
  for (float* p : pinned) urf_pinned_free(p);
  for (auto& bufs : repacked) for (float* p : bufs) urf_pinned_free(p);
  return 0;
}
