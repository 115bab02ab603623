// tests/kat/lomuto_check.cpp — urban_road_filter_b200/csrc/urf_lomuto.cuh (the reference tie order k_lomuto_rings computes
// on the device) run sequentially with SeqLomuto, against lomuto_sort of the CPU oracle (oracle/urf_oracle.cpp, compiled
// into this program as it is), which restates the reference's quicksort (lidar_segmentation.cpp:70-93).
// Arrays: random with ties (sizes 0..20000), NaN anywhere (as the pivot too), all-equal, non-decreasing, non-increasing,
// rotated, and dual-return rings (interleaved / appended, both azimuth directions); `-f file` adds rings from a file
// (records: int32 n, then n float32). Prints mismatches=..., and for the sensor-ordered rings the partition count and
// the element steps (elements of every subproblem taken from the stack).
// usage: lomuto_check [rounds] [-f rings.bin]
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "../../oracle/urf_oracle.cpp"
#include "../../urban_road_filter_b200/csrc/urf_lomuto.cuh"

static long g_cases = 0, g_bad = 0;

// one ring: the device's inputs (azimuth bits, rank in (bits, position) order as k_sort_rings leaves it), then both sorts
static bool check(const std::vector<float>& a, const char* stat) {
  const int n = (int)a.size();
  std::vector<unsigned> az(n), rk(n), s0(n), s1(n), s2(n);
  std::vector<int> by(n), perm(n);
  for (int i = 0; i < n; i++) { memcpy(&az[i], &a[i], 4); by[i] = i; perm[i] = i; }
  std::stable_sort(by.begin(), by.end(), [&](int x, int y) { return az[x] < az[y]; });
  for (int r = 0; r < n; r++) rk[by[r]] = (unsigned)r;
  urf::LomutoArrays w{az.data(), rk.data(), s0.data(), s1.data(), s2.data()};
  urf::LomutoShared sh{};
  urf::lomuto_ring<urf::SeqLomuto>(w, n, sh);
  lomuto_sort(a, perm);
  g_cases++;
  for (int i = 0; i < n; i++)
    if ((int)s0[i] != perm[i]) {
      if (g_bad++ < 5) fprintf(stderr, "n=%d (%s): position %d holds %u, the quicksort put %d there\n", n, stat ? stat : "random", i, s0[i], perm[i]);
      return false;
    }
  if (stat) printf("stat %s n=%d partitions=%lld steps=%lld\n", stat, n, sh.partitions, sh.steps);
  return true;
}

// a sensor ring of m columns starting at azimuth `start`, turning up (dir = 1) or down (-1); dual: every column twice,
// the second return right after the first (interleaved) or all second returns after the scan (appended)
static std::vector<float> sensor_ring(int m, float start, int dir, int dual, bool interleave) {
  std::vector<float> col(m), out;
  for (int c = 0; c < m; c++) {
    float v = start + dir * (360.0f / m) * c;
    v = std::fmod(v + 720.0f, 360.0f);
    col[c] = v;
  }
  if (!dual) return col;
  if (interleave) for (float v : col) { out.push_back(v); out.push_back(v); }
  else { out = col; out.insert(out.end(), col.begin(), col.end()); }
  return out;
}

int main(int argc, char** argv) {
  int rounds = 3000;
  const char* file = nullptr;
  for (int i = 1; i < argc; i++) {
    if (!strcmp(argv[i], "-f") && i + 1 < argc) file = argv[++i];
    else rounds = atoi(argv[i]);
  }
  std::mt19937 g(20261016);
  const float qnan = std::numeric_limits<float>::quiet_NaN();
  for (int round = 0; round < rounds; round++) {
    const int n = round < 64 ? round : (int)(g() % (round % 100 == 0 ? 20001 : 2000));
    const int distinct = 1 + (int)(g() % (round % 3 == 0 ? 3 : (round % 3 == 1 ? 50 : 5000)));
    std::vector<float> a(n);
    for (float& x : a) x = 0.125f * (float)(g() % distinct);
    switch (round % 6) {
      case 1: std::sort(a.begin(), a.end()); break;
      case 2: std::sort(a.begin(), a.end()); std::reverse(a.begin(), a.end()); break;
      case 3: std::sort(a.begin(), a.end()); if (n) std::rotate(a.begin(), a.begin() + g() % n, a.end()); break;
      default: break;
    }
    if (n && round % 5 == 0) { const int k = 1 + (int)(g() % 3); for (int t = 0; t < k; t++) a[g() % n] = qnan; }
    if (n && round % 7 == 0) a[n - 1] = qnan;                      // NaN pivot of the first partition
    check(a, nullptr);
  }
  for (int n : {2, 3, 17, 1000, 7000}) {
    check(std::vector<float>(n, 37.25f), nullptr);                                    // all equal
    std::vector<float> v(n, qnan);
    check(v, nullptr);                                                                 // all NaN
    v.assign(n, 5.0f); v[n / 2] = qnan; check(v, nullptr);
  }
  char name[96];
  for (int m : {64, 900, 2048})
    for (int dir : {1, -1})
      for (int dual = 0; dual < 2; dual++)
        for (int il = 0; il < (dual ? 2 : 1); il++)
          for (float start : {0.0f, 123.4f}) {
            snprintf(name, sizeof(name), "%s_%s_m%d_%s_start%g", dual ? (il ? "dual_interleaved" : "dual_appended") : "single",
                     dir > 0 ? "up" : "down", m, "ring", start);
            check(sensor_ring(m, start, dir, dual, il), name);
          }
  if (file) {
    FILE* fp = fopen(file, "rb");
    if (!fp) { fprintf(stderr, "cannot open %s\n", file); return 2; }
    int n, k = 0;
    while (fread(&n, 4, 1, fp) == 1) {
      std::vector<float> a(n);
      if (n && fread(a.data(), 4, n, fp) != (size_t)n) { fprintf(stderr, "short file\n"); return 2; }
      snprintf(name, sizeof(name), "file_ring%d", k++);
      check(a, name);
    }
    fclose(fp);
  }
  printf("cases=%ld mismatches=%ld\n", g_cases, g_bad);
  return g_bad ? 1 : 0;
}
