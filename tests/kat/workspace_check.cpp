// workspace_check: the per-scan workspace layout of urf_workspace.cuh, without a GPU. Over a grid of capacities
// (max_points, max_batch), launch strides, batches, stream-group counts, host chunkings and channel counts it checks that
//   1. every view of every sub-batch, out to the farthest element its kernels index for that extent, lies inside its
//      allocation;
//   2. the views of the sub-batches of one launch (and the scans inside one view) are pairwise disjoint, array by array;
//   3. the two host slots share no per-slot array;
//   4. the capacity sizes equal the known answers below.
// The arrays are "allocated" at made-up addresses by the same alloc_arrays / class split the library uses; nothing is
// dereferenced. Prints "cases=N failures=F" last; exits 1 on a failure.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../urban_road_filter_b200/csrc/urf_workspace.cuh"

using namespace urf;

namespace {

const char* const kNames[] = {"in",  "alpha_v", "mark", "ringid", "sect",    "label", "label8",   "bpt",  "sr",   "sz",  "sidx", "ssrz",
                              "ssl", "az",      "d2",   "baz",    "roadlist", "roadcnt", "Tf",     "Tb",   "lut",  "order", "epos", "lomuto",
                              "sortbuf", "hist", "firstidx", "cmin", "cmax", "ne",     "newY",     "n",    "out",  "tab"};
static_assert(sizeof(kNames) / sizeof(kNames[0]) == kArrays, "one name per array");

long long g_cases = 0, g_fail = 0;
void fail(const char* what, int i, long long a, long long b, long long c) {
  if (g_fail++ < 20) std::printf("FAIL %s array=%s %lld %lld %lld\n", what, kNames[i], a, b, c);
}

// Farthest element + 1 that the kernels index in one scan's slice, restated from their index expressions
size_t reach(Kind k, size_t S, size_t C) {
  const size_t T = (S + kChunk - 1) / kChunk;
  switch (k) {
    case Kind::Point: return S;                                     // point i < n <= S
    case Kind::Pair: return 2 * (S - 1) + 2;                      // sortbuf[2 * i], [2 * i + 1]
    case Kind::Warp: return ((S - 1) >> 5) + 1;                     // roadcnt[i >> 5]
    case Kind::ChunkRows: return (T - 1) * C + C;                   // hist row (chunk), ring k < C
    case Kind::TTable: return (size_t)(kTStride - 1) * C + C;       // (j, k) at j * C + k
    case Kind::DegBins: return (C - 1) * kDegBins + kDegBins;       // (k, bin) at k * kDegBins + bin
    case Kind::DegSum: return (C - 1) * (kDegBins + 1) + kDegBins + 1;
    case Kind::Elev: return kElevBins + 1;
    case Kind::RingList: return kRingKeys + 1;                      // count, then up to kRingKeys rings
    case Kind::Scan: return 1;
    case Kind::Shared: return 0;
  }
  return 0;
}

struct Alloc {
  uintptr_t base = 0;
  size_t bytes = 0;
};

// A context's arrays at made-up addresses: the workspace with slot 0's arrays (urf_create), the on-demand arrays, and
// slot 1 (the first asynchronous batch); every array records its allocation.
struct Ctx {
  Extent cap;
  size_t B;
  DevBuffers ws{}, s0{}, s1{};
  Alloc a_ws[kArrays], a_s0[kArrays], a_s1[kArrays];
  size_t elems[kArrays] = {};                                       // capacity elements per array
  uintptr_t next = uintptr_t(1) << 40;

  template <class Pick> void alloc(DevBuffers& d, Alloc* a, Pick pick) {
    alloc_arrays(d, cap, B, pick, [&](int i, auto& p, size_t count) {
      const size_t bytes = count * sizeof(*p);
      p = reinterpret_cast<std::remove_reference_t<decltype(p)>>(next);
      a[i] = {next, bytes};
      elems[i] = count;
      next += (bytes + 256 + 4095) & ~size_t(4095);
      return 0;
    });
  }
  Ctx(int max_points, int max_batch) : cap(capacity_extent((max_points + kChunk - 1) / kChunk * kChunk)), B(max_batch) {
    alloc(ws, a_ws, created_with_context);                           // the library's allocations, in its order
    alloc(s0, a_s0, slot_array);
    alloc(ws, a_ws, tie_order_array);
    alloc(s0, a_s0, label8_array);
    alloc(s1, a_s1, slot_array);
    alloc(s1, a_s1, label8_array);
    ws = slot_view(ws, s0);
  }
};

// the allocation each member of a view of slot `slot` must lie in
const Alloc& home(const Ctx& x, int slot, int i, unsigned c) { return (c & kSlot) ? (slot ? x.a_s1[i] : x.a_s0[i]) : x.a_ws[i]; }

// One launch of `batch` scans of stride S split into sub-batches [b[j], b[j + 1]): checks 1 and 2
void check_launch(const Ctx& x, int slot, int S, int channels, const std::vector<int>& b) {
  g_cases++;
  const DevBuffers base = slot ? slot_view(x.ws, x.s1) : x.ws;
  const Extent e = launch_extent(S, channels);
  std::vector<std::pair<size_t, size_t>> spans(b.size() - 1);
  for_each_array([&](int i, auto m, Kind k, unsigned c) {
    if (k == Kind::Shared) return;
    const Alloc& a = home(x, slot, i, c);
    const size_t el = sizeof(*(base.*m)), slice = slice_elems(k, e), r = reach(k, e.S, e.C);
    if (r > slice) fail("scans-overlap", i, S, channels, (long long)r - (long long)slice);
    for (size_t j = 0; j + 1 < b.size(); j++) {
      const DevBuffers v = scan_view(base, b[j], e);
      const uintptr_t p = reinterpret_cast<uintptr_t>(v.*m);
      if (p < a.base || (p - a.base) % el) { fail("view-outside", i, S, b[j], 0); continue; }
      const size_t lo = (p - a.base) / el, hi = lo + (size_t)(b[j + 1] - b[j] - 1) * slice + r;
      if (hi * el > a.bytes) fail("past-allocation", i, S, b[j], (long long)(hi * el - a.bytes));
      spans[j] = {lo, hi};
    }
    for (size_t j = 0; j < spans.size(); j++)
      for (size_t l = j + 1; l < spans.size(); l++)
        if (spans[j].first < spans[l].second && spans[l].first < spans[j].second) fail("sub-batches-overlap", i, S, b[j], b[l]);
  });
}

void check_capacity(int max_points, int max_batch) {
  const Ctx x(max_points, max_batch);
  const int mp = (int)x.cap.S;
  const size_t P = (size_t)mp * max_batch;
  static const int kS[] = {1, 2, 31, 32, 33, 255, 256, 257, 511, 512, 513, 1000, 4096, 65536, 130000, 300001, 1 << 24};
  static const int kBatch[] = {1, 2, 3, 5, 16, 17, 31, 32, 33, 64, 100, 128, 1000, 4096, 65535};
  static const int kChannels[] = {1, 7, 32, 64, 128, 255, 256};
  std::vector<int> S_list;
  for (int S : kS) if (S <= mp) S_list.push_back(S);
  S_list.push_back(mp);
  if (mp > 1) S_list.push_back(mp - 1);
  for (int S : S_list)
    for (int batch : kBatch) {
      if (batch > max_batch || (size_t)S * batch > P) continue;
      for (int C : kChannels) {
        // device-resident batches: G stream groups (the library takes G only when batch >= 2 G), in slot 0's arrays
        for (int G = 1; G <= 16; G++) {
          if (G > 1 && batch < 2 * G) break;
          std::vector<int> b;
          for (int g = 0; g < G; g++) { int b0, b1; group_bounds(g, G, batch, &b0, &b1); b.push_back(b0); if (g == G - 1) b.push_back(b1); }
          check_launch(x, 0, S, C, b);
        }
        // host-buffer batches: chunks at a stride of whole 256-point blocks, in either host slot
        if (S % 256 == 0)
          for (int slot = 0; slot < 2; slot++) {
            std::vector<int> b;
            for (int b0 = 0, chunk = host_chunk(batch); b0 < batch; b0 += chunk) b.push_back(b0);
            b.push_back(batch);
            check_launch(x, slot, S, C, b);
            std::vector<int> each;                                  // the per-scan views of the result copies
            for (int s = 0; s <= batch && s <= 8; s++) each.push_back(s);
            check_launch(x, slot, S, C, each);
          }
      }
    }
  // 3. the host slots share no per-slot array, and neither shares one with the workspace
  g_cases++;
  for_each_array([&](int i, auto, Kind, unsigned c) {
    if (!(c & kSlot)) return;
    const Alloc &a = x.a_s0[i], &b = x.a_s1[i];
    if (!a.bytes || !b.bytes || (a.base < b.base + b.bytes && b.base < a.base + a.bytes)) fail("slots-share", i, max_points, max_batch, 0);
    if (x.a_ws[i].bytes) fail("slot-array-in-workspace", i, max_points, max_batch, 0);
  });
}

// 4. capacity elements per array: the sizes the library has always allocated
struct Known {
  int max_points, max_batch;
  unsigned long long P, roadcnt, ttab, elev, lomuto, hist, degbins, degsum, newY, rawb0;
};
const Known kKnown[] = {
    {1, 1, 512ull, 18ull, 93184ull, 4097ull, 257ull, 256ull, 92416ull, 92672ull, 512ull, 32768ull},
    {1000, 7, 7168ull, 232ull, 652288ull, 28679ull, 1799ull, 3584ull, 646912ull, 648704ull, 1024ull, 65536ull},
    {130000, 128, 16646144ull, 520321ull, 11927552ull, 524416ull, 32896ull, 8323072ull, 11829248ull, 11862016ull, 130048ull, 8323072ull},
    {100000, 2048, 205520896ull, 6424577ull, 190840832ull, 8390656ull, 526336ull, 102760448ull, 189267968ull, 189792256ull, 100352ull,
     6422528ull},
    {16777216, 127, 2130706432ull, 66584704ull, 11834368ull, 520319ull, 32639ull, 1065353216ull, 11736832ull, 11769344ull, 16777216ull,
     1073741824ull},
    {512, 65535, 33553920ull, 1114096ull, 6106813440ull, 268496895ull, 16842495ull, 16776960ull, 6056482560ull, 6073259520ull, 512ull,
     32768ull},
};

void check_known(const Known& k) {
  g_cases++;
  const Ctx x(k.max_points, k.max_batch);
  for (int i = 0; i < kArrays; i++) {
    const char* n = kNames[i];
    unsigned long long want = k.P;
    if (!std::strcmp(n, "roadcnt")) want = k.roadcnt;
    else if (!std::strcmp(n, "Tf") || !std::strcmp(n, "Tb")) want = k.ttab;
    else if (!std::strcmp(n, "lut") || !std::strcmp(n, "firstidx")) want = k.elev;
    else if (!std::strcmp(n, "lomuto")) want = k.lomuto;
    else if (!std::strcmp(n, "sortbuf")) want = 2 * k.P;
    else if (!std::strcmp(n, "hist")) want = k.hist;
    else if (!std::strcmp(n, "cmin") || !std::strcmp(n, "cmax")) want = k.degbins;
    else if (!std::strcmp(n, "ne")) want = k.degsum;
    else if (!std::strcmp(n, "newY")) want = k.newY;
    else if (!std::strcmp(n, "n") || !std::strcmp(n, "out") || !std::strcmp(n, "tab")) want = (unsigned long long)k.max_batch;
    if (x.elems[i] != want) fail("capacity", i, k.max_points, (long long)x.elems[i], (long long)want);
  }
  // slot 0's record staging (max_points records of URF_MAX_POINT_STEP bytes) and the ring-id buffers of the slots (P)
  if (capacity_elems(Kind::Point, x.cap, 1) * URF_MAX_POINT_STEP != k.rawb0) fail("capacity-rawb", 0, k.max_points, 0, 0);
  if (capacity_elems(Kind::Point, x.cap, k.max_batch) != k.P) fail("capacity-ring", 0, k.max_points, 0, 0);
}

}  // namespace

int main() {
  for (const Known& k : kKnown) check_known(k);
  static const int kMaxPoints[] = {1, 100, 512, 513, 1000, 4096, 65536, 130000, 300001, 1 << 20, 1 << 24};
  static const int kMaxBatch[] = {1, 2, 3, 16, 33, 128, 1000, 65535};
  for (int mp : kMaxPoints)
    for (int mb : kMaxBatch)
      if ((long long)(mp + kChunk) * mb < (1ll << 31)) check_capacity(mp, mb);
  std::printf("cases=%lld failures=%lld\n", g_cases, g_fail);
  return g_fail ? 1 : 0;
}
