// urf_workspace.cuh — the per-scan layout of the device arrays (DevBuffers), stated once. Every per-scan array holds one
// slice per scan, back to back, whose length depends on the array's kind and the launch's extent (S points of stride, T
// chunks, C channels). Allocation, sub-batch views, the kernels' per-scan bases and the debug fetch all take it from here.
#pragma once
#include <algorithm>

#include "urf_logic.cuh"

namespace urf {

// Elements of one scan's slice, per kind; templates on the integer type, so every kernel keeps its own width
template <class I> URF_HD constexpr I point_slice(I S) { return S; }                 // in, label, alpha_v, ...
template <class I> URF_HD constexpr I pair_slice(I S) { return 2 * S; }              // sortbuf: two 64-bit keys per point
template <class I> URF_HD constexpr I warp_slice(I S) { return (S + 31) >> 5; }      // roadcnt: one count per input warp
template <class I> URF_HD constexpr I chunk_rows(I T) { return T; }                  // hist: T rows of C counters
template <class I> URF_HD constexpr I ttab_slice(I C) { return C * kTStride; }       // Tf, Tb
template <class I> URF_HD constexpr I degbin_slice(I C) { return C * kDegBins; }     // cmin, cmax
template <class I> URF_HD constexpr I degsum_slice(I C) { return C * (kDegBins + 1); }   // ne
constexpr int kElevSlice = kElevBins + 1, kRingListSlice = kRingKeys + 1;   // lut, firstidx; lomuto

enum class Kind { Point, Pair, Warp, ChunkRows, TTable, DegBins, DegSum, Elev, RingList, Scan, Shared };
struct Extent { size_t S, T, C; };
inline Extent launch_extent(int S, int channels) { return {(size_t)S, (size_t)(S + kChunk - 1) / kChunk, (size_t)channels}; }
inline Extent capacity_extent(int max_points) { return launch_extent(max_points, URF_MAX_CHANNELS); }

// elements of one scan's slice of an array of kind k (in Kind order); 0 for newY, which all scans share
inline size_t slice_elems(Kind k, Extent e) {
  const size_t n[] = {point_slice(e.S), pair_slice(e.S), warp_slice(e.S), chunk_rows(e.T) * e.C, ttab_slice(e.C),
                      degbin_slice(e.C), degsum_slice(e.C), kElevSlice, kRingListSlice, 1, 0};
  return n[(int)k];
}
// elements allocated for B scans at capacity: roadcnt keeps B + 1 of slack, newY one entry per point of one scan
inline size_t capacity_elems(Kind k, Extent cap, size_t B) {
  return k == Kind::Shared ? cap.S : B * slice_elems(k, cap) + (k == Kind::Warp ? B + 1 : 0);
}

// Classes (bits): workspace, per host slot, on demand, shared. Each allocation takes what its predicate selects: urf_create
// the workspace and slot 0, the first asynchronous batch slot 1, the first call that needs them the on-demand arrays.
enum : unsigned { kWork = 1, kSlot = 2, kOnDemand = 4, kShared = 8 };
constexpr bool created_with_context(unsigned c) { return !(c & (kSlot | kOnDemand)); }
constexpr bool slot_array(unsigned c) { return c == kSlot; }
constexpr bool tie_order_array(unsigned c) { return c == (kWork | kOnDemand); }
constexpr bool label8_array(unsigned c) { return c == (kSlot | kOnDemand); }

// Calls f(index, member, kind, class) for every pointer member of DevBuffers in declaration order; returns their number
template <class F> constexpr int for_each_array(F&& f) {
  using D = DevBuffers;
  constexpr Kind P = Kind::Point;
  int i = 0;
  auto v = [&](auto m, Kind k, unsigned c) { f(i++, m, k, c); };
  v(&D::in, P, kSlot); v(&D::alpha_v, P, kWork); v(&D::mark, P, kWork); v(&D::ringid, P, kWork); v(&D::sect, P, kWork);
  v(&D::label, P, kSlot); v(&D::label8, P, kSlot | kOnDemand); v(&D::bpt, P, kWork); v(&D::sr, P, kWork); v(&D::sz, P, kWork);
  v(&D::sidx, P, kWork); v(&D::ssrz, P, kWork); v(&D::ssl, P, kWork); v(&D::az, P, kWork); v(&D::d2, P, kWork);
  v(&D::baz, P, kWork); v(&D::roadlist, P, kWork); v(&D::roadcnt, Kind::Warp, kWork);
  v(&D::Tf, Kind::TTable, kWork); v(&D::Tb, Kind::TTable, kWork); v(&D::lut, Kind::Elev, kWork); v(&D::order, P, kSlot);
  v(&D::epos, P, kWork | kOnDemand); v(&D::lomuto, Kind::RingList, kWork | kOnDemand); v(&D::sortbuf, Kind::Pair, kWork);
  v(&D::hist, Kind::ChunkRows, kWork); v(&D::firstidx, Kind::Elev, kWork);
  v(&D::cmin, Kind::DegBins, kWork); v(&D::cmax, Kind::DegBins, kWork); v(&D::ne, Kind::DegSum, kWork);
  v(&D::newY, Kind::Shared, kShared); v(&D::n, Kind::Scan, kSlot); v(&D::out, Kind::Scan, kSlot); v(&D::tab, Kind::Scan, kWork);
  return i;
}
constexpr int kArrays = for_each_array([](int, auto, Kind, unsigned) {});
static_assert(sizeof(DevBuffers) == kArrays * sizeof(void*), "for_each_array must list every member of DevBuffers");

// View of `a` for the sub-batch that starts at scan b0 of a launch of extent e: every per-scan array advanced by b0 slices
inline DevBuffers scan_view(const DevBuffers& a, int b0, Extent e) {
  DevBuffers v = a;
  for_each_array([&](int, auto m, Kind k, unsigned) { if (v.*m) v.*m += (size_t)b0 * slice_elems(k, e); });
  return v;
}
// `ws` with host slot `slot`'s per-slot arrays in place of its own
inline DevBuffers slot_view(const DevBuffers& ws, const DevBuffers& slot) {
  DevBuffers v = ws;
  for_each_array([&](int, auto m, Kind, unsigned c) { if (c & kSlot) v.*m = slot.*m; });
  return v;
}
// Allocates the arrays of `d` that pick(class) selects for B scans at capacity through alloc(index, d's member (a
// reference), element count); stops at the first failure and returns its code
template <class Pick, class Alloc> int alloc_arrays(DevBuffers& d, Extent cap, size_t B, Pick pick, Alloc&& alloc) {
  int rc = 0;
  for_each_array([&](int i, auto m, Kind k, unsigned c) { if (rc == 0 && pick(c)) rc = alloc(i, d.*m, capacity_elems(k, cap, B)); });
  return rc;
}

// stream group g of G takes scans [b0, b1) of a device-resident batch; host chunks are batch / 16 scans, at least 4
inline void group_bounds(int g, int G, int batch, int* b0, int* b1) { *b0 = (g * batch + G - 1) / G; *b1 = ((g + 1) * batch + G - 1) / G; }
inline int host_chunk(int batch) { return batch >= 16 ? std::max(4, (batch + 15) / 16) : batch; }

}  // namespace urf
