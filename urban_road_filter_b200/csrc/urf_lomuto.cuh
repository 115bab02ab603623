// urf_lomuto.cuh — the reference's tie order for one ring: the permutation its unstable Lomuto quicksort leaves
// (lidar_segmentation.cpp:70-93, called at :289-291; pivot = last element, float `<`), computed by a group of threads.
//
// Only rings with a float-equal pair or a NaN azimuth need it: without them the sorted order is unique and k_sort_rings
// already produced it. Subproblems (low, high) are taken from an explicit stack, the whole group on one subproblem (the
// two halves of a partition are independent, so the processing order does not change the result). Three shortcuts:
//   1. size <= 1: nothing to do;
//   2. no element has a tie partner in the ring and none is NaN: the subproblem's elements hold consecutive ranks of the
//      ring's (azimuth, position) order (every ancestor pivot lies outside their value range), so they are placed by rank;
//   3. non-decreasing (so no NaN): Lomuto swaps the pivot with the first element of its run of equals and recurses, which
//      rotates every maximal run of equal values right by one — its last element first, the others in their order.
// Any other subproblem gets one partition with pivot p = a[high], in parallel: the elements < p go to the front in their
// order (a prefix count). The elements >= p pass through the scan as a FIFO window: an element >= p appends itself to a
// log, an element < p met after the first >= p element (position f) pops the window's front and appends it again. The log
// entry of scan position j is therefore j - f, and the copy a pop appends refers to entry h = (elements < p in [f, j)), an
// earlier one, so the log is resolved by pointer jumping. The window is log[h_end:]; the segment ends as
// less + [pivot] + window[1:] + [window[0]]. (Stored by scan position, entry f + h sits at low + lr, lr = elements < p in
// [low, j), and the window's front at the pivot's final position.)
//
// The same template runs on the device (CtaGroup: one CTA) and sequentially on the host (SeqLomuto), where
// tests/kat/lomuto_check.cpp compares it with the restated quicksort of the CPU oracle.
#pragma once
#include <stdint.h>

#include "urf_logic.cuh"

namespace urf {

constexpr unsigned kLomutoCare = 0x80000000u;   // rank flag: the element has a tie partner in its ring or is NaN
constexpr unsigned kLomutoPtr = 0x80000000u;    // log entry: a copy of the entry at the low 31 bits, not an element
constexpr int kLomutoStack = 64;                // pending subproblems; pushing the larger half first bounds it by log2(n) + 1

// Work arrays of one ring of n points, each [n]. Elements are ring positions (bucket order, = input order in the ring).
struct LomutoArrays {
  const unsigned* az;   // azimuth bits by element
  unsigned* rk;         // in: rank of the element in (azimuth bits, position) order, NaN last; the setup adds kLomutoCare
  unsigned* s0;         // out: element by output position
  unsigned* s1;         // scratch
  unsigned* s2;         // scratch: the partition's log
};

// State the group shares (shared memory on the device).
struct LomutoShared {
  int stk[kLomutoStack][2];
  int top, low, high;
  long long partitions, steps;   // statistics: partitions, and elements of every subproblem taken from the stack
};

URF_HD float lomuto_val(const LomutoArrays& w, unsigned e) { return bitsf(w.az[e]); }

// The ring's Lomuto permutation into w.s0; G provides rank(), size(), sync(), any(p), count(p, &total) (exclusive count of
// p over the group, with the group's total) and min(v). Every member of the group calls it.
#pragma nv_exec_check_disable
template <class G>
URF_HD void lomuto_ring(const LomutoArrays& w, int n, LomutoShared& sh) {
  const int r0 = G::rank(), gs = G::size();
  // setup: the inverse of the rank permutation in s1, then the tie / NaN flag of every element
  for (int t = r0; t < n; t += gs) w.s1[w.rk[t]] = (unsigned)t;
  G::sync();
  for (int t = r0; t < n; t += gs) {
    const unsigned a = w.az[t], r = w.rk[t];
    const float v = bitsf(a);
    const bool care = v != v || (r > 0 && w.az[w.s1[r - 1]] == a) || (r + 1 < (unsigned)n && w.az[w.s1[r + 1]] == a);
    w.s0[t] = (unsigned)t;
    if (care) w.rk[t] = r | kLomutoCare;
  }
  if (r0 == 0) { sh.top = 0; if (n > 1) { sh.stk[0][0] = 0; sh.stk[0][1] = n - 1; sh.top = 1; } }
  G::sync();
  for (;;) {
    if (r0 == 0) {
      if (sh.top == 0) sh.low = -1;
      else { sh.top--; sh.low = sh.stk[sh.top][0]; sh.high = sh.stk[sh.top][1]; }
    }
    G::sync();
    const int low = sh.low, high = sh.high;
    if (low < 0) break;
    if (r0 == 0) sh.steps += high - low + 1;
    bool nan = false, care = false, up = true;
    for (int j = low + r0; j <= high; j += gs) {
      const unsigned e = w.s0[j];
      const float v = lomuto_val(w, e);
      nan |= v != v;
      care |= (w.rk[e] & kLomutoCare) != 0;
      if (j < high) up &= v <= lomuto_val(w, w.s0[j + 1]);
    }
    nan = G::any(nan); care = G::any(care); up = !G::any(!up);   // (the barriers also order the stack reads above)
    if (!nan && !care) {                                          // shortcut 2: place by rank
      int rmin = 0x7fffffff;
      for (int j = low + r0; j <= high; j += gs) { const int r = (int)w.rk[w.s0[j]]; rmin = r < rmin ? r : rmin; }
      rmin = G::min(rmin);
      for (int j = low + r0; j <= high; j += gs) { const unsigned e = w.s0[j]; w.s1[low + ((int)w.rk[e] - rmin)] = e; }
      G::sync();
      for (int j = low + r0; j <= high; j += gs) w.s0[j] = w.s1[j];
      G::sync();
      continue;
    }
    if (up) {                                                     // shortcut 3: every run of equals rotated right by one
      for (int j = low + r0; j <= high; j += gs) {
        const unsigned e = w.s0[j];
        const float v = lomuto_val(w, e);
        if (j < high && lomuto_val(w, w.s0[j + 1]) == v) { w.s1[j + 1] = e; continue; }
        int lo = low, hi = j;                                     // last of its run: to the run's first position
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (lomuto_val(w, w.s0[mid]) < v) lo = mid + 1; else hi = mid; }
        w.s1[lo] = e;
      }
      G::sync();
      for (int j = low + r0; j <= high; j += gs) w.s0[j] = w.s1[j];
      G::sync();
      continue;
    }
    // one partition with pivot a[high]
    const unsigned pe = w.s0[high];
    const float p = lomuto_val(w, pe);
    int carry = 0, f = -1;                                        // elements < p so far, first position of an element >= p
    for (int t0 = low; t0 < high; t0 += gs) {
      const int j = t0 + r0;
      const unsigned e = j < high ? w.s0[j] : 0u;
      const bool less = j < high && lomuto_val(w, e) < p;
      int tot = 0;
      const int lr = carry + G::count(less, &tot);               // elements < p in [low, j)
      if (f < 0) { const int m = G::min(j < high && !less ? j : 0x7fffffff); if (m != 0x7fffffff) f = m; }
      if (j < high) {
        if (less) w.s1[low + lr] = e;
        if (f >= 0 && j >= f) w.s2[j] = less ? ((unsigned)(low + lr) | kLomutoPtr) : e;   // entry f + h, h = lr - (f - low)
      }
      carry += tot;
    }
    G::sync();
    const int pi = low + carry;                                   // the pivot's final position
    if (f >= 0) {
      unsigned *src = w.s2, *dst = w.s0;                           // s0[low..high] is free: less in s1, the rest in the log
      for (;;) {
        bool more = false;
        for (int j = f + r0; j < high; j += gs) {
          unsigned v = src[j];
          if (v & kLomutoPtr) { v = src[v & ~kLomutoPtr]; more |= (v & kLomutoPtr) != 0; }
          dst[j] = v;
        }
        more = G::any(more);
        unsigned* t = src; src = dst; dst = t;
        if (!more) break;
      }
      if (src != w.s2) {
        for (int j = f + r0; j < high; j += gs) w.s2[j] = src[j];
        G::sync();
      }
    }
    // the window is log[pi:] (pops so far: the L - (f - low) elements < p after f): its front goes last, the rest in place
    for (int q = low + r0; q <= high; q += gs)
      w.s0[q] = q < pi ? w.s1[q] : q == pi ? pe : q == high ? w.s2[pi] : w.s2[q];
    if (r0 == 0) {
      sh.partitions++;
      const int a0 = low, a1 = pi - 1, b0 = pi + 1, b1 = high;    // larger half first: the smaller one is taken next
      const bool aBig = a1 - a0 > b1 - b0;
      if (aBig && a1 > a0) { sh.stk[sh.top][0] = a0; sh.stk[sh.top][1] = a1; sh.top++; }
      if (b1 > b0) { sh.stk[sh.top][0] = b0; sh.stk[sh.top][1] = b1; sh.top++; }
      if (!aBig && a1 > a0) { sh.stk[sh.top][0] = a0; sh.stk[sh.top][1] = a1; sh.top++; }
    }
    G::sync();
  }
}

// One thread on the host: the sequential run of the same code.
struct SeqLomuto {
  static URF_HDM int rank() { return 0; }
  static URF_HDM int size() { return 1; }
  static URF_HDM void sync() {}
  static URF_HDM bool any(bool p) { return p; }
  static URF_HDM int count(bool p, int* total) { *total = p ? 1 : 0; return 0; }
  static URF_HDM int min(int v) { return v; }
};

}  // namespace urf
