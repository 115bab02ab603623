// urf_kernels.cuh — sm_90a kernels of the per-scan road/curb classification path (pipeline v2).
//
// Every kernel takes the batch index from blockIdx.y (or blockIdx.x for one-CTA-per-scan kernels): a launch covers a
// whole batch of scans laid out back to back with `S` points of stride. Everything that decides a label is computed by
// the host+device functions of urf_logic.cuh (bit-identical to the x86-64 -O2 build of the reference, file:line cited
// there); the kernels add indexing, staging, atomics and synchronisation.
//
// Pipeline (DESIGN.md has the picture):
//   k_reset -> k_points -> k_register -> k_assign -> k_scan_offsets (+ exact re-registration of refuted scans)
//   -> k_scatter -> k_star_sort (near-first) -> k_star_sort_big (large sectors, exact fallback) -> k_star_scan
//   -> k_star_refine (sectors without an edge in their prefix: full sort, walk resumed)
//   -> k_ring_detect -> k_tab1 -> k_reach -> k_tab2 -> k_label (input order) -> k_markers1 (one CTA per scan; scans
//   above 300,000 points: k_markers_grid<1> -> k_markers_grid<2> -> k_verts)
//   [-> k_sort_rings when the emission order is requested]
//   Reference tie order (urf_set_tie_order): k_sort_rings -> k_lomuto_rings run in front of k_label instead, always.
//   PointCloud2 entry points: k_unpack_cloud2_batch in front, k_pack_count -> k_pack_scan -> k_pack_write behind
#pragma once
#include <type_traits>

#include "urf_device.cuh"
#include "urf_logic.cuh"
#include "urf_lomuto.cuh"
#include "urf_stdsort.cuh"
#include "urf_workspace.cuh"

namespace urf {

__constant__ float c_beam_d[kSectKeys];
__constant__ float c_beam_o[kSectKeys];
__constant__ unsigned char c_beam_yx[kSectKeys];

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }
// 32-bit offset of scan b inside the batch-major arrays (urf_create keeps max_batch * max_points below 2^31): array
// accesses then cost one IMAD.WIDE instead of 64-bit multiply/add chains
__device__ __forceinline__ unsigned scan_base(int b, int S) { return (unsigned)b * point_slice((unsigned)S); }

// Inclusive prefix sums over the warp's lanes of N values per lane at once (N independent sums, one shuffle ladder).
// Every lane of the warp calls it.
template <int N, class T>
__device__ __forceinline__ void warp_inclusive_sum(T (&x)[N]) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    T u[N];
#pragma unroll
    for (int i = 0; i < N; i++) u[i] = __shfl_up_sync(0xffffffffu, x[i], d);
    if (lane_id() >= d)
#pragma unroll
      for (int i = 0; i < N; i++) x[i] += u[i];
  }
}
// Append to a list in shared memory: the slot of a flagged lane, in lane order after the *counter entries taken before
// (one shared atomic per warp). Every lane of the warp calls it; a lane without the flag gets a value it must not use.
template <class T>
__device__ __forceinline__ T warp_append(bool flag, T* counter) {
  const unsigned bal = __ballot_sync(0xffffffffu, flag);
  T base = 0;
  if (lane_id() == 0 && bal) base = atomicAdd(counter, (T)__popc(bal));
  return __shfl_sync(0xffffffffu, base, 0) + (T)__popc(bal & ((1u << lane_id()) - 1u));
}

// The thread groups that sort together in memory: the whole CTA, or one warp.
// The CTA-wide helpers (exclusive_sum, count, min) share one contract: every thread of the CTA calls them, the CTA has at
// most 32 warps, and the scratch is the helper's own function-scope __shared__ array for 32 warps. A helper holds every
// barrier it needs, the last one after its final read of that scratch, so two calls may follow each other without a
// barrier of the caller's between them. Shared memory the caller writes after a call still wants the caller's barrier.
struct CtaGroup {
  static __device__ __forceinline__ unsigned rank() { return threadIdx.x; }
  static __device__ __forceinline__ unsigned size() { return blockDim.x; }
  static __device__ __forceinline__ void sync() { __syncthreads(); }
  static __device__ __forceinline__ bool any(bool p) { return __syncthreads_or(p); }
  // x[i] becomes the sum of x[i] over the threads before this one (thread order); total[i] = the sum over the CTA
  template <int N, class T>
  static __device__ __forceinline__ void exclusive_sum(T (&x)[N], T (&total)[N]) {
    __shared__ T s_w[N][32];
    const int lane = lane_id(), warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    T inc[N];
#pragma unroll
    for (int i = 0; i < N; i++) inc[i] = x[i];
    warp_inclusive_sum(inc);
    if (lane == 31)
#pragma unroll
      for (int i = 0; i < N; i++) s_w[i][warp] = inc[i];
    __syncthreads();
#pragma unroll
    for (int i = 0; i < N; i++) {                          // lane w holds warp w's total
      const T c = lane < nw ? s_w[i][lane] : (T)0;
      x[i] = __reduce_add_sync(0xffffffffu, lane < warp ? c : (T)0) + inc[i] - x[i];
      total[i] = __reduce_add_sync(0xffffffffu, c);
    }
    __syncthreads();
  }
  // exclusive count of p over the threads before this one, and the CTA's total
  static __device__ __forceinline__ int count(bool p, int* total) {
    __shared__ int s_w[32];
    const unsigned bal = __ballot_sync(0xffffffffu, p);
    const int lane = lane_id(), warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    if (lane == 0) s_w[warp] = __popc(bal);
    __syncthreads();
    const int c = lane < nw ? s_w[lane] : 0;
    const int before = __reduce_add_sync(0xffffffffu, lane < warp ? c : 0);
    *total = __reduce_add_sync(0xffffffffu, c);
    __syncthreads();
    return before + __popc(bal & ((1u << lane) - 1u));
  }
  static __device__ __forceinline__ int min(int v) {
    __shared__ int s_w[32];
    v = __reduce_min_sync(0xffffffffu, v);
    if (lane_id() == 0) s_w[threadIdx.x >> 5] = v;
    __syncthreads();
    v = __reduce_min_sync(0xffffffffu, lane_id() < (int)(blockDim.x >> 5) ? s_w[lane_id()] : 0x7fffffff);
    __syncthreads();
    return v;
  }
};
struct WarpGroup {
  static __device__ __forceinline__ int rank() { return lane_id(); }
  static __device__ __forceinline__ int size() { return 32; }
  static __device__ __forceinline__ void sync() { __syncwarp(); }
  static __device__ __forceinline__ bool any(bool p) { return __any_sync(0xffffffffu, p); }
};

// Bitonic sort of npad (power of two) keys in shared or global memory by thread group G; all its threads must call.
template <class G, class T>
__device__ void group_bitonic(T* a, int npad) {
  for (int k = 2; k <= npad; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = G::rank(); t < (npad >> 1); t += G::size()) {
        int i = 2 * t - (t & (j - 1));
        int l = i + j;
        bool up = (i & k) == 0;
        T x = a[i], y = a[l];
        if ((x > y) == up) { a[i] = y; a[l] = x; }
      }
      G::sync();
    }
  }
}

__device__ __forceinline__ int next_pow2(int n) { int p = 1; while (p < n) p <<= 1; return p; }

// A detector found input point idx of scan b to be a curb point (star_shaped_search.cpp:146, x_zero_method.cpp:66,
// z_zero_method.cpp:71): mark it and, if it sits in a ring bucket (k = its ring, or -1 = look it up), enter its azimuth
// into the curb aggregates of that ring's integer-degree bin — what blindSpots reads. NaN azimuths fall out.
__device__ __forceinline__ void curb_hit(const DevBuffers& buf, const DevParams& prm, int b, unsigned gb, int idx, int k) {
  buf.mark[gb + (unsigned)idx] = 2;
  if (k < 0) k = buf.ringid[gb + (unsigned)idx];
  if (k < 0) return;                                   // not in array3D: the mark is never read (lidar_segmentation.cpp:241)
  const float a = buf.az[gb + (unsigned)idx];
  if (a >= 0.0f) {
    const unsigned o = (unsigned)b * degbin_slice((unsigned)prm.channels) + (unsigned)k * kDegBins + (unsigned)deg_bin(a);
    atomicMin(&buf.cmin[o], fbits(a));
    atomicMax(&buf.cmax[o], fbits(a));
  }
}
// ring of bucket position p: rings are contiguous in bucket order, ring_start has kRingKeys + 1 non-decreasing entries
__device__ __forceinline__ int ring_of_position(const int* __restrict__ ring_start, int p) {
  int lo = 0, hi = kRingKeys;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (ring_start[mid] <= p) lo = mid + 1; else hi = mid; }
  return lo - 1;
}

// ---------------------------------------------------------------------------------------------------------------------
// k_reset: per-call initialisation of the per-scan tables.
__global__ void k_reset(DevBuffers buf, DevParams prm) {
  const int b = blockIdx.y;
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  const int nth = gridDim.x * blockDim.x;
  ScanOut& o = buf.out[b];
  ScanTab& t = buf.tab[b];
  if (tid == 0) {
    o.n_in = buf.n[b]; o.n_roi = 0; o.n_rings = 0; o.n_order = 0; o.n_road = 0; o.n_curb = 0; o.n_vert = 0; o.flags = 0;
  }
  for (int i = tid; i <= kRingKeys; i += nth) o.ring_start[i] = 0;
  for (int i = tid; i < kRingKeys; i += nth) { t.maxs[i] = 0ull; t.maxdist[i] = 0u; t.angle[i] = 0.f; t.regidx[i] = 0x7fffffff; t.regorder[i] = 0x7fffffff; }
  for (int i = tid; i < kDegBins; i += nth) { t.cutbest[i] = ~0ull; t.dmax[i] = 0u; t.best[i] = ~0ull; }
  for (int i = tid; i < kSectKeys; i += nth) t.sect_cnt[i] = 0;
  if (tid == 0) { t.nbig = 0; t.nslow = 0; t.nrefine = 0; }
  if (tid == 0 && buf.lomuto) buf.lomuto[(size_t)b * kRingListSlice] = 0;
  unsigned* fi = buf.firstidx + (size_t)b * kElevSlice;
  for (int i = tid; i <= kElevBins; i += nth) fi[i] = 0xffffffffu;
  const size_t nb = degbin_slice((size_t)prm.channels);
  unsigned* cmin = buf.cmin + (size_t)b * nb;
  unsigned* cmax = buf.cmax + (size_t)b * nb;
  for (size_t i = tid; i < nb; i += nth) { cmin[i] = 0x7f800000u; cmax[i] = 0u; }
}

// ---------------------------------------------------------------------------------------------------------------------
// k_points: everything that depends on one input point alone — ROI crop predicate, range and elevation angle
// (lidar_segmentation.cpp:106-113,148-166), planar range and azimuth (:245-269; the squares are shared with the range) and
// the star sector (star_shaped_search.cpp:164-173). Also records, per fine elevation bin, the first input index that
// falls into it (speculation input for k_register).
// A few CTAs per scan (the grid is at most one resident wave, see launch_pipeline), each over a contiguous range of
// whole tiles of kPtsTile points; thread t takes points t and t + 256 of a tile, and the next tile's records are loaded
// into registers while the current one is computed. The first index per elevation bin, the ROI count and the sector
// counts are kept in shared memory and added to the scan's global ones once per CTA: one global atomic per touched bin /
// sector instead of one per point / warp.
constexpr int kPtsThreads = 256;
constexpr int kPtsPerThread = 2;                                 // records per thread per tile
constexpr int kPtsTile = kPtsThreads * kPtsPerThread;
__global__ void __launch_bounds__(kPtsThreads) k_points(DevBuffers buf, DevParams prm, int S) {
  __shared__ unsigned s_first[kElevBins + 1];                    // CTA's smallest ROI input index per fine elevation bin
  __shared__ int s_scnt[kSectKeys];                              // CTA's points per star sector
  __shared__ int s_roi;
  const int b = blockIdx.y;
  const int n = buf.n[b];
  const int tiles = (n + kPtsTile - 1) / kPtsTile;
  const int per = (tiles + gridDim.x - 1) / gridDim.x;
  const int t0 = blockIdx.x * per, t1 = min(tiles, t0 + per);
  if (t0 >= t1) return;                                          // uniform in the CTA
  for (int e = threadIdx.x; e <= kElevBins; e += kPtsThreads) s_first[e] = 0xffffffffu;
  for (int s = threadIdx.x; s < kSectKeys; s += kPtsThreads) s_scnt[s] = 0;
  if (threadIdx.x == 0) s_roi = 0;
  const unsigned gb = scan_base(b, S);
  float4 cur[kPtsPerThread], nxt[kPtsPerThread];
#pragma unroll
  for (int j = 0; j < kPtsPerThread; ++j) {
    const int i = t0 * kPtsTile + j * kPtsThreads + (int)threadIdx.x;
    if (i < n) cur[j] = __ldg(&buf.in[gb + (unsigned)i]);
  }
  __syncthreads();
  int roi = 0;
  for (int t = t0; t < t1; ++t) {
    if (t + 1 < t1) {
#pragma unroll
      for (int j = 0; j < kPtsPerThread; ++j) {
        const int i = (t + 1) * kPtsTile + j * kPtsThreads + (int)threadIdx.x;
        if (i < n) nxt[j] = __ldg(&buf.in[gb + (unsigned)i]);
      }
    }
#pragma unroll
    for (int j = 0; j < kPtsPerThread; ++j) {
      const int i = t * kPtsTile + j * kPtsThreads + (int)threadIdx.x;
      int sec = -1;
      if (i < n) {
        const unsigned g = gb + (unsigned)i;
        const float4 p = cur[j];
        const int keep = roi_keep(prm, p.x, p.y, p.z);
        float a = -1.0f;
        if (keep) {
          float d, az;
          point_angles(p.x, p.y, p.z, &a, &d, &az);
          unsigned* fi = s_first + elev_bin(a);
          if (*fi > (unsigned)i) atomicMin(fi, (unsigned)i);    // plain (possibly stale) read: a stale value is only larger
          if (a == 0.0f) atomicOr(&buf.out[b].flags, F_ZERO_ALPHA);
          if (az != az) atomicOr(&buf.out[b].flags, F_NAN_AZIMUTH);   // x == y == 0 inside the ROI
          if (prm.star) sec = star_sector(prm, p.x, p.y, c_beam_d, c_beam_o, c_beam_yx);   // star_shaped_search.cpp:164-173
          buf.az[g] = az;
          buf.d2[g] = d;
          roi++;
        }
        buf.alpha_v[g] = a;
        buf.mark[g] = 0;
        buf.sect[g] = (short)sec;
      }
      // per-sector point counts of the (unordered) sector partition: one atomic per group of equal sectors in the warp
      const unsigned peers = __match_any_sync(0xffffffffu, sec);
      if (sec >= 0 && lane_id() == __ffs(peers) - 1) atomicAdd(&s_scnt[sec], __popc(peers));
    }
#pragma unroll
    for (int j = 0; j < kPtsPerThread; ++j) cur[j] = nxt[j];
  }
  roi = __reduce_add_sync(0xffffffffu, roi);
  if (lane_id() == 0 && roi) atomicAdd(&s_roi, roi);
  __syncthreads();
  unsigned* fi = buf.firstidx + (size_t)b * kElevSlice;
  for (int e = threadIdx.x; e <= kElevBins; e += kPtsThreads) {
    const unsigned v = s_first[e];
    if (v != 0xffffffffu) atomicMin(&fi[e], v);
  }
  for (int s = threadIdx.x; s < kSectKeys; s += kPtsThreads)
    if (s_scnt[s]) atomicAdd(&buf.tab[b].sect_cnt[s], s_scnt[s]);
  if (threadIdx.x == 0 && s_roi) atomicAdd(&buf.out[b].n_roi, s_roi);
}

// ---------------------------------------------------------------------------------------------------------------------
// Ring registration, lidar_segmentation.cpp:136-139,170-196: a point registers its elevation angle iff no VISIBLE
// registered angle lies within `interval` of it and fewer than `channels` angles are registered. "Visible": the
// reference's scan stops at the first angle[j] == 0, so once an angle of exactly 0 is registered, it and everything
// registered after it are never compared again.
//
// Exact path (any input): rounds of "find the first uncovered point after the last registrant" with a CTA-wide min.
__device__ void register_exact_cta(const float* __restrict__ alpha, int n, float interval, int channels, float* s_vis,
                                   float* s_reg, int* s_idx, int* out_m) {
  int m = 0, vis = 0, i_last = -1;
  bool frozen = false;
  while (m < channels) {
    int local = 0x7fffffff;
    for (int i = i_last + 1 + threadIdx.x; i < n; i += blockDim.x) {
      const float a = alpha[i];
      if (a < 0.0f) continue;
      bool cov = false;
      for (int t = 0; t < vis; t++) {
        if (fabsf(__fsub_rn(s_vis[t], a)) <= interval) { cov = true; break; }   // :179
      }
      if (!cov) { local = i; break; }
    }
    const int istar = CtaGroup::min(local);
    if (istar == 0x7fffffff) break;
    const float a = alpha[istar];
    if (threadIdx.x == 0) { s_reg[m] = a; s_idx[m] = istar; if (!frozen && a != 0.0f) s_vis[vis] = a; }
    if (!frozen) { if (a == 0.0f) frozen = true; else vis++; }
    m++;
    i_last = istar;
    __syncthreads();
  }
  *out_m = m;
}

// Sort the m registered (angle, regidx) pairs by angle (:205), publish them and build the elevation-bin lookup table
// k_assign starts its ring search from. Angles are >= 0 so their bits order them.
__device__ void publish_rings_cta(ScanTab& tab, ScanOut& out, unsigned short* lut, float interval, const float* s_reg,
                                  const int* s_idx, int m, unsigned long long* s_keys, float* s_sorted) {
  for (int t = threadIdx.x; t < kRingKeys; t += blockDim.x)
    s_keys[t] = t < m ? (((unsigned long long)fbits(s_reg[t]) << 32) | (unsigned)s_idx[t]) : ~0ull;
  __syncthreads();
  group_bitonic<CtaGroup>(s_keys, kRingKeys);
  for (int t = threadIdx.x; t < kRingKeys; t += blockDim.x) {
    if (t < m) {
      const float a = bitsf((unsigned)(s_keys[t] >> 32));
      s_sorted[t] = a;
      tab.angle[t] = a;
      tab.regidx[t] = (int)(unsigned)s_keys[t];
      tab.regorder[t] = s_idx[t];
    } else { s_sorted[t] = 0.f; tab.angle[t] = 0.f; tab.regidx[t] = 0x7fffffff; tab.regorder[t] = 0x7fffffff; }
  }
  if (threadIdx.x == 0) out.n_rings = m;
  __syncthreads();
  for (int e = threadIdx.x; e <= kElevBins; e += blockDim.x) lut[e] = (unsigned short)ring_lut_entry(s_sorted, m, interval, e);
}

// k_register: one CTA (256 threads) per scan. Fast path: the greedy registration is run over "candidates" only — the
// first point of every non-empty fine elevation bin, in input order. That is a speculation (a registrant need not be
// the first of its bin); k_assign verifies it against every point and k_scan_offsets repairs a failed speculation (exact greedy, in-kernel).
__global__ void __launch_bounds__(256) k_register(DevBuffers buf, DevParams prm, int S) {
  const int b = blockIdx.x;
  const int n = buf.n[b];
  ScanOut& out = buf.out[b];
  ScanTab& tab = buf.tab[b];
  const float* alpha = buf.alpha_v + (size_t)b * point_slice(S);
  __shared__ unsigned s_cand[kMaxCand];
  __shared__ float s_calpha[kMaxCand];
  __shared__ float s_vis[kRingKeys];
  __shared__ float s_reg[kRingKeys];
  __shared__ float s_sorted[kRingKeys];
  __shared__ int s_idx[kRingKeys];
  __shared__ unsigned long long s_keys[kRingKeys];
  __shared__ int s_cnt, s_m;
  if (out.n_roi < 30) {                      // lidar_segmentation.cpp:124-126: nothing happens for this scan
    if (threadIdx.x == 0) out.n_rings = 0;
    return;
  }
  bool exact = prm.force_exact || (out.flags & F_ZERO_ALPHA);
  if (!exact) {
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    const unsigned* fi = buf.firstidx + (size_t)b * kElevSlice;
    for (int t = threadIdx.x; t <= kElevBins; t += blockDim.x) {
      const unsigned v = fi[t];
      if (v != 0xffffffffu) { int s = atomicAdd(&s_cnt, 1); if (s < kMaxCand) s_cand[s] = v; }
    }
    __syncthreads();
    const int cnt = s_cnt;
    if (cnt > kMaxCand) exact = true;        // uniform across the CTA
    else {
      const int npad = next_pow2(cnt < 2 ? 2 : cnt);
      for (int t = cnt + threadIdx.x; t < npad; t += blockDim.x) s_cand[t] = 0xffffffffu;
      __syncthreads();
      group_bitonic<CtaGroup>(s_cand, npad);
      for (int t = threadIdx.x; t < cnt; t += blockDim.x) s_calpha[t] = alpha[s_cand[t]];
      __syncthreads();
      if (threadIdx.x < 32) {
        int m = 0;
        for (int c = 0; c < cnt && m < prm.channels; c++) {
          const float a = s_calpha[c];
          bool cov = false;
          for (int t = lane_id(); t < m; t += 32)
            if (fabsf(__fsub_rn(s_reg[t], a)) <= prm.interval) cov = true;          // :179
          cov = __any_sync(0xffffffffu, cov);
          if (!cov) {
            if (lane_id() == 0) { s_reg[m] = a; s_idx[m] = (int)s_cand[c]; }
            m++;
            __syncwarp();
          }
        }
        if (lane_id() == 0) s_m = m;
      }
      __syncthreads();
    }
  }
  if (exact) {
    int m;
    register_exact_cta(alpha, n, prm.interval, prm.channels, s_vis, s_reg, s_idx, &m);
    if (threadIdx.x == 0) { s_m = m; atomicOr(&out.flags, F_EXACT_REG); }
    __syncthreads();
  }
  publish_rings_cta(tab, out, buf.lut + (size_t)b * kElevSlice, prm.interval, s_reg, s_idx, s_m, s_keys, s_sorted);
}

// ---------------------------------------------------------------------------------------------------------------------
// k_assign: per input point — ring index (lidar_segmentation.cpp:226-233: first sorted angle within `interval`) and the
// per-warp-chunk ring histogram of the stable ring partition. assign_chunk is one warp's chunk of kChunk points; cnt is
// the warp's zeroed shared histogram. Returns true (per lane) where the speculated registration is refuted.
__device__ __forceinline__ bool assign_chunk(const DevBuffers& buf, const DevParams& prm, int b, int S, int T, int chunk, int n, bool live,
                                             bool verify, const float* s_angle, const int* s_regidx, const int* regorder, int R,
                                             const unsigned short* __restrict__ lut, unsigned* cnt, int lane) {
  bool violation = false;
  // two halves of eight iterations: the eight elevation loads are issued together, then the eight table look-ups they
  // address, and only then the (short, shared-memory) ring searches — two memory round trips per half instead of sixteen
  constexpr int H = 8;
  static_assert((kChunk / 32) % H == 0, "chunk iterations come in groups of H");
#pragma unroll 1
  for (int h0 = 0; h0 < kChunk / 32; h0 += H) {
    float av[H];
    unsigned short start[H];
#pragma unroll
    for (int u = 0; u < H; u++) {
      const int i = chunk * kChunk + (h0 + u) * 32 + lane;
      av[u] = i < n ? buf.alpha_v[scan_base(b, S) + (unsigned)i] : -1.0f;
    }
#pragma unroll
    for (int u = 0; u < H; u++) start[u] = (live && av[u] >= 0.0f) ? lut[elev_bin(av[u])] : (unsigned short)0;
#pragma unroll
    for (int u = 0; u < H; u++) {
      const int i = chunk * kChunk + (h0 + u) * 32 + lane;
      int ring = -1;
      if (i < n) {
        const float a = av[u];
        const bool kept = live && a >= 0.0f;
        if (kept) {
          int lo;
          ring = assign_ring_from(s_angle, R, a, prm.interval, start[u], &lo);
          if (verify && registration_violation(s_angle, s_regidx, regorder, R, prm.channels, prm.interval, a, i, lo)) violation = true;
        }
        buf.ringid[scan_base(b, S) + (unsigned)i] = kept ? (short)ring : (short)-2;   // -2: not part of the ROI cloud (k_label writes URF_LABEL_OUTSIDE)
      }
      // histogram: a ring-major scan puts one ring into a warp (one add of 32), a column-major one 32 different rings
      // (32 conflict-free shared atomics); results unused, so no read-modify-write chain between iterations
      const int ring0 = __shfl_sync(0xffffffffu, ring, 0);
      if (__all_sync(0xffffffffu, ring == ring0)) { if (lane == 0 && ring0 >= 0) atomicAdd(&cnt[ring0], 32u); }
      else if (ring >= 0) atomicAdd(&cnt[ring], 1u);
    }
  }
  __syncwarp();
  // rows are `channels` counters wide: ring ids are below n_rings <= channels
  const int C = prm.channels;
  unsigned* row = buf.hist + ((size_t)b * chunk_rows(T) + chunk) * C;
  for (int t = lane; t < C; t += 32) row[t] = cnt[t];
  return violation;
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32) k_assign(DevBuffers buf, DevParams prm, int S, int T) {
  const int b = blockIdx.y;
  ScanOut& out = buf.out[b];
  const int flags = out.flags;
  const int n = buf.n[b];
  const int warp = threadIdx.x >> 5, lane = lane_id();
  const int chunk = blockIdx.x * kWarpsPerBlock + warp;
  __shared__ float s_angle[kRingKeys];
  __shared__ int s_regidx[kRingKeys];
  __shared__ unsigned s_cnt[kWarpsPerBlock][kRingKeys];
  ScanTab& tab = buf.tab[b];
  const int R = out.n_rings;
  for (int t = threadIdx.x; t < kRingKeys; t += blockDim.x) { s_angle[t] = tab.angle[t]; s_regidx[t] = tab.regidx[t]; }
  for (int t = lane; t < kRingKeys; t += 32) s_cnt[warp][t] = 0;
  __syncthreads();
  if (chunk * kChunk >= n) return;             // whole warp; no block-level sync follows
  const bool violation = assign_chunk(buf, prm, b, S, T, chunk, n, out.n_roi >= 30, !(flags & F_EXACT_REG), s_angle, s_regidx, tab.regorder, R,
                                      buf.lut + (size_t)b * kElevSlice, s_cnt[warp], lane);
  if (__any_sync(0xffffffffu, violation) && lane == 0) atomicOr(&out.flags, F_SPEC_VIOLATION);
}

// ---------------------------------------------------------------------------------------------------------------------
// k_scan_offsets: one CTA per scan turns hist[chunk][ring] (rows of `channels` counters) into exclusive scatter offsets
// (ring-major bases + prefix over chunks), publishes ring_start, and turns the sector counts into sect_start + scatter
// cursors. Each warp owns a range of rows; a lane keeps kScanOffBatch rows of its column in flight. The ring bases and
// the sector starts are CTA-wide scans with one ring and one sector per thread. 512 threads at no more than 64 registers
// take at most half of an SM, so CTAs of the other stream groups run beside it.
// In front of that it repairs a scan whose speculated registration k_assign refuted (F_SPEC_VIOLATION, rare): the exact
// registration, then ring ids and chunk histograms of the whole scan again, one chunk per warp at a time.
constexpr int kScanOffThreads = 512, kScanOffWarps = kScanOffThreads / 32;
constexpr int kScanOffBatch = 16;
static_assert(kRingKeys < kScanOffThreads && kSectKeys <= kScanOffThreads, "one ring_start entry and one sector per thread");
__global__ void __launch_bounds__(kScanOffThreads, 2) k_scan_offsets(DevBuffers buf, DevParams prm, int S, int T) {
  __shared__ unsigned s_part[kScanOffWarps][kRingKeys];     // per-warp partial sums, then per-warp exclusive prefixes
  __shared__ unsigned s_base[kRingKeys];
  const int b = blockIdx.x;
  const int n = buf.n[b];
  const int C = prm.channels;
  const int rows = (n + kChunk - 1) / kChunk;
  const int warp = threadIdx.x >> 5, lane = lane_id();
  {
    ScanOut& out = buf.out[b];
    const int flags = out.flags;
    if ((flags & F_SPEC_VIOLATION) && !(flags & F_EXACT_REG)) {      // uniform across the CTA
      __shared__ float s_vis[kRingKeys], s_reg[kRingKeys], s_sorted[kRingKeys];
      __shared__ int s_idx[kRingKeys];
      __shared__ unsigned long long s_keys[kRingKeys];
      __shared__ int s_m;
      int m;
      register_exact_cta(buf.alpha_v + (size_t)b * point_slice(S), n, prm.interval, prm.channels, s_vis, s_reg, s_idx, &m);
      if (threadIdx.x == 0) s_m = m;
      __syncthreads();
      const unsigned short* lut = buf.lut + (size_t)b * kElevSlice;
      publish_rings_cta(buf.tab[b], out, buf.lut + (size_t)b * kElevSlice, prm.interval, s_reg, s_idx, s_m, s_keys, s_sorted);
      __syncthreads();                                                // s_sorted = the sorted angles, lut written
      const int R = s_m;
      for (int c0 = 0; c0 < rows; c0 += kScanOffWarps) {
        for (int t = lane; t < kRingKeys; t += 32) s_part[warp][t] = 0;
        __syncwarp();
        if (c0 + warp < rows) assign_chunk(buf, prm, b, S, T, c0 + warp, n, true, false, s_sorted, nullptr, nullptr, R, lut, s_part[warp], lane);
        __syncwarp();
      }
      if (threadIdx.x == 0) out.flags = flags | F_EXACT_REG;
      __syncthreads();                                                // the histogram rows are read back below
    }
  }
  ScanTab& tab = buf.tab[b];
  const unsigned scnt = threadIdx.x < kSectKeys ? (unsigned)tab.sect_cnt[threadIdx.x] : 0u;   // in flight during the row sums
  const int rpw = (rows + kScanOffWarps - 1) / kScanOffWarps;
  const int r0 = min(rows, warp * rpw), r1 = min(rows, (warp + 1) * rpw);
  unsigned* hist = buf.hist + (size_t)b * chunk_rows(T) * C;
  for (int key = lane; key < C; key += 32) {
    unsigned s = 0;
    for (int r = r0; r < r1; r += kScanOffBatch) {
      unsigned v[kScanOffBatch];
#pragma unroll
      for (int u = 0; u < kScanOffBatch; u++) v[u] = r + u < r1 ? hist[(size_t)(r + u) * C + key] : 0u;
#pragma unroll
      for (int u = 0; u < kScanOffBatch; u++) s += v[u];
    }
    s_part[warp][key] = s;
  }
  __syncthreads();
  unsigned rtot = 0;                              // total of ring threadIdx.x
  if (threadIdx.x < C)
    for (int w = 0; w < kScanOffWarps; w++) { const unsigned v = s_part[w][threadIdx.x]; s_part[w][threadIdx.x] = rtot; rtot += v; }
  // CTA-wide exclusive scans of the ring totals (-> ring bases) and of the sector counts (-> sector starts)
  unsigned x[2] = {rtot, scnt}, all[2];
  CtaGroup::exclusive_sum(x, all);
  const unsigned xr = x[0], xs = x[1], all_r = all[0], all_s = all[1];
  ScanOut& o = buf.out[b];
  if (threadIdx.x < C) s_base[threadIdx.x] = xr;
  if (threadIdx.x <= kRingKeys) o.ring_start[threadIdx.x] = (int)(threadIdx.x < C ? xr : all_r);
  if (threadIdx.x < kSectKeys) { tab.sect_start[threadIdx.x] = (int)xs; tab.sect_cur[threadIdx.x] = (int)xs; }
  if (threadIdx.x == 0) { o.n_order = (int)all_r; tab.sect_start[kSectKeys] = (int)all_s; }
  __syncthreads();
  for (int key = lane; key < C; key += 32) {
    unsigned run = s_base[key] + s_part[warp][key];
    for (int r = r0; r < r1; r += kScanOffBatch) {
      unsigned v[kScanOffBatch];
#pragma unroll
      for (int u = 0; u < kScanOffBatch; u++) v[u] = r + u < r1 ? hist[(size_t)(r + u) * C + key] : 0u;
#pragma unroll
      for (int u = 0; u < kScanOffBatch; u++)
        if (r + u < r1) { hist[(size_t)(r + u) * C + key] = run; run += v[u]; }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// k_scatter: stable scatter of every point into its ring bucket (input order inside a ring, lidar_segmentation.cpp:221-
// 277) and unordered scatter into its star sector (the radius sort that follows breaks ties by input index, which is the
// push_back order of star_shaped_search.cpp:173). One warp per chunk of kChunk points, kScatterWarps chunks per CTA.
// Sectors: every point takes a rank inside its sector from a CTA-wide shared counter; after a barrier one thread per
// sector that occurs in the CTA reserves the CTA's slots from the scan's sector cursor with ONE global atomic (all of them
// in flight together), and after a second barrier the records are written to base + rank.
// Ring buckets are written coalesced: the warp first ranks its chunk by ring in shared memory, then walks the chunk in
// ring order so that consecutive lanes write consecutive bucket slots.
// Input records: each warp's chunk (up to kChunk 16-byte records, 8 KB) is copied into shared memory once, at kernel
// entry, by one bulk asynchronous copy (cp.async.bulk, completion counted on a per-warp mbarrier). The copy runs while
// the warp ranks its points; the ring-order gather and the sector pass then read the records from shared memory.
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(count) : "memory");
  asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");   // the initialised barrier is visible to the copy engine
}
// one bulk copy of `bytes` (a multiple of 16, both addresses 16-byte aligned) that completes phase 0 of `bar`
__device__ __forceinline__ void bulk_copy_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(dst), m = (unsigned)__cvta_generic_to_shared(bar);
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(m), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
               ::"r"(d), "l"(src), "r"(bytes), "r"(m) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned phase) {
  const unsigned m = (unsigned)__cvta_generic_to_shared(bar);
  unsigned done;
  do {
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}\n"
                 : "=r"(done) : "r"(m), "r"(phase) : "memory");
  } while (!done);
}
constexpr int kScatterWarps = 4;     // chunks per CTA: 8 KB input tile per warp, four CTAs per SM
constexpr size_t kScatterSmem = (size_t)kScatterWarps * kChunk * sizeof(float4);   // dynamic: the input tiles
__global__ void __launch_bounds__(kScatterWarps * 32, 4) k_scatter(DevBuffers buf, DevParams prm, int S, int T) {
  const int b = blockIdx.y;
  const int n = buf.n[b];
  const int warp = threadIdx.x >> 5, lane = lane_id();
  const int chunk = blockIdx.x * kScatterWarps + warp;
  extern __shared__ float4 s_tiles[];                             // [kScatterWarps][kChunk] input records of the chunk
  __shared__ unsigned long long s_bar[kScatterWarps];             // per warp: its tile has arrived
  __shared__ unsigned s_delta[kScatterWarps][kChunk];             // bucket slot of ring-ordered slot t, minus t
  __shared__ unsigned s_lcnt[kScatterWarps][kRingKeys];           // per-ring count, then exclusive local start
  __shared__ unsigned short s_perm[kScatterWarps][kChunk];        // chunk-local point index in ring order
  __shared__ int s_scnt[kSectKeys], s_sbase[kSectKeys];           // sector: points of this CTA, first slot reserved for them
  const float4* tile = s_tiles + warp * kChunk;
  unsigned* delta = s_delta[warp];
  unsigned* lcnt = s_lcnt[warp];
  unsigned short* perm = s_perm[warp];
  ScanTab& tab = buf.tab[b];
  const bool live = chunk * kChunk < n;                           // a warp past the end only takes part in the barriers
  const unsigned* row = buf.hist + ((size_t)b * chunk_rows(T) + chunk) * prm.channels;
  const unsigned gb = scan_base(b, S), g0 = gb + (unsigned)chunk * kChunk;
  if (live && lane == 0) {                                        // clipped at the end of the scan
    mbar_init(&s_bar[warp], 1);
    bulk_copy_g2s(s_tiles + warp * kChunk, buf.in + g0, (unsigned)min(kChunk, n - chunk * kChunk) * sizeof(float4), &s_bar[warp]);
  }
  for (int t = threadIdx.x; t < kSectKeys; t += blockDim.x) s_scnt[t] = 0;
  for (int t = lane; t < kRingKeys; t += 32) lcnt[t] = 0;
  __syncthreads();
  const unsigned lt = (1u << lane) - 1u;
  unsigned packed[kChunk / 32];                 // (ring + 1) << 16 | rank inside the chunk's ring group
  unsigned spack[kChunk / 32];                  // (sector + 1) << 16 | rank inside the CTA's sector group
  if (live) {
    // all sixteen ring / sector loads of a lane are issued together before anything depends on them (groups of four
    // measured slower: four CTAs per SM hold half the warps the kernel had before it staged its input)
    constexpr int GRP = kChunk / 32;
#pragma unroll
    for (int h = 0; h < kChunk / 32 / GRP; h++) {
      short rr[GRP], ss[GRP];
#pragma unroll
      for (int u = 0; u < GRP; u++) {
        const int li = (h * GRP + u) * 32 + lane;
        const bool in = chunk * kChunk + li < n;
        rr[u] = in ? buf.ringid[g0 + li] : (short)-1;
        ss[u] = in ? buf.sect[g0 + li] : (short)-1;
      }
#pragma unroll
      for (int u = 0; u < GRP; u++) {
        const int it = h * GRP + u;
        // sector rank (any order will do): one shared atomic for a warp that sits in one sector (column-major scans: 32
        // rings of one azimuth), else one per lane
        const int sec = ss[u];
        const int sec0 = __shfl_sync(0xffffffffu, sec, 0);
        int srank = 0;
        if (__all_sync(0xffffffffu, sec == sec0)) {
          int sb = 0;
          if (lane == 0 && sec0 >= 0) sb = atomicAdd(&s_scnt[sec0], 32);
          srank = __shfl_sync(0xffffffffu, sb, 0) + lane;
        } else if (sec >= 0) srank = atomicAdd(&s_scnt[sec], 1);
        spack[it] = sec >= 0 ? (((unsigned)(sec + 1) << 16) | (unsigned)srank) : 0u;
        // stable rank inside the ring: the group's first lane takes the group's slots from the warp's ring counter with a
        // shared atomic (same-address atomics of one warp apply in program order, so iteration order = input order; nothing
        // else orders the iterations, the sixteen of them pipeline), lanes add their position inside the group
        // groups of equal rings in the warp. The two sensor layouts need no MATCH (its latency was the kernel's largest
        // stall): ring-major input puts ONE ring into a warp, column-major input 32 DIFFERENT rings in ascending or
        // descending order (all distinct: every lane is its own group); anything else takes __match_any_sync
        const int ring = rr[u];
        const int rprev = __shfl_up_sync(0xffffffffu, ring, 1), ring0 = __shfl_sync(0xffffffffu, ring, 0);
        unsigned peers;
        if (__all_sync(0xffffffffu, ring == ring0)) peers = 0xffffffffu;
        else if (__all_sync(0xffffffffu, lane == 0 || ring > rprev) || __all_sync(0xffffffffu, lane == 0 || ring < rprev)) peers = 1u << lane;
        else peers = __match_any_sync(0xffffffffu, ring);
        const int leader = __ffs(peers) - 1;
        unsigned rb = 0;
        if (ring >= 0 && lane == leader) rb = atomicAdd(&lcnt[ring], (unsigned)__popc(peers));
        rb = __shfl_sync(0xffffffffu, rb, leader);
        packed[it] = ring >= 0 ? (((unsigned)(ring + 1) << 16) | (rb + __popc(peers & lt))) : 0u;
      }
    }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < kSectKeys; t += blockDim.x) {     // one reservation per sector present in this CTA
    const int c = s_scnt[t];
    s_sbase[t] = c > 0 ? atomicAdd(&tab.sect_cur[t], c) : 0;
  }
  int total = 0;
  if (live) {
    // exclusive scan of the chunk's ring counts -> local starts (runs while the reservations are in flight)
    {
      unsigned v[kRingKeys / 32], sum = 0;
#pragma unroll
      for (int j = 0; j < kRingKeys / 32; j++) { v[j] = lcnt[lane * (kRingKeys / 32) + j]; sum += v[j]; }
      unsigned inc[1] = {sum};
      warp_inclusive_sum(inc);
      unsigned run = inc[0] - sum;
      __syncwarp();
#pragma unroll
      for (int j = 0; j < kRingKeys / 32; j++) { lcnt[lane * (kRingKeys / 32) + j] = run; run += v[j]; }
    }
    __syncwarp();
#pragma unroll
    for (int it = 0; it < kChunk / 32; it++) {
      const unsigned pk = packed[it];
      if (pk) {
        const int ring = (int)(pk >> 16) - 1;
        const unsigned lstart = lcnt[ring];
        const int slot = lstart + (pk & 0xffffu);
        perm[slot] = (unsigned short)(it * 32 + lane);
        delta[slot] = __ldg(&row[ring]) - lstart;        // global offset of the chunk's ring group - its local start
      }
      total += __popc(__ballot_sync(0xffffffffu, pk != 0));
    }
    __syncwarp();
    mbar_wait(&s_bar[warp], 0);                                   // the chunk's input records are in `tile`
    // walk the chunk in ring order
    for (int t = lane; t < total; t += 32) {
      const int li = perm[t];
      const float4 p = tile[li];
      const unsigned dst = gb + delta[t] + (unsigned)t;
      buf.bpt[dst] = make_float4(p.x, p.y, p.z, __int_as_float(chunk * kChunk + li));
      // (azimuth, input index) in bucket order: all k_sort_rings reads
      if (prm.want_order) buf.baz[dst] = make_uint2(fbits(buf.az[g0 + li]), (unsigned)(chunk * kChunk + li));
    }
  }
  __syncthreads();                                                // s_sbase is complete
  if (live) {
    // sector records: r, z, input index into their three arrays
#pragma unroll
    for (int it = 0; it < kChunk / 32; it++) {
      const unsigned sp = spack[it];
      if (sp) {
        const int sec = (int)(sp >> 16) - 1;
        const int li = it * 32 + lane;
        const float4 p = tile[li];
        const unsigned dst = gb + (unsigned)(s_sbase[sec] + (int)(sp & 0xffffu));
        buf.sr[dst] = star_radius(p.x, p.y);
        buf.sz[dst] = p.z;
        buf.sidx[dst] = (unsigned)(chunk * kChunk + li);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Star-shaped search, sort by planar radius (star_shaped_search.cpp:109). Order: (r, input index) — the reference's
// introsort order for equal r is unspecified; ties raise F_TIE_SECTOR.
//
// Records: the unsorted sector is three arrays in slot order (sr, sz, sidx: radius, height, input index); a sort writes
// ssrz = (r, z) in radius order, all the edge search reads, and ssl = per sorted position the slot the point came from
// (the input index is sidx[slot], looked up only for the one point a walk marks) — or, from the exact fallback, which
// sorts by (radius, input index) and has no slot, the input index with bit 31 set. star_input_index resolves either.
//
// Register-resident bitonic network: thread t owns elements t*EPL .. t*EPL+EPL-1 (32-bit radius bits + the element's slot
// in the unsorted sector as payload). Strides below EPL are register-only compare-exchanges, strides below 32*EPL go
// through warp shuffles, larger strides (multi-warp CTAs only) exchange through shared memory. One warp sorts up to 1024
// points (k_star_sort: one sector per warp at a time, warp-uniform control flow around the shuffles; k_star_refine), eight
// warps up to 8192 (k_star_sort_big / k_star_refine, work lists). Returns true when two points share a
// radius: their order is what the reference's std::sort leaves (urf_stdsort.cuh), which the network does not see — such a
// sector, like any sector beyond 8192 points, is redone by slow_sort_sector.
constexpr int kWarpCap = 1024, kCtaCap = 8192;
constexpr int kNetCap = 512;                          // widest single-warp network of k_star_sort (16 elements per lane)
constexpr unsigned kSslIndex = 0x80000000u;           // ssl entry holds an input index (exact fallback), not a slot

// The record arrays of one sector: the unsorted side (sr, sz) is read from element o on, the sorted side (ssrz, ssl)
// written from element at on. 32-bit element offsets into the buffers of the kernel parameter instead of four 64-bit
// pointers: the sorts run at their register limit.
struct SectorRecs {
  const DevBuffers& buf;
  unsigned o;        // b * S + sector base
  unsigned at;       // o + the sorted positions in front of what a sort writes
  __device__ __forceinline__ const float* r() const { return buf.sr + o; }
  __device__ __forceinline__ unsigned key(int e) const { return fbits(buf.sr[o + (unsigned)e]); }
  // sorted position e: radius bits k of the point at `slot`
  __device__ __forceinline__ void put(int e, unsigned k, unsigned slot) const {
    buf.ssrz[at + (unsigned)e] = make_float2(bitsf(k), buf.sz[o + slot]);
    buf.ssl[at + (unsigned)e] = slot;
  }
};
__device__ __forceinline__ SectorRecs sector_recs(const DevBuffers& buf, int b, int S, int base, int at = 0) {
  const unsigned o = scan_base(b, S) + (unsigned)base;
  return SectorRecs{buf, o, o + (unsigned)at};
}
// input index of the point at sorted position e of the sector that starts at element o = b * S + base
__device__ __forceinline__ int star_input_index(const DevBuffers& buf, unsigned o, int e) {
  const unsigned l = buf.ssl[o + (unsigned)e];
  return (l & kSslIndex) ? (int)(l & ~kSslIndex) : (int)buf.sidx[o + l];
}

// LIST: the n elements to sort are given as (radius bits, slot) pairs in s_xk / s_xe instead of being all of
// d.r[0 .. n) — the near-first prefix.
// STAGED (k_star_sort: one warp, LIST, s_xk = the warp's key stage): s_xe == nullptr means that s_xk holds the radius bits
// of all of d.r[0 .. n) in slot order; the records are stored through s_xk in sorted order (see below).
template <int EPL, int WARPS, bool LIST = false, bool STAGED = false>
__device__ __forceinline__ bool bitonic_sector(const SectorRecs& d, int n, int tid, unsigned* s_xk, unsigned* s_xe) {
  constexpr int THREADS = WARPS * 32;                // sorts up to THREADS * EPL elements
  // LIST with WARPS > 1: the list lives in the exchange buffers; every thread has taken its entries into registers before
  // the barrier in front of the first cross-warp exchange lets anybody overwrite them
  const int lane = tid & 31;
  unsigned key[EPL], el[EPL];
#pragma unroll
  for (int r = 0; r < EPL; r++) {
    const int e = tid * EPL + r;
    key[r] = 0xffffffffu; el[r] = 0u;
    if (e < n) {
      if (LIST) { key[r] = s_xk[e]; el[r] = (STAGED && s_xe == nullptr) ? (unsigned)e : s_xe[e]; }
      else { key[r] = d.key(e); el[r] = (unsigned)e; }
    }
  }
  // intra-thread compare-exchange network for strides EPL/2 .. 1 of merge phase k (compile-time register indices)
  auto intra = [&](int k_over_epl, auto kc) {
    constexpr int K = decltype(kc)::value;             // K > 0: merge phase k = K < EPL (direction depends on r only)
#pragma unroll
    for (int j = (K > 0 ? K : EPL) >> 1; j > 0; j >>= 1) {
#pragma unroll
      for (int r = 0; r < EPL; r++) {
        if ((r & j) == 0) {
          const bool asc = K > 0 ? ((r & K) == 0) : ((tid & k_over_epl) == 0);
          const bool sw = (key[r] > key[r | j]) == asc;
          const unsigned ka = sw ? key[r | j] : key[r], kb = sw ? key[r] : key[r | j];
          const unsigned ea = sw ? el[r | j] : el[r], eb = sw ? el[r] : el[r | j];
          key[r] = ka; key[r | j] = kb; el[r] = ea; el[r | j] = eb;
        }
      }
    }
  };
  // phases k = 2 .. EPL/2: entirely inside the thread
  if (EPL > 2) intra(0, std::integral_constant<int, 2>());
  if (EPL > 4) intra(0, std::integral_constant<int, 4>());
  if (EPL > 8) intra(0, std::integral_constant<int, 8>());
  if (EPL > 16) intra(0, std::integral_constant<int, 16>());
  // phases k = EPL .. N: thread-level strides (shuffles / shared memory, runtime loop), then the intra-thread strides
  for (int ke = 1; ke <= THREADS; ke <<= 1) {          // ke = k / EPL
    for (int tj = ke >> 1; tj > 0; tj >>= 1) {         // partner thread = tid ^ tj
      const bool keep_min = ((tid & tj) == 0) == ((tid & ke) == 0);
      if (tj < 32) {
#pragma unroll
        for (int r = 0; r < EPL; r++) {
          const unsigned o = __shfl_xor_sync(0xffffffffu, key[r], tj);
          const unsigned oe = __shfl_xor_sync(0xffffffffu, el[r], tj);
          const bool take = (o < key[r]) == keep_min;            // branch-free; taking an equal key is harmless
          key[r] = take ? o : key[r];
          el[r] = take ? oe : el[r];
        }
      } else {                                         // partner in another warp: exchange through shared memory
        __syncthreads();
#pragma unroll
        for (int r = 0; r < EPL; r++) { s_xk[r * THREADS + tid] = key[r]; s_xe[r * THREADS + tid] = el[r]; }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < EPL; r++) {
          const unsigned o = s_xk[r * THREADS + (tid ^ tj)], oe = s_xe[r * THREADS + (tid ^ tj)];
          const bool take = (o < key[r]) == keep_min;
          key[r] = take ? o : key[r];
          el[r] = take ? oe : el[r];
        }
      }
    }
    intra(ke, std::integral_constant<int, 0>());
  }
  // write out + tie detection against the predecessor in sorted order
  unsigned prev0 = __shfl_up_sync(0xffffffffu, key[EPL - 1], 1);
  if (WARPS > 1) {
    __syncthreads();
    if (lane == 31) s_xk[tid >> 5] = key[EPL - 1];
    __syncthreads();
    if (lane == 0 && tid > 0) prev0 = s_xk[(tid >> 5) - 1];
  }
  bool tie = false;
  if constexpr (STAGED) {
    static_assert(!STAGED || (WARPS == 1 && LIST && EPL <= 16), "STAGED: single-warp list sorts of up to 16 elements per lane");
#pragma unroll
    for (int r = 0; r < EPL; r++) {
      const int e = tid * EPL + r;
      const unsigned prev = r > 0 ? key[r - 1] : prev0;
      if (e < n && e > 0 && prev == key[r]) tie = true;
    }
    // the list is in registers now: its buffer takes the (key, slot) pairs in sorted order — slots in s_xk[0 .. 32 * EPL),
    // keys kNetCap words above — so that consecutive lanes write consecutive records (a lane's own EPL records are EPL
    // records apart). Word r of lane t goes to t * EPL + (r ^ swz(t)): the XOR spreads the 32 lanes' words of one r over
    // all 32 banks. Only z is gathered: r is the key.
    static_assert(!STAGED || 32 * EPL <= kNetCap, "STAGED: the keys go kNetCap words above the slots");
    constexpr int TPW = 32 / EPL;                      // lanes per 32 consecutive elements
    __syncwarp();
#pragma unroll
    for (int r = 0; r < EPL; r++) {
      const int w = tid * EPL + (r ^ ((tid / TPW) & (EPL - 1)));
      s_xk[w] = el[r];
      s_xk[kNetCap + w] = key[r];
    }
    __syncwarp();
#pragma unroll
    for (int r = 0; r < EPL; r++) {
      const int e = r * 32 + tid, t = e / EPL;
      const int w = t * EPL + ((e & (EPL - 1)) ^ ((t / TPW) & (EPL - 1)));
      if (e < n) d.put(e, s_xk[kNetCap + w], s_xk[w]);
    }
    __syncwarp();
  } else {
#pragma unroll
    for (int r = 0; r < EPL; r++) {
      const int e = tid * EPL + r;
      const unsigned prev = r > 0 ? key[r - 1] : prev0;
      if (e < n) {
        d.put(e, key[r], el[r]);
        if (e > 0 && prev == key[r]) tie = true;
      }
    }
  }
  return tie;
}

// A near-first prefix of m of a sector's n points is worth sorting on its own (instead of the whole sector).
__device__ __forceinline__ bool near_prefix(int m, int n) { return m >= 32 && 4 * m <= 3 * n; }

// Near-first selection (see k_star_sort): the pivot is the 18th smallest of 32 evenly spaced samples of the sector's
// radius bits kb[0 .. n); returns the number m of points below it. Only when that prefix is what k_star_sort will sort
// (near_prefix(m, n) and m <= kNetCap) are its (radius bits, slot) pairs written, IN PLACE of the keys and in any order:
// radius bits to kb[0 .. m), slots to kb[kNetCap .. kNetCap + m). Otherwise kb is left as it was (the whole sector is
// sorted from it, or it goes to k_star_sort_big).
template <int EPL>
__device__ __forceinline__ int select_near(unsigned* kb, int n, int lane, int pivot_rank) {
  const unsigned mine = kb[(int)(((unsigned)lane * (unsigned)n) >> 5)];
  unsigned key[EPL];
#pragma unroll
  for (int r = 0; r < EPL; r++) {
    const int e = r * 32 + lane;
    key[r] = e < n ? kb[e] : 0xffffffffu;
  }
  int rank = 0;                                        // ranks of the samples are a permutation (ties broken by lane)
#pragma unroll
  for (int j = 0; j < 32; j++) { const unsigned o = __shfl_sync(0xffffffffu, mine, j); rank += (o < mine) || (o == mine && j < lane); }
  const unsigned pivot = __shfl_sync(0xffffffffu, mine, __ffs(__ballot_sync(0xffffffffu, rank == pivot_rank)) - 1);
  int m = 0;                                           // padding keys are 0xffffffff: never below the pivot
#pragma unroll
  for (int r = 0; r < EPL; r++) m += __popc(__ballot_sync(0xffffffffu, key[r] < pivot));
  if (!near_prefix(m, n) || m > kNetCap) return m;     // warp-uniform
  __syncwarp();                                        // every lane holds its keys: the list may overwrite them
  const unsigned lt = (1u << lane) - 1u;
  int pos0 = 0;
#pragma unroll
  for (int r = 0; r < EPL; r++) {
    const bool sel = key[r] < pivot;
    const unsigned bs = __ballot_sync(0xffffffffu, sel);
    const int pos = pos0 + __popc(bs & lt);
    if (sel) { kb[pos] = key[r]; kb[kNetCap + pos] = (unsigned)(r * 32 + lane); }
    pos0 += __popc(bs);
  }
  __syncwarp();
  return m;
}

// The other side of a near-first split, for k_star_refine: the (radius bits, slot) pairs of the points whose radius lies
// ABOVE `kmax` (the largest radius of the sorted prefix; prefix radii are all below the pivot, the rest at or above it),
// appended to the shared lists in any order. Returns their number.
template <int EPL>
__device__ __forceinline__ int select_far(const float* __restrict__ sr, int n, int lane, unsigned* s_pk, unsigned* s_pe, unsigned kmax) {
  unsigned key[EPL];
#pragma unroll
  for (int r = 0; r < EPL; r++) {
    const int e = r * 32 + lane;
    key[r] = e < n ? fbits(sr[e]) : 0u;                // padding: radius bits 0 are never above kmax
  }
  const unsigned lt = (1u << lane) - 1u;
  int m = 0;
#pragma unroll
  for (int r = 0; r < EPL; r++) {
    const bool sel = key[r] > kmax;
    const unsigned bs = __ballot_sync(0xffffffffu, sel);
    if (sel) { const int pos = m + __popc(bs & lt); s_pk[pos] = key[r]; s_pe[pos] = (unsigned)(r * 32 + lane); }
    m += __popc(bs);
  }
  __syncwarp();
  return m;
}

// Near-first sort. The edge search (k_star_scan) walks a sector outwards and stops at its first edge point, so the far
// part of a sector is usually never looked at. Sectors above kPrefixMin points are therefore split at a pivot radius (the
// 18th smallest of 32 evenly spaced samples): points below the pivot are compacted into shared memory and sorted (about
// half the sector -> a network of half the width, ~40 % of the compare-exchanges); the rest is not written at all.
// tab.sorted_len tells k_star_scan how far it may walk; a sector whose walk reaches the end of the sorted prefix
// without an edge is put on tab.refine and redone in full (k_star_refine: full sort + star_resume_walk_warp). Exact either
// way: every point of the prefix is closer than every point behind it.
constexpr int kPrefixMin = 128;

// 4- and 16-byte asynchronous global -> shared copies (cp.async): the copy needs no register, and the warp goes on
// working while it is in flight
__device__ __forceinline__ void cp_async4(unsigned* s, const float* g) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"((unsigned)__cvta_generic_to_shared(s)), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async16(unsigned* s, const float* g) {      // both addresses 16-byte aligned
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"((unsigned)__cvta_generic_to_shared(s)), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

// One sector of k_star_sort, by one warp; kb[0 .. n) holds its radius bits (slot order), kb has kWarpCap words of room
// (the list of the near-first prefix and the sorted hand-out both use kb[kNetCap ..)). Sectors of more than kWarpCap
// points, and sorts wider than kNetCap elements, go to k_star_sort_big's lists; equal radii to the exact fallback.
__device__ __forceinline__ void star_sort_sector(const DevBuffers& buf, const DevParams& prm, int S, int b, int s, int base, int n,
                                                 unsigned* kb, int lane) {
  ScanTab& tab = buf.tab[b];
  if (lane == 0) tab.sorted_len[s] = n;
  if (n <= 0) return;
  const SectorRecs d = sector_recs(buf, b, S, base);
  if (n == 1) { if (lane == 0) d.put(0, d.key(0), 0u); return; }
  if (n > kWarpCap) {                                                   // hand over to the CTA sort / the fallback
    if (lane == 0) {
      if (n <= kCtaCap) tab.biglist[atomicAdd(&tab.nbig, 1)] = (unsigned short)s;
      else tab.slowlist[atomicAdd(&tab.nslow, 1)] = (unsigned short)s;
    }
    return;
  }
  int m = 0;
  if (prm.star_prefix && n > kPrefixMin) {
    if (n <= 256) m = select_near<8>(kb, n, lane, prm.star_pivot);
    else if (n <= 512) m = select_near<16>(kb, n, lane, prm.star_pivot);
    else m = select_near<32>(kb, n, lane, prm.star_pivot);
  }
  const bool near = near_prefix(m, n);                                  // worth it: sort the near part only
  const int len = near ? m : n;
  if (len > kNetCap) {                                                  // a wide network: eight warps do it (k_star_sort_big)
    if (lane == 0) tab.biglist[atomicAdd(&tab.nbig, 1)] = (unsigned short)s;
    return;
  }
  unsigned* pe = near ? kb + kNetCap : nullptr;                         // whole sector: the keys in kb are in slot order
  bool tie;
  if (len <= 128) tie = bitonic_sector<4, 1, true, true>(d, len, lane, kb, pe);
  else if (len <= 256) tie = bitonic_sector<8, 1, true, true>(d, len, lane, kb, pe);
  else tie = bitonic_sector<16, 1, true, true>(d, len, lane, kb, pe);
  if (near && lane == 0) tab.sorted_len[s] = m;
  if (__any_sync(0xffffffffu, tie) && lane == 0) tab.slowlist[atomicAdd(&tab.nslow, 1)] = (unsigned short)s;   // sets F_TIE_SECTOR there
}

// k_star_sort: the radius sort of the sectors of a batch. Every warp walks the flat (scan, sector) index q = warp,
// warp + W, ... (W = warps in the grid; the loop counter is warp-uniform, so the shuffle network needs no convergence
// barriers) and keeps the next sector's memory traffic in flight while it sorts the current one: the radius bits of the
// next sector (sr, contiguous) are copied into the warp's other shared-memory stage with cp.async — 16 bytes per copy for
// the aligned middle, 4 for the head and tail; the keys land at word (address / 4) mod 4 of the stage so that both sides of
// a 16-byte copy are aligned — and the offsets of the sector after that are loaded into registers. A one-warp CTA per
// sector (the previous form) exposed the offset load, the key loads and the record gather one after the other on every
// sector, with at most 32 warps per SM (the resident-CTA limit) to cover them.
// (Measured and dropped before: a keys-only network — one SHFL + two VIMNMX per remote compare-exchange instead of two
// SHFL, a compare and two selects — with the payload recovered by a binary search of every key in the sorted keys: 30 %
// fewer instructions, but 0.7 % slower per step.)
constexpr int kSortWarps = 8;                                                              // warps per CTA
constexpr int kStage = kWarpCap + 4;                                                       // words per key stage
constexpr size_t kStarSortSmem = (size_t)kSortWarps * 2 * kStage * sizeof(unsigned);      // 64.25 KB: two key stages per warp
__global__ void __launch_bounds__(kSortWarps * 32, 3) k_star_sort(DevBuffers buf, DevParams prm, int S, int B) {
  extern __shared__ unsigned s_dyn[];                                   // 16-byte aligned, like every stage (kStage % 4 == 0)
  const int lane = lane_id(), warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0);
  unsigned* const stage = s_dyn + (size_t)warp * 2 * kStage;
  const int Q = B * kSectKeys, W = gridDim.x * kSortWarps;
  // (base, size) of sector q: lanes 0 and 1 load the two offsets, the shuffles hand them to the warp
  auto offsets = [&](int q, int& base, int& n) {
    int v = 0;
    if (q < Q && lane < 2) { const int b = q / kSectKeys; v = buf.tab[b].sect_start[q - b * kSectKeys + lane]; }
    base = __shfl_sync(0xffffffffu, v, 0);
    n = __shfl_sync(0xffffffffu, v, 1) - base;
  };
  // radii of sector q, and the word of a stage its keys start at: sr[base] sits that many words past a 16-byte boundary
  auto radii = [&](int q, int base) { return buf.sr + (size_t)(q / kSectKeys) * S + base; };
  auto key_word = [](const float* g) { return (int)((reinterpret_cast<uintptr_t>(g) >> 2) & 3); };
  // radius bits of sector q into stage st (one commit group per call, empty when there is nothing to stage)
  auto stage_keys = [&](int q, int base, int n, unsigned* st) {
    if (q < Q && n > 1 && n <= kWarpCap) {
      const float* g = radii(q, base);
      const int off = key_word(g);
      unsigned* kb = st + off;
      const int h = min(n, (4 - off) & 3);                              // head: up to the first 16-byte boundary
      const int nv = (n - h) >> 2, t0 = h + 4 * nv;                     // 16-byte middle, then a tail of up to 3
      for (int v = lane; v < nv; v += 32) cp_async16(kb + h + 4 * v, g + h + 4 * v);
      if (lane < h + (n - t0)) { const int e = lane < h ? lane : t0 + (lane - h); cp_async4(kb + e, g + e); }
    }
    cp_async_commit();
  };
  int q = blockIdx.x * kSortWarps + warp;
  int base, n, nbase, nn;
  offsets(q, base, n);
  stage_keys(q, base, n, stage);
  offsets(q + W, nbase, nn);
  for (int it = 0; q < Q; q += W, it ^= 1) {
    stage_keys(q + W, nbase, nn, stage + (it ^ 1) * kStage);            // that stage's last reader finished (__syncwarp below)
    int base2, n2;
    offsets(q + 2 * W, base2, n2);
    cp_async_wait<1>();                                                 // this lane's copies of sector q have landed ...
    __syncwarp();                                                       // ... and every other lane's
    const int b = q / kSectKeys;
    star_sort_sector(buf, prm, S, b, q - b * kSectKeys, base, n, stage + it * kStage + key_word(radii(q, base)), lane);
    __syncwarp();
    base = nbase; n = nn; nbase = base2; nn = n2;
  }
  cp_async_wait<0>();
}

// Exact fallback sort of one sector by thread group G, the whole CTA or one warp (bitonic; shared memory up to `cap` keys,
// global scratch beyond, which only a CTA reaches): sectors larger than kCtaCap and sectors holding EQUAL radii. Keys are
// (radius bits, input index). Without equal radii any correct sort gives the reference's order. With them (F_TIE_SECTOR)
// the reference's order is what libstdc++'s introsort leaves when it sorts the sector's points in push_back (= input)
// order by radius alone (star_shaped_search.cpp:109): the points are put back into input order (second bitonic pass, keyed
// by index) and ONE thread runs the restated std::sort (urf_stdsort.cuh) over them.
template <class G>
__device__ void slow_sort_sector(const DevBuffers& buf, int b, int S, int base, int n, unsigned long long* s_keys, int cap) {
  const size_t o = (size_t)b * point_slice(S) + base;
  const int npad = next_pow2(n < 2 ? 2 : n);
  unsigned long long* keys = npad <= cap ? s_keys : buf.sortbuf + pair_slice(o);
  G::sync();
  for (int t = G::rank(); t < npad; t += G::size())
    keys[t] = t < n ? (((unsigned long long)fbits(buf.sr[o + t]) << 32) | buf.sidx[o + t]) : ~0ull;
  G::sync();
  group_bitonic<G>(keys, npad);
  bool tie = false;
  for (int t = G::rank() + 1; t < n; t += G::size()) if ((unsigned)(keys[t - 1] >> 32) == (unsigned)(keys[t] >> 32)) tie = true;
  if (G::any(tie)) {                                     // uniform: reproduce std::sort's order of the equal radii
    for (int t = G::rank(); t < n; t += G::size()) { const unsigned long long k = keys[t]; keys[t] = (k << 32) | (k >> 32); }
    G::sync();
    group_bitonic<G>(keys, npad);                        // ascending input index = push_back order (padding keys stay last)
    for (int t = G::rank(); t < n; t += G::size()) { const unsigned long long k = keys[t]; keys[t] = (k << 32) | (k >> 32); }
    G::sync();
    if (G::rank() == 0) { urfsort::std_sort(keys, n); atomicOr(&buf.out[b].flags, F_TIE_SECTOR); }
    G::sync();
  }
  // write the records in key order (z comes from the input record of that index)
  for (int t = G::rank(); t < n; t += G::size()) {
    const unsigned long long k = keys[t];
    const unsigned idx = (unsigned)k;
    buf.ssrz[o + t] = make_float2(bitsf((unsigned)(k >> 32)), buf.in[(size_t)b * point_slice(S) + idx].z);
    buf.ssl[o + t] = idx | kSslIndex;
  }
  G::sync();
}

// Near-first selection for the eight-warp sort (see k_star_sort): pivot = the 144th smallest of 256 evenly spaced
// samples (56 %), the (radius bits, slot) pairs below it appended to the shared lists in any order. Returns their number.
template <int EPL>
__device__ __forceinline__ int select_near_cta(const float* __restrict__ sr, int n, int tid, unsigned* s_pk, unsigned* s_pe, unsigned* s_misc, int pivot_rank) {
  const unsigned mine = fbits(sr[(int)(((unsigned)tid * (unsigned)n) >> 8)]);
  unsigned key[EPL];
#pragma unroll
  for (int r = 0; r < EPL; r++) {
    const int e = r * 256 + tid;
    key[r] = e < n ? fbits(sr[e]) : 0xffffffffu;
  }
  __syncthreads();                                     // the lists are free (previous sector done)
  s_pk[tid] = mine;
  if (tid == 0) s_misc[1] = 0u;
  __syncthreads();
  int rank = 0;                                        // ranks of the samples are a permutation (ties broken by thread)
  for (int j = 0; j < 256; j++) { const unsigned o = s_pk[j]; rank += (o < mine) || (o == mine && j < tid); }
  if (rank == pivot_rank) s_misc[0] = mine;
  __syncthreads();
  const unsigned pivot = s_misc[0];
  __syncthreads();                                     // everybody has read the samples: the lists may be overwritten
#pragma unroll
  for (int r = 0; r < EPL; r++) {
    const bool sel = key[r] < pivot;                   // padding keys are 0xffffffff: never selected
    const unsigned pos = warp_append(sel, &s_misc[1]);
    if (sel) { s_pk[pos] = key[r]; s_pe[pos] = (unsigned)(r * 256 + tid); }
  }
  __syncthreads();
  return (int)s_misc[1];
}

// eight-warp register network on a whole sector (LIST = false) or on the m listed elements (LIST = true); true = radius
// tie, or more than kCtaCap elements (nothing sorted: beyond the networks)
template <bool LIST>
__device__ __forceinline__ bool sort_sector_cta(const SectorRecs& d, int n, int tid, unsigned* s_xk, unsigned* s_xe) {
  if (n <= 1024) return bitonic_sector<4, 8, LIST>(d, n, tid, s_xk, s_xe);
  if (n <= 2048) return bitonic_sector<8, 8, LIST>(d, n, tid, s_xk, s_xe);
  if (n <= 4096) return bitonic_sector<16, 8, LIST>(d, n, tid, s_xk, s_xe);
  if (n <= kCtaCap) return bitonic_sector<32, 8, LIST>(d, n, tid, s_xk, s_xe);
  return true;
}

// k_star_sort_big: the sectors k_star_sort handed over. tab.biglist (1025 .. kCtaCap points): eight-warp register
// network, near-first like the single-warp sort (only the points below a sampled pivot radius are sorted, sorted_len tells
// k_star_scan how far it may walk), redone at once in full by the exact fallback when it meets equal radii; tab.slowlist
// (larger sectors, and sectors in which the single-warp sort met equal radii): exact fallback, whole sector.
constexpr size_t kStarCtaSmem = 2 * sizeof(unsigned) * kCtaCap;            // 64 KB: exchange buffers / 8192 64-bit keys
__global__ void __launch_bounds__(256) k_star_sort_big(DevBuffers buf, DevParams prm, int S) {
  extern __shared__ unsigned s_dyn[];
  const int b = blockIdx.y;
  ScanTab& tab = buf.tab[b];
  unsigned* s_xk = s_dyn;
  unsigned* s_xe = s_dyn + kCtaCap;
  __shared__ int s_tie;
  __shared__ unsigned s_misc[2];
  const int nbig = tab.nbig, nslow = tab.nslow;
  for (int w = blockIdx.x; w < nbig; w += gridDim.x) {
    const int s = tab.biglist[w];
    const int base = tab.sect_start[s], n = tab.sect_start[s + 1] - base;
    const SectorRecs d = sector_recs(buf, b, S, base);
    if (threadIdx.x == 0) s_tie = 0;
    int m = 0;
    if (prm.star_prefix) {
      if (n <= 2048) m = select_near_cta<8>(d.r(), n, threadIdx.x, s_xk, s_xe, s_misc, 8 * prm.star_pivot + 7);
      else if (n <= 4096) m = select_near_cta<16>(d.r(), n, threadIdx.x, s_xk, s_xe, s_misc, 8 * prm.star_pivot + 7);
      else m = select_near_cta<32>(d.r(), n, threadIdx.x, s_xk, s_xe, s_misc, 8 * prm.star_pivot + 7);
    }
    const bool near = m >= 256 && 4 * m <= 3 * n;                          // uniform: m comes from shared memory
    const bool tie = near ? sort_sector_cta<true>(d, m, threadIdx.x, s_xk, s_xe) : sort_sector_cta<false>(d, n, threadIdx.x, s_xk, s_xe);
    if (near && threadIdx.x == 0) tab.sorted_len[s] = m;
    // the tie flag goes through shared memory rather than __syncthreads_or: with the reduction barrier here ptxas emits
    // every network twice (128 registers instead of 127, 13 % more instructions, 2 % slower on C5 sectors)
    __syncthreads();
    if (tie) s_tie = 1;
    __syncthreads();
    const bool redo = s_tie != 0;
    __syncthreads();
    if (redo) {
      if (threadIdx.x == 0) tab.sorted_len[s] = n;
      slow_sort_sector<CtaGroup>(buf, b, S, base, n, reinterpret_cast<unsigned long long*>(s_dyn), kCtaCap);
    }
  }
  for (int w = blockIdx.x; w < nslow; w += gridDim.x) {
    const int s = tab.slowlist[w];
    const int base = tab.sect_start[s], n = tab.sect_start[s + 1] - base;
    if (threadIdx.x == 0) tab.sorted_len[s] = n;
    slow_sort_sector<CtaGroup>(buf, b, S, base, n, reinterpret_cast<unsigned long long*>(s_dyn), kCtaCap);
  }
}

// resumed walk of a refined sector (entry w of tab.refine, starting at o = b * S + base) over its completely sorted points
// by one WARP (all 32 lanes call it): per tile of 32 points every lane computes what does not depend on the recurrence for
// one point (slope, radius step, 1 / i: the IEEE divisions), then all lanes run the dependent part of the 32 points in lock
// step on their own copy of the state (values handed round by shuffles), so control flow stays uniform. star_step is the
// same arithmetic point by point.
__device__ __forceinline__ void star_resume_walk_warp(const DevBuffers& buf, const DevParams& prm, ScanTab& tab, int b, int S, int w, int s,
                                                      unsigned o, int n, int lane) {
  const float2* dst = buf.ssrz + o;
  if (lane == 0) tab.sorted_len[s] = n;
  StarState st;
  st.avg = tab.resume[w][0]; st.dev = tab.resume[w][1]; st.nan = tab.resume[w][2];
  const int n0 = __float_as_int(tab.resume[w][3]);     // >= 32: a prefix is never shorter
  st.bx = 0.f; st.by = 0.f;                            // unused: slopes come from the points themselves
  int hit = -1;
  for (int t0 = n0; t0 < n && hit < 0; t0 += 32) {
    const int e = min(t0 + lane, n - 1);
    const float2 p = dst[e], pp = dst[e - 1];
    float dx;
    const float slp = star_slope(pp.x, pp.y, p.x, p.y, &dx);
    const float dxk = __fmul_rn(dx, prm.kdist);
    const float inv = star_inv(e);
    const int cnt = min(32, n - t0);
    for (int j = 0; j < cnt; j++) {
      const float sj = __shfl_sync(0xffffffffu, slp, j), dj = __shfl_sync(0xffffffffu, dxk, j), ij = __shfl_sync(0xffffffffu, inv, j);
      if (star_update(prm, st, t0 + j, sj, dj, ij)) { hit = t0 + j; break; }
    }
  }
  if (hit >= 0 && lane == 0) curb_hit(buf, prm, b, scan_base(b, S), star_input_index(buf, o, hit), -1);   // star_shaped_search.cpp:146
}

// k_star_refine: second pass for the sectors whose edge search ran off their sorted prefix (tab.refine, filled by
// k_star_scan): the rest of the sector is sorted behind the prefix (single-warp path; the CTA path sorts the whole sector
// again), then one warp resumes the walk at point n0 with the saved running mean / deviation — the first n0 points of
// the full order are the prefix already walked (all of them are closer than the rest). Sectors of up to kWarpCap points:
// one WARP per sector (register network, exact fallback on equal radii in the warp's shared memory), the eight warps of a
// CTA working on eight sectors; larger sectors: the whole CTA sorts, one sector at a time, and its warp 0 walks.
// Two CTAs per SM stated explicitly: with the bound left implicit ptxas also settles on 128 registers but spills.
__global__ void __launch_bounds__(256, 2) k_star_refine(DevBuffers buf, DevParams prm, int S) {
  extern __shared__ unsigned s_dyn[];
  const int b = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  ScanTab& tab = buf.tab[b];
  const int nref = tab.nrefine;
  unsigned long long* wkeys = reinterpret_cast<unsigned long long*>(s_dyn) + (size_t)warp * kWarpCap;   // 8 x 8 KB
  for (int w = blockIdx.x * 8 + warp; w < nref; w += gridDim.x * 8) {
    const int s = tab.refine[w];
    const int base = tab.sect_start[s], n = tab.sect_start[s + 1] - base;
    if (n > kWarpCap) continue;                                            // second loop
    const unsigned o = scan_base(b, S) + (unsigned)base;
    // sorted positions [0, n0) already hold the n0 closest points in order (the walked prefix): only the rest is sorted,
    // behind it
    const int n0 = __float_as_int(tab.resume[w][3]);
    const SectorRecs d = sector_recs(buf, b, S, base, n0);
    unsigned* s_pk = reinterpret_cast<unsigned*>(wkeys);
    unsigned* s_pe = s_pk + kWarpCap;
    const unsigned kmax = fbits(buf.ssrz[o + n0 - 1].x);
    int m;
    if (n <= 256) m = select_far<8>(d.r(), n, lane, s_pk, s_pe, kmax);
    else if (n <= 512) m = select_far<16>(d.r(), n, lane, s_pk, s_pe, kmax);
    else m = select_far<32>(d.r(), n, lane, s_pk, s_pe, kmax);
    bool tie;
    if (m != n - n0) tie = true;                                           // cannot happen (prefix = everything below the pivot); exact path if it does
    else if (m <= 128) tie = bitonic_sector<4, 1, true>(d, m, lane, s_pk, s_pe);
    else if (m <= 256) tie = bitonic_sector<8, 1, true>(d, m, lane, s_pk, s_pe);
    else if (m <= 512) tie = bitonic_sector<16, 1, true>(d, m, lane, s_pk, s_pe);
    else tie = bitonic_sector<32, 1, true>(d, m, lane, s_pk, s_pe);
    __syncwarp();
    if (__any_sync(0xffffffffu, tie)) slow_sort_sector<WarpGroup>(buf, b, S, base, n, wkeys, kWarpCap);   // equal radii: whole sector, std::sort's order
    __syncwarp();
    star_resume_walk_warp(buf, prm, tab, b, S, w, s, o, n, lane);
    __syncwarp();
  }
  __syncthreads();
  for (int w = blockIdx.x; w < nref; w += gridDim.x) {
    const int s = tab.refine[w];
    const int base = tab.sect_start[s], n = tab.sect_start[s + 1] - base;
    if (n <= kWarpCap) continue;                                           // done above
    if (__syncthreads_or(sort_sector_cta<false>(sector_recs(buf, b, S, base), n, tid, s_dyn, s_dyn + kCtaCap)))   // ties, or above kCtaCap
      slow_sort_sector<CtaGroup>(buf, b, S, base, n, reinterpret_cast<unsigned long long*>(s_dyn), kCtaCap);
    // both ways a barrier follows the last record written. The walk reads only global records and touches no shared
    // memory: the next sector's sort may start beside it

    if (warp == 0) star_resume_walk_warp(buf, prm, tab, b, S, w, s, scan_base(b, S) + (unsigned)base, n, lane);
  }
}

// k_star_scan: one lane per sector walks its radius-sorted points with the reference's running mean / average absolute
// deviation recurrence (star_shaped_search.cpp:112-150) and marks the first edge point. Per 32-point tile the warp first
// computes, 32 points of one sector at a time, everything that does not depend on the recurrence (slope, radius step,
// 1 / i — including the IEEE divisions) into shared memory; the serial walk is then a dozen dependent float operations
// per point.
constexpr int kScanWarps = 2;
__global__ void __launch_bounds__(kScanWarps * 32) k_star_scan(DevBuffers buf, DevParams prm, int S) {
  const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = lane_id();
  __shared__ float s_slp[kScanWarps][32][33];
  __shared__ float s_dxk[kScanWarps][32][33];
  __shared__ float s_inv[kScanWarps][32][33];
  ScanTab& tab = buf.tab[b];
  const int s = (blockIdx.x * kScanWarps + warp) * 32 + lane;
  int base = 0, n = 0, whole = 0;
  if (s < kSectKeys) {
    base = tab.sect_start[s]; whole = tab.sect_start[s + 1] - base;
    n = min(whole, tab.sorted_len[s]);               // walk the sorted prefix only
  }
  const float2* all = buf.ssrz + (size_t)b * point_slice(S);
  StarState st;
  star_init(st, 0.f, 0.f);
  bool done = n <= 1;                                                   // star_shaped_search.cpp:112
  int hit = -1;
  int nmax = n;
  for (int o = 16; o > 0; o >>= 1) nmax = max(nmax, __shfl_xor_sync(0xffffffffu, nmax, o));
  for (int t0 = 0; t0 < nmax; t0 += 32) {
    // stage tile [t0, t0 + 32) of all 32 sector rows: 8 rows at a time so that the 16 loads of a group are in flight
    // together (one L2 round trip per group instead of one per row). (Tried and dropped as slower, when the sorted records
    // were 16 bytes: 16 rows at a time with 8-byte loads and the predecessor taken from the left neighbour by shuffle.)
    for (int q0 = 0; q0 < 32; q0 += 8) {
      float2 p[8], pp[8];
      bool ok[8];
#pragma unroll
      for (int u = 0; u < 8; u++) {
        const int q = q0 + u;
        const int qn = __shfl_sync(0xffffffffu, n, q), qbase = __shfl_sync(0xffffffffu, base, q);
        const int qdone = __shfl_sync(0xffffffffu, (int)done, q);
        const int e = t0 + lane;
        ok[u] = !qdone && e < qn && e >= 1;
        const int at = ok[u] ? qbase + e : 1;
        p[u] = all[at]; pp[u] = all[at - 1];
      }
#pragma unroll
      for (int u = 0; u < 8; u++) {
        if (ok[u]) {
          float dx;
          s_slp[warp][q0 + u][lane] = star_slope(pp[u].x, pp[u].y, p[u].x, p[u].y, &dx);
          s_dxk[warp][q0 + u][lane] = __fmul_rn(dx, prm.kdist);
          s_inv[warp][q0 + u][lane] = star_inv(t0 + lane);
        }
      }
    }
    __syncwarp();
    if (!done) {
      const int e1 = min(32, n - t0);
      for (int e = (t0 == 0 ? 1 : 0); e < e1; e++) {
        const int i = t0 + e;
        if (star_update(prm, st, i, s_slp[warp][lane][e], s_dxk[warp][lane][e], s_inv[warp][lane][e])) { hit = i; done = true; break; }
      }
      if (t0 + 32 >= n) done = true;
    }
    __syncwarp();
    if (__all_sync(0xffffffffu, done)) break;
  }
  if (hit >= 0) curb_hit(buf, prm, b, scan_base(b, S), star_input_index(buf, scan_base(b, S) + (unsigned)base, hit), -1);   // star_shaped_search.cpp:146
  else if (n < whole) {                               // ran off the sorted prefix: sort in full, k_star_refine continues from here
    const int w = atomicAdd(&tab.nrefine, 1);
    tab.refine[w] = (unsigned short)s;
    tab.resume[w][0] = st.avg; tab.resume[w][1] = st.dev; tab.resume[w][2] = st.nan; tab.resume[w][3] = __int_as_float(n);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// k_ring_detect: one thread per ring-bucket position: the x-zero test for which this point is the middle point p2
// (x_zero_method.cpp:30-67), the z-zero test centred on it (z_zero_method.cpp:21-72), and the ring's largest planar range
// (maxDistance, lidar_segmentation.cpp:271-274, as the largest double sum — see planar_sum_bits). The CTA stages its 256
// bucket positions plus a halo of curb_points on each side in shared memory as three coordinate arrays (plain global
// reads when curb_points exceeds kHalo). Both detectors are a cheap height gate followed by an expensive angle test
// (four double square roots, a double divide, acosf); about one point in eight passes a gate, scattered over most warps,
// so every thread evaluates only the gates and the CTA compacts the survivors into a work list that full warps then run
// the angle tests over (x-zero items from thread 0 upwards, z-zero items from thread 255 downwards). Points found to be
// curb points are marked in input order and entered into the curb bins (curb_hit); nothing else is written per point.
constexpr int kHalo = 32;

// Threads 0 .. 2 kHalo - 1 of a ring-detector CTA: the kHalo bucket records on either side of the tile [p0, p0 + T) into
// the tile slots [0, kHalo) and [kHalo + T, T + 2 kHalo) of the coordinate arrays, zeros outside the ordered points [0, N).
template <int T>
__device__ __forceinline__ void load_halo(const float4* bucket, int p0, int N, float* s_x, float* s_y, float* s_z) {
  const int tid = threadIdx.x;
  if (tid < 2 * kHalo) {
    const int ph = tid < kHalo ? p0 - kHalo + tid : p0 + T + tid - kHalo;
    const int sh = tid < kHalo ? tid : T + tid;
    float4 h = make_float4(0.f, 0.f, 0.f, 0.f);
    if (ph >= 0 && ph < N) h = bucket[ph];
    s_x[sh] = h.x; s_y[sh] = h.y; s_z[sh] = h.z;
  }
}
// Warp-aggregated 64-bit atomicMax (MIN = false) or atomicMin (MIN = true) of v into a[key] from the lanes that hold a
// value; the other lanes pass v = 0 (max) or ~0 (min). One atomic, from lane 0, when every holder has the same key, else
// one per holder; either only where it would move a[key] past cur, the value the lane last read there (0 for a max that
// read nothing). The warp reduces the high words first, then the low words of the lanes that hold the extreme high word.
template <bool MIN>
__device__ __forceinline__ void warp_atomic64(unsigned long long* a, bool holds, int key, unsigned long long v,
                                              unsigned long long cur) {
  const unsigned long long idle = MIN ? ~0ull : 0ull;
  const unsigned hm = __ballot_sync(0xffffffffu, holds);
  if (!hm) return;
  const int key0 = __shfl_sync(0xffffffffu, key, __ffs(hm) - 1);
  if (__all_sync(0xffffffffu, !holds || key == key0)) {
    const unsigned hi = (unsigned)(v >> 32), mh = MIN ? __reduce_min_sync(0xffffffffu, hi) : __reduce_max_sync(0xffffffffu, hi);
    const unsigned lo = hi == mh ? (unsigned)v : (unsigned)idle;
    const unsigned ml = MIN ? __reduce_min_sync(0xffffffffu, lo) : __reduce_max_sync(0xffffffffu, lo);
    const unsigned long long cur0 = __shfl_sync(0xffffffffu, cur, __ffs(hm) - 1);
    if (lane_id() == 0) {                                           // results unused: REDs
      const unsigned long long r = ((unsigned long long)mh << 32) | ml;
      if (MIN ? cur0 > r : cur0 < r) { if (MIN) atomicMin(&a[key0], r); else atomicMax(&a[key0], r); }
    }
  } else if (holds && (MIN ? cur > v : cur < v)) {
    if (MIN) atomicMin(&a[key], v); else atomicMax(&a[key], v);
  }
}
__global__ void __launch_bounds__(256, 8) k_ring_detect(DevBuffers buf, DevParams prm, int S) {
  const int b = blockIdx.y;
  const ScanOut& out = buf.out[b];
  const int p0 = blockIdx.x * 256, tid = threadIdx.x, p = p0 + tid;
  const unsigned gb = scan_base(b, S);
  const float4* bucket = buf.bpt + gb;
  // inside the scan's slot whatever n_order is, so the load need not wait for it
  const float4 me0 = p < S ? bucket[p] : make_float4(0.f, 0.f, 0.f, 0.f);
  const int N = out.n_order;
  __shared__ float s_x[256 + 2 * kHalo], s_y[256 + 2 * kHalo], s_z[256 + 2 * kHalo];
  __shared__ int s_rs[kRingKeys + 2];                     // ring_start of the rings this CTA touches, indexed by ring - k_lo
  __shared__ int s_base[256];                             // ring_start of each thread's ring
  __shared__ unsigned short s_item[512];                  // x-zero work items grow from 0 up, z-zero items from 511 down
  __shared__ unsigned char s_hit[256];
  __shared__ int s_klo, s_nx, s_nz;
  if (p0 >= N) return;
  if (tid < 32) {                                         // rings are contiguous in bucket order: first .. last ring of the CTA
    const int k_lo = ring_of_position(out.ring_start, p0), k_hi = ring_of_position(out.ring_start, min(p0 + 255, N - 1));
    if (tid == 0) { s_klo = k_lo; s_nx = 0; s_nz = 0; }
    for (int t = tid; t <= k_hi - k_lo + 1; t += 32) s_rs[t] = out.ring_start[k_lo + t];
  }
  const bool tiled = prm.curbPoints <= kHalo;
  const bool act = p < N;
  const float4 me = act ? me0 : make_float4(0.f, 0.f, 0.f, 0.f);
  if (tiled) {                                            // one bucket record per thread + a halo record for the first 64 threads
    s_x[kHalo + tid] = me.x; s_y[kHalo + tid] = me.y; s_z[kHalo + tid] = me.z;
    load_halo<256>(bucket, p0, N, s_x, s_y, s_z);
    s_hit[tid] = 0;
  }
  __syncthreads();
  int k = -1;
  bool hit = false, need_x = false, need_z = false;
  if (act) {
    int r = 0;
    while (p >= s_rs[r + 1]) r++;                         // p < N = the last staged entry at the latest
    k = s_klo + r;
    const int base = s_rs[r], n = s_rs[r + 1] - base, m = p - base;
    if (tiled) {
      s_base[tid] = base;
      const int off = base - (p0 - kHalo);                // ring-local index q lives at tile slot off + q
      const RingSoA ring{s_x + off, s_y + off, s_z + off};
      need_x = prm.x_zero && xzero_pre_t<0>(prm, ring, n, m);
      need_z = prm.z_zero && zzero_pre_t<0>(prm, ring, n, m);
    } else {                                              // huge curb_points: straight from global memory
      const float4* ring = bucket + base;
      hit = (prm.x_zero && xzero_mark_t<0>(prm, ring, n, m, buf.newY)) ||             // x_zero_method.cpp:66
            (prm.z_zero && zzero_mark_t<0>(prm, ring, n, m));                         // z_zero_method.cpp:71
    }
  }
  if (tiled) {
    const int ox = warp_append(need_x, &s_nx), oz = warp_append(need_z, &s_nz);
    if (need_x) s_item[ox] = (unsigned short)tid;
    if (need_z) s_item[511 - oz] = (unsigned short)tid;
    __syncthreads();
    const int nx = s_nx, nz = s_nz;
    for (int it = tid; it < nx; it += 256) {                            // x-zero angle tests, x_zero_method.cpp:35-61
      const int t = s_item[it], base = s_base[t], off = base - (p0 - kHalo);
      const RingSoA ring{s_x + off, s_y + off, s_z + off};
      if (xzero_post(prm, ring, p0 + t - base, buf.newY)) s_hit[t] = 1;
    }
    for (int it = 255 - tid; it < nz; it += 256) {                      // z-zero angle tests, z_zero_method.cpp:23-66
      const int t = s_item[511 - it], base = s_base[t], off = base - (p0 - kHalo);
      const RingSoA ring{s_x + off, s_y + off, s_z + off};
      if (zzero_post_t<0>(prm, ring, p0 + t - base)) s_hit[t] = 1;
    }
    __syncthreads();
    hit = act && s_hit[tid];                                            // x_zero_method.cpp:66, z_zero_method.cpp:71
  }
  if (hit) curb_hit(buf, prm, b, gb, __float_as_int(me.w), k);
  // maxDistance[k], lidar_segmentation.cpp:271-274
  warp_atomic64<false>(buf.tab[b].maxs, k >= 0, k, planar_sum_bits(me.x, me.y), 0ull);
}

// k_ring_detect4: the same work for the default curb_points = 5 with FOUR consecutive bucket positions per thread (tile of
// 1024 positions + halo per CTA). The two height gates of a position only read z: of its own ring, 5 positions to either
// side (z-zero) and at -2 / +3 (x-zero). Four consecutive positions share a window of 14 heights, which the thread fetches
// with five 16-byte shared-memory loads instead of 4 x 14 scalar ones; ring lookup, work-list compaction and the maximum of
// the planar sums are amortised over the four positions as well. The gates restate xzero_pre_t<5> / zzero_pre_t<5> on the
// register window (called through a view on it, they made the kernel 2 % slower on an H100 80GB HBM3 at 700 W).
constexpr int kTile4 = 1024;
__global__ void __launch_bounds__(256, 6) k_ring_detect4(DevBuffers buf, DevParams prm, int S) {
  constexpr int CP = 5;
  const int b = blockIdx.y;
  const ScanOut& out = buf.out[b];
  const int p0 = blockIdx.x * kTile4, tid = threadIdx.x;
  const unsigned gb = scan_base(b, S);
  const float4* bucket = buf.bpt + gb;
  // inside the scan's slot whatever n_order is, so the loads need not wait for it
  float4 rec[4];
#pragma unroll
  for (int j = 0; j < 4; j++) { const int q = p0 + tid + 256 * j; rec[j] = q < S ? bucket[q] : make_float4(0.f, 0.f, 0.f, 0.f); }
  const int N = out.n_order;
  __shared__ __align__(16) float s_x[kTile4 + 2 * kHalo], s_y[kTile4 + 2 * kHalo], s_z[kTile4 + 2 * kHalo];
  __shared__ int s_rs[kRingKeys + 2];                     // ring_start of the rings this CTA touches, indexed by ring - k_lo
  __shared__ unsigned short s_itx[kTile4], s_itz[kTile4]; // x-zero / z-zero work items: tile positions that passed the gate
  __shared__ __align__(4) unsigned char s_hit[kTile4];
  __shared__ int s_klo, s_nx, s_nz;
  if (p0 >= N) return;
  if (tid < 32) {                                         // rings are contiguous in bucket order: first .. last ring of the CTA
    const int k_lo = ring_of_position(out.ring_start, p0), k_hi = ring_of_position(out.ring_start, min(p0 + kTile4 - 1, N - 1));
    if (tid == 0) { s_klo = k_lo; s_nx = 0; s_nz = 0; }
    for (int t = tid; t <= k_hi - k_lo + 1; t += 32) s_rs[t] = out.ring_start[k_lo + t];
  }
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int t = tid + 256 * j;
    const bool in = p0 + t < N;
    s_x[kHalo + t] = in ? rec[j].x : 0.f; s_y[kHalo + t] = in ? rec[j].y : 0.f; s_z[kHalo + t] = in ? rec[j].z : 0.f;
    s_hit[t] = 0;
  }
  load_halo<kTile4>(bucket, p0, N, s_x, s_y, s_z);
  __syncthreads();
  // the thread's four consecutive positions t0 .. t0 + 3 of the tile; heights of tile slots t0 - 8 .. t0 + 11
  const int t0 = 4 * tid;
  float zw[20];
#pragma unroll
  for (int v = 0; v < 5; v++) {
    const float4 f = *reinterpret_cast<const float4*>(&s_z[kHalo + t0 - 8 + 4 * v]);
    zw[4 * v] = f.x; zw[4 * v + 1] = f.y; zw[4 * v + 2] = f.z; zw[4 * v + 3] = f.w;
  }
  const float4 fx = *reinterpret_cast<const float4*>(&s_x[kHalo + t0]), fy = *reinterpret_cast<const float4*>(&s_y[kHalo + t0]);
  const float xs[4] = {fx.x, fx.y, fx.z, fx.w}, ys[4] = {fy.x, fy.y, fy.z, fy.w};
  int r = 0;                                              // ring (relative to s_klo) of the current position
  unsigned nx_mask = 0, nz_mask = 0;
  unsigned long long smax = 0ull;                         // largest planar sum among the thread's positions of ring rmax
  int rmax = -1;
  const int kbase = s_klo;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int p = p0 + t0 + j;
    if (p >= N) break;
    while (p >= s_rs[r + 1]) r++;                         // p < N = the last staged entry at the latest
    const int base = s_rs[r], n = s_rs[r + 1] - base, m = p - base;
    const float z = zw[8 + j];
    // z-zero gate, zzero_pre_t<5> on the register window (z_zero_method.cpp:38-40,47-49,67-69)
    if (prm.z_zero && m >= CP && m <= (n - 1) - CP) {
      const float az0 = fabsf(z);
      float max1 = az0, max2 = az0;
#pragma unroll
      for (int u = 1; u <= CP; u++) { const float v = fabsf(zw[8 + j - u]); if (v > max1) max1 = v; }
#pragma unroll
      for (int u = 1; u <= CP; u++) { const float v = fabsf(zw[8 + j + u]); if (v > max2) max2 = v; }
      if ((__fsub_rn(max1, az0) >= prm.curbHeight || __fsub_rn(max2, az0) >= prm.curbHeight) && (double)fabsf(__fsub_rn(max1, max2)) >= 0.05)
        nz_mask |= 1u << j;
    }
    // x-zero gate, xzero_pre_t<5> with this point as p2 = j + cp / 2 (x_zero_method.cpp:62-64)
    const int jx = m - CP / 2;
    if (prm.x_zero && jx >= CP && jx <= (n - 1) - CP) {
      const float za = zw[8 + j - CP / 2], zc = zw[8 + j - CP / 2 + CP];
      if ((fabsf(__fsub_rn(za, z)) >= prm.curbHeight || fabsf(__fsub_rn(zc, z)) >= prm.curbHeight) && (double)fabsf(__fsub_rn(za, zc)) >= 0.05)
        nx_mask |= 1u << j;
    }
    // maxDistance: the thread keeps the maximum for the ring of its last position; an earlier ring's goes out at once
    const unsigned long long sb = planar_sum_bits(xs[j], ys[j]);
    if (r != rmax) {
      if (rmax >= 0) atomicMax(&buf.tab[b].maxs[kbase + rmax], smax);
      rmax = r; smax = sb;
    } else if (sb > smax) smax = sb;
  }
  // compaction of the gate survivors into the two work lists (one shared counter bump per warp and list)
  {
    const int cx = __popc(nx_mask), cz = __popc(nz_mask);
    int pc[2] = {cx, cz};                                 // inclusive warp scans of the per-thread counts
    warp_inclusive_sum(pc);
    const int px = pc[0], pz = pc[1];
    int wx = 0, wz = 0;
    if (lane_id() == 31) { if (px) wx = atomicAdd(&s_nx, px); if (pz) wz = atomicAdd(&s_nz, pz); }
    wx = __shfl_sync(0xffffffffu, wx, 31); wz = __shfl_sync(0xffffffffu, wz, 31);
    int ox = wx + px - cx, oz = wz + pz - cz;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      if (nx_mask & (1u << j)) s_itx[ox++] = (unsigned short)(t0 + j);
      if (nz_mask & (1u << j)) s_itz[oz++] = (unsigned short)(t0 + j);
    }
  }
  // warp-level maximum of the planar sums when the whole warp ended in one ring, else one atomic per thread
  {
    const int r0 = __shfl_sync(0xffffffffu, rmax, 0);
    if (__all_sync(0xffffffffu, rmax == r0)) {
      if (r0 >= 0) {
        const unsigned hi = (unsigned)(smax >> 32), mh = __reduce_max_sync(0xffffffffu, hi);
        const unsigned ml = __reduce_max_sync(0xffffffffu, hi == mh ? (unsigned)smax : 0u);
        if (lane_id() == 0) atomicMax(&buf.tab[b].maxs[kbase + r0], ((unsigned long long)mh << 32) | ml);
      }
    } else if (rmax >= 0) atomicMax(&buf.tab[b].maxs[kbase + rmax], smax);
  }
  __syncthreads();
  const int nx = s_nx, nz = s_nz;
  auto ring_base = [&](int t) {                           // ring start of tile position t (a tile spans few rings)
    const int p = p0 + t;
    int a = 0;
    while (p >= s_rs[a + 1]) a++;
    return s_rs[a];
  };
  for (int it = tid; it < nx; it += 256) {                              // x-zero angle tests, x_zero_method.cpp:35-61
    const int t = s_itx[it];
    const int base = ring_base(t), off = base - (p0 - kHalo);
    const RingSoA ring{s_x + off, s_y + off, s_z + off};
    if (xzero_post(prm, ring, p0 + t - base, buf.newY)) s_hit[t] = 1;
  }
  for (int it = tid; it < nz; it += 256) {                              // z-zero angle tests, z_zero_method.cpp:23-66
    const int t = s_itz[it];
    const int base = ring_base(t), off = base - (p0 - kHalo);
    const RingSoA ring{s_x + off, s_y + off, s_z + off};
    if (zzero_post_t<CP>(prm, ring, p0 + t - base)) s_hit[t] = 1;
  }
  __syncthreads();
  const unsigned hits = *reinterpret_cast<const unsigned*>(&s_hit[t0]);  // x_zero_method.cpp:66, z_zero_method.cpp:71
  if (hits) {
    int rr = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int p = p0 + t0 + j;
      if (p >= N) break;
      while (p >= s_rs[rr + 1]) rr++;
      if ((hits >> (8 * j)) & 0xffu) curb_hit(buf, prm, b, gb, __float_as_int(bucket[p].w), kbase + rr);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// blindSpots as tables (urf_logic.cuh: CurbView, window_blocked, build_T_row, covered_T). Three short kernels — a cluster
// of eight CTAs per scan running the three phases behind cluster barriers was tried and was slower than the three
// launches (C2 x 128: the 722 window tests of a scan want more than eight CTAs' worth of warps at once).
// k_tab1: per scan — prefix counts of non-empty curb bins per ring, maxDistance / arc widths, q1..q4, reach := n_rings.
__global__ void __launch_bounds__(256) k_tab1(DevBuffers buf, DevParams prm) {
  const int b = blockIdx.y;
  const ScanOut& out = buf.out[b];
  ScanTab& tab = buf.tab[b];
  const int R = out.n_rings;
  const int warp = threadIdx.x >> 5, lane = lane_id();
  if (blockIdx.x == 0) for (int t = threadIdx.x; t < 2 * kDegBins; t += blockDim.x) tab.reach[t / kDegBins][t % kDegBins] = R;
  if (R <= 0) return;
  const size_t nb = degbin_slice((size_t)prm.channels);
  const unsigned* cmin = buf.cmin + (size_t)b * nb;
  unsigned short* ne = buf.ne + (size_t)b * degsum_slice((size_t)prm.channels);
  for (int k = blockIdx.x * 8 + warp; k < R; k += gridDim.x * 8) {        // one warp per ring: 12 x 32 bins with a running carry
    unsigned carry = 0;
    for (int c = 0; c < (kDegBins + 31) / 32; c++) {
      const int bin = c * 32 + lane;
      const unsigned f = bin < kDegBins && cmin[(size_t)k * kDegBins + bin] != 0x7f800000u;
      const unsigned bal = __ballot_sync(0xffffffffu, f);
      if (bin < kDegBins) ne[(size_t)k * (kDegBins + 1) + bin] = (unsigned short)(carry + __popc(bal & ((1u << lane) - 1u)));
      carry += __popc(bal);
    }
    if (lane == 0) ne[(size_t)k * (kDegBins + 1) + kDegBins] = (unsigned short)carry;
  }
  if (blockIdx.x != 0) return;
  const float arc = arc_distance(prm, maxdist_from_bits(tab.maxs[0]));   // blind_spots.cpp:65
  for (int k = threadIdx.x; k < R; k += blockDim.x) {
    const float md = maxdist_from_bits(tab.maxs[k]);                     // lidar_segmentation.cpp:271-274
    tab.maxdist[k] = fbits(md);
    tab.A[k] = ring_width(arc, md);                                      // :142
  }
  if (threadIdx.x < 4) {
    CurbView cv{cmin, buf.cmax + (size_t)b * nb, ne};
    tab.q[threadIdx.x] = blind_quarter(prm, cv, R, threadIdx.x);         // :13-57 (reads the curb bins only)
  }
}

// k_reach: one warp per (direction, window start i): lanes test 32 rings at a time whether ring k holds a curb point
// inside window i and stop at the first blocked ring — reach[dir][i] (blind_spots.cpp:107-171 / :216-280 stop there too).
__global__ void __launch_bounds__(256) k_reach(DevBuffers buf, DevParams prm) {
  const int b = blockIdx.y;
  const ScanOut& out = buf.out[b];
  ScanTab& tab = buf.tab[b];
  const int R = out.n_rings;
  const int w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = lane_id();
  if (w >= 2 * kDegBins || R <= 0) return;
  const int dir = w / kDegBins, i = w % kDegBins;
  if (dir == 0 ? i > prm.fwd_last : i < prm.bwd_first) return;          // outside the loop range: never accepted anyway
  const size_t nb = degbin_slice((size_t)prm.channels);
  CurbView cv{buf.cmin + (size_t)b * nb, buf.cmax + (size_t)b * nb, buf.ne + (size_t)b * degsum_slice((size_t)prm.channels)};
  int reach = R;
  for (int k0 = 0; k0 < R; k0 += 32) {
    const int k = k0 + lane;
    const bool blocked = k < R && window_blocked(prm, cv, tab.A[k], dir, i, k);
    const unsigned bal = __ballot_sync(0xffffffffu, blocked);
    if (bal) { reach = k0 + __ffs(bal) - 1; break; }
  }
  if (lane == 0) tab.reach[dir][i] = reach;
}

// k_tab2: one warp per (ring, direction) builds a row of a threshold table with a warp max/min scan over the 361
// window starts (same result as the sequential build_T_row of urf_logic.cuh). Degree-major layout in memory: entry (j, k)
// at (j * channels + k) — a warp of k_label reads one or a few contiguous runs whether the sensor emits column-major (32
// rings at one azimuth) or ring-major (one ring, a few degrees). A CTA builds the rows of kTab2Rings consecutive rings in
// shared memory and writes them out transposed, kTab2Rings consecutive floats per degree.
constexpr int kTab2Rings = 16;
__global__ void __launch_bounds__(kTab2Rings * 64) k_tab2(DevBuffers buf, DevParams prm) {
  const int b = blockIdx.y;
  const ScanOut& out = buf.out[b];
  const ScanTab& tab = buf.tab[b];
  __shared__ float s_T[2][kDegBins][kTab2Rings + 1];     // +1: the row writes of a warp (stride kTab2Rings + 1) avoid bank conflicts
  const int w = threadIdx.x >> 5, lane = lane_id();
  const int kl = w >> 1, dir = w & 1;
  const int k0 = blockIdx.x * kTab2Rings, k = k0 + kl;
  const int R = out.n_rings;
  if (k0 >= R) return;
  constexpr int NCH = (kDegBins + 31) / 32;
  if (k < R) {
    const double A = tab.A[k];
    if (dir == 0) {
      int carry = -1;
      for (int c = 0; c < NCH; c++) {
        const int j = c * 32 + lane;
        int m = (j < kDegBins && accepted_fwd(prm, tab.reach[0], tab.q, k, j)) ? j : -1;
        for (int d = 1; d < 32; d <<= 1) { const int v = __shfl_up_sync(0xffffffffu, m, d); if (lane >= d) m = max(m, v); }
        m = max(m, carry);
        if (j < kDegBins) s_T[0][j][kl] = T_fwd_value(prm, k, m, A);
        carry = __shfl_sync(0xffffffffu, m, 31);
      }
    } else {
      int carry = 361;
      for (int c = NCH - 1; c >= 0; c--) {
        const int j = c * 32 + lane;
        int m = (j < kDegBins && accepted_bwd(prm, tab.reach[1], tab.q, k, j)) ? j : 361;
        for (int d = 1; d < 32; d <<= 1) { const int v = __shfl_down_sync(0xffffffffu, m, d); if (lane + d < 32) m = min(m, v); }
        m = min(m, carry);
        if (j < kDegBins) s_T[1][j][kl] = T_bwd_value(prm, k, m, A);
        carry = __shfl_sync(0xffffffffu, m, 0);
      }
    }
  }
  __syncthreads();
  const size_t ch = prm.channels;
  const size_t o = (size_t)b * ttab_slice(ch) + k0;
  const int nk = min(kTab2Rings, R - k0);
  for (int t = threadIdx.x; t < 2 * kDegBins * kTab2Rings; t += blockDim.x) {
    const int kk = t % kTab2Rings, j = (t / kTab2Rings) % kDegBins, d = t / (kTab2Rings * kDegBins);
    if (kk < nk) (d == 0 ? buf.Tf : buf.Tb)[o + (size_t)j * ch + kk] = s_T[d][j][kk];
  }
}

// k_label: final label per input point, in input order (coalesced): -1 outside the ROI cloud, 2 where a detector marked
// the point, 1 where a blindSpots window covers it (two threshold look-ups, covered_from), else 0. Also the counts, per
// degree bin the first non-road point in the reference's scan order (ring, azimuth; equal azimuths in input order), and
// the road points for the marker search: every warp owns the 32 list slots at its own position (roadlist[warp * 32 ..],
// count in roadcnt[warp]) — no running counter, so no atomic with a return value and no barrier in this kernel.
// A warp handles kLabelGroups consecutive groups of 32 input points (one point of each per lane) and makes two memory
// round trips for all of them together: every point's ring / azimuth / range / mark, then every threshold entry and bin
// key. Loads are issued whatever the ring id says (values of points outside the ROI are dropped; the buffers are zeroed
// at allocation and the reads stay inside the scan's slot), so that nothing in a round trip waits for another load.
constexpr int kLabelGroups = 2;
// REF (reference tie order): a point's place in the scan order is its emission position epos, not its input index.
constexpr int kLabelThreads = 256;
template <bool REF>
__global__ void __launch_bounds__(kLabelThreads) k_label(DevBuffers buf, DevParams prm, int S) {
  constexpr int G = kLabelGroups;
  const int b = blockIdx.y;
  ScanOut& out = buf.out[b];
  ScanTab& tab = buf.tab[b];
  const int n = buf.n[b];
  const int lane = lane_id();
  const int w0 = (blockIdx.x * kLabelThreads + (threadIdx.x & ~31)) * G;     // first input point of the warp
  if (w0 >= n) return;                                  // whole warp past the end of the scan
  const unsigned gb = scan_base(b, S);
  int k[G], m[G], pos[G];
  float a[G], d[G];
#pragma unroll
  for (int u = 0; u < G; u++) {
    const int i = w0 + u * 32 + lane;
    const bool in = i < n;
    const unsigned g = gb + (unsigned)i;
    k[u] = in ? buf.ringid[g] : -2;                     // -2 past the end too: such a point gets no label
    a[u] = in ? buf.az[g] : 0.f;
    d[u] = in ? buf.d2[g] : 0.f;
    m[u] = in ? buf.mark[g] : 0;
    pos[u] = REF ? (in && k[u] >= 0 ? buf.epos[g] : 0) : i;
  }
  // the two threshold entries (degree-major table, see k_tab2) and the bin's current first-non-road key of every point
  float tf[G], tb[G];
  unsigned long long cb[G];
  int bin[G];
  const unsigned ob = (unsigned)b * ttab_slice((unsigned)prm.channels);
#pragma unroll
  for (int u = 0; u < G; u++) {
    const bool valid = k[u] >= 0 && a[u] >= 0.0f;
    int j = 0, jc = 0;
    if (valid) T_indices(a[u], &j, &jc);
    bin[u] = valid ? j : -1;                            // j == deg_bin(a)
    tf[u] = valid ? buf.Tf[ob + (unsigned)k[u] + (unsigned)j * prm.channels] : 0.f;
    tb[u] = valid ? buf.Tb[ob + (unsigned)k[u] + (unsigned)jc * prm.channels] : 0.f;
    cb[u] = valid ? __ldcg(&tab.cutbest[j]) : 0ull;     // from L2: L1 would keep serving the value of the first look
  }
  unsigned nroad = 0, ncurb = 0;
#pragma unroll
  for (int u = 0; u < G; u++) {
    const int i = w0 + u * 32 + lane;
    if (w0 + u * 32 >= n) break;                        // warp-uniform: this group and the ones after it lie past the end
    const unsigned g = gb + (unsigned)i;
    int lab = -2;                                       // -2: past the end of the scan
    unsigned long long key = ~0ull;                     // first-non-road key of this point (~0 = none)
    if (i < n) {
      lab = k[u] == -2 ? URF_LABEL_OUTSIDE : URF_LABEL_NONE;
      if (k[u] >= 0) {
        const bool valid = bin[u] >= 0;
        lab = m[u] == 2 ? 2 : (valid && covered_from(a[u], tf[u], tb[u])) ? 1 : 0;   // covered_T of urf_logic.cuh with the loads hoisted
        if (valid && lab != 1) key = best_key(k[u], fbits(a[u]), pos[u]);   // lidar_segmentation.cpp:318: non-road point in bin [i, i+1)
      }
      buf.label[g] = lab;
      if (buf.label8) buf.label8[g] = (signed char)lab;
      if (prm.want_order && i >= out.n_order) buf.order[g] = -1;   // defined tail of the emission order (k_sort_rings writes [0, n_order))
    }
    // first non-road point per bin: atomicMin of the keys. A column-major scan puts the 32 rings of one azimuth — one bin —
    // into a group, a ring-major one a few neighbouring bins: when all keys of the group belong to one bin only their
    // minimum goes out (one atomic per group instead of one per point). A key loaded before an earlier group of this warp
    // lowered it is only larger: the atomic then goes out needlessly, never wrongly.
    warp_atomic64<true>(tab.cutbest, key != ~0ull, bin[u], key, cb[u]);
    const unsigned br = __ballot_sync(0xffffffffu, lab == 1), bc = __ballot_sync(0xffffffffu, lab == 2);
    nroad += __popc(br);
    ncurb += __popc(bc);
    if (lane == 0) buf.roadcnt[(size_t)b * warp_slice(S) + (unsigned)(i >> 5)] = (unsigned char)__popc(br);
    if (lab == 1)
      buf.roadlist[gb + (unsigned)(i & ~31) + (unsigned)__popc(br & ((1u << lane) - 1u))] =
          make_uint4((unsigned)bin[u] | ((unsigned)k[u] << 16), fbits(a[u]), fbits(d[u]), (unsigned)pos[u]);
  }
  if (lane == 0) {                                      // results unused: fire-and-forget
    if (nroad) atomicAdd(&out.n_road, (int)nroad);
    if (ncurb) atomicAdd(&out.n_curb, (int)ncurb);
  }
}

// k_markers1: marker candidate vertices, lidar_segmentation.cpp:305-351, over the road points k_label listed (32 slots per
// warp of input points, count in roadcnt) — ONE CTA of 1024 threads per scan, everything in its own shared memory:
//   pass 1  farthest candidate road point per bin (candidates: road points scanned before the bin's first non-road point)
//   pass 2  first candidate in scan order that reaches that distance (`d > maxDistanceRoad` is strict, :329)
//   then    the per-bin winners are compacted in bin order into markerPointsArray (:343-350)
// In each pass a warp takes 32 list segments at a time, scans their counts and spreads the entries evenly over its lanes
// (entry e of the 32 segments belongs to the segment whose exclusive count prefix is the last one <= e), four entries in
// flight per lane. Scans above kMarkSingleMax (urf_api.cu) points take k_markers_grid instead.
constexpr int kMark1Threads = 1024;
template <int PASS>
__device__ __forceinline__ void markers_pass(const uint4* __restrict__ list, const unsigned char* __restrict__ cnt, int nseg,
                                             const unsigned long long* s_cut, unsigned* s_dmax, unsigned long long* s_best) {
  const int lane = lane_id(), nwarps = (blockDim.x >> 5) * gridDim.x;       // warps of all CTAs that share this scan
  const int warp = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int cpre[4];                                          // counts of the warp's next four sweeps, loaded together
  for (int seg0 = warp * 32, sw = 0; seg0 < nseg; seg0 += nwarps * 32, sw++) {
    if ((sw & 3) == 0) {
#pragma unroll
      for (int u = 0; u < 4; u++) { const int sg = seg0 + u * nwarps * 32 + lane; cpre[u] = sg < nseg ? cnt[sg] : 0; }
    }
    const int c = (sw & 3) == 0 ? cpre[0] : (sw & 3) == 1 ? cpre[1] : (sw & 3) == 2 ? cpre[2] : cpre[3];
    int inc[1] = {c};
    warp_inclusive_sum(inc);
    const int excl = inc[0] - c, total = __shfl_sync(0xffffffffu, inc[0], 31);
    for (int e0 = 0; e0 < total; e0 += 128) {
      uint4 ent[4];
      bool ok[4];
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const int e = e0 + u * 32 + lane;
        int lo = 0;                                      // last segment whose exclusive prefix is <= e (skips empty segments)
#pragma unroll
        for (int step = 16; step > 0; step >>= 1) {
          const int ex = __shfl_sync(0xffffffffu, excl, lo + step < 32 ? lo + step : 31);
          if (lo + step < 32 && ex <= e) lo += step;
        }
        const int r = e - __shfl_sync(0xffffffffu, excl, lo);
        ok[u] = e < total;
        ent[u] = ok[u] ? list[(seg0 + lo) * 32 + r] : make_uint4(0u, 0u, 0u, 0u);
      }
#pragma unroll
      for (int u = 0; u < 4; u++) {
        if (!ok[u]) continue;
        const uint4 q = ent[u];
        const int bin = q.x & 0xffff, k = q.x >> 16;
        if (PASS == 1) {
          if (marker_candidate(s_cut[bin], k, q.y, (int)q.w) && s_dmax[bin] < q.z) atomicMax(&s_dmax[bin], q.z);
        } else if (q.z != 0u && q.z == s_dmax[bin] && marker_candidate(s_cut[bin], k, q.y, (int)q.w)) {
          const unsigned long long key = best_key(k, q.y, (int)q.w);
          if (s_best[bin] > key) atomicMin(&s_best[bin], key);
        }
      }
    }
  }
}
// The per-bin winners best[] (~0 = none) compacted in bin order into markerPointsArray (:343-350), with redPoints where
// the bin has a first non-road point cut[] (:320,348), and a zeroed tail. One bin per thread: the CTA has at least
// kDegBins threads.
template <bool REF>
__device__ __forceinline__ void write_vertices(const DevBuffers& buf, int b, int S, const unsigned long long* best,
                                               const unsigned long long* cut) {
  ScanOut& out = buf.out[b];
  const int i = threadIdx.x;
  const bool has = i < kDegBins && best[i] != ~0ull;
  int total;
  const int slot = CtaGroup::count(has, &total);
  if (has) {
    int p = (int)(best[i] & 0xffffffull);               // input index of the winner (REF: its emission position)
    if (REF) p = buf.order[(size_t)b * point_slice(S) + p];
    const float4 q = buf.in[(size_t)b * point_slice(S) + p];
    out.vert[slot][0] = q.x; out.vert[slot][1] = q.y; out.vert[slot][2] = q.z;
    out.vert[slot][3] = cut[i] != ~0ull ? 1.0f : 0.0f;
  }
  if (i == 0) out.n_vert = total;
  if (i >= total && i < URF_MAX_VERTS) { out.vert[i][0] = 0.f; out.vert[i][1] = 0.f; out.vert[i][2] = 0.f; out.vert[i][3] = 0.f; }   // defined tail
}
template <bool REF>
__global__ void __launch_bounds__(kMark1Threads) k_markers1(DevBuffers buf, int S) {
  const int b = blockIdx.y;                            // grid (1, B)
  const ScanTab& tab = buf.tab[b];
  __shared__ unsigned long long s_cut[kDegBins], s_best[kDegBins];
  __shared__ unsigned s_dmax[kDegBins];
  const int tid = threadIdx.x;
  for (int t = tid; t < kDegBins; t += kMark1Threads) { s_cut[t] = tab.cutbest[t]; s_dmax[t] = 0u; s_best[t] = ~0ull; }
  __syncthreads();
  const int n = buf.n[b];
  const int nseg = (n + 31) >> 5;
  const unsigned char* cnt = buf.roadcnt + (size_t)b * warp_slice(S);
  const uint4* list = buf.roadlist + scan_base(b, S);
  markers_pass<1>(list, cnt, nseg, s_cut, s_dmax, s_best);
  __syncthreads();
  markers_pass<2>(list, cnt, nseg, s_cut, s_dmax, s_best);
  __syncthreads();
  write_vertices<REF>(buf, b, S, s_best, s_cut);
}

// The same search for LARGE scans (hundreds of thousands of road points want more than one CTA): a grid of CTAs per scan,
// every CTA aggregates its share per degree bin in shared memory and merges into the scan's global arrays with atomics;
// pass 1, pass 2 and the vertex compaction are three launches.
constexpr int kMarkGridThreads = 256;
template <int PASS>
__global__ void __launch_bounds__(kMarkGridThreads) k_markers_grid(DevBuffers buf, int S) {
  const int b = blockIdx.y;
  ScanTab& tab = buf.tab[b];
  __shared__ unsigned long long s_cut[kDegBins], s_best[kDegBins];
  __shared__ unsigned s_dmax[kDegBins];
  const int tid = threadIdx.x;
  for (int t = tid; t < kDegBins; t += kMarkGridThreads) {
    s_cut[t] = tab.cutbest[t]; s_best[t] = ~0ull;
    s_dmax[t] = PASS == 1 ? 0u : tab.dmax[t];          // pass 2 compares with the merged maxima of pass 1
  }
  __syncthreads();
  const int n = buf.n[b];
  const int nseg = (n + 31) >> 5;
  const unsigned char* cnt = buf.roadcnt + (size_t)b * warp_slice(S);
  const uint4* list = buf.roadlist + scan_base(b, S);
  markers_pass<PASS>(list, cnt, nseg, s_cut, s_dmax, s_best);
  __syncthreads();
  for (int t = tid; t < kDegBins; t += kMarkGridThreads) {
    if (PASS == 1) { const unsigned v = s_dmax[t]; if (v) atomicMax(&tab.dmax[t], v); }
    else { const unsigned long long v = s_best[t]; if (v != ~0ull) atomicMin(&tab.best[t], v); }
  }
}
// k_verts: the vertex compaction of k_markers1 on the merged winners (tab.best)
template <bool REF>
__global__ void __launch_bounds__(384) k_verts(DevBuffers buf, int S) {
  const int b = blockIdx.x;
  const ScanTab& tab = buf.tab[b];
  write_vertices<REF>(buf, b, S, tab.best, tab.cutbest);
}

// ---------------------------------------------------------------------------------------------------------------------
// k_sort_rings (only when the emission order is requested): per-ring sort by azimuth, lidar_segmentation.cpp:70-93,289-291.
// Tie policy: (azimuth, input order) — the reference's Lomuto quicksort is unstable; ties raise F_TIE_AZIMUTH.
// One CTA per ring. Rings of up to kRingFast points take a counting sort in shared memory: azimuths are spread over
// kRingBins equal-width bins between the ring's smallest and largest azimuth (a monotone map, so bin order = azimuth
// order), a histogram + exclusive scan places every point in its bin, and the few points that share a bin (LiDAR rings
// are close to uniform in azimuth) are ordered by one thread with an insertion sort on (azimuth bits, position). A ring
// with a crowded bin (more than kBinCap points) or more than kRingFast points falls back to the CTA-wide bitonic sort on
// 64-bit (azimuth bits, position) keys. Both paths produce the same total order.
// REF (reference tie order): also the emission position of every point (epos), and the rings whose order is not unique —
// a tied pair or a NaN azimuth — listed for k_lomuto_rings.
constexpr int kRingSmemKeys = 6144;                     // 48 KB of dynamic shared memory: four CTAs per SM
constexpr int kRingFast = 4096, kRingBins = 4096, kBinCap = 48;
constexpr int kSortThreads = 512;
__device__ __forceinline__ void lomuto_enlist(const DevBuffers& buf, int b, int k, bool weird) {
  if (__syncthreads_or(weird) && threadIdx.x == 0) {
    int* l = buf.lomuto + (size_t)b * kRingListSlice;
    l[1 + atomicAdd(l, 1)] = k;
  }
}
template <bool REF>
__global__ void __launch_bounds__(kSortThreads) k_sort_rings(DevBuffers buf, int S) {
  extern __shared__ unsigned long long s_rkeys[];
  const int b = blockIdx.y, k = blockIdx.x;
  ScanOut& out = buf.out[b];
  if (k >= out.n_rings) return;
  const int base = out.ring_start[k], n = out.ring_start[k + 1] - base;
  if (n <= 0) return;
  const size_t gb = (size_t)b * point_slice(S), g0 = gb + base;
  const int tid = threadIdx.x;
  if (n <= kRingFast) {
    unsigned* s_az = reinterpret_cast<unsigned*>(s_rkeys);            // [kRingFast] azimuth bits by ring position
    unsigned* s_cnt = s_az + kRingFast;                               // [kRingBins] bin counts, then exclusive starts
    unsigned short* s_rank = reinterpret_cast<unsigned short*>(s_cnt + kRingBins);   // [kRingFast] arrival rank inside the bin
    unsigned short* s_slot = s_rank + kRingFast;                      // [kRingFast] ring position by sorted position
    __shared__ unsigned s_lo, s_hi, s_over;
    if (tid == 0) { s_lo = 0xffffffffu; s_hi = 0u; s_over = 0u; }
    for (int t = tid; t < kRingBins; t += kSortThreads) s_cnt[t] = 0u;
    __syncthreads();
    unsigned lo = 0xffffffffu, hi = 0u;
    for (int t0 = tid; t0 < n; t0 += 4 * kSortThreads) {             // four coalesced loads in flight per thread
      unsigned av[4];
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const int t = t0 + u * kSortThreads;
        av[u] = t < n ? buf.baz[g0 + t].x : 0u;                      // (azimuth, input index) in bucket order, written by k_scatter
      }
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const int t = t0 + u * kSortThreads;
        if (t < n) {
          s_az[t] = av[u];
          if (av[u] <= 0x7f800000u) { lo = min(lo, av[u]); hi = max(hi, av[u]); }   // azimuths are >= +0: their bits order them; NaN stays out
        }
      }
    }
    lo = __reduce_min_sync(0xffffffffu, lo); hi = __reduce_max_sync(0xffffffffu, hi);
    if (lane_id() == 0) { atomicMin(&s_lo, lo); atomicMax(&s_hi, hi); }
    __syncthreads();
    const float flo = bitsf(s_lo), fhi = bitsf(s_hi);
    const float scale = fhi > flo ? __fdiv_rn((float)(kRingBins - 2), __fsub_rn(fhi, flo)) : 0.0f;
    auto bin_of = [&](unsigned a) -> int {                           // monotone in a; NaN azimuths go to the last bin
      if (a > 0x7f800000u) return kRingBins - 1;
      const int v = __float2int_rz(__fmul_rn(__fsub_rn(bitsf(a), flo), scale));
      return v < 0 ? 0 : (v > kRingBins - 2 ? kRingBins - 2 : v);
    };
    for (int t = tid; t < n; t += kSortThreads) s_rank[t] = (unsigned short)atomicAdd(&s_cnt[bin_of(s_az[t])], 1u);
    __syncthreads();
    {   // exclusive scan over the bins: consecutive bins per thread, then the CTA-wide scan of the threads' sums
      constexpr int PER = kRingBins / kSortThreads;
      unsigned v[PER], run[1] = {0}, all[1], mx = 0;
#pragma unroll
      for (int j = 0; j < PER; j++) { v[j] = s_cnt[tid * PER + j]; run[0] += v[j]; mx = max(mx, v[j]); }
      if (mx > (unsigned)kBinCap) s_over = 1u;
      CtaGroup::exclusive_sum(run, all);
#pragma unroll
      for (int j = 0; j < PER; j++) { s_cnt[tid * PER + j] = run[0]; run[0] += v[j]; }
    }
    __syncthreads();
    if (!s_over) {
      for (int t = tid; t < n; t += kSortThreads) s_slot[s_cnt[bin_of(s_az[t])] + s_rank[t]] = (unsigned short)t;
      __syncthreads();
      constexpr int PER = kRingBins / kSortThreads;
      for (int j = 0; j < PER; j++) {                                  // order the points that share a bin
        const int bin = tid * PER + j;
        const int s0 = (int)s_cnt[bin], s1 = bin + 1 < kRingBins ? (int)s_cnt[bin + 1] : n;
        for (int e = s0 + 1; e < s1; e++) {
          const unsigned short cur = s_slot[e];
          const unsigned ca = s_az[cur];
          int f = e - 1;
          while (f >= s0) {
            const unsigned short o = s_slot[f];
            const unsigned oa = s_az[o];
            if (oa < ca || (oa == ca && o < cur)) break;
            s_slot[f + 1] = o; f--;
          }
          s_slot[f + 1] = cur;
        }
      }
      __syncthreads();
      bool tie = false, nan = false;
      for (int p = tid; p < n; p += kSortThreads) {
        const unsigned short slot = s_slot[p];
        const int idx = (int)buf.baz[g0 + slot].y;                   // the ring's pairs are in L2 from the first pass
        buf.order[g0 + p] = idx;
        if (REF) { buf.epos[gb + idx] = base + p; nan |= s_az[slot] > 0x7f800000u; }
        if (p > 0 && s_az[s_slot[p - 1]] == s_az[slot]) tie = true;
      }
      if (tie) atomicOr(&out.flags, F_TIE_AZIMUTH);
      if (REF) lomuto_enlist(buf, b, k, tie || nan);
      return;
    }
    __syncthreads();                                                   // the fallback reuses the shared memory
  }
  const int npad = next_pow2(n < 2 ? 2 : n);
  unsigned long long* keys = npad <= kRingSmemKeys ? s_rkeys : buf.sortbuf + pair_slice(g0);
  for (int t = tid; t < npad; t += blockDim.x)
    keys[t] = t < n ? (((unsigned long long)buf.baz[g0 + t].x << 32) | (unsigned)t) : ~0ull;
  __syncthreads();
  group_bitonic<CtaGroup>(keys, npad);
  bool tie = false, nan = false;
  for (int t = tid; t < n; t += blockDim.x) {
    const unsigned long long key = keys[t];
    const int idx = (int)buf.baz[g0 + (unsigned)key].y;
    buf.order[g0 + t] = idx;
    if (REF) { buf.epos[gb + idx] = base + t; nan |= (unsigned)(key >> 32) > 0x7f800000u; }
    if (t > 0 && (unsigned)(keys[t - 1] >> 32) == (unsigned)(key >> 32)) tie = true;
  }
  if (tie) atomicOr(&out.flags, F_TIE_AZIMUTH);
  if (REF) lomuto_enlist(buf, b, k, tie || nan);
}

// ---------------------------------------------------------------------------------------------------------------------
// k_lomuto_rings (reference tie order only): the rings k_sort_rings listed get the order of the reference's Lomuto
// quicksort (urf_lomuto.cuh), one CTA per listed ring (grid: channels x B, CTAs past the list return). It overwrites the
// ring's segment of `order` and the emission positions of its points. The work arrays (five words per point) sit in
// shared memory up to kLomutoSmemPts points, else in the ring's own 16-byte segment of sortbuf plus its slots of
// roadlist, which k_label only fills afterwards.
constexpr int kLomutoThreads = 512;
constexpr int kLomutoSmemPts = 4096;
constexpr size_t kLomutoSmem = (size_t)5 * kLomutoSmemPts * sizeof(unsigned);   // 80 KB
__global__ void __launch_bounds__(kLomutoThreads) k_lomuto_rings(DevBuffers buf, int S) {
  extern __shared__ unsigned s_lw[];
  __shared__ LomutoShared sh;
  const int b = blockIdx.y;
  const int* list = buf.lomuto + (size_t)b * kRingListSlice;
  if ((int)blockIdx.x >= list[0]) return;
  const int k = list[1 + blockIdx.x];
  const ScanOut& out = buf.out[b];
  const int base = out.ring_start[k], n = out.ring_start[k + 1] - base;
  const unsigned gb = scan_base(b, S), g0 = gb + (unsigned)base;
  const bool smem = n <= kLomutoSmemPts;
  unsigned* w = smem ? s_lw : reinterpret_cast<unsigned*>(buf.sortbuf + pair_slice((size_t)g0));
  for (int t = threadIdx.x; t < n; t += blockDim.x) {
    const uint2 q = buf.baz[g0 + t];
    w[t] = q.x;
    w[n + t] = (unsigned)(buf.epos[gb + q.y] - base);      // rank in k_sort_rings' order
  }
  if (threadIdx.x == 0) { sh.partitions = 0; sh.steps = 0; }
  __syncthreads();
  LomutoArrays a;
  a.az = w; a.rk = w + n; a.s0 = w + 2 * n; a.s1 = w + 3 * n;
  a.s2 = smem ? s_lw + 4 * n : reinterpret_cast<unsigned*>(buf.roadlist + g0);
  lomuto_ring<CtaGroup>(a, n, sh);
  for (int p = threadIdx.x; p < n; p += blockDim.x) {
    const int idx = (int)buf.baz[g0 + a.s0[p]].y;
    buf.order[g0 + p] = idx;
    buf.epos[gb + idx] = base + p;
  }
}

// k_unpack_cloud2_batch: PointCloud2 record -> (x, y, z, intensity) float4 (SURVEY.md §8 f1) for a batch: scan
// b = blockIdx.y, its records at raw + b * S * step_max, its points at dst + b * S. Scan b's format is fmt[b] (a batch of
// mixed formats, urf_process_cloud2_batch_mixed: the per-scan table in device memory), or with fmt == NULL `one` for every
// scan (step_max == one.point_step). Byte-wise loads when a field is not 4-byte aligned (Velodyne's 22-byte records).
// off_intensity < 0: no intensity field, 0 is stored.
__device__ __forceinline__ float load_f32_unaligned(const unsigned char* p) {
  if ((reinterpret_cast<size_t>(p) & 3) == 0) return *reinterpret_cast<const float*>(p);
  const unsigned v = (unsigned)p[0] | ((unsigned)p[1] << 8) | ((unsigned)p[2] << 16) | ((unsigned)p[3] << 24);
  return __uint_as_float(v);
}
__global__ void __launch_bounds__(256) k_unpack_cloud2_batch(const unsigned char* __restrict__ raw, float4* __restrict__ dst,
                                                              const int* __restrict__ n, int S, int step_max, urf_cloud2_format one,
                                                              const urf_cloud2_format* __restrict__ fmt) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n[b]) return;
  const urf_cloud2_format f = fmt ? fmt[b] : one;
  const unsigned char* rec = raw + (size_t)b * point_slice(S) * step_max + (size_t)i * f.point_step;
  dst[(size_t)b * point_slice(S) + i] = make_float4(load_f32_unaligned(rec + f.off_x), load_f32_unaligned(rec + f.off_y),
                                                    load_f32_unaligned(rec + f.off_z),
                                                    f.off_intensity >= 0 ? load_f32_unaligned(rec + f.off_intensity) : 0.f);
}

// ---------------------------------------------------------------------------------------------------------------------
// Output clouds packed on the device (SURVEY.md §8 f1, scan 0 of the buffers): what lidar_segmentation.cpp:354-367 and
// :605-608 push into cloud_filtered_Road / _High / _ProbablyRoad and what :120 leaves in cloud_filtered_Box, as 32-byte
// pcl::PointXYZI records (x, y, z, 1.0f | intensity, 0, 0, 0) in the reference's emission order:
//   road = points of `order` (ring-major, ascending azimuth) with label 1, curb = label 2 (stored behind road in the same
//   buffer), roi = label >= 0 in input order, road_probably = ring 10 of `order`.
// Three kernels: per-tile counts -> exclusive scan over tiles -> stable per-tile compaction.
constexpr int kPackTile = 1024;
__device__ __forceinline__ void pack_flags(const DevBuffers& buf, const ScanOut& out, int e, bool* road, bool* curb, bool* roi, int* idx) {
  *road = *curb = *roi = false; *idx = 0;
  if (out.n_roi < 30) return;                                            // nothing is published, lidar_segmentation.cpp:124-126
  if (e < out.n_order) { *idx = buf.order[e]; const int lab = buf.label[*idx]; *road = lab == 1; *curb = lab == 2; }
  if (e < out.n_in) *roi = buf.label[e] >= 0;
}
__global__ void __launch_bounds__(256) k_pack_count(DevBuffers buf, int* __restrict__ cnt, int tiles) {
  __shared__ int s_c[3];
  const ScanOut& out = buf.out[0];
  if (threadIdx.x < 3) s_c[threadIdx.x] = 0;
  __syncthreads();
  int c0 = 0, c1 = 0, c2 = 0;
  for (int j = 0; j < kPackTile / 256; j++) {
    bool road, curb, roi; int idx;
    pack_flags(buf, out, blockIdx.x * kPackTile + j * 256 + threadIdx.x, &road, &curb, &roi, &idx);
    c0 += road; c1 += curb; c2 += roi;
  }
  c0 = __reduce_add_sync(0xffffffffu, c0); c1 = __reduce_add_sync(0xffffffffu, c1); c2 = __reduce_add_sync(0xffffffffu, c2);
  if (lane_id() == 0) { atomicAdd(&s_c[0], c0); atomicAdd(&s_c[1], c1); atomicAdd(&s_c[2], c2); }
  __syncthreads();
  if (threadIdx.x < 3) cnt[threadIdx.x * tiles + blockIdx.x] = s_c[threadIdx.x];
}
// one CTA: exclusive scan of the three per-tile count rows in place; tot[0..3] = road, curb, roi, road_probably counts
__global__ void __launch_bounds__(1024) k_pack_scan(DevBuffers buf, int* __restrict__ cnt, int tiles, int* __restrict__ tot) {
  for (int row = 0; row < 3; row++) {
    int carry = 0;                                                       // tiles of the earlier rounds
    for (int t0 = 0; t0 < tiles; t0 += 1024) {
      const int t = t0 + threadIdx.x;
      int x[1] = {t < tiles ? cnt[row * tiles + t] : 0}, all[1];
      CtaGroup::exclusive_sum(x, all);
      if (t < tiles) cnt[row * tiles + t] = carry + x[0];
      carry += all[0];
    }
    if (threadIdx.x == 0) tot[row] = carry;
  }
  if (threadIdx.x == 0) {
    const ScanOut& out = buf.out[0];
    tot[3] = out.n_roi < 30 ? 0 : out.ring_start[11] - out.ring_start[10];     // lidar_segmentation.cpp:605-608
  }
}
__device__ __forceinline__ void pack_record(float4* __restrict__ dst, int pos, const float4 p) {
  dst[2 * (size_t)pos] = make_float4(p.x, p.y, p.z, 1.0f);               // PCL_ADD_POINT4D: data[3] = 1.0f
  dst[2 * (size_t)pos + 1] = make_float4(p.w, 0.f, 0.f, 0.f);            // intensity + padding
}
__global__ void __launch_bounds__(256) k_pack_write(DevBuffers buf, const int* __restrict__ cnt, int tiles, const int* __restrict__ tot,
                                                     float4* __restrict__ road_curb, float4* __restrict__ roi_dst, float4* __restrict__ prob) {
  const ScanOut& out = buf.out[0];
  int road_pos = cnt[blockIdx.x], curb_pos = tot[0] + cnt[tiles + blockIdx.x], roi_pos = cnt[2 * tiles + blockIdx.x];
  const int rs10 = out.ring_start[10], rs11 = out.n_roi < 30 ? rs10 : out.ring_start[11];
  for (int j = 0; j < kPackTile / 256; j++) {
    const int e = blockIdx.x * kPackTile + j * 256 + threadIdx.x;
    bool road, curb, roi; int idx;
    pack_flags(buf, out, e, &road, &curb, &roi, &idx);
    int total;
    const int r0 = CtaGroup::count(road, &total);
    if (road) pack_record(road_curb, road_pos + r0, buf.in[idx]);
    road_pos += total;
    const int r1 = CtaGroup::count(curb, &total);
    if (curb) pack_record(road_curb, curb_pos + r1, buf.in[idx]);
    curb_pos += total;
    const int r2 = CtaGroup::count(roi, &total);
    if (roi) pack_record(roi_dst, roi_pos + r2, buf.in[e]);
    roi_pos += total;
    if (e >= rs10 && e < rs11) pack_record(prob, e - rs10, buf.in[idx]);
  }
}

// Device-side evaluation of the emulated libm (test hook: urf_test_math).
__global__ void k_test_math(const float* a, const float* bb, float* o, int n, int which) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float r;
  switch (which) {
    case 0: r = urfm::asinf_glibc(a[i]); break;
    case 1: r = urfm::acosf_glibc(a[i]); break;
    case 2: r = urfm::atan2f_glibc(a[i], bb[i]); break;
    default: r = urfm::atanf_glibc(a[i]); break;
  }
  o[i] = r;
}

}  // namespace urf
