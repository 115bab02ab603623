// urf_api.cu — host side of liburf_b200.so: context, parameter narrowing, pipeline launcher and the C-ABI of include/urf.h.
// There is no CPU fallback in this library: without a CUDA device every compute entry point returns an error.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <array>
#include <memory>
#include <string>
#include <vector>

#include "urf_kernels.cuh"
#include "urf_host.hpp"
#include "urf_queue_internal.hpp"

using namespace urf;

constexpr int kMaxBatch = 65535;   // scans per context: the largest grid y dimension

// Owners of CUDA resources: each handle is released by its deleter when its owner goes
template <class T, cudaError_t (*F)(T*)> struct CudaDel { void operator()(T* p) const { F(p); } };
template <class T> using DevMem = std::unique_ptr<T, CudaDel<void, cudaFree>>;
template <class T> using HostMem = std::unique_ptr<T, CudaDel<void, cudaFreeHost>>;
using Stream = std::unique_ptr<CUstream_st, CudaDel<CUstream_st, cudaStreamDestroy>>;
using Event = std::unique_ptr<CUevent_st, CudaDel<CUevent_st, cudaEventDestroy>>;
using GraphExec = std::unique_ptr<CUgraphExec_st, CudaDel<CUgraphExec_st, cudaGraphExecDestroy>>;
using ArrayMem = std::array<DevMem<unsigned char>, kArrays>;   // owners of a DevBuffers' arrays, in for_each_array order

struct urf_ctx {
  int device = 0;
  int max_points = 0;      // per scan, rounded up to kChunk
  int max_batch = 0;
  size_t P = 0;            // max_batch * max_points
  int Tmax = 0;
  Stream stream;                       // compute
  Stream s_in, s_out;                  // H2D / D2H copy streams of the pipelined host-buffer path
  // Sub-batches of a device-resident call run on separate lanes (scans are independent, so their short, partly
  // latency-bound kernels overlap); lane kGroups is the context's own stream. Between k_scatter and k_tab1 the ring
  // detector runs on the lane's side stream, next to the star-shaped search
  // (H100 (400 W), C2 x 128: 1.95 / 2.06 ms per step with, 2.11 / 1.99 without (within noise)).
  static constexpr int kGroups = 16;
  struct Lane { cudaStream_t st = nullptr; Stream own, side; Event join, sfork, sjoin; };   // lane kGroups: no own, no join
  Lane lane[kGroups + 1];
  Event ev_fork;                       // the context stream's fork to the lanes
  int sort_ctas = 0;                  // resident CTAs of k_star_sort on the whole device (its grid: the warps walk the sectors)
  int pts_ctas = 0;                    // resident CTAs of k_points on the whole device (its grid: the scans share them)
  // H100 (400 W), C2 x 128: 1 stream 1.628 ms (one run), 2 streams 1.630 (median of six); 3 and 4 streams slower (DESIGN.md §6).
  // The groups do not hide each other's one-CTA-per-scan stages: descending stream priorities (1.683 ms) and a start
  // staggered by one k_points (1.631) were tried and dropped
  int groups = 2;
  // CUDA graph of the kernel sequence for small host-buffer batches (launch latency dominates there); re-captured when
  // the shape, the parameters or an option change
  bool use_graph = true;
  GraphExec gexec;
  int g_B = -1, g_S = -1, g_order = -1, g_launches = 0;
  unsigned long long g_version = 0, version = 1;
  std::vector<Event> ev_in, ev_comp;   // per chunk: input landed / results ready
  Event ev0, ev1;                      // the device-resident pair
  DevBuffers buf{};                    // the workspace, with slot 0's arrays
  ArrayMem mem;                        // owners of the workspace arrays of buf (slot 0's own theirs)
  // A host-buffer batch between its enqueue and its finish (urf_enqueue_batch / urf_finish_batch; the synchronous entry
  // points are one enqueue and one finish, always in slot 0). A slot holds what the batch's copies touch while the other
  // batch's kernels run; the per-point workspace is shared, and the kernels of both batches queue on `stream`.
  // Slot 0 is the context's own set (from urf_create); slot 1 is allocated by the first asynchronous call.
  struct HostSlot {
    DevBuffers dev{};                  // the per-slot arrays (class kSlot); label8 (int8 labels) is allocated when a caller
    ArrayMem mem;                      // first asks for it
    // record staging of the PointCloud2 / packed-xyz entry points: slot 0 has max_points * URF_MAX_POINT_STEP bytes from
    // urf_create, so single scans never allocate; re-allocated at P * step bytes by the first batch that needs more
    DevMem<unsigned char> rawb;
    size_t rawb_bytes = 0;
    // per-scan record formats of a mixed batch (urf_*_cloud2_batch_mixed), max_batch entries each, allocated by the slot's
    // first mixed batch; the chunks copy their slices on s_in with their point counts
    DevMem<urf_cloud2_format> fmt;
    HostMem<urf_cloud2_format> h_fmt;
    DevMem<int> ring;                 // ring ids for the caller; none in slot 0 before the first asynchronous call: the sort
                                       // scratch (buf.sortbuf) takes them, see ring_chunk
    HostMem<int> h_n; HostMem<ScanOut> h_out;   // pinned copies of n and out
    Event ev0, ev1, ev_done;           // bracket the batch's kernels; after its last copy to the host
    // the batch in flight; gen and C are the parameter generation and `channels` it was enqueued with (urf_set_params_next
    // may change the context's while it runs)
    int batch = 0, S = 0, launches = 0, C = 0;
    int32_t gen = 0;
    urf_result* outs = nullptr;
    urf_clouds* clouds = nullptr;
  };
  HostSlot hs[2];
  int hs_head = 0, hs_count = 0;       // oldest host batch in flight, number in flight (0..2)
  DevMem<float4> pack;                 // packed output clouds (urf_process_cloud2_packed): 3 * max_points 32-byte records, allocated on first use
  DevMem<int> packcnt, packtot;        // [3][tiles] per-tile counts / offsets, [4] cloud sizes
  HostMem<int> h_packtot;              // pinned copy
  int tie_order = URF_TIES_INPUT_ORDER;   // urf_set_tie_order; the reference order's buffers (buf.epos, buf.lomuto) are
                                          // allocated by the first switch to it
  urf_params params{};
  DevParams dp{};                      // copied by value into every launch: a batch keeps the parameters it was enqueued with
  int32_t gen = 0;                     // parameter generation (urf_set_params_next); 0 until the first one
  int32_t dev_gen = 0;                 // generation of the device-resident batch (urf_enqueue_batch_device*)
  // asynchronous enqueues stage their point counts in a ring of pinned rows, each guarded by the event of its H2D copy,
  // so back-to-back enqueues with different counts never overwrite a row whose copy has not run yet
  static constexpr int kNRing = 8;
  HostMem<int> h_nring;                // [kNRing][max_batch]
  Event ev_nring[kNRing];
  int nring_pos = 0;
  int last_B = 0, last_S = 0, last_C = 0;   // scans, stride and channels of the last finished call (urf_debug_fetch)
  int launches = 0;
  float last_ms = 0.f;                 // device ms of the last finished host batch (timing_host)
  bool timing_valid = false, timing_host = false;
  std::string err;
  // optional per-kernel CUDA-event timing (urf_set_option(ctx, 1, 1)); events live on the ctx stream
  bool profile = false;
  int kslots = 1, kslot = 0;           // event slots: consecutive calls cycle through them so K steps can be timed without syncing
  std::vector<Event> kev;              // [kslots][kMaxKernels + 1]; the last event of a slot closes the pipeline
  std::vector<const char*> knames;
  std::vector<int> kcounts;            // kernels recorded per slot
  int kcount = 0;
};

namespace {

// URF code of a CUDA status; the text of a failed call is kept for urf_last_cuda_error
int cuda_rc(urf_ctx* ctx, cudaError_t e, const char* call) {
  if (e == cudaSuccess) return URF_OK;
  ctx->err = std::string(call) + ": " + cudaGetErrorString(e);
  return e == cudaErrorMemoryAllocation ? URF_ERR_NOMEM : URF_ERR_CUDA;
}

#define CK(call)                                                                                   \
  do {                                                                                             \
    const int rc_ = cuda_rc(ctx, (call), #call);                                                   \
    if (rc_ != URF_OK) return rc_;                                                                 \
  } while (0)

template <class T> int dalloc(urf_ctx* ctx, DevMem<T>& owner, size_t count) {
  void* q = nullptr;
  CK(cudaMalloc(&q, count * sizeof(T) + 256));
  owner.reset(static_cast<T*>(q));
  // zero once: some kernels load ahead of the bound they check, and slots a call does not fill must read as defined (on the
  // context's stream, waited for: the legacy default stream is not ordered against the non-blocking streams used next)
  CK(cudaMemsetAsync(q, 0, count * sizeof(T) + 256, ctx->stream.get()));
  CK(cudaStreamSynchronize(ctx->stream.get()));
  return URF_OK;
}

// Hands the arrays allocated in `from`, and their owners, over to `to`
void adopt(DevBuffers& to, ArrayMem& to_mem, const DevBuffers& from, ArrayMem& from_mem) {
  for_each_array([&](int i, auto m, Kind, unsigned) { if (from.*m) { to.*m = from.*m; to_mem[i] = std::move(from_mem[i]); } });
}

// The arrays of `d` that `pick` selects, for max_batch scans at capacity, each owned by its entry of `mem`
template <class Pick> int alloc_owned(urf_ctx* ctx, DevBuffers& d, ArrayMem& mem, Pick pick) {
  return alloc_arrays(d, capacity_extent(ctx->max_points), ctx->max_batch, pick, [&](int i, auto& p, size_t count) {
    const int rc = dalloc(ctx, mem[i], count * sizeof(*p));
    if (rc == URF_OK) p = reinterpret_cast<std::remove_reference_t<decltype(p)>>(mem[i].get());
    return rc;
  });
}

// a new handle, held by `owner` (empty when the call fails)
cudaError_t new_stream(Stream& owner) { cudaStream_t h = nullptr; const cudaError_t e = cudaStreamCreateWithFlags(&h, cudaStreamNonBlocking); owner.reset(h); return e; }
cudaError_t new_event(Event& owner, unsigned flags = cudaEventDisableTiming) { cudaEvent_t h = nullptr; const cudaError_t e = cudaEventCreateWithFlags(&h, flags); owner.reset(h); return e; }
template <class T> cudaError_t new_pinned(HostMem<T>& owner, size_t count) { void* p = nullptr; const cudaError_t e = cudaMallocHost(&p, sizeof(T) * count); owner.reset(static_cast<T*>(p)); return e; }
// the pinned result rows and the events of a host slot
cudaError_t init_slot(urf_ctx* ctx, urf_ctx::HostSlot& h) {
  cudaError_t e = new_pinned(h.h_n, ctx->max_batch);
  if (e == cudaSuccess) e = new_pinned(h.h_out, ctx->max_batch);
  if (e == cudaSuccess) e = new_event(h.ev0, cudaEventDefault);
  if (e == cudaSuccess) e = new_event(h.ev1, cudaEventDefault);
  return e == cudaSuccess ? new_event(h.ev_done) : e;
}

__global__ void k_ring32(DevBuffers buf, int* dst, int S) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < buf.n[b]) dst[(size_t)b * point_slice(S) + i] = max((int)buf.ringid[(size_t)b * point_slice(S) + i], -1);
}

constexpr int kMaxKernels = 32;
constexpr int kMarkSingleMax = 300000;   // scans above this many points take the multi-CTA marker search
thread_local std::string g_create_err;

// Enqueues the kernel sequence for B scans of stride S from `buf` on `lane` and stores the number of kernels launched in
// *launched.
int launch_pipeline(urf_ctx* ctx, const DevBuffers& buf, int B, int S, bool want_order, const urf_ctx::Lane& lane, int* launched) {
  DevParams dp = ctx->dp;
  // reference tie order: the emission order decides the marker search's scan order, so the ring sort always runs, in
  // front of k_label (into the context's own order buffer when the caller asked for none)
  const bool ref = ctx->tie_order == URF_TIES_REFERENCE;
  dp.want_order = want_order || ref ? 1 : 0;
  cudaStream_t st = lane.st;
  const int T = (S + kChunk - 1) / kChunk;
  if (T > ctx->Tmax) return URF_ERR_CAPACITY;
  int L = 0;
  ctx->kcount = 0;
  const dim3 gpts((S + 255) / 256, B), gchunk((T + kWarpsPerBlock - 1) / kWarpsPerBlock, B);
  // K(name, launch): one kernel launch; with profiling on, an event is recorded in front of it
#define K(name, ...)                                                                         \
  do {                                                                                       \
    if (ctx->profile && ctx->kcount < kMaxKernels) {                                         \
      ctx->knames[ctx->kcount] = name;                                                       \
      CK(cudaEventRecord(ctx->kev[(size_t)ctx->kslot * (kMaxKernels + 1) + ctx->kcount].get(), st)); \
      ctx->kcount++;                                                                         \
    }                                                                                        \
    __VA_ARGS__;                                                                             \
    L++;                                                                                     \
  } while (0)
  K("k_reset", k_reset<<<dim3(8, B), 256, 0, st>>>(buf, dp));
  // k_points: at most one resident wave of CTAs over the launch's scans (a second, partial wave would take as long as
  // the first), a contiguous range of whole tiles each
  const int gp = std::max(1, std::min(ctx->pts_ctas / B, (S + kPtsTile - 1) / kPtsTile));
  K("k_points", k_points<<<dim3(gp, B), kPtsThreads, 0, st>>>(buf, dp, S));
  K("k_register", k_register<<<B, 256, 0, st>>>(buf, dp, S));
  K("k_assign", k_assign<<<gchunk, kWarpsPerBlock * 32, 0, st>>>(buf, dp, S, T));
  K("k_scan_offsets", k_scan_offsets<<<B, kScanOffThreads, 0, st>>>(buf, dp, S, T));   // + exact re-registration of refuted scans
  K("k_scatter", k_scatter<<<dim3((T + kScatterWarps - 1) / kScatterWarps, B), kScatterWarps * 32, kScatterSmem, st>>>(buf, dp, S, T));
  // the ring detector next to the star-shaped search: both only read what k_scatter left and add curb hits (idempotent
  // marks, atomic min / max aggregates); k_tab1 is the first reader of the aggregates. Per-kernel timing keeps every
  // kernel on `st`, where K records its events, and without the star-shaped search there is nothing to overlap.
  const bool fork = dp.star && !ctx->profile;
  cudaStream_t st_ring = fork ? lane.side.get() : st;
  if (fork) {
    CK(cudaEventRecord(lane.sfork.get(), st));
    CK(cudaStreamWaitEvent(st_ring, lane.sfork.get(), 0));
  }
  // k_ring_detect never sees curb_points = 5, so it runs the detectors' runtime (<0>) instantiations only
  if (dp.curbPoints == 5)              // four positions per thread (default curb_points only)
    K("k_ring_detect4", k_ring_detect4<<<dim3((S + kTile4 - 1) / kTile4, B), 256, 0, st_ring>>>(buf, dp, S));
  else K("k_ring_detect", k_ring_detect<<<gpts, 256, 0, st_ring>>>(buf, dp, S));
  if (fork) CK(cudaEventRecord(lane.sjoin.get(), st_ring));
  if (dp.star) {
    const int gbig = std::max(4, std::min(kSectKeys, 2048 / B));
    const dim3 gscan((kSectKeys + kScanWarps * 32 - 1) / (kScanWarps * 32), B);
    // as many CTAs as can be resident at once, the sectors dealt out by a static stride: the sectors of a launch are of
    // similar size (every scan of a batch comes from one sensor), so the shares are even; a work counter would cost one
    // same-address atomic per sector (46 k per C2 launch). A CTA that starts late because the other stream or the ring
    // detector holds SMs finishes its share late; the two-stream step times in DESIGN.md §6 include that.
    const int gsort = std::min(ctx->sort_ctas, (B * kSectKeys + kSortWarps - 1) / kSortWarps);
    K("k_star_sort", k_star_sort<<<gsort, kSortWarps * 32, kStarSortSmem, st>>>(buf, dp, S, B));
    K("k_star_sort_big", k_star_sort_big<<<dim3(gbig, B), 256, kStarCtaSmem, st>>>(buf, dp, S));
    K("k_star_scan", k_star_scan<<<gscan, kScanWarps * 32, 0, st>>>(buf, dp, S));
    if (dp.star_prefix)            // sectors whose edge search ran off the near-first prefix: full sort, search resumed
      K("k_star_refine", k_star_refine<<<dim3(std::max(8, std::min(kSectKeys / 8, 8192 / B)), B), 256, kStarCtaSmem, st>>>(buf, dp, S));
  }
  if (fork) CK(cudaStreamWaitEvent(st, lane.sjoin.get(), 0));
  K("k_tab1", k_tab1<<<dim3((dp.channels + 7) / 8, B), 256, 0, st>>>(buf, dp));
  K("k_reach", k_reach<<<dim3((2 * kDegBins + 7) / 8, B), 256, 0, st>>>(buf, dp));
  K("k_tab2", k_tab2<<<dim3((dp.channels + kTab2Rings - 1) / kTab2Rings, B), kTab2Rings * 64, 0, st>>>(buf, dp));
  const dim3 glabel((S + kLabelThreads * kLabelGroups - 1) / (kLabelThreads * kLabelGroups), B), gsort(dp.channels, B);
  if (ref) {
    K("k_sort_rings", k_sort_rings<true><<<gsort, kSortThreads, kRingSmemKeys * sizeof(unsigned long long), st>>>(buf, S));
    K("k_lomuto_rings", k_lomuto_rings<<<gsort, kLomutoThreads, kLomutoSmem, st>>>(buf, S));
    K("k_label", k_label<true><<<glabel, kLabelThreads, 0, st>>>(buf, dp, S));
  } else K("k_label", k_label<false><<<glabel, kLabelThreads, 0, st>>>(buf, dp, S));
  if (S > kMarkSingleMax) {            // large scans: a grid of CTAs per scan, three launches
    const dim3 gm(std::max(1, std::min(64, S / 16384)), B);
    K("k_markers_grid1", k_markers_grid<1><<<gm, kMarkGridThreads, 0, st>>>(buf, S));
    K("k_markers_grid2", k_markers_grid<2><<<gm, kMarkGridThreads, 0, st>>>(buf, S));
    if (ref) K("k_verts", k_verts<true><<<B, 384, 0, st>>>(buf, S));
    else K("k_verts", k_verts<false><<<B, 384, 0, st>>>(buf, S));
  } else if (ref) K("k_markers1", k_markers1<true><<<dim3(1, B), kMark1Threads, 0, st>>>(buf, S));
  else K("k_markers1", k_markers1<false><<<dim3(1, B), kMark1Threads, 0, st>>>(buf, S));   // one CTA per scan
  if (want_order && !ref) K("k_sort_rings", k_sort_rings<false><<<gsort, kSortThreads, kRingSmemKeys * sizeof(unsigned long long), st>>>(buf, S));
#undef K
  if (ctx->profile) {
    CK(cudaEventRecord(ctx->kev[(size_t)ctx->kslot * (kMaxKernels + 1) + kMaxKernels].get(), st));
    ctx->kcounts[ctx->kslot] = ctx->kcount;
    ctx->kslot = (ctx->kslot + 1) % ctx->kslots;
  }
  CK(cudaGetLastError());
  *launched = L;
  return URF_OK;
}

// Small host-buffer batches replay the kernel sequence as one CUDA graph (launch latency dominates there). Makes
// ctx->gexec the graph of this shape, captured from ctx->buf itself (the graph keeps its pointers) and re-captured when
// the shape, the parameters or an option change.
int update_graph(urf_ctx* ctx, int B, int S, bool want_order) {
  if (ctx->gexec && ctx->g_B == B && ctx->g_S == S && ctx->g_order == (int)want_order && ctx->g_version == ctx->version) return URF_OK;
  ctx->gexec.reset();
  cudaGraph_t graph = nullptr;
  CK(cudaStreamBeginCapture(ctx->stream.get(), cudaStreamCaptureModeThreadLocal));
  int L = 0;
  const int rc = launch_pipeline(ctx, ctx->buf, B, S, want_order, ctx->lane[urf_ctx::kGroups], &L);
  const cudaError_t e = cudaStreamEndCapture(ctx->stream.get(), &graph);
  if (rc != URF_OK || e != cudaSuccess || !graph) { if (graph) cudaGraphDestroy(graph); ctx->err = "graph capture failed"; return rc != URF_OK ? rc : URF_ERR_CUDA; }
  cudaGraphExec_t exec = nullptr;
  const cudaError_t ei = cudaGraphInstantiate(&exec, graph, 0);
  cudaGraphDestroy(graph); ctx->gexec.reset(exec);
  if (ei != cudaSuccess) { ctx->err = cudaGetErrorString(ei); return URF_ERR_CUDA; }
  ctx->g_B = B; ctx->g_S = S; ctx->g_order = (int)want_order; ctx->g_version = ctx->version; ctx->g_launches = L;
  return URF_OK;
}

// with_ring_start = false leaves the caller's ring_start untouched; gen: the parameter generation the scan ran with
void fill_result(const ScanOut& o, urf_result* r, bool with_ring_start, int32_t gen) {
  r->n_in = o.n_in; r->n_roi = o.n_roi;
  r->flags = o.flags & F_PUBLIC_MASK; r->params_gen = gen;
  if (o.n_roi < 30) {                       // lidar_segmentation.cpp:124-126
    r->status = URF_TOO_FEW_POINTS;
    r->n_rings = 0; r->n_order = 0; r->n_road = 0; r->n_curb = 0; r->n_vert = 0;
    if (with_ring_start && r->ring_start) for (int k = 0; k <= URF_MAX_CHANNELS; k++) r->ring_start[k] = 0;
    return;
  }
  r->status = URF_OK;
  r->n_rings = o.n_rings; r->n_order = o.n_order; r->n_road = o.n_road; r->n_curb = o.n_curb; r->n_vert = o.n_vert;
  std::memcpy(r->vert, o.vert, sizeof(float) * 4 * (size_t)o.n_vert);
  if (with_ring_start && r->ring_start) std::memcpy(r->ring_start, o.ring_start, sizeof(int) * (URF_MAX_CHANNELS + 1));
}

}  // namespace

extern "C" {

int urf_version(void) { return URF_VERSION; }

const char* urf_strerror(int code) {
  switch (code) {
    case URF_OK: return "ok";
    case URF_TOO_FEW_POINTS: return "fewer than 30 points in the ROI: nothing published";
    case URF_ERR_INVALID: return "invalid argument";
    case URF_ERR_NO_DEVICE: return "no CUDA device (this library has no CPU fallback)";
    case URF_ERR_CUDA: return "CUDA error";
    case URF_ERR_NOMEM: return "out of device or pinned memory";
    case URF_ERR_CAPACITY: return "scan or batch larger than the context was created for";
    case URF_ERR_TIMEOUT: return "timed out";
    case URF_ERR_CLOSED: return "queue closed";
    default: return "unknown error";
  }
}

const char* urf_last_cuda_error(const urf_ctx* ctx) {
  if (ctx) return ctx->err.c_str();
  return g_create_err.empty() ? "null context" : g_create_err.c_str();     // text of this thread's last failed urf_create
}

void urf_default_params(urf_params* p) {
  if (!p) return;
  std::memset(p, 0, sizeof(*p));
  std::snprintf(p->fixed_frame, sizeof(p->fixed_frame), "left_os1/os1_lidar");
  std::snprintf(p->topic_name, sizeof(p->topic_name), "/left_os1/os1_cloud_node/points");
  p->x_zero_method = 1; p->z_zero_method = 1; p->star_shaped_method = 1; p->blind_spots = 1; p->xDirection = 0;
  p->interval = 0.18; p->curb_height = 0.05; p->curb_points = 5; p->beamZone = 30;
  p->min_x = 0; p->max_x = 30; p->min_y = -10; p->max_y = 10; p->min_z = -3; p->max_z = -1;
  p->cylinder_deg_x = 150; p->cylinder_deg_z = 140; p->curb_slope_deg = 50;
  p->kdev_param = 1.225; p->kdist_param = 2; p->starbeam_filter = 0; p->dmin_param = 10;
  p->simple_poly_allow = 1; p->poly_s_param = 0.7; p->poly_z_manual = -1.5; p->poly_z_avg_allow = 1;
  p->channels = 64;
}

int urf_create(urf_ctx** out, int device, int max_points, int max_batch) {
  if (!out || max_points < 1 || max_batch < 1 || max_points > (1 << 24)) return URF_ERR_INVALID;
  if ((long long)(max_points + kChunk) * max_batch >= (1ll << 31)) return URF_ERR_CAPACITY;   // kernels use 32-bit offsets
  if (max_batch > kMaxBatch) return URF_ERR_CAPACITY;          // every kernel takes its scan from blockIdx.y
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) return URF_ERR_NO_DEVICE;
  urf_ctx* ctx = new urf_ctx();
  // the context dies with the failure: its error text survives in a per-thread slot that urf_last_cuda_error(NULL) returns
  auto fail = [&](int rc) { g_create_err = ctx->err.empty() ? std::string(urf_strerror(rc)) : ctx->err; urf_destroy(ctx); return rc; };
  ctx->device = device;
  if (cudaSetDevice(device) != cudaSuccess) return fail(URF_ERR_NO_DEVICE);
  ctx->max_points = ((max_points + kChunk - 1) / kChunk) * kChunk;
  ctx->max_batch = max_batch;
  ctx->P = (size_t)ctx->max_points * max_batch;
  ctx->Tmax = ctx->max_points / kChunk;
  int rc;
#define TRY(x) do { rc = (x); if (rc != URF_OK) return fail(rc); } while (0)
#define CKF(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { ctx->err = cudaGetErrorString(e_); return fail(URF_ERR_CUDA); } } while (0)
  for (Stream* s : {&ctx->stream, &ctx->s_in, &ctx->s_out}) CKF(new_stream(*s));
  for (int g = 0; g <= urf_ctx::kGroups; g++) {
    urf_ctx::Lane& l = ctx->lane[g];
    if (g < urf_ctx::kGroups) { CKF(new_stream(l.own)); CKF(new_event(l.join)); }
    l.st = g < urf_ctx::kGroups ? l.own.get() : ctx->stream.get();
    CKF(new_stream(l.side)); CKF(new_event(l.sfork)); CKF(new_event(l.sjoin));
  }
  CKF(new_event(ctx->ev_fork)); CKF(new_event(ctx->ev0, cudaEventDefault)); CKF(new_event(ctx->ev1, cudaEventDefault));
  DevBuffers& b = ctx->buf;
  urf_ctx::HostSlot& h0 = ctx->hs[0];
  TRY(alloc_owned(ctx, b, ctx->mem, created_with_context));
  TRY(alloc_owned(ctx, h0.dev, h0.mem, slot_array));
  b = slot_view(b, h0.dev);
  h0.rawb_bytes = capacity_elems(Kind::Point, capacity_extent(ctx->max_points), 1) * URF_MAX_POINT_STEP;
  TRY(dalloc(ctx, h0.rawb, h0.rawb_bytes));
  CKF(init_slot(ctx, h0));
  CKF(new_pinned(ctx->h_nring, (size_t)max_batch * urf_ctx::kNRing));
  for (Event& e : ctx->ev_nring) CKF(new_event(e));
  {
    std::vector<float> ny;
    host_newY(ny, ctx->max_points);
    CKF(cudaMemcpy(b.newY, ny.data(), sizeof(float) * ny.size(), cudaMemcpyHostToDevice));
    float bd[kSectKeys], bo[kSectKeys], Kfi;
    unsigned char byx[kSectKeys];
    host_beam_init(bd, bo, byx, &Kfi);
    CKF(cudaMemcpyToSymbol(c_beam_d, bd, sizeof(bd)));
    CKF(cudaMemcpyToSymbol(c_beam_o, bo, sizeof(bo)));
    CKF(cudaMemcpyToSymbol(c_beam_yx, byx, sizeof(byx)));
    ctx->dp.Kfi = Kfi;
  }
  CKF(cudaFuncSetAttribute(k_star_sort, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kStarSortSmem));
  {
    int sms = 0, per_sm = 0;
    CKF(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, ctx->device));
    CKF(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_star_sort, kSortWarps * 32, kStarSortSmem));
    ctx->sort_ctas = std::max(1, sms * per_sm);
    CKF(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_points, kPtsThreads, 0));
    ctx->pts_ctas = std::max(1, sms * per_sm);
  }
  CKF(cudaFuncSetAttribute(k_star_sort_big, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kStarCtaSmem));
  CKF(cudaFuncSetAttribute(k_star_refine, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kStarCtaSmem));
  CKF(cudaFuncSetAttribute(k_scatter, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kScatterSmem));
  CKF(cudaFuncSetAttribute(k_scatter, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));   // four CTAs per SM
  CKF(cudaFuncSetAttribute(k_sort_rings<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kRingSmemKeys * sizeof(unsigned long long))));
  CKF(cudaFuncSetAttribute(k_sort_rings<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kRingSmemKeys * sizeof(unsigned long long))));
  CKF(cudaFuncSetAttribute(k_lomuto_rings, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kLomutoSmem));
  urf_default_params(&ctx->params);
  const char* fe = std::getenv("URF_FORCE_EXACT_REGISTRATION");
  narrow_params(&ctx->params, &ctx->dp, ctx->dp.Kfi, fe && fe[0] == '1', 0);
  ctx->last_C = ctx->dp.channels;
  ctx->dp.star_prefix = 1;                                  // near-first star sort (option 4 turns it off)
  ctx->dp.star_pivot = 17;
#undef TRY
#undef CKF
  *out = ctx;
  return URF_OK;
}

void urf_destroy(urf_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  // host batches still in flight copy into the caller's buffers on s_in / s_out: wait for them too
  for (const Stream* s : {&ctx->s_in, &ctx->stream, &ctx->s_out}) if (*s) cudaStreamSynchronize(s->get());
  delete ctx;
}

void* urf_pinned_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  return p;
}
void urf_pinned_free(void* p) { if (p) cudaFreeHost(p); }

int urf_set_params(urf_ctx* ctx, const urf_params* p) {
  if (!ctx || !p || ctx->hs_count) return URF_ERR_INVALID;
  int rc = validate_params(p);
  if (rc != URF_OK) return rc;
  ctx->params = *p;
  narrow_params(p, &ctx->dp, ctx->dp.Kfi, ctx->dp.force_exact, 0);
  ctx->version++;
  return URF_OK;
}

// Nothing between an enqueue and its finish reads ctx->params or ctx->dp: launch_pipeline copies dp into the kernels'
// arguments, the strides of the batch's copies are fixed at the enqueue, and what the finish needs is in its HostSlot. A
// changed set bumps `version`, so the next graphed batch re-captures; that can only be a slot-0 batch, whose previous graph
// launch was finished with slot 0's last batch, so the old executable graph is no longer running when it is replaced.
int urf_set_params_next(urf_ctx* ctx, const urf_params* p) {
  if (!ctx || !p) return URF_ERR_INVALID;
  const int rc = validate_params(p);
  if (rc != URF_OK) return rc;
  ctx->params = *p;
  narrow_params(p, &ctx->dp, ctx->dp.Kfi, ctx->dp.force_exact, 0);
  ctx->version++;
  return ++ctx->gen;
}

int urf_get_params(const urf_ctx* ctx, urf_params* p) {
  if (!ctx || !p) return URF_ERR_INVALID;
  *p = ctx->params;
  return URF_OK;
}

// test/diagnostic options: 0 = force exact ring registration (0/1); 1 = per-kernel CUDA-event timing (slots, 0 = off);
// 2 = number of compute streams a device-resident batch is spread over (1..4); 3 = CUDA graph for small batches (0/1);
// 4 = near-first star sort (0/1, default 1); 10 = near-first pivot rank (3..28 of 32 samples).
// 5, 6, 7, 8, 9, 11 and 12 are retired numbers, accepted and ignored: they selected scheduling and kernel variants
// (sub-batch size, batch graph, shared workspace slots, ring detector and marker search variants, ring detector on the
// pipeline's own stream, star sort network width) that measured no better than the defaults, which are all that is left.
int urf_set_option(urf_ctx* ctx, int option, int value) {
  if (!ctx || ctx->hs_count) return URF_ERR_INVALID;
  CK(cudaSetDevice(ctx->device));
  ctx->version++;
  if (option == 0) { ctx->dp.force_exact = value != 0; ctx->version++; return URF_OK; }
  if (option == 4) { ctx->dp.star_prefix = value != 0; ctx->version++; return URF_OK; }
  if (option == 3) { ctx->use_graph = value != 0; return URF_OK; }
  if (option == 2) { ctx->groups = value < 1 ? 1 : (value > urf_ctx::kGroups ? urf_ctx::kGroups : value); return URF_OK; }
  if ((option >= 5 && option <= 9) || option == 11 || option == 12) return URF_OK;
  if (option == 10) { ctx->dp.star_pivot = value < 3 ? 3 : (value > 28 ? 28 : value); return URF_OK; }
  if (option == 1) {                   // value = number of event slots (0 = off)
    CK(cudaStreamSynchronize(ctx->stream.get()));         // events of the previous setting may still be pending
    if (ctx->gexec) { ctx->gexec.reset(); ctx->g_B = -1; }
    ctx->kev.clear();
    ctx->profile = value > 0;
    ctx->kslots = value > 0 ? value : 1;
    ctx->kslot = 0;
    if (ctx->profile) {
      ctx->kev.resize((size_t)ctx->kslots * (kMaxKernels + 1));
      for (Event& e : ctx->kev) {
        const cudaError_t ce = new_event(e, cudaEventDefault);
        if (ce != cudaSuccess) {                           // leave the option off
          ctx->kev.clear(); ctx->profile = false; ctx->kslots = 1;
          ctx->err = std::string("cudaEventCreate: ") + cudaGetErrorString(ce);
          return URF_ERR_CUDA;
        }
      }
      ctx->knames.assign(kMaxKernels, "");
      ctx->kcounts.assign(ctx->kslots, 0);
    }
    return URF_OK;
  }
  return URF_ERR_INVALID;
}

int urf_set_tie_order(urf_ctx* ctx, int mode) {
  if (!ctx || ctx->hs_count || (mode != URF_TIES_INPUT_ORDER && mode != URF_TIES_REFERENCE)) return URF_ERR_INVALID;
  CK(cudaSetDevice(ctx->device));
  if (mode == URF_TIES_REFERENCE && !ctx->buf.lomuto) {   // 4 bytes per point of capacity plus one ring list per scan
    DevBuffers d{};
    ArrayMem mem;                                          // freed on a failure
    if (const int rc = alloc_owned(ctx, d, mem, tie_order_array); rc != URF_OK) return rc;
    adopt(ctx->buf, ctx->mem, d, mem);
  }
  ctx->tie_order = mode;
  ctx->version++;                                          // the captured graph holds the other launch sequence
  return URF_OK;
}

int urf_get_tie_order(const urf_ctx* ctx, int* mode) {
  if (!ctx || !mode) return URF_ERR_INVALID;
  *mode = ctx->tie_order;
  return URF_OK;
}

int urf_mq_set_tie_order(urf_mq* mq, int mode) {
  if (!mq || (mode != URF_TIES_INPUT_ORDER && mode != URF_TIES_REFERENCE)) return URF_ERR_INVALID;
  return urf_internal::mq_apply_idle(mq, [](urf_ctx* c, const void* m) { return urf_set_tie_order(c, *static_cast<const int*>(m)); }, &mode);
}

void* urf_stream(urf_ctx* ctx) { return ctx ? (void*)ctx->stream.get() : nullptr; }

float urf_last_device_ms(const urf_ctx* c) {
  urf_ctx* ctx = const_cast<urf_ctx*>(c);
  if (!ctx || !ctx->timing_valid) return -1.f;
  if (ctx->timing_host) return ctx->last_ms;
  float ms = -1.f;
  if (cudaEventSynchronize(ctx->ev1.get()) != cudaSuccess) return -1.f;
  if (cudaEventElapsedTime(&ms, ctx->ev0.get(), ctx->ev1.get()) != cudaSuccess) return -1.f;
  return ms;
}

int urf_last_launch_count(const urf_ctx* ctx) { return ctx ? ctx->launches : 0; }

// With option 1 on: number of kernels of the last call, and name / device milliseconds of kernel `idx` (event before it to
// the event before the next kernel, or to the end-of-pipeline event for the last one). Waits for the stream.
int urf_profile_count(const urf_ctx* ctx) { return ctx && ctx->profile ? ctx->kcounts[0] : 0; }
int urf_profile_slots(const urf_ctx* ctx) { return ctx && ctx->profile ? ctx->kslots : 0; }
// name / device milliseconds of kernel `idx` in event slot `slot` (the slot's calls must have completed)
int urf_profile_get(urf_ctx* ctx, int slot, int idx, const char** name, float* ms) {
  if (!ctx || !ctx->profile || slot < 0 || slot >= ctx->kslots || idx < 0 || idx >= ctx->kcounts[slot]) return URF_ERR_INVALID;
  const size_t o = (size_t)slot * (kMaxKernels + 1);
  cudaEvent_t next = (idx + 1 < ctx->kcounts[slot] ? ctx->kev[o + idx + 1] : ctx->kev[o + kMaxKernels]).get();
  CK(cudaEventSynchronize(next));
  CK(cudaEventElapsedTime(ms, ctx->kev[o + idx].get(), next));
  if (name) *name = ctx->knames[idx];
  return URF_OK;
}

int urf_enqueue_batch_device_ex(urf_ctx* ctx, const float* d_xyzi, int stride_points, const int* n, int batch, int32_t* d_label,
                                int32_t* d_order) {
  if (!ctx || ctx->hs_count || !d_xyzi || !n || !d_label || batch < 1 || stride_points < 1) return URF_ERR_INVALID;
  if (batch > ctx->max_batch || (size_t)stride_points * batch > ctx->P || stride_points > ctx->max_points) return URF_ERR_CAPACITY;
  CK(cudaSetDevice(ctx->device));
  for (int b = 0; b < batch; b++) if (n[b] < 0 || n[b] > stride_points) return URF_ERR_INVALID;
  int* row = ctx->h_nring.get() + (size_t)ctx->nring_pos * ctx->max_batch;
  CK(cudaEventSynchronize(ctx->ev_nring[ctx->nring_pos].get()));   // the copy that last used this row (kNRing enqueues ago) is done
  std::memcpy(row, n, sizeof(int) * batch);
  CK(cudaMemcpyAsync(ctx->buf.n, row, sizeof(int) * batch, cudaMemcpyHostToDevice, ctx->stream.get()));
  CK(cudaEventRecord(ctx->ev_nring[ctx->nring_pos].get(), ctx->stream.get()));
  ctx->nring_pos = (ctx->nring_pos + 1) % urf_ctx::kNRing;
  const bool want_order = d_order != nullptr;
  DevBuffers bufv = ctx->buf;                                 // the caller's buffers instead of the context's own
  bufv.in = reinterpret_cast<float4*>(const_cast<float*>(d_xyzi));
  bufv.label = d_label;
  if (want_order) bufv.order = d_order;
  const int G = (ctx->profile || batch < 2 * ctx->groups) ? 1 : ctx->groups;   // per-kernel event timing needs one stream
  int launches = 0;
  CK(cudaEventRecord(ctx->ev0.get(), ctx->stream.get()));
  if (G == 1) {
    const int rc = launch_pipeline(ctx, bufv, batch, stride_points, want_order, ctx->lane[urf_ctx::kGroups], &launches);
    if (rc != URF_OK) return rc;
  } else {
    // fork: the ctx stream hands one of G near-equal sub-batches (group_bounds) to each lane and joins them again, so
    // callers still see ONE stream. Scans are independent.
    CK(cudaEventRecord(ctx->ev_fork.get(), ctx->stream.get()));
    for (int g = 0; g < G; g++) CK(cudaStreamWaitEvent(ctx->lane[g].st, ctx->ev_fork.get(), 0));
    const Extent e = launch_extent(stride_points, ctx->dp.channels);
    for (int g = 0; g < G; g++) {
      int b0, b1, L = 0;
      group_bounds(g, G, batch, &b0, &b1);
      const int rc = launch_pipeline(ctx, scan_view(bufv, b0, e), b1 - b0, stride_points, want_order, ctx->lane[g], &L);
      if (rc != URF_OK) return rc;
      launches += L;
    }
    for (int g = 0; g < G; g++) {
      CK(cudaEventRecord(ctx->lane[g].join.get(), ctx->lane[g].st));
      CK(cudaStreamWaitEvent(ctx->stream.get(), ctx->lane[g].join.get(), 0));
    }
  }
  CK(cudaEventRecord(ctx->ev1.get(), ctx->stream.get()));
  ctx->launches = launches;
  ctx->timing_valid = true;
  ctx->timing_host = false;
  ctx->last_B = batch; ctx->last_S = stride_points; ctx->last_C = ctx->dp.channels;
  ctx->dev_gen = ctx->gen;
  return URF_OK;
}

int urf_enqueue_batch_device(urf_ctx* ctx, const float* d_xyzi, int stride_points, const int* n, int batch, int32_t* d_label) {
  return urf_enqueue_batch_device_ex(ctx, d_xyzi, stride_points, n, batch, d_label, nullptr);
}

int urf_finish_batch_device(urf_ctx* ctx, urf_result* outs) {
  if (!ctx || ctx->hs_count) return URF_ERR_INVALID;
  CK(cudaSetDevice(ctx->device));
  const int B = ctx->last_B;
  ScanOut* h_out = ctx->hs[0].h_out.get();
  if (outs) CK(cudaMemcpyAsync(h_out, ctx->buf.out, sizeof(ScanOut) * B, cudaMemcpyDeviceToHost, ctx->stream.get()));
  CK(cudaStreamSynchronize(ctx->stream.get()));
  if (outs) for (int b = 0; b < B; b++) fill_result(h_out[b], &outs[b], false, ctx->dev_gen);
  return URF_OK;
}

int urf_process_batch_device(urf_ctx* ctx, const float* d_xyzi, int stride_points, const int* n, int batch,
                             int32_t* d_label, urf_result* outs) {
  int rc = urf_enqueue_batch_device(ctx, d_xyzi, stride_points, n, batch, d_label);
  if (rc != URF_OK) return rc;
  return urf_finish_batch_device(ctx, outs);
}

namespace {
// Shared body of the host-buffer batch entry points. step == 0: data[b] holds n[b] (x, y, z, intensity) float4 records that
// are copied straight into the input buffer; step > 0: data[b] holds n[b] records of `step` bytes with FLOAT32 x / y / z /
// intensity at the given byte offsets (oi < 0: none) — the raw bytes cross PCIe and are unpacked on the device.
// fmt (or NULL): scan b's records have the format fmt[b] instead (step and the offsets are then ignored); a batch whose
// formats are all equal runs as the one-format call.
// label8 (or NULL): per scan an int8 HOST buffer for the labels (one byte per point instead of four).
// clouds (or NULL, batch == 1 only): the four published clouds of the scan, packed on the device.
// Enqueues the batch into the next free host slot and returns; finish_batch waits for it and fills outs.
int enqueue_batch(urf_ctx* ctx, const void* const* data, const int* n, int batch, int step, int ox, int oy, int oz, int oi,
                  const urf_cloud2_format* fmt, urf_result* outs, int8_t* const* label8, urf_clouds* clouds) {
  if (!ctx || !data || !n || !outs || batch < 1) return URF_ERR_INVALID;
  if (batch > ctx->max_batch || ctx->hs_count == 2) return URF_ERR_CAPACITY;
  if (fmt) {                                                  // step becomes the batch's largest point_step
    bool mixed = false;
    step = 0;
    for (int b = 0; b < batch; b++) {
      if (urf::check_cloud2_format(fmt[b]) != URF_OK) return URF_ERR_INVALID;
      step = std::max(step, (int)fmt[b].point_step);
      mixed |= std::memcmp(&fmt[b], &fmt[0], sizeof(urf_cloud2_format)) != 0;
    }
    ox = fmt[0].off_x; oy = fmt[0].off_y; oz = fmt[0].off_z; oi = fmt[0].off_intensity;
    if (!mixed) fmt = nullptr;
  } else if (step != 0 && urf::check_cloud2_format(step, ox, oy, oz, oi) != URF_OK) {
    return URF_ERR_INVALID;
  }
  CK(cudaSetDevice(ctx->device));
  const int slot = (ctx->hs_head + ctx->hs_count) % 2;
  urf_ctx::HostSlot& h = ctx->hs[slot];                       // free: its last batch was finished, its copies are done
  if (fmt && !h.fmt) {                                        // the slot's first mixed batch: its format tables
    DevMem<urf_cloud2_format> d;
    HostMem<urf_cloud2_format> hf;
    int rc = dalloc(ctx, d, (size_t)ctx->max_batch);
    if (rc == URF_OK) rc = cuda_rc(ctx, new_pinned(hf, (size_t)ctx->max_batch), "cudaMallocHost");
    if (rc != URF_OK) return rc;
    h.fmt = std::move(d); h.h_fmt = std::move(hf);
  }
  if (fmt) std::memcpy(h.h_fmt.get(), fmt, sizeof(urf_cloud2_format) * (size_t)batch);
  int nmax = 1;
  bool want_order = clouds != nullptr, want_ring = false, want_l8 = false;
  for (int b = 0; b < batch; b++) {
    if (n[b] < 0 || (n[b] > 0 && !data[b])) return URF_ERR_INVALID;
    if (n[b] > ctx->max_points) return URF_ERR_CAPACITY;
    nmax = n[b] > nmax ? n[b] : nmax;
    want_order |= outs[b].order != nullptr;
    want_ring |= outs[b].ring != nullptr;
    want_l8 |= label8 && label8[b];
    h.h_n.get()[b] = n[b];
  }
  const int S = ((nmax + 255) / 256) * 256;
  const Extent cap = capacity_extent(ctx->max_points), e = launch_extent(S, ctx->dp.channels);
  const size_t pts = slice_elems(Kind::Point, e);             // per scan: points of the input, ring ids, record staging
  if ((size_t)batch * S * step > h.rawb_bytes) {              // records of a batch beyond the staging buffer: P * step bytes
    CK(cudaStreamSynchronize(ctx->stream.get()));
    h.rawb.reset(); h.rawb_bytes = 0;                         // the old buffer goes first
    const size_t bytes = capacity_elems(Kind::Point, cap, ctx->max_batch) * step;
    if (const int rc = dalloc(ctx, h.rawb, bytes); rc != URF_OK) return rc;
    h.rawb_bytes = bytes;
  }
  if (want_l8 && !h.dev.label8)
    if (const int rc = alloc_owned(ctx, h.dev, h.mem, label8_array); rc != URF_OK) return rc;
  if (clouds && !ctx->pack) {                                  // first packed call: 96 bytes per point of capacity
    const int tiles = (std::max(ctx->max_points, 1) + kPackTile - 1) / kPackTile;
    DevMem<float4> pack;                                       // all or nothing: freed on a failure
    DevMem<int> packcnt, packtot; HostMem<int> h_packtot;
    int rc = dalloc(ctx, pack, (size_t)6 * ctx->max_points);
    if (rc == URF_OK) rc = dalloc(ctx, packcnt, (size_t)3 * tiles);
    if (rc == URF_OK) rc = dalloc(ctx, packtot, 4);
    if (rc == URF_OK) rc = cuda_rc(ctx, new_pinned(h_packtot, 4), "cudaMallocHost");
    if (rc != URF_OK) return rc;
    ctx->pack = std::move(pack); ctx->packcnt = std::move(packcnt); ctx->packtot = std::move(packtot); ctx->h_packtot = std::move(h_packtot);
  }
  cudaStream_t st = ctx->stream.get();
  DevBuffers bufv = slot_view(ctx->buf, h.dev);               // slot 0: the same pointers as ctx->buf
  if (!want_l8) bufv.label8 = nullptr;
  // Software pipeline over chunks of scans: H2D of chunk c+1 (s_in), kernels of chunk c (stream) and D2H of chunk c-1
  // (s_out) overlap; scans are independent, every chunk owns its slice of every buffer.
  // Chunks of batch / 16 scans. (Tried and dropped: smaller chunks at both ends of the call — a shorter pipeline fill and
  // drain on paper, slower in practice — and copies running only three chunks ahead of the launches.)
  std::vector<int> cb;                                        // chunk c = scans [cb[c], cb[c + 1])
  for (int b0 = 0, chunk = host_chunk(batch); b0 < batch; b0 += chunk) cb.push_back(b0);
  cb.push_back(batch);
  const int nchunks = (int)cb.size() - 1;
  for (int c = (int)ctx->ev_in.size(); c < nchunks; c++) {
    Event in, comp;
    CK(new_event(in)); CK(new_event(comp));
    ctx->ev_in.push_back(std::move(in)); ctx->ev_comp.push_back(std::move(comp));
  }
  // ring ids of chunk c: until the first asynchronous call, slot 0 writes them into the chunk's private slice of the sort
  // scratch (16 bytes per point), free once the chunk's sorts are done; from then on every slot has a buffer of its own,
  // because the next batch's sorts overwrite the scratch while this batch's ring ids are still being copied out
  const bool ring_in_scratch = !h.ring;
  auto ring_chunk = [&](const DevBuffers& v, int b0) { return ring_in_scratch ? reinterpret_cast<int*>(v.sortbuf) : h.ring.get() + b0 * pts; };
  // the graph holds ctx->buf's pointers, which are slot 0's
  const bool graphed = slot == 0 && nchunks == 1 && batch <= 8 && !want_l8 && ctx->use_graph && !ctx->profile;
  if (graphed) {
    const int rc = update_graph(ctx, batch, S, want_order);
    if (rc != URF_OK) return rc;
  }
  // every host-to-device copy of the call is queued first (the copies depend on nothing): the copy engine then never waits
  // for this thread to get through a chunk's kernel launches and result copies
  for (int c = 0; c < nchunks; c++) {
    const int b0 = cb[c], nb = cb[c + 1] - b0;
    CK(cudaMemcpyAsync(scan_view(bufv, b0, e).n, h.h_n.get() + b0, sizeof(int) * nb, cudaMemcpyHostToDevice, ctx->s_in.get()));
    if (fmt) CK(cudaMemcpyAsync(h.fmt.get() + b0, h.h_fmt.get() + b0, sizeof(urf_cloud2_format) * nb, cudaMemcpyHostToDevice, ctx->s_in.get()));
    for (int b = b0; b < b0 + nb; b++) {
      if (n[b] <= 0) continue;
      const size_t bytes = (size_t)(fmt ? fmt[b].point_step : step) * (size_t)n[b];
      if (step == 0) CK(cudaMemcpyAsync(scan_view(bufv, b, e).in, data[b], sizeof(float) * 4 * (size_t)n[b], cudaMemcpyHostToDevice, ctx->s_in.get()));
      else CK(cudaMemcpyAsync(h.rawb.get() + b * pts * step, data[b], bytes, cudaMemcpyHostToDevice, ctx->s_in.get()));
    }
    CK(cudaEventRecord(ctx->ev_in[c].get(), ctx->s_in.get()));
  }
  int launches = 0;
  for (int c = 0; c < nchunks; c++) {
    const int b0 = cb[c], nb = cb[c + 1] - b0;
    CK(cudaStreamWaitEvent(st, ctx->ev_in[c].get(), 0));
    const DevBuffers view = scan_view(bufv, b0, e);
    if (step != 0)
      k_unpack_cloud2_batch<<<dim3((S + 255) / 256, nb), 256, 0, st>>>(h.rawb.get() + b0 * pts * step, view.in, view.n, S, step,
                                                                        urf_cloud2_format{step, ox, oy, oz, oi}, fmt ? h.fmt.get() + b0 : nullptr);
    // ev0 / ev1 bracket the kernels of the whole call: before the first chunk's pipeline, after the last one's
    int L = graphed ? ctx->g_launches : 0;
    int rc = c == 0 ? cuda_rc(ctx, cudaEventRecord(h.ev0.get(), st), "cudaEventRecord(ev0)") : URF_OK;
    if (rc == URF_OK)
      rc = graphed ? cuda_rc(ctx, cudaGraphLaunch(ctx->gexec.get(), st), "cudaGraphLaunch")
                   : launch_pipeline(ctx, view, nb, S, want_order, ctx->lane[urf_ctx::kGroups], &L);
    if (rc == URF_OK && c == nchunks - 1) rc = cuda_rc(ctx, cudaEventRecord(h.ev1.get(), st), "cudaEventRecord(ev1)");
    if (rc != URF_OK) {                                 // nothing of this call may still be writing into the caller's buffers
      cudaStreamSynchronize(ctx->s_in.get()); cudaStreamSynchronize(st); cudaStreamSynchronize(ctx->s_out.get());
      return rc;
    }
    launches += L;
    if (want_ring) k_ring32<<<dim3((S + 255) / 256, nb), 256, 0, st>>>(view, ring_chunk(view, b0), S);
    if (clouds) {                                       // batch == 1: pack scan 0, sizes to the host with the results
      const int nt = (std::max(n[0], 1) + kPackTile - 1) / kPackTile;
      float4* pack = ctx->pack.get();
      k_pack_count<<<nt, 256, 0, st>>>(ctx->buf, ctx->packcnt.get(), nt);
      k_pack_scan<<<1, 1024, 0, st>>>(ctx->buf, ctx->packcnt.get(), nt, ctx->packtot.get());
      k_pack_write<<<nt, 256, 0, st>>>(ctx->buf, ctx->packcnt.get(), nt, ctx->packtot.get(), pack, pack + 2 * (size_t)ctx->max_points,
                                       pack + 4 * (size_t)ctx->max_points);
      launches += 3;
      CK(cudaMemcpyAsync(ctx->h_packtot.get(), ctx->packtot.get(), sizeof(int) * 4, cudaMemcpyDeviceToHost, st));
    }
    cudaStream_t so = ctx->s_out.get();
    CK(cudaEventRecord(ctx->ev_comp[c].get(), st));
    CK(cudaStreamWaitEvent(so, ctx->ev_comp[c].get(), 0));
    CK(cudaMemcpyAsync(h.h_out.get() + b0, view.out, sizeof(ScanOut) * nb, cudaMemcpyDeviceToHost, so));
    for (int b = b0; b < b0 + nb; b++) {
      if (n[b] <= 0) continue;
      const DevBuffers v = scan_view(bufv, b, e);
      if (outs[b].label) CK(cudaMemcpyAsync(outs[b].label, v.label, sizeof(int) * (size_t)n[b], cudaMemcpyDeviceToHost, so));
      if (label8 && label8[b]) CK(cudaMemcpyAsync(label8[b], v.label8, (size_t)n[b], cudaMemcpyDeviceToHost, so));
      if (outs[b].ring) CK(cudaMemcpyAsync(outs[b].ring, ring_chunk(view, b0) + (b - b0) * pts, sizeof(int) * (size_t)n[b], cudaMemcpyDeviceToHost, so));
      if (outs[b].order) CK(cudaMemcpyAsync(outs[b].order, v.order, sizeof(int) * (size_t)n[b], cudaMemcpyDeviceToHost, so));
    }
  }
  // s_out waited for the last chunk's kernels: ev_done covers every copy and kernel of the batch
  CK(cudaEventRecord(h.ev_done.get(), ctx->s_out.get()));
  h.batch = batch; h.S = S; h.launches = launches; h.outs = outs; h.clouds = clouds;
  h.C = ctx->dp.channels; h.gen = ctx->gen;
  ctx->hs_count++;
  return URF_OK;
}

// Waits for the oldest host batch in flight and fills its outs (the slot is free again whatever the outcome).
int finish_batch(urf_ctx* ctx) {
  if (!ctx || ctx->hs_count == 0) return URF_ERR_INVALID;
  urf_ctx::HostSlot& h = ctx->hs[ctx->hs_head];
  ctx->hs_count--;
  ctx->hs_head = ctx->hs_count ? 1 - ctx->hs_head : 0;       // idle: the next batch (and every synchronous call) takes slot 0
  CK(cudaSetDevice(ctx->device));
  CK(cudaEventSynchronize(h.ev_done.get()));
  cudaStream_t st = ctx->stream.get();
  urf_clouds* clouds = h.clouds;
  if (clouds) {                                              // sizes are known now: copy exactly the records that exist
    const int* t = ctx->h_packtot.get();
    const float4* d_rc = ctx->pack.get();
    const float4 *d_roi = d_rc + 2 * (size_t)ctx->max_points, *d_prob = d_rc + 4 * (size_t)ctx->max_points;
    clouds->n_road = t[0]; clouds->n_curb = t[1]; clouds->n_roi = t[2]; clouds->n_road_probably = t[3];
    const size_t rec = sizeof(urf_point_xyzi);
    if (clouds->road && t[0] > 0) CK(cudaMemcpyAsync(clouds->road, d_rc, rec * t[0], cudaMemcpyDeviceToHost, st));
    if (clouds->curb && t[1] > 0) CK(cudaMemcpyAsync(clouds->curb, d_rc + 2 * (size_t)t[0], rec * t[1], cudaMemcpyDeviceToHost, st));
    if (clouds->roi && t[2] > 0) CK(cudaMemcpyAsync(clouds->roi, d_roi, rec * t[2], cudaMemcpyDeviceToHost, st));
    if (clouds->road_probably && t[3] > 0) CK(cudaMemcpyAsync(clouds->road_probably, d_prob, rec * t[3], cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  float ms = -1.f;
  if (cudaEventElapsedTime(&ms, h.ev0.get(), h.ev1.get()) != cudaSuccess) ms = -1.f;
  ctx->last_ms = ms;
  ctx->launches = h.launches;
  ctx->timing_valid = true;
  ctx->timing_host = true;
  ctx->last_B = h.batch; ctx->last_S = h.S; ctx->last_C = h.C;
  urf_result* outs = h.outs;
  for (int b = 0; b < h.batch; b++) {
    fill_result(h.h_out.get()[b], &outs[b], true, h.gen);
    if (outs[b].status == URF_TOO_FEW_POINTS && outs[b].ring) for (int i = 0; i < h.h_n.get()[b]; i++) outs[b].ring[i] = -1;
  }
  return URF_OK;
}

// The second host slot, and slot 0's own ring-id buffer (include/urf.h: 32 bytes of device memory per point of capacity),
// on the first asynchronous call (nothing is in flight then).
int alloc_second_slot(urf_ctx* ctx) {
  if (ctx->hs[1].ev_done) return URF_OK;
  CK(cudaSetDevice(ctx->device));
  const size_t P = capacity_elems(Kind::Point, capacity_extent(ctx->max_points), ctx->max_batch);
  urf_ctx::HostSlot t;                                      // all or nothing: freed on a failure
  DevMem<int> ring0;
  int rc = alloc_owned(ctx, t.dev, t.mem, slot_array);
  if (rc == URF_OK) rc = dalloc(ctx, t.ring, P);
  if (rc == URF_OK) rc = dalloc(ctx, ring0, P);
  if (rc == URF_OK) rc = cuda_rc(ctx, init_slot(ctx, t), "pinned rows and events of host slot 1");   // ev_done marks it complete
  if (rc != URF_OK) return rc;
  ctx->hs[1] = std::move(t);
  ctx->hs[0].ring = std::move(ring0);
  return URF_OK;
}

// The synchronous entry points: one enqueue and one finish, refused while asynchronous batches are in flight.
int process_batch_impl(urf_ctx* ctx, const void* const* data, const int* n, int batch, int step, int ox, int oy, int oz, int oi,
                       const urf_cloud2_format* fmt, urf_result* outs, int8_t* const* label8, urf_clouds* clouds) {
  if (ctx && ctx->hs_count) return URF_ERR_INVALID;
  const int rc = enqueue_batch(ctx, data, n, batch, step, ox, oy, oz, oi, fmt, outs, label8, clouds);
  return rc != URF_OK ? rc : finish_batch(ctx);
}

int enqueue_async(urf_ctx* ctx, const void* const* data, const int* n, int batch, int step, int ox, int oy, int oz, int oi,
                  const urf_cloud2_format* fmt, urf_result* outs, int8_t* const* label8) {
  if (!ctx) return URF_ERR_INVALID;
  const int rc = alloc_second_slot(ctx);
  return rc != URF_OK ? rc : enqueue_batch(ctx, data, n, batch, step, ox, oy, oz, oi, fmt, outs, label8, nullptr);
}
}  // namespace

int urf_enqueue_batch(urf_ctx* ctx, const float* const* xyzi, const int* n, int batch, urf_result* outs, int8_t* const* label8) {
  return enqueue_async(ctx, reinterpret_cast<const void* const*>(xyzi), n, batch, 0, 0, 0, 0, -1, nullptr, outs, label8);
}

int urf_enqueue_cloud2_batch(urf_ctx* ctx, const void* const* data, const int* n_points, int batch, int point_step, int off_x, int off_y,
                             int off_z, int off_intensity, urf_result* outs, int8_t* const* label8) {
  if (point_step == 0) return URF_ERR_INVALID;
  return enqueue_async(ctx, data, n_points, batch, point_step, off_x, off_y, off_z, off_intensity, nullptr, outs, label8);
}

// the mixed entry points take their step and offsets from fmt; a batch of one format runs as the one-format call
int urf_enqueue_cloud2_batch_mixed(urf_ctx* ctx, const void* const* data, const int* n_points, const urf_cloud2_format* fmt, int batch,
                                   urf_result* outs, int8_t* const* label8) {
  if (!fmt) return URF_ERR_INVALID;
  return enqueue_async(ctx, data, n_points, batch, 0, 0, 0, 0, -1, fmt, outs, label8);
}

int urf_process_cloud2_batch_mixed(urf_ctx* ctx, const void* const* data, const int* n_points, const urf_cloud2_format* fmt, int batch,
                                   urf_result* outs, int8_t* const* label8) {
  if (!fmt) return URF_ERR_INVALID;
  return process_batch_impl(ctx, data, n_points, batch, 0, 0, 0, 0, -1, fmt, outs, label8, nullptr);
}

int urf_finish_batch(urf_ctx* ctx) { return finish_batch(ctx); }

int urf_process_batch(urf_ctx* ctx, const float* const* xyzi, const int* n, int batch, urf_result* outs) {
  return process_batch_impl(ctx, reinterpret_cast<const void* const*>(xyzi), n, batch, 0, 0, 0, 0, -1, nullptr, outs, nullptr, nullptr);
}

int urf_process_batch_xyz(urf_ctx* ctx, const float* const* xyz, const int* n, int batch, urf_result* outs, int8_t* const* label8) {
  return process_batch_impl(ctx, reinterpret_cast<const void* const*>(xyz), n, batch, 12, 0, 4, 8, -1, nullptr, outs, label8, nullptr);
}

// the record entry points reject point_step 0 themselves: the body reads step 0 as float4 input
int urf_process_cloud2_batch(urf_ctx* ctx, const void* const* data, const int* n_points, int batch, int point_step, int off_x, int off_y,
                             int off_z, int off_intensity, urf_result* outs, int8_t* const* label8) {
  if (point_step == 0) return URF_ERR_INVALID;
  return process_batch_impl(ctx, data, n_points, batch, point_step, off_x, off_y, off_z, off_intensity, nullptr, outs, label8, nullptr);
}

int urf_process_cloud2(urf_ctx* ctx, const void* data, int n, int point_step, int off_x, int off_y, int off_z, urf_result* out) {
  if (point_step == 0) return URF_ERR_INVALID;
  return process_batch_impl(ctx, &data, &n, 1, point_step, off_x, off_y, off_z, -1, nullptr, out, nullptr, nullptr);
}

int urf_process_cloud2_packed(urf_ctx* ctx, const void* data, int n, int point_step, int off_x, int off_y, int off_z,
                              int off_intensity, urf_result* out, urf_clouds* clouds) {
  if (!clouds || point_step == 0) return URF_ERR_INVALID;
  return process_batch_impl(ctx, &data, &n, 1, point_step, off_x, off_y, off_z, off_intensity, nullptr, out, nullptr, clouds);
}

int urf_process(urf_ctx* ctx, const float* xyzi, int n, urf_result* out) {
  const float* ptrs[1] = {xyzi};
  return urf_process_batch(ctx, ptrs, &n, 1, out);
}

// ---- test hooks (not part of the reference-facing surface) ------------------------------------------------------------
// Evaluate the device build of the emulated libm: which = 0 asinf(a), 1 acosf(a), 2 atan2f(a, b), 3 atanf(a).
int urf_test_math(int device, int which, const float* a, const float* b, float* out, int n) {
  if (cudaSetDevice(device) != cudaSuccess) return URF_ERR_NO_DEVICE;
  float *da = nullptr, *db = nullptr, *dout = nullptr;
  if (cudaMalloc(&da, sizeof(float) * n) != cudaSuccess || cudaMalloc(&db, sizeof(float) * n) != cudaSuccess ||
      cudaMalloc(&dout, sizeof(float) * n) != cudaSuccess)
    return URF_ERR_NOMEM;
  cudaMemcpy(da, a, sizeof(float) * n, cudaMemcpyHostToDevice);
  cudaMemcpy(db, b ? b : a, sizeof(float) * n, cudaMemcpyHostToDevice);
  k_test_math<<<(n + 255) / 256, 256>>>(da, db, dout, n, which);
  cudaError_t e = cudaMemcpy(out, dout, sizeof(float) * n, cudaMemcpyDeviceToHost);
  cudaFree(da); cudaFree(db); cudaFree(dout);
  return e == cudaSuccess ? URF_OK : URF_ERR_CUDA;
}

// Copy a device-side intermediate of scan `b` of the last call into host memory (stage-level differential tests).
//   what: 0 alpha_v[f32,n]  1 mark[u8,n] (all detectors)  2 ringid[i16,n]  3 sect[i16,n]  4 az[f32,n]  5 d2[f32,n]
//         (4, 5: defined for ROI points only)  8 ScanTab (raw)  9 star sort work lists [i32,2]: sectors handed to the
//         eight-warp sort (nbig) and to the exact fallback (nslow)  10 sectors completed by k_star_refine [i32,1]
//         (nrefine: their edge search ran off the near-first prefix)  11 Tf, 12 Tb: the blindSpots threshold tables as
//         k_tab2 left them [f32, kDegBins * channels], degree-major (entry (j, k) at j * channels + k; rows k >= n_rings
//         are not written)  13 firstidx [u32, kElevBins + 1]: the smallest ROI input index per fine elevation bin as
//         k_points left it (0xffffffff = empty bin)
int urf_debug_fetch(urf_ctx* ctx, int b, int what, void* dst, size_t bytes) {
  if (!ctx || !dst || b < 0 || b >= ctx->last_B) return URF_ERR_INVALID;
  CK(cudaSetDevice(ctx->device));
  CK(cudaStreamSynchronize(ctx->stream.get()));
  const DevBuffers v = scan_view(ctx->buf, b, launch_extent(ctx->last_S, ctx->last_C));
  const void* src = nullptr;
  auto clamp = [&](size_t most) { if (bytes > most) bytes = most; };
  switch (what) {
    case 0: src = v.alpha_v; break;  case 1: src = v.mark; break;  case 2: src = v.ringid; break;
    case 3: src = v.sect; break;     case 4: src = v.az; break;    case 5: src = v.d2; break;
    case 8: src = v.tab; clamp(sizeof(ScanTab)); break;
    case 9: src = &v.tab->nbig; clamp(2 * sizeof(int)); break;
    case 10: src = &v.tab->nrefine; clamp(sizeof(int)); break;
    case 11: case 12: src = what == 11 ? v.Tf : v.Tb; clamp(sizeof(float) * ctx->last_C * kDegBins); break;
    case 13: src = v.firstidx; clamp(sizeof(unsigned) * kElevSlice); break;
    default: return URF_ERR_INVALID;
  }
  CK(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
  return URF_OK;
}

size_t urf_debug_sizeof_tab(void) { return sizeof(ScanTab); }

}  // extern "C"
