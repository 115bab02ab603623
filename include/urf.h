/*
 * urf.h — C-ABI of liburf_b200.so: the H100-native (sm_90a) replacement for the per-scan road/curb classification path of
 * jkk-research/urban_road_filter.
 *
 * Reference interface replaced (all paths relative to the reference repo root):
 *   - void Detector::filtered(const pcl::PointCloud<pcl::PointXYZI>&)      include/urban_road_filter/data_structures.hpp:118,
 *     defined src/lidar_segmentation.cpp:95-622 (hot path = :95-367; marker tail = :369-602)      -> urf_process / urf_process_batch
 *   - void paramsCallback(LidarFiltersConfig&, uint32_t)  src/main.cpp:4-34 (fields cfg/LidarFilters.cfg:10-84) -> urf_set_params
 *   - Detector::Detector / Detector::beam_init            src/lidar_segmentation.cpp:51-65, src/star_shaped_search.cpp:32-66 -> urf_create
 *   - the five publishers (road, curb, roi, road_probably, road_marker) src/lidar_segmentation.cpp:55-59,601,618-621
 *     -> urf_result (labels + emission order + marker vertices) and urf_build_markers (line strips)
 *
 * Plain C: pointers and sizes only, no C++/torch types. One urf_ctx owns one CUDA device, one stream and all device and
 * pinned staging memory (allocated in urf_create, never in urf_process*). A ctx is not thread-safe; use one per thread.
 * There is NO CPU fallback: every entry point that computes fails with URF_ERR_CUDA / URF_ERR_NO_DEVICE without a GPU.
 */
#ifndef URF_H_
#define URF_H_

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define URF_VERSION 100
#define URF_MAX_VERTS 361        /* one candidate vertex per 1-degree bin 0..360, lidar_segmentation.cpp:305 */
#define URF_STAR_SECTORS 360     /* `rep`, star_shaped_search.cpp:8 */
#define URF_MAX_CHANNELS 256     /* upper bound accepted for urf_params.channels */

/* status / error codes (the reference has none: it is `void` and silently returns, lidar_segmentation.cpp:124-126) */
enum {
  URF_OK = 0,
  URF_TOO_FEW_POINTS = 1,        /* fewer than 30 points in the ROI: the reference publishes nothing for this scan */
  URF_ERR_INVALID = -1,          /* bad argument (NULL, n > max_points, batch > max_batch, bad param range) */
  URF_ERR_NO_DEVICE = -2,        /* no CUDA device / device index out of range */
  URF_ERR_CUDA = -3,             /* a CUDA call failed; urf_last_cuda_error() has the text */
  URF_ERR_NOMEM = -4,            /* device or pinned allocation failed */
  URF_ERR_CAPACITY = -5          /* scan larger than the ctx was created for */
};

/* Label encoding = `short isCurbPoint` of the reference (data_structures.hpp:44) plus -1 for "not in the ROI cloud". */
enum { URF_LABEL_OUTSIDE = -1, URF_LABEL_NONE = 0, URF_LABEL_ROAD = 1, URF_LABEL_CURB = 2 };

/*
 * The 27 dynamic_reconfigure parameters, same names, types and defaults as cfg/LidarFilters.cfg:10-84
 * (double_t -> double, int_t -> int, bool_t -> int 0/1, str_t -> char[]). Like src/main.cpp:12-32 the library narrows
 * every double to float when it is applied. `channels` is the reference's global `int channels = 64`
 * (src/lidar_segmentation.cpp:4), exposed because 128/256-ring sensors need it.
 */
typedef struct urf_params {
  char   fixed_frame[128];       /* glue only */
  char   topic_name[128];        /* glue only */
  int    x_zero_method;
  int    z_zero_method;
  int    star_shaped_method;
  int    blind_spots;
  int    xDirection;             /* 0 bothX, 1 positiveX, 2 negativeX */
  double interval;
  double curb_height;
  int    curb_points;
  double beamZone;
  double min_x, max_x, min_y, max_y, min_z, max_z;
  double cylinder_deg_x;
  double cylinder_deg_z;
  double curb_slope_deg;
  double kdev_param;
  double kdist_param;
  int    starbeam_filter;
  int    dmin_param;
  int    simple_poly_allow;      /* marker tail only */
  double poly_s_param;           /* marker tail only */
  double poly_z_manual;          /* marker tail only */
  int    poly_z_avg_allow;       /* marker tail only */
  int    channels;               /* 1..URF_MAX_CHANNELS, default 64 */
} urf_params;

/*
 * Per-scan result. The caller owns every buffer; pointer members may be NULL when that output is not wanted.
 *   label[i]  (i < n_in)  : URF_LABEL_* of input point i (input order).
 *   ring[i]   (i < n_in)  : index of the point's ring in ascending-elevation order (= first index of array3D,
 *                           lidar_segmentation.cpp:226-238), -1 if outside the ROI or no registered ring matches.
 *   order[k]  (k < n_order): input index of the k-th point in the reference's emission order (ring-major, ascending
 *                           azimuth — the order of lidar_segmentation.cpp:354-367). road cloud = points of `order` with
 *                           label 1, curb cloud = label 2, road_probably = the segment of ring 10.
 *   ring_start[r] (r <= n_rings): offset of ring r inside `order` (ring_start[n_rings] == n_order); caller provides
 *                           URF_MAX_CHANNELS+1 ints or NULL.
 *   vert      : marker candidate vertices (x, y, z, redFlag) exactly as markerPointsArray is filled by
 *               lidar_segmentation.cpp:305-351, BEFORE the flag smoothing of :381-415.
 */
typedef struct urf_result {
  int32_t  status;               /* URF_OK or URF_TOO_FEW_POINTS (all other outputs then describe "nothing published") */
  int32_t  n_in;
  int32_t  n_roi;                /* `piece`, lidar_segmentation.cpp:120 */
  int32_t  n_rings;              /* `index`, lidar_segmentation.cpp:139 */
  int32_t  n_order;              /* points that were assigned a ring */
  int32_t  n_road;               /* label 1 count */
  int32_t  n_curb;               /* label 2 count */
  int32_t  n_vert;               /* `cM`, lidar_segmentation.cpp:300 */
  int32_t  flags;                /* bit0: exact-fallback ring registration ran; bit1: sector-radius ties present among the
                                    points the star search sorted (the near-first sort leaves the far part of a sector
                                    unsorted; ties there are neither seen nor relevant); bit2: ring-azimuth ties present
                                    (bit1 / bit2: tie policy differs from the reference's unstable sorts); bit3: a ROI point
                                    with x == y == 0 exists (azimuth NaN: it belongs to no window or bin here, while in the
                                    reference it truncates the window scans of its ring) */
  int32_t  reserved;
  int32_t* label;                /* [n_in] or NULL */
  int32_t* ring;                 /* [n_in] or NULL */
  int32_t* order;                /* [n_in] or NULL */
  int32_t* ring_start;           /* [URF_MAX_CHANNELS + 1] or NULL */
  float    vert[URF_MAX_VERTS][4];
} urf_result;

/* One line strip of the road_marker MarkerArray (lidar_segmentation.cpp:417-598). */
typedef struct urf_strip {
  int32_t id;                    /* Marker.id */
  int32_t action;                /* 0 = ADD, 2 = DELETE (ghost removal, :592-597) */
  int32_t red;                   /* 1 = red (1,0,0,1), 0 = green (0,1,0,1) */
  int32_t first;                 /* first point index in the points array */
  int32_t count;                 /* number of points */
} urf_strip;

typedef struct urf_ctx urf_ctx;

/* Fill *p with the defaults of cfg/LidarFilters.cfg (and channels = 64). */
void urf_default_params(urf_params* p);

/* Create a context on CUDA device `device` able to process scans of up to max_points input points, up to max_batch
 * scans per urf_process_batch call. Replaces Detector::Detector + beam_init (lidar_segmentation.cpp:51-65).
 * max_points above 2^24 is URF_ERR_INVALID; max_batch above 65535 (the kernels' grid y limit) is URF_ERR_CAPACITY. */
int urf_create(urf_ctx** out, int device, int max_points, int max_batch);
void urf_destroy(urf_ctx* ctx);

/* Replaces paramsCallback (src/main.cpp:4-34). Takes effect for the next urf_process* call. */
int urf_set_params(urf_ctx* ctx, const urf_params* p);
int urf_get_params(const urf_ctx* ctx, urf_params* p);

/* Replaces one Detector::filtered() call. xyzi = n points of 4 floats (x, y, z, intensity) in HOST memory: the first
 * 16 bytes of each pcl::PointXYZI record once the PointCloud2 has been deserialised. Synchronous. */
int urf_process(urf_ctx* ctx, const float* xyzi, int n, urf_result* out);

/* Same as urf_process, but takes the raw `data` bytes of a sensor_msgs/PointCloud2 message (what pcl_ros deserialises
 * for the reference's callback, lidar_segmentation.cpp:53,95): n_points records of point_step bytes in HOST memory, with
 * x / y / z (FLOAT32) at byte offsets off_x / off_y / off_z inside a record (Ouster: 48-byte records, Velodyne: 22 or 32).
 * Records need not be 4-byte aligned. The bytes are copied to the device as they are and unpacked there (SURVEY.md §8 f1);
 * point_step must be in [12, URF_MAX_POINT_STEP]. Synchronous. */
#define URF_MAX_POINT_STEP 64
int urf_process_cloud2(urf_ctx* ctx, const void* data, int n_points, int point_step, int off_x, int off_y, int off_z,
                       urf_result* out);

/* One pcl::PointXYZI record as the reference stores it in its output clouds (32 bytes, PCL_ADD_POINT4D + intensity). */
typedef struct urf_point_xyzi {
  float x, y, z, w;              /* w = data[3] = 1.0f, as PCL's constructor leaves it */
  float intensity, pad[3];
} urf_point_xyzi;

/* The four output clouds of one scan, packed on the device in the reference's emission order (SURVEY.md §8 f1):
 *   road          = cloud_filtered_Road          lidar_segmentation.cpp:354-361 (label 1; ring-major, ascending azimuth)
 *   curb          = cloud_filtered_High          lidar_segmentation.cpp:362-366 (label 2; same order)
 *   roi           = cloud_filtered_Box           lidar_segmentation.cpp:114-120 (every ROI point, input order)
 *   road_probably = cloud_filtered_ProbablyRoad  lidar_segmentation.cpp:605-608 (ring 10, ascending azimuth)
 * Each pointer is a caller-owned HOST buffer with room for n_points records, or NULL to skip that cloud; n_* are set
 * by the call (all 0 when status == URF_TOO_FEW_POINTS). */
typedef struct urf_clouds {
  urf_point_xyzi* road;
  urf_point_xyzi* curb;
  urf_point_xyzi* roi;
  urf_point_xyzi* road_probably;
  int32_t n_road, n_curb, n_roi, n_road_probably;
} urf_clouds;

/* urf_process_cloud2 with the output side on the device too: instead of (or besides) labels and the emission order, the
 * call returns the four clouds the reference publishes, ready to be wrapped in PointCloud2 messages; only the records
 * that exist cross PCIe. off_intensity = byte offset of the FLOAT32 intensity field, or -1 (intensity 0). out->label /
 * ring / order may be NULL. The first packed call allocates 96 bytes of device memory per point of capacity. */
int urf_process_cloud2_packed(urf_ctx* ctx, const void* data, int n_points, int point_step, int off_x, int off_y, int off_z,
                              int off_intensity, urf_result* out, urf_clouds* clouds);

/* `batch` independent scans (distinct clouds, same params), HOST buffers. xyzi[b] has n[b] points; outs[b] as above. */
int urf_process_batch(urf_ctx* ctx, const float* const* xyzi, const int* n, int batch, urf_result* outs);

/* Lean variants for callers that are bound by PCIe (opt-in additions; urf_process_batch above stays the drop-in for
 * Detector::filtered): the label path never reads intensity and a label is one of four values, so
 *   urf_process_batch_xyz   takes packed (x, y, z) FLOAT32 triples — 12 bytes per point cross PCIe instead of 16 — and
 *   label8[b] (int8 HOST buffers of n[b] bytes, or label8 == NULL / label8[b] == NULL) receives the labels as one byte per
 *   point (same URF_LABEL_* values) instead of four. outs[b].label / ring / order are still honoured when non-NULL.
 *   urf_process_cloud2_batch is urf_process_cloud2 for `batch` scans of one sensor format: the raw PointCloud2 records of
 *   every scan cross PCIe as they are and are unpacked on the device (off_intensity < 0: no intensity field). */
int urf_process_batch_xyz(urf_ctx* ctx, const float* const* xyz, const int* n, int batch, urf_result* outs, int8_t* const* label8);
int urf_process_cloud2_batch(urf_ctx* ctx, const void* const* data, const int* n_points, int batch, int point_step, int off_x,
                             int off_y, int off_z, int off_intensity, urf_result* outs, int8_t* const* label8);

/* Device-resident variant used to time the kernels without PCIe: d_xyzi is a DEVICE pointer to the scans stored back to
 * back (scan b starts at point offset b*stride_points, has n[b] points), d_label a DEVICE pointer with the same layout
 * (int32 per point) that receives the labels. Small per-scan metadata (counts, vertices) is still returned in outs[b]
 * (label/ring/order pointers in outs[] are ignored). Runs on the ctx stream; returns after the stream is idle. */
int urf_process_batch_device(urf_ctx* ctx, const float* d_xyzi, int stride_points, const int* n, int batch,
                             int32_t* d_label, urf_result* outs);

/* Asynchronous pair for the above (enqueue on the ctx stream / wait + read back metadata), so callers can bracket the
 * enqueue with their own CUDA events on urf_stream(). */
int urf_enqueue_batch_device(urf_ctx* ctx, const float* d_xyzi, int stride_points, const int* n, int batch,
                             int32_t* d_label);
/* As urf_enqueue_batch_device, plus the emission order: d_order (DEVICE, int32, same layout as d_label, or NULL) receives
 * for every scan b the input indices of its n_order ring-assigned points in the reference's emission order (ring-major,
 * ascending azimuth, lidar_segmentation.cpp:289-291,354-367) — i.e. the per-ring azimuth sort runs as part of the call. */
int urf_enqueue_batch_device_ex(urf_ctx* ctx, const float* d_xyzi, int stride_points, const int* n, int batch,
                                int32_t* d_label, int32_t* d_order);
int urf_finish_batch_device(urf_ctx* ctx, urf_result* outs);
void* urf_stream(urf_ctx* ctx);            /* cudaStream_t of the ctx */
/* CUDA-event timing of everything enqueued by the last urf_enqueue/process call: total ms on the ctx stream. */
float urf_last_device_ms(const urf_ctx* ctx);
/* Number of kernel launches issued by the last urf_process* / urf_enqueue* call. */
int urf_last_launch_count(const urf_ctx* ctx);

/* Marker tail (lidar_segmentation.cpp:371-598) as a host routine: flag smoothing, strip splitting, optional
 * Douglas-Peucker simplification, zavg, ghost DELETE markers. `ghostcount` is the reference's global (:23) kept by the
 * caller between scans. points_xyz receives 3 doubles per point (geometry_msgs::Point); returns the number of strips
 * written (<= max_strips), or a negative error. n_points_out receives the number of points written. */
int urf_build_markers(const urf_params* p, const float (*vert)[4], int n_vert, int* ghostcount,
                      urf_strip* strips, int max_strips, double* points_xyz, int max_points, int* n_points_out);

/* Pinned (page-locked) host memory for callers that stage scans themselves: urf_process* copies from such buffers
 * asynchronously at full PCIe rate. NULL without a CUDA device. */
void* urf_pinned_alloc(size_t bytes);
void urf_pinned_free(void* p);

/*
 * Streaming ingest (SURVEY.md §8 f4). The reference node subscribes with queue size 1 (lidar_segmentation.cpp:53): while
 * Detector::filtered() runs, newer scans replace each other and all but the last are dropped. urf_queue keeps that
 * contract available (URF_QUEUE_DROP_OLDEST) but makes it rare: producers (one per LiDAR topic / driver thread) copy
 * their scan into one of `slots` pinned staging buffers and return at once; one worker thread owns the ctx and runs
 * every scan that is pending — up to `max_batch` of them per urf_process_batch call, whose chunked three-stream pipeline
 * overlaps the H2D copy of one chunk with the kernels of the previous one — and consumers take the results in
 * submission order. The ctx must have been created with max_batch >= the queue's max_batch and must not be used by
 * anyone else until urf_queue_destroy returns.
 */
typedef struct urf_queue urf_queue;
/* policy of urf_queue_create*: BLOCK or DROP_OLDEST, optionally OR-ed with URF_QUEUE_LABEL8 — int8 label slots (max_points
 * bytes per slot instead of 4 * max_points; the worker fetches one-byte labels from the device, the int32 label copy is not
 * issued). On such a queue urf_queue_next widens the labels into the caller's int32 buffer, urf_queue_next_view returns
 * URF_ERR_INVALID (there is no int32 array to point at) and urf_queue_next_batch lends int8_t views. */
enum { URF_QUEUE_BLOCK = 0, URF_QUEUE_DROP_OLDEST = 1, URF_QUEUE_LABEL8 = 2 };
enum { URF_ERR_TIMEOUT = -6, URF_ERR_CLOSED = -7 };
typedef struct urf_queue_stats {
  uint64_t submitted, processed, dropped, delivered, batches;
  int32_t  largest_batch, pending, reserved;
} urf_queue_stats;

int urf_queue_create(urf_queue** out, urf_ctx* ctx, int max_points, int slots, int max_batch, int policy);
/* Copy scan (n points of x, y, z, intensity) into a free slot. `tag` comes back with the result (sequence number,
 * sensor id, stamp). No free slot: URF_QUEUE_BLOCK waits up to timeout_ms (< 0: forever) and returns URF_ERR_TIMEOUT;
 * URF_QUEUE_DROP_OLDEST discards the oldest scan whose processing has not started (it is never delivered) — if every
 * slot is already being processed or waiting to be collected it waits like BLOCK. Results are ordered by the moment a
 * submit call finished copying (with one producer: submission order). */
int urf_queue_submit(urf_queue* q, const float* xyzi, int n, uint64_t tag, int timeout_ms);
/* Next result in submission order (dropped scans are skipped). out->label (n ints) may be NULL; ring / order /
 * ring_start are not produced by the queue. URF_ERR_TIMEOUT when nothing finished within timeout_ms (< 0: wait),
 * URF_ERR_CLOSED once the queue is closed and drained. A scan whose processing failed returns that error code. */
int urf_queue_next(urf_queue* q, uint64_t* tag, urf_result* out, int timeout_ms);
/* urf_queue_next without the copy of the labels: *label_view points at the n_in labels inside the queue's staging slot
 * (NULL for a failed scan); the slot stays reserved until the consumer's next urf_queue_next / _next_view call on this queue
 * or urf_queue_release_view. out->label is ignored. One consumer thread at a time may hold a view. */
int urf_queue_next_view(urf_queue* q, uint64_t* tag, urf_result* out, const int32_t** label_view, int timeout_ms);
/* Batched delivery: one wake-up and one lock round for every scan that is ready, instead of one per scan. Waits up to
 * timeout_ms (< 0: forever) until the oldest live scan is done, then lends out the run of consecutive finished scans that
 * starts with it, in submission order, at most max_results of them (it never skips a scan that is not done yet; dropped
 * scans are skipped as by urf_queue_next). Returns how many it lent (>= 1), or URF_ERR_TIMEOUT / URF_ERR_CLOSED as
 * urf_queue_next. For scan j: tags[j], rcs[j] (URF_OK, or the error code of the batch the scan failed in), outs[j] (counts,
 * flags and the n_vert vertices; pointer members set to NULL) and label_views[j], which points at the n_in labels inside
 * the queue's slot — int8_t with URF_QUEUE_LABEL8, int32_t otherwise — or is NULL for a failed scan. tags, rcs and
 * label_views may be NULL. Every lent slot stays reserved until the consumer's next urf_queue_next* call on this queue or
 * urf_queue_release_view, so the views stay valid until then. */
int urf_queue_next_batch(urf_queue* q, int max_results, uint64_t* tags, int32_t* rcs, urf_result* outs, const void** label_views,
                         int timeout_ms);
/* Gives back every slot lent by urf_queue_next_view / urf_queue_next_batch. */
void urf_queue_release_view(urf_queue* q);
int urf_queue_get_stats(urf_queue* q, urf_queue_stats* st);
/* Stop accepting scans: blocked and later urf_queue_submit calls return URF_ERR_CLOSED; the worker still finishes what
 * is pending and urf_queue_next keeps delivering until the queue is drained, then returns URF_ERR_CLOSED. */
void urf_queue_close(urf_queue* q);
/* urf_queue_close, then waits for the worker and frees everything (undelivered results are discarded). No other thread
 * may be inside a urf_queue_* call on this queue any more: close first, let producers and consumers return, then destroy. */
void urf_queue_destroy(urf_queue* q);

/* As urf_queue_submit, but the scan is NOT copied: `xyzi` is used in place by the worker's host-to-device copy and must stay
 * valid and unchanged until the scan's result has been delivered by urf_queue_next (pinned memory — urf_pinned_alloc —
 * gives asynchronous copies at full PCIe rate). Removes the producer-side memcpy, the host limiter of a single ingest thread. */
int urf_queue_submit_ref(urf_queue* q, const float* xyzi, int n, uint64_t tag, int timeout_ms);

/* A queue whose scans are raw sensor_msgs/PointCloud2 records of ONE sensor format (what the node's subscriber receives,
 * lidar_segmentation.cpp:53,95): producers hand in the `data` bytes of a message with urf_queue_submit_cloud2, the worker
 * runs everything pending through urf_process_cloud2_batch (records unpacked on the device). urf_queue_next as above. */
int urf_queue_create_cloud2(urf_queue** out, urf_ctx* ctx, int max_points, int slots, int max_batch, int policy, int point_step,
                            int off_x, int off_y, int off_z, int off_intensity);
int urf_queue_submit_cloud2(urf_queue* q, const void* data, int n_points, uint64_t tag, int timeout_ms);

/* Test hook: the same queue around a caller-supplied batch function with urf_process_batch's signature (`user` is passed
 * as its ctx argument) and malloc'ed instead of pinned staging — the queue mechanics can then be exercised without a GPU.
 * With URF_QUEUE_LABEL8 the function still writes int32 labels (outs[b].label); the queue narrows them into its int8 slots. */
typedef int (*urf_queue_process_fn)(void* user, const float* const* xyzi, const int* n, int batch, urf_result* outs);
int urf_queue_create_with(urf_queue** out, urf_queue_process_fn fn, void* user, int max_points, int slots, int max_batch,
                          int policy);

/*
 * Multi-GPU ingest (BASELINE config 4: one continuous scan stream sharded across the GPUs of a box). The reference is one
 * subscriber in one process (lidar_segmentation.cpp:53); urf_mq is one submit / next interface over N devices: it creates
 * a context and a urf_queue (above) per device, hands every scan to the device with the fewest scans in flight, and
 * delivers the results in the order the submissions completed. Scans are independent, so no data moves between devices.
 * Any number of producer threads; ONE consumer thread. urf_mq_submit_ref is the no-copy variant (see urf_queue_submit_ref).
 * urf_mq_set_params applies to all devices and is only accepted while nothing is in flight (like the reference's
 * paramsCallback between two scan callbacks).
 */
typedef struct urf_mq urf_mq;
#define URF_MQ_MAX_DEVICES 16
typedef struct urf_mq_stats {
  int32_t  n_devices, pending;
  uint64_t submitted[URF_MQ_MAX_DEVICES], delivered[URF_MQ_MAX_DEVICES], batches[URF_MQ_MAX_DEVICES];
  int32_t  largest_batch[URF_MQ_MAX_DEVICES];
} urf_mq_stats;
int urf_mq_create(urf_mq** out, const int* devices, int n_devices, int max_points, int slots_per_device, int max_batch,
                  const urf_params* params /* or NULL: cfg defaults */);
int urf_mq_set_params(urf_mq* mq, const urf_params* p);
int urf_mq_submit(urf_mq* mq, const float* xyzi, int n, uint64_t tag, int timeout_ms);
int urf_mq_submit_ref(urf_mq* mq, const float* xyzi, int n, uint64_t tag, int timeout_ms);
int urf_mq_next(urf_mq* mq, uint64_t* tag, urf_result* out, int timeout_ms);
int urf_mq_next_view(urf_mq* mq, uint64_t* tag, urf_result* out, const int32_t** label_view, int timeout_ms);   /* see urf_queue_next_view */
/* urf_queue_next_batch over all devices: lends the run of finished scans at the front of the global order (one call may
 * take scans from several devices, in the global order), at most max_results of them. Every lent slot, on whichever device,
 * stays reserved until the consumer's next urf_mq_next* call. The mq lock is taken twice per call, whatever the count. */
int urf_mq_next_batch(urf_mq* mq, int max_results, uint64_t* tags, int32_t* rcs, urf_result* outs, const void** label_views,
                      int timeout_ms);
/* urf_mq_create with int8 label slots on every device (URF_QUEUE_LABEL8; urf_mq_next_view then returns URF_ERR_INVALID). */
int urf_mq_create_label8(urf_mq** out, const int* devices, int n_devices, int max_points, int slots_per_device, int max_batch,
                         const urf_params* params /* or NULL: cfg defaults */);
int urf_mq_get_stats(urf_mq* mq, urf_mq_stats* st);
void urf_mq_close(urf_mq* mq);
void urf_mq_destroy(urf_mq* mq);
/* Test hook: N stand-in devices around a caller-supplied batch function (users[j] is passed to it for device j). */
int urf_mq_create_with(urf_mq** out, urf_queue_process_fn fn, void* const* users, int n_devices, int max_points,
                       int slots_per_device, int max_batch);
int urf_mq_create_with_label8(urf_mq** out, urf_queue_process_fn fn, void* const* users, int n_devices, int max_points,
                              int slots_per_device, int max_batch);

const char* urf_strerror(int code);
/* Text of the last failed CUDA call of `ctx`; with ctx == NULL: why this thread's last urf_create failed. */
const char* urf_last_cuda_error(const urf_ctx* ctx);
int urf_version(void);

#ifdef __cplusplus
}
#endif
#endif /* URF_H_ */
