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
                                    reference it truncates the window scans of its ring). With the reference tie order
                                    (urf_set_tie_order below) bit2 is reported whether or not `order` is requested, and
                                    the order it marks is the reference's own */
  union {                        /* anonymous: `reserved` keeps its name for existing callers */
    int32_t reserved;
    int32_t params_gen;          /* parameter generation the scan ran with (urf_set_params_next, urf_queue_update_params,
                                    urf_mq_update_params); 0 until the first such update */
  };
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

/* Replaces paramsCallback (src/main.cpp:4-34). Takes effect for the next urf_process* call. Refused (URF_ERR_INVALID)
 * while host batches are in flight; it leaves the parameter generation (urf_set_params_next) as it is. */
int urf_set_params(urf_ctx* ctx, const urf_params* p);
/*
 * paramsCallback for a context with host batches in flight: validates p (URF_ERR_INVALID, nothing changed, for a bad set)
 * and applies it to every urf_enqueue* / urf_process* call made after it returns. Batches already enqueued keep the
 * parameters they were enqueued with, and their urf_finish_batch fills outs exactly as the synchronous call with those
 * parameters would (channels-dependent sizes included). Returns the context's new parameter generation (1, 2, ...), which
 * every result of a later call reports in urf_result.params_gen; results report 0 until the first call. urf_set_params
 * does not advance the generation: a caller that numbers its sets uses this call only.
 */
int urf_set_params_next(urf_ctx* ctx, const urf_params* p);
int urf_get_params(const urf_ctx* ctx, urf_params* p);

/*
 * Tie order of the emission order (urf_result.order, the packed clouds) and of the marker vertices where a ring holds
 * equal azimuths (dual-return modes, duplicated points, rings merged by a large `interval`):
 *   URF_TIES_INPUT_ORDER (default): equal azimuths in input order, NaN azimuths last. Labels never depend on the tie order.
 *   URF_TIES_REFERENCE: the order the reference's unstable Lomuto quicksort leaves (lidar_segmentation.cpp:70-93,
 *     289-291) on every ring that holds a float-equal pair or a NaN azimuth — its road, curb and road_probably clouds and
 *     its marker vertices (:313-335) bit for bit. Costs the ring sort on every call (even without `order`) and, per
 *     ring with ties, about one CTA-wide partition per point in the worst case (DESIGN.md §6).
 *     Not covered: a NaN azimuth (x == y == 0) still truncates the reference's blindSpots window scans, so with
 *     blind_spots on, labels of such scans can differ (flags bit3).
 * The setting applies to the next urf_process* / urf_enqueue* call. The first switch to URF_TIES_REFERENCE allocates 4
 * bytes of device memory per point of capacity (URF_ERR_NOMEM if that fails); urf_process* never allocates for it.
 * A urf_queue uses its ctx's setting; urf_mq_set_tie_order sets it on every device, only while nothing is in flight.
 */
enum { URF_TIES_INPUT_ORDER = 0, URF_TIES_REFERENCE = 1 };
int urf_set_tie_order(urf_ctx* ctx, int mode);
int urf_get_tie_order(const urf_ctx* ctx, int* mode);

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

/*
 * Several sensor formats in one batch (a vehicle with Ouster and Velodyne LiDARs): only the unpack on the device reads the
 * record format, so one batch can carry scans of different formats. A format is what a PointCloud2's `fields` and
 * `point_step` give: FLOAT32 x / y / z at off_x / off_y / off_z and intensity at off_intensity (or -1: none) inside a record
 * of point_step bytes. A float4 scan is the format {16, 0, 4, 8, 12}.
 */
typedef struct urf_cloud2_format {
  int32_t point_step, off_x, off_y, off_z, off_intensity;
} urf_cloud2_format;
#define URF_MAX_FORMATS 8        /* formats of one urf_queue_create_formats / urf_mq_create_formats table */
/* urf_process_cloud2_batch where scan b's records have the format fmt[b]. Every fmt[b] passes the checks of
 * urf_process_cloud2 (URF_ERR_INVALID otherwise); outs and label8 as urf_process_cloud2_batch, and every output of scan b is
 * bit for bit what urf_process_cloud2_batch gives for that scan alone in its own format, in both tie orders. The records of
 * scan b are staged on the device at b * stride * step_max bytes, step_max being the batch's largest point_step (the staging
 * buffer grows as for urf_process_cloud2_batch); the formats cross PCIe with the point counts, 20 bytes per scan. A batch
 * whose scans all have one format runs exactly as urf_process_cloud2_batch. */
int urf_process_cloud2_batch_mixed(urf_ctx* ctx, const void* const* data, const int* n_points, const urf_cloud2_format* fmt,
                                   int batch, urf_result* outs, int8_t* const* label8);

/*
 * Asynchronous host-buffer batches: urf_enqueue_batch (float4 scans, as urf_process_batch) and urf_enqueue_cloud2_batch
 * (PointCloud2 records, as urf_process_cloud2_batch) queue the copies and kernels of a batch and return at once;
 * urf_finish_batch waits for the OLDEST batch in flight and fills its outs[] (and label8[] buffers). While batch N runs,
 * the caller can hand over batch N+1: its input copies overlap batch N's kernels, its kernels follow them on the same
 * stream, and batch N's result copies overlap batch N+1's kernels.
 *   - A context holds at most TWO host batches in flight: a third enqueue returns URF_ERR_CAPACITY; urf_finish_batch with
 *     nothing in flight returns URF_ERR_INVALID.
 *   - Every output (labels, int8 labels, ring, order, ring_start, counts, flags, vertices) is bit for bit what
 *     urf_process_batch / urf_process_cloud2_batch give for the same scans, in both tie orders. label8 as in
 *     urf_process_batch_xyz; label8 == NULL: no int8 labels.
 *   - The input buffers, the outs array and every buffer it or label8 points at must stay valid and unchanged until the
 *     batch's urf_finish_batch returns. Copies from pinned memory (urf_pinned_alloc) run asynchronously. A copy to or from
 *     pageable memory makes the call wait for it: with pageable outs the enqueue returns only once the batch's results
 *     are on the host, and nothing overlaps.
 *   - While host batches are in flight, urf_process*, urf_enqueue_batch_device*, urf_finish_batch_device, urf_set_params,
 *     urf_set_tie_order and urf_set_option return URF_ERR_INVALID (urf_set_params_next changes the parameters of the next
 *     enqueue). urf_destroy waits for them (their outs are not filled).
 *   - urf_last_device_ms and urf_last_launch_count describe the last finished batch.
 * The first asynchronous call allocates a second set of the buffers a batch's copies touch, and a ring-id buffer for the
 * first set (which until then keeps ring ids in sort scratch that the next batch's kernels overwrite): 32 bytes of device
 * memory per point of capacity (input, labels, order, two ring-id buffers), plus 1 byte per point once int8 labels are
 * asked for and point_step bytes per point once records are given, and two small pinned arrays per scan of max_batch.
 * No batch waits for another batch's copies.
 */
int urf_enqueue_batch(urf_ctx* ctx, const float* const* xyzi, const int* n, int batch, urf_result* outs, int8_t* const* label8);
int urf_enqueue_cloud2_batch(urf_ctx* ctx, const void* const* data, const int* n_points, int batch, int point_step, int off_x,
                             int off_y, int off_z, int off_intensity, urf_result* outs, int8_t* const* label8);
/* urf_process_cloud2_batch_mixed without waiting: finished by urf_finish_batch, two batches in flight as above. The fmt
 * array is read during the call only. */
int urf_enqueue_cloud2_batch_mixed(urf_ctx* ctx, const void* const* data, const int* n_points, const urf_cloud2_format* fmt,
                                   int batch, urf_result* outs, int8_t* const* label8);
int urf_finish_batch(urf_ctx* ctx);

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
 * every scan that is pending — up to `max_batch` of them per batch, whose chunked three-stream pipeline overlaps the H2D
 * copy of one chunk with the kernels of the previous one, with two batches in flight (urf_enqueue_batch /
 * urf_finish_batch: the next batch is enqueued before the worker waits for the oldest) — and consumers take the results
 * in submission order. A scan counts as started (DROP_OLDEST no longer drops it) once its batch has been enqueued. The ctx must have been created with max_batch >= the queue's max_batch and must not be used by
 * anyone else until urf_queue_destroy returns; parameters of a running queue change through urf_queue_update_params.
 */
typedef struct urf_queue urf_queue;
/* policy of urf_queue_create*: BLOCK or DROP_OLDEST, optionally OR-ed with URF_QUEUE_LABEL8 and/or URF_QUEUE_ORDER (any
 * other bit: URF_ERR_INVALID).
 *   URF_QUEUE_LABEL8 — int8 label slots (max_points bytes per slot instead of 4 * max_points; the worker fetches one-byte
 *   labels from the device, the int32 label copy is not issued). On such a queue urf_queue_next widens the labels into the
 *   caller's int32 buffer, urf_queue_next_view returns URF_ERR_INVALID (there is no int32 array to point at) and
 *   urf_queue_next_batch lends int8_t views.
 *   URF_QUEUE_ORDER — every scan also delivers its emission order and ring offsets (urf_result.order / ring_start), from
 *   which a consumer rebuilds the road, curb and road_probably clouds in the reference's order. Each slot holds
 *   int32 order[max_points] and int32 ring_start[URF_MAX_CHANNELS + 1] besides its labels: 4 bytes per point plus 1,028
 *   bytes (pinned on a real queue, malloc'ed for a stand-in). The worker passes both to the batch call, so every batch runs
 *   the per-ring azimuth sort and copies 4 bytes per input point more to the host. order and ring_start are bit for bit
 *   what urf_process_batch (float4 queues) or urf_process_cloud2_batch (record queues) give for the same scan, under the
 *   ctx's tie order and the parameter generation the scan ran with (channels may differ between generations: n_rings + 1
 *   entries of ring_start are meaningful). For URF_TOO_FEW_POINTS, n_order == 0 and ring_start is all zeros.
 *   Without the bit the worker passes NULL for both and every delivered order / ring_start pointer is NULL. */
enum { URF_QUEUE_BLOCK = 0, URF_QUEUE_DROP_OLDEST = 1, URF_QUEUE_LABEL8 = 2, URF_QUEUE_ORDER = 4 };
enum { URF_ERR_TIMEOUT = -6, URF_ERR_CLOSED = -7 };
typedef struct urf_queue_stats {
  uint64_t submitted, processed, dropped, delivered, batches;
  int32_t  largest_batch, pending;
  int32_t  most_in_flight;       /* most batches the worker had enqueued at once (2 on a real context once a run was
                                    enqueued behind another; a synchronous stand-in: 1) */
} urf_queue_stats;

int urf_queue_create(urf_queue** out, urf_ctx* ctx, int max_points, int slots, int max_batch, int policy);
/* Copy scan (n points of x, y, z, intensity) into a free slot. `tag` comes back with the result (sequence number,
 * sensor id, stamp). No free slot: URF_QUEUE_BLOCK waits up to timeout_ms (< 0: forever) and returns URF_ERR_TIMEOUT;
 * URF_QUEUE_DROP_OLDEST discards the oldest scan whose processing has not started (it is never delivered) — if every
 * slot is already being processed or waiting to be collected it waits like BLOCK. Results are ordered by the moment a
 * submit call finished copying (with one producer: submission order). */
int urf_queue_submit(urf_queue* q, const float* xyzi, int n, uint64_t tag, int timeout_ms);
/* Next result in submission order (dropped scans are skipped). out->label (n ints) may be NULL. With URF_QUEUE_ORDER,
 * out->order (room for n ints) and out->ring_start (room for URF_MAX_CHANNELS + 1 ints) may be non-NULL on entry: they
 * receive n_order and n_rings + 1 entries. The caller's label / order / ring_start pointers stay in *out. Without the bit
 * order and ring_start are set to NULL; ring is never produced by the queue. URF_ERR_TIMEOUT when nothing finished within
 * timeout_ms (< 0: wait), URF_ERR_CLOSED once the queue is closed and drained. A scan whose processing failed returns that
 * error code. */
int urf_queue_next(urf_queue* q, uint64_t* tag, urf_result* out, int timeout_ms);
/* urf_queue_next without the copy of the labels: *label_view points at the n_in labels inside the queue's staging slot
 * (NULL for a failed scan); the slot stays reserved until the consumer's next urf_queue_next / _next_view call on this queue
 * or urf_queue_release_view. out->label is ignored. With URF_QUEUE_ORDER out->order and out->ring_start point into the
 * same slot, read-only and valid as long as the label view (NULL for a failed scan). One consumer thread at a time may
 * hold a view. */
int urf_queue_next_view(urf_queue* q, uint64_t* tag, urf_result* out, const int32_t** label_view, int timeout_ms);
/* Batched delivery: one wake-up and one lock round for every scan that is ready, instead of one per scan. Waits up to
 * timeout_ms (< 0: forever) until the oldest live scan is done, then lends out the run of consecutive finished scans that
 * starts with it, in submission order, at most max_results of them (it never skips a scan that is not done yet; dropped
 * scans are skipped as by urf_queue_next). Returns how many it lent (>= 1), or URF_ERR_TIMEOUT / URF_ERR_CLOSED as
 * urf_queue_next. For scan j: tags[j], rcs[j] (URF_OK, or the error code of the batch the scan failed in), outs[j] (counts,
 * flags and the n_vert vertices; label and ring set to NULL; order and ring_start as below) and label_views[j], which
 * points at the n_in labels inside the queue's slot — int8_t with URF_QUEUE_LABEL8, int32_t otherwise — or is NULL for a
 * failed scan. With URF_QUEUE_ORDER outs[j].order (n_order entries) and outs[j].ring_start (n_rings + 1 entries) point
 * into the same slot, read-only, NULL for a failed scan; without it they are NULL. tags, rcs and label_views may be NULL.
 * Every lent slot stays reserved until the consumer's next urf_queue_next* call on this queue or urf_queue_release_view,
 * so the views stay valid until then. */
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
/* As urf_queue_submit_cloud2, but the records are NOT copied: `data` (n_points * point_step bytes) is used in place by the
 * worker's host-to-device copy and must stay valid and unchanged until the scan's result has been delivered, as for
 * urf_queue_submit_ref. A float4 queue refuses record submits (URF_ERR_INVALID), and a record queue refuses
 * urf_queue_submit / urf_queue_submit_ref. */
int urf_queue_submit_cloud2_ref(urf_queue* q, const void* data, int n_points, uint64_t tag, int timeout_ms);

/*
 * Parameter update on a running queue, with no drain (the reference's paramsCallback, which runs between two scan
 * callbacks on the node's one spinner thread). Validates p (URF_ERR_INVALID, nothing changed, for a bad set; URF_ERR_CLOSED
 * after urf_queue_close) and returns the queue's new generation (1, 2, ...; generation 0 is what the ctx had at creation):
 *   - every scan runs with the generation in force when it was accepted (the moment that also fixes delivery order): with
 *     one producer, scans submitted after the call returns use p, scans submitted before it the sets before;
 *   - a batch never mixes generations: the worker ends a run at the first pending scan of another generation, and applies
 *     a run's set to the ctx (urf_set_params_next) just before enqueueing it, while the other batch may still be in flight;
 *   - every result reports its generation in urf_result.params_gen, so that the consumer can pass the right set (poly_*
 *     fields) to urf_build_markers.
 * Only the urf_params fields: the tie order and urf_set_option keep their rule (ctx idle).
 */
int urf_queue_update_params(urf_queue* q, const urf_params* p);

/* Test hook: the same queue around a caller-supplied batch function with urf_process_batch's signature (`user` is passed
 * as its ctx argument) and malloc'ed instead of pinned staging — the queue mechanics can then be exercised without a GPU.
 * With URF_QUEUE_LABEL8 the function still writes int32 labels (outs[b].label); the queue narrows them into its int8 slots.
 * With URF_QUEUE_ORDER outs[b].order / ring_start point into the slot, for the function to fill (and NULL without it). */
typedef int (*urf_queue_process_fn)(void* user, const float* const* xyzi, const int* n, int batch, urf_result* outs);
int urf_queue_create_with(urf_queue** out, urf_queue_process_fn fn, void* user, int max_points, int slots, int max_batch,
                          int policy);
/* Test hook: the worker schedule of a real queue (two batches in flight) around stand-ins for urf_enqueue_batch and
 * urf_finish_batch: `enqueue` (urf_process_batch's signature) takes a batch and may keep the pointers it is given until the
 * batch is finished; `finish(user)` completes the OLDEST batch enqueued, fills its outs, and returns its status. The
 * worker never has more than two batches enqueued. Staging and int8 narrowing as urf_queue_create_with. */
typedef int (*urf_queue_finish_fn)(void* user);
int urf_queue_create_with_async(urf_queue** out, urf_queue_process_fn enqueue, urf_queue_finish_fn finish, void* user, int max_points,
                                int slots, int max_batch, int policy);
/* Test hook: a stand-in queue has no ctx, so its worker calls fn(user, set, generation) where a real queue's worker calls
 * urf_set_params_next: before the first batch of each generation it runs (fn == NULL: none). A non-zero return fails that
 * batch with the code, as a refused enqueue does. URF_ERR_INVALID on a queue around a ctx. */
typedef int (*urf_queue_params_fn)(void* user, const urf_params* p, int32_t gen);
int urf_queue_set_params_hook(urf_queue* q, urf_queue_params_fn fn);
/* Test hook: a record queue (urf_queue_create_cloud2: same format checks, same submits) around a synchronous stand-in, as
 * urf_queue_create_with. The batch function gets the raw record pointers in its `xyzi` argument: xyzi[b] points at
 * n[b] * point_step bytes (the queue's slot, or with urf_queue_submit_cloud2_ref the caller's own buffer), never 4-byte
 * aligned float4 points. Its `user` argument, and the parameter hook's, is a urf_cloud2_user the queue owns: the record
 * format and the caller's `user`, valid until urf_queue_destroy. */
typedef struct urf_cloud2_user {
  void*   user;                  /* the creator's `user` (urf_mq_create_cloud2_with: users[j] for device j, or NULL) */
  int32_t point_step, off_x, off_y, off_z, off_intensity;
} urf_cloud2_user;
int urf_queue_create_cloud2_with(urf_queue** out, urf_queue_process_fn fn, void* user, int max_points, int slots, int max_batch,
                                 int policy, int point_step, int off_x, int off_y, int off_z, int off_intensity);

/*
 * A queue for the PointCloud2 records of SEVERAL sensor formats (one queue for every LiDAR of a vehicle): a table of
 * 1..URF_MAX_FORMATS formats at creation (each passes urf_queue_create_cloud2's checks, URF_ERR_INVALID otherwise), and each
 * submit names its scan's format by its index in the table. The worker runs what is pending through
 * urf_enqueue_cloud2_batch_mixed, so a batch mixes formats freely (never parameter generations), and every result is bit for
 * bit what urf_process_cloud2_batch gives for that scan alone in its own format. A float4 producer shares the queue by
 * registering {16, 0, 4, 8, 12}.
 *   - Slots hold max_points * (the table's largest point_step) bytes each.
 *   - urf_queue_submit_format copies n_points records of format `fmt` into a slot; urf_queue_submit_format_ref uses them in
 *     place, with urf_queue_submit_cloud2_ref's lifetime contract. fmt outside the table: URF_ERR_INVALID; n_points >
 *     max_points: URF_ERR_CAPACITY.
 *   - A formats queue refuses urf_queue_submit, urf_queue_submit_ref and urf_queue_submit_cloud2* (URF_ERR_INVALID), and every
 *     other queue refuses the _format submits.
 *   - Policy, delivery (urf_queue_next / _next_view / _next_batch, URF_QUEUE_LABEL8, URF_QUEUE_ORDER), DROP_OLDEST,
 *     urf_queue_update_params generations, the ctx's tie order, stats, close and destroy are those of a record queue.
 */
int urf_queue_create_formats(urf_queue** out, urf_ctx* ctx, int max_points, int slots, int max_batch, int policy,
                             const urf_cloud2_format* formats, int n_formats);
int urf_queue_submit_format(urf_queue* q, int fmt, const void* data, int n_points, uint64_t tag, int timeout_ms);
int urf_queue_submit_format_ref(urf_queue* q, int fmt, const void* data, int n_points, uint64_t tag, int timeout_ms);
/* Test hook: a formats queue around a synchronous stand-in, as urf_queue_create_cloud2_with. xyzi[b] points at scan b's raw
 * bytes (the queue's slot, or the caller's buffer after urf_queue_submit_format_ref). The batch function's `user`, and the
 * parameter hook's, is a urf_formats_user the queue owns, valid until urf_queue_destroy: the creator's `user`, the format
 * table (the queue's copy) and `fmt`, which during a batch call points at the format index of each of its scans. */
typedef struct urf_formats_user {
  void*                    user;           /* the creator's `user` (urf_mq_create_formats_with: users[j] for device j, or NULL) */
  const urf_cloud2_format* formats;        /* [n_formats] */
  int32_t                  n_formats;
  const int32_t*           fmt;            /* [batch]: fmt[b] is scan b's index into formats; valid during the call only */
} urf_formats_user;
int urf_queue_create_formats_with(urf_queue** out, urf_queue_process_fn fn, void* user, int max_points, int slots, int max_batch,
                                  int policy, const urf_cloud2_format* formats, int n_formats);

/*
 * Multi-GPU ingest (BASELINE config 4: one continuous scan stream sharded across the GPUs of a box). The reference is one
 * subscriber in one process (lidar_segmentation.cpp:53); urf_mq is one submit / next interface over N devices: it creates
 * a context and a urf_queue (above) per device, hands every scan to the device with the fewest scans in flight, and
 * delivers the results in the order the submissions completed. Scans are independent, so no data moves between devices.
 * Any number of producer threads; ONE consumer thread. urf_mq_submit_ref is the no-copy variant (see urf_queue_submit_ref).
 * urf_mq_set_params (and urf_mq_set_tie_order) applies to all devices and is only accepted while nothing is in flight (like the reference's
 * paramsCallback between two scan callbacks). urf_mq_update_params changes the parameters of a running mq (below).
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
int urf_mq_set_tie_order(urf_mq* mq, int mode);   /* urf_set_tie_order on every device; the same in-flight rule */
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
/* urf_mq_create with the device queues' slot options: policy = URF_QUEUE_BLOCK, optionally OR-ed with URF_QUEUE_LABEL8
 * and/or URF_QUEUE_ORDER (urf_mq_next / _next_view / _next_batch then deliver order and ring_start as urf_queue_next* do).
 * URF_QUEUE_DROP_OLDEST and unknown bits return URF_ERR_INVALID: the mq has no drop policy. */
int urf_mq_create_policy(urf_mq** out, const int* devices, int n_devices, int max_points, int slots_per_device, int max_batch,
                         const urf_params* params /* or NULL: cfg defaults */, int policy);
/* urf_queue_update_params over all devices, at one point of the global order: every scan before it in the delivery order
 * runs with the earlier sets, every scan after it with p. Returns the mq's generation (1, 2, ...), which the results of every
 * device report in params_gen. Waits while a producer is inside a submit call (the update takes every device's submit lock). */
int urf_mq_update_params(urf_mq* mq, const urf_params* p);
/* urf_mq_create_policy whose scans are raw sensor_msgs/PointCloud2 records of ONE sensor format: every device gets a context
 * and a urf_queue_create_cloud2 queue, and the records cross PCIe as they are and are unpacked on the device
 * (urf_process_cloud2_batch), so a producer hands in a message's `data` without repacking it. Format checks as
 * urf_queue_create_cloud2, policy as urf_mq_create_policy; both are checked before any device is set up. Producers call
 * urf_mq_submit_cloud2 (copy into the device queue's pinned slot) or urf_mq_submit_cloud2_ref (no copy: `data` must stay
 * valid and unchanged until the scan's result has been delivered). A record mq refuses urf_mq_submit / urf_mq_submit_ref
 * and a float4 mq refuses the record submits (URF_ERR_INVALID); n_points > max_points is URF_ERR_CAPACITY. Device choice,
 * delivery order, urf_mq_next / _next_view / _next_batch, urf_mq_update_params generations, urf_mq_set_tie_order,
 * urf_mq_get_stats, close and destroy are those of a float4 mq, and every result is bit for bit what
 * urf_process_cloud2_batch gives for the same records under the device context's tie order and the scan's generation. */
int urf_mq_create_cloud2(urf_mq** out, const int* devices, int n_devices, int max_points, int slots_per_device, int max_batch,
                         const urf_params* params /* or NULL: cfg defaults */, int policy, int point_step, int off_x, int off_y,
                         int off_z, int off_intensity);
int urf_mq_submit_cloud2(urf_mq* mq, const void* data, int n_points, uint64_t tag, int timeout_ms);
int urf_mq_submit_cloud2_ref(urf_mq* mq, const void* data, int n_points, uint64_t tag, int timeout_ms);
int urf_mq_get_stats(urf_mq* mq, urf_mq_stats* st);
void urf_mq_close(urf_mq* mq);
void urf_mq_destroy(urf_mq* mq);
/* Test hook: N stand-in devices around a caller-supplied batch function (users[j] is passed to it for device j). */
int urf_mq_create_with(urf_mq** out, urf_queue_process_fn fn, void* const* users, int n_devices, int max_points,
                       int slots_per_device, int max_batch);
int urf_mq_create_with_label8(urf_mq** out, urf_queue_process_fn fn, void* const* users, int n_devices, int max_points,
                              int slots_per_device, int max_batch);
int urf_mq_create_with_policy(urf_mq** out, urf_queue_process_fn fn, void* const* users, int n_devices, int max_points,
                              int slots_per_device, int max_batch, int policy);   /* policy as urf_mq_create_policy */
/* Test hook: urf_mq_create_cloud2 over N stand-in devices, each a urf_queue_create_cloud2_with queue around fn (its
 * urf_cloud2_user carries users[j] for device j). */
int urf_mq_create_cloud2_with(urf_mq** out, urf_queue_process_fn fn, void* const* users, int n_devices, int max_points,
                              int slots_per_device, int max_batch, int policy, int point_step, int off_x, int off_y, int off_z,
                              int off_intensity);
/* urf_mq_create_policy whose device queues are urf_queue_create_formats queues of one format table: one context, one worker
 * and one set of pinned slots per device carry every sensor format, and the scans of all of them share one device choice
 * and one delivery order. Table and policy checks as urf_queue_create_formats and urf_mq_create_policy, made before any
 * device is set up. urf_mq_submit_format / _format_ref name the scan's format as urf_queue_submit_format does (same
 * refusals); a formats mq refuses urf_mq_submit, urf_mq_submit_ref and urf_mq_submit_cloud2*, and every other mq the _format
 * submits. Device choice, delivery, generations, urf_mq_set_tie_order, stats, close and destroy are those of a record mq, and
 * every result is bit for bit what urf_process_cloud2_batch gives for that scan alone in its own format. */
int urf_mq_create_formats(urf_mq** out, const int* devices, int n_devices, int max_points, int slots_per_device, int max_batch,
                          const urf_params* params /* or NULL: cfg defaults */, int policy, const urf_cloud2_format* formats,
                          int n_formats);
int urf_mq_submit_format(urf_mq* mq, int fmt, const void* data, int n_points, uint64_t tag, int timeout_ms);
int urf_mq_submit_format_ref(urf_mq* mq, int fmt, const void* data, int n_points, uint64_t tag, int timeout_ms);
/* Test hook: urf_mq_create_formats over N stand-in devices, each a urf_queue_create_formats_with queue around fn (its
 * urf_formats_user carries users[j] for device j). */
int urf_mq_create_formats_with(urf_mq** out, urf_queue_process_fn fn, void* const* users, int n_devices, int max_points,
                               int slots_per_device, int max_batch, int policy, const urf_cloud2_format* formats, int n_formats);
/* Test hook: urf_queue_set_params_hook on every stand-in device (fn gets users[j] for device j). URF_ERR_INVALID on real devices. */
int urf_mq_set_params_hook(urf_mq* mq, urf_queue_params_fn fn);

const char* urf_strerror(int code);
/* Text of the last failed CUDA call of `ctx`; with ctx == NULL: why this thread's last urf_create failed. */
const char* urf_last_cuda_error(const urf_ctx* ctx);
int urf_version(void);

#ifdef __cplusplus
}
#endif
#endif /* URF_H_ */
