// urf_params.hpp — the range check of a urf_params set, shared by the context (urf_api.cu, through urf_host.hpp) and the
// streaming queues (urf_queue.cpp, urf_mq.cpp), which validate an update when it is made rather than when a batch applies it,
// and the record format checks, which the queues make at creation and the context at every record batch.
// Plain host C++: no CUDA header, so the ThreadSanitizer builds of the queues compile it with g++ alone.
#pragma once
#include <cmath>

#include "../../include/urf.h"

namespace urf {

inline int validate_params(const urf_params* p) {
  auto fin = [](double v) { return std::isfinite(v); };
  if (p->channels < 1 || p->channels > URF_MAX_CHANNELS) return URF_ERR_INVALID;
  if (p->xDirection < 0 || p->xDirection > 2) return URF_ERR_INVALID;
  if (!(p->interval > 0) || !fin(p->interval)) return URF_ERR_INVALID;
  if (p->curb_points < 1 || p->curb_points > 4096) return URF_ERR_INVALID;
  if (!(p->beamZone > 0) || !(p->beamZone <= 360)) return URF_ERR_INVALID;
  if (!fin(p->curb_height) || !fin(p->cylinder_deg_x) || !fin(p->cylinder_deg_z) || !fin(p->curb_slope_deg) ||
      !fin(p->kdev_param) || !fin(p->kdist_param))
    return URF_ERR_INVALID;
  if (!fin(p->min_x) || !fin(p->max_x) || !fin(p->min_y) || !fin(p->max_y) || !fin(p->min_z) || !fin(p->max_z))
    return URF_ERR_INVALID;
  return URF_OK;
}

// The record format checks of every record entry point, batch and queue: URF_OK when point_step is in
// [12, URF_MAX_POINT_STEP] and the FLOAT32 x / y / z (and intensity, when off_intensity >= 0) lie inside a record.
inline int check_cloud2_format(int point_step, int off_x, int off_y, int off_z, int off_intensity) {
  if (point_step < 12 || point_step > URF_MAX_POINT_STEP) return URF_ERR_INVALID;
  for (int o : {off_x, off_y, off_z}) if (o < 0 || o + 4 > point_step) return URF_ERR_INVALID;
  if (off_intensity >= 0 && off_intensity + 4 > point_step) return URF_ERR_INVALID;
  return URF_OK;
}
inline int check_cloud2_format(const urf_cloud2_format& f) {
  return check_cloud2_format(f.point_step, f.off_x, f.off_y, f.off_z, f.off_intensity);
}
// A format table of urf_queue_create_formats / urf_mq_create_formats: 1..URF_MAX_FORMATS entries, each passing the checks.
inline int check_format_table(const urf_cloud2_format* f, int n) {
  if (!f || n < 1 || n > URF_MAX_FORMATS) return URF_ERR_INVALID;
  for (int i = 0; i < n; i++) if (check_cloud2_format(f[i]) != URF_OK) return URF_ERR_INVALID;
  return URF_OK;
}

}  // namespace urf
