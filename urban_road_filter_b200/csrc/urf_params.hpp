// urf_params.hpp — the range check of a urf_params set, shared by the context (urf_api.cu, through urf_host.hpp) and the
// streaming queues (urf_queue.cpp, urf_mq.cpp), which validate an update when it is made rather than when a batch applies it.
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

}  // namespace urf
