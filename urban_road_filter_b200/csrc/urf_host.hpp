// urf_host.hpp — host-only helpers shared by liburf_b200 (urf_api.cu) and the CPU model check (tests/kat/model_check.cpp):
// parameter validation (urf_params.hpp) and narrowing (src/main.cpp:4-34), beam_init (star_shaped_search.cpp:32-66), newY ramp.
#pragma once
#include <cmath>
#include <vector>

#include "urf_device.cuh"
#include "urf_params.hpp"

namespace urf {

// star_shaped_search.cpp:32-66 beam_init(): same libm calls and narrowing as the reference, evaluated on the host.
inline void host_beam_init(float* d, float* o, unsigned char* yx, float* Kfi) {
  const int rep = 360;             // :8
  const float width = 0.2f;        // :9
  float fi, off = 0.5 * width;     // :35
  for (int i = 0; i < rep; i++) {
    fi = i * 2 * M_PI / rep;                                   // :38
    if (std::abs(std::tan(fi)) > 1) {                          // :39
      yx[i] = 1;
      d[i] = std::tan(0.5 * M_PI - fi);                        // :42
      o[i] = std::abs(off / std::sin(fi));                     // :43
    } else {
      yx[i] = 0;
      d[i] = std::tan(fi);                                     // :48
      o[i] = std::abs(off / std::cos(fi));                     // :49
    }
  }
  *Kfi = rep / (2 * M_PI);                                     // :65
}

// x_zero_method.cpp:24-27: newY[j] = newY[j-1] + 0.0100 (double add narrowed to float); depends on j only
inline void host_newY(std::vector<float>& ny, int count) {
  ny.assign(count > 0 ? count : 1, 0.f);
  for (int j = 1; j < count; j++) ny[j] = ny[j - 1] + 0.0100;
}

inline void narrow_params(const urf_params* p, DevParams* q, float Kfi, int force_exact, int want_order) {
  // src/main.cpp:5-32: every double lands in a float global
  q->x_zero = p->x_zero_method != 0; q->z_zero = p->z_zero_method != 0; q->star = p->star_shaped_method != 0;
  q->blind = p->blind_spots != 0; q->xDirection = p->xDirection;
  q->interval = (float)p->interval; q->curbHeight = (float)p->curb_height; q->curbPoints = p->curb_points;
  q->beamZone = (float)p->beamZone;
  q->angleFilter1 = (float)p->cylinder_deg_x; q->angleFilter2 = (float)p->cylinder_deg_z;
  const float angleFilter3 = (float)p->curb_slope_deg;
  q->slope_param = angleFilter3 * (M_PI / 180);                        // star_shaped_search.cpp:160
  q->min_X = (float)p->min_x; q->max_X = (float)p->max_x; q->min_Y = (float)p->min_y; q->max_Y = (float)p->max_y;
  q->min_Z = (float)p->min_z; q->max_Z = (float)p->max_z;
  q->kdev = (float)p->kdev_param; q->kdist = (float)p->kdist_param;
  q->starbeam = p->starbeam_filter != 0; q->dmin = p->dmin_param; q->channels = p->channels;
  q->Kfi = Kfi;
  // blind_spots.cpp:68 `i <= 360 - params::beamZone` (int vs float) and :177 `i >= 0 + params::beamZone`
  const float lim_f = 360 - q->beamZone, lim_b = 0 + q->beamZone;
  q->fwd_last = -1; q->fwd_special = -1; q->bwd_first = 361; q->bwd_special = -1;
  for (int i = 0; i <= 360 && i <= lim_f; i++) { q->fwd_last = i; if (i == lim_f) q->fwd_special = i; }
  for (int i = 360; i >= 0 && i >= lim_b; --i) { q->bwd_first = i; if (i == lim_b) q->bwd_special = i; }
  q->force_exact = force_exact;
  q->want_order = want_order;
}

}  // namespace urf
