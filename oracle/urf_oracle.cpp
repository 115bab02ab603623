// oracle/urf_oracle.cpp — TEST INFRASTRUCTURE ONLY. CPU restatement ("port") of the reference's per-scan road/curb
// classification path, used to check the CUDA path where the unmodified reference (oracle/_ref) is too slow or absent.
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may load this library.
//
// PARITY PINNING: the reference has no tests or golden vectors (SURVEY.md §4). This restatement is pinned against
// outputs of the reference itself: tests/test_oracle.py diffs it against oracle/_ref/liburf_ref.so (the unmodified
// reference sources) where that library exists, and against tests/golden/*.npz (generated from oracle/_ref by
// tests/golden/make_golden.py) everywhere.
//
// Platform definition of "the reference's result": x86-64, g++ -std=c++17 -O2 (CMakeLists.txt:5, no FMA contraction),
// glibc 2.39 libm, libstdc++ std::sort. Built with -ffp-contract=off; calls the same libm functions.
//
// Every block cites the reference lines it follows (paths relative to the reference repo).
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "../include/urf.h"

// Optional per-input-point intermediates for stage-level differential tests (all indexed by INPUT index; entries of
// points that never reach the stage keep the fill value the caller put there).
struct urf_oracle_debug {
  float* alpha_v;     // elevation angle, lidar_segmentation.cpp:162/165
  float* az;          // ring azimuth `alpha`, :254-269
  float* d2;          // planar range `d`, :245
  int8_t* star_mark;  // 2 where starShapedSearch marked the point (:146), else 0
  int8_t* det_label;  // label after star/x-zero/z-zero, before blindSpots (ring-assigned points only)
  float* ring_angle;  // [URF_MAX_CHANNELS] sorted registered angles (:205)
  float* max_dist;    // [URF_MAX_CHANNELS] maxDistance per ring (:271-274)
  // blindSpots / star-shaped search inputs (each may be NULL)
  int16_t* sector;    // star sector of the point (star_shaped_search.cpp:164-173, after the wrap); -1 outside the ROI or
                      // removed by the beam filter (:73-107); untouched when the star search is off
  float* q;           // [4] q1..q4 (blind_spots.cpp:13-57)
  double* A;          // [URF_MAX_CHANNELS] arcDistance / ((maxDistance[k] * M_PI) / 180) (:142), written for k >= 1
  int* reach;         // [2][361] rings window start i accepted in the forward (:68-174) / backward (:177-283) loop:
                      // 0 when ring 0 holds a curb point, n_rings when no ring does; -1 where the loop skips i or i is blind
};

namespace {

struct P {  // narrowed parameters, src/main.cpp:5-32 (double -> float / int / bool)
  bool x_zero, z_zero, star, blind;
  int xDirection;
  float interval, curbHeight;
  int curbPoints;
  float beamZone, angleFilter1, angleFilter2, angleFilter3;
  float min_X, max_X, min_Y, max_Y, min_Z, max_Z;
  float kdev, kdist;
  bool starbeam;
  int dmin;
  int channels;
};

P narrow(const urf_params* p) {
  P q;
  q.x_zero = p->x_zero_method != 0; q.z_zero = p->z_zero_method != 0; q.star = p->star_shaped_method != 0;
  q.blind = p->blind_spots != 0; q.xDirection = p->xDirection;
  q.interval = (float)p->interval; q.curbHeight = (float)p->curb_height; q.curbPoints = p->curb_points;
  q.beamZone = (float)p->beamZone;
  q.angleFilter1 = (float)p->cylinder_deg_x; q.angleFilter2 = (float)p->cylinder_deg_z; q.angleFilter3 = (float)p->curb_slope_deg;
  q.min_X = (float)p->min_x; q.max_X = (float)p->max_x; q.min_Y = (float)p->min_y; q.max_Y = (float)p->max_y;
  q.min_Z = (float)p->min_z; q.max_Z = (float)p->max_z;
  q.kdev = (float)p->kdev_param; q.kdist = (float)p->kdist_param; q.starbeam = p->starbeam_filter != 0;
  q.dmin = p->dmin_param; q.channels = p->channels;
  return q;
}

struct Ring {  // one row of array3D (lidar_segmentation.cpp:207), SoA
  std::vector<float> x, y, z, d, alpha;
  std::vector<short> label;
  std::vector<int> id;   // input index
  int n() const { return (int)x.size(); }
};

// star_shaped_search.cpp:32-66 beam_init(): per-sector rectangle parameters
struct Beam { bool yx; float o, d; };
void beam_init(Beam* beams, float* Kfi) {
  const int rep = 360;             // :8
  const float width = 0.2f;        // :9
  float fi, off = 0.5 * width;     // :35
  for (int i = 0; i < rep; i++) {
    fi = i * 2 * M_PI / rep;                                 // :38
    if (std::abs(std::tan(fi)) > 1) {                        // :39  (float overloads -> tanf)
      beams[i].yx = true;
      beams[i].d = std::tan(0.5 * M_PI - fi);                // :42  (double tan)
      beams[i].o = std::abs(off / std::sin(fi));             // :43  (sinf)
    } else {
      beams[i].yx = false;
      beams[i].d = std::tan(fi);                             // :48  (tanf)
      beams[i].o = std::abs(off / std::cos(fi));             // :49  (cosf)
    }
  }
  *Kfi = rep / (2 * M_PI);                                   // :65
}

struct Polar { int id; float r; };
bool ptcmpr(const Polar& a, const Polar& b) { return a.r < b.r; }   // star_shaped_search.cpp:22-25

// star_shaped_search.cpp:155-181 + beamfunc :68-153. mark2D[i] := 2 for the <=360 detected points (ROI order).
// Returns the number of sectors that hold an exact radius tie among their (filtered) points.
// sector_out (or NULL): per ROI point its sector, -1 when the beam filter drops it.
int star_shaped(const P& prm, const std::vector<float>& X, const std::vector<float>& Y, const std::vector<float>& Z,
                std::vector<short>& mark2D, std::vector<short>* sector_out = nullptr) {
  static Beam beams[360];
  static float Kfi = 0;
  static bool init = false;
  if (!init) { beam_init(beams, &Kfi); init = true; }
  const int s = (int)X.size();
  float slope_param = prm.angleFilter3 * (M_PI / 180);       // :160
  std::vector<std::vector<Polar>> sect(360);
  for (int i = 0; i < s; i++) {
    float r = std::sqrt(X[i] * X[i] + Y[i] * Y[i]);           // :164 (float expr -> sqrtf)
    float fi = std::atan2(Y[i], X[i]);                        // :166 (atan2f)
    if (fi < 0) fi += 2 * M_PI;                               // :168-169 (double add, narrowed)
    int f = (int)(fi * Kfi);                                  // :171
    if (f >= 360) f = 0;   // reference dereferences a null beamp[360] here (UB, SURVEY.md §7.4 H5); we wrap to sector 0
    if (f < 0) f = 0;
    sect[f].push_back(Polar{i, r});                           // :173
    if (sector_out) (*sector_out)[i] = (short)f;
  }
  int tie_sectors = 0;
  for (int tid = 0; tid < 360; tid++) {
    std::vector<Polar>& v = sect[tid];
    if (prm.starbeam) {                                       // :73-107 rectangular beam filter (order preserving erase)
      std::vector<Polar> kept;
      const Beam& b = beams[tid];
      for (const Polar& q : v) {
        bool keep;
        if (b.yx) {
          float c = b.d * Y[q.id];                            // :79
          keep = (c - b.o) < X[q.id] && X[q.id] < (c + b.o);  // :80
        } else {
          float c = b.d * X[q.id];                            // :95
          keep = (c - b.o) < Y[q.id] && Y[q.id] < (c + b.o);  // :96
        }
        if (keep) kept.push_back(q);
        else if (sector_out) (*sector_out)[q.id] = -1;
      }
      v.swap(kept);
    }
    std::sort(v.begin(), v.end(), ptcmpr);                    // :109 (same libstdc++ introsort => same tie order)
    const int n = (int)v.size();
    bool tie = false;
    for (int i = 1; i < n; i++) if (v[i].r == v[i - 1].r) tie = true;
    tie_sectors += tie;
    if (n > 1) {                                              // :112
      float kdev = prm.kdev, kdist = prm.kdist;
      int dmin = prm.dmin;
      float avg = 0, dev = 0, nan = 0;                        // :118
      float ax, ay, bx, by, slp;
      bx = v[0].r;
      by = Z[v[0].id];
      for (int i = 1; i < n; i++) {                           // :123
        ax = bx; bx = v[i].r; ay = by; by = Z[v[i].id];
        slp = (by - ay) / (bx - ax);                          // :27-30,129
        if (std::isnan(slp)) nan++;                           // :131-132
        else {
          avg *= i - nan - 1;                                 // :135
          avg += slp;                                         // :136
          avg *= 1 / (i - nan);                               // :137
          dev *= i - nan - 1;                                 // :138
          dev += std::abs(slp - avg);                         // :139
          dev *= 1 / (i - nan);                               // :140
        }
        if (slp > slope_param ||                              // :142
            (i > dmin && (slp * slp - avg * avg) * kdev * ((bx - ax) * kdist) > dev)) {   // :143
          mark2D[v[i].id] = 2;                                // :146
          break;
        }
      }
    }
  }
  return tie_sectors;
}

// lidar_segmentation.cpp:70-93: Lomuto quicksort on alpha, restated on a permutation array with an explicit stack.
void lomuto_sort(const std::vector<float>& alpha, std::vector<int>& perm) {
  std::vector<std::pair<int, int>> st;
  st.emplace_back(0, (int)perm.size() - 1);
  while (!st.empty()) {
    auto [low, high] = st.back();
    st.pop_back();
    if (low < high) {                                         // :87
      float pivot = alpha[perm[high]];                        // :72
      int i = low - 1;
      for (int j = low; j <= high - 1; j++) {
        if (alpha[perm[j]] < pivot) { i++; std::swap(perm[i], perm[j]); }   // :75-78
      }
      std::swap(perm[i + 1], perm[high]);                     // :80
      int pi = i + 1;
      // recursion order (:90-91) does not change the result; both halves are independent
      st.emplace_back(pi + 1, high);
      st.emplace_back(low, pi - 1);
    }
  }
}

template <class T> void apply_perm(std::vector<T>& v, const std::vector<int>& perm) {
  std::vector<T> t(v.size());
  for (size_t i = 0; i < v.size(); i++) t[i] = v[perm[i]];
  v.swap(t);
}

// x_zero_method.cpp:7-70
void x_zero(const P& prm, std::vector<Ring>& rings) {
  const int cp = prm.curbPoints;
  for (Ring& g : rings) {
    const int n = g.n();
    std::vector<float> newY(std::max(n, 1), 0.0f);
    for (int j = 1; j < n; j++) newY[j] = newY[j - 1] + 0.0100;   // :24-27 (double add, narrowed)
    for (int j = cp; j <= (n - 1) - cp; j++) {                    // :30
      int p2 = j + cp / 2, p3 = j + cp;
      float d = std::sqrt(std::pow(g.x[p3] - g.x[j], 2) + std::pow(g.y[p3] - g.y[j], 2));   // :35-37
      if (d < 5.0000) {
        float x1 = std::sqrt(std::pow(newY[p2] - newY[j], 2) + std::pow(g.z[p2] - g.z[j], 2));    // :42-44
        float x2 = std::sqrt(std::pow(newY[p3] - newY[p2], 2) + std::pow(g.z[p3] - g.z[p2], 2));  // :45-47
        float x3 = std::sqrt(std::pow(newY[p3] - newY[j], 2) + std::pow(g.z[p3] - g.z[j], 2));    // :48-50
        float bracket = (std::pow(x3, 2) - std::pow(x1, 2) - std::pow(x2, 2)) / (-2 * x1 * x2);  // :52
        if (bracket < -1) bracket = -1; else if (bracket > 1) bracket = 1;
        float alpha = std::acos(bracket) * 180 / M_PI;                                            // :58
        if (alpha <= prm.angleFilter1 &&
            (std::abs(g.z[j] - g.z[p2]) >= prm.curbHeight || std::abs(g.z[p3] - g.z[p2]) >= prm.curbHeight) &&
            std::abs(g.z[j] - g.z[p3]) >= 0.05) {                                                 // :61-64
          g.label[p2] = 2;
        }
      }
    }
  }
}

// z_zero_method.cpp:5-75
void z_zero(const P& prm, std::vector<Ring>& rings) {
  const int cp = prm.curbPoints;
  for (Ring& g : rings) {
    const int n = g.n();
    for (int j = cp; j <= (n - 1) - cp; j++) {                    // :21
      float d = std::sqrt(std::pow(g.x[j + cp] - g.x[j - cp], 2) + std::pow(g.y[j + cp] - g.y[j - cp], 2));   // :23-25
      if (d < 5.0000) {
        float max1, max2, va1, va2, vb1, vb2;
        max1 = max2 = std::abs(g.z[j]);                           // :31
        va1 = va2 = vb1 = vb2 = 0;
        for (int k = j - 1; k >= j - cp; k--) {                   // :35-41
          va1 = va1 + (g.x[k] - g.x[j]);
          va2 = va2 + (g.y[k] - g.y[j]);
          if (std::abs(g.z[k]) > max1) max1 = std::abs(g.z[k]);
        }
        for (int k = j + 1; k <= j + cp; k++) {                   // :44-50
          vb1 = vb1 + (g.x[k] - g.x[j]);
          vb2 = vb2 + (g.y[k] - g.y[j]);
          if (std::abs(g.z[k]) > max2) max2 = std::abs(g.z[k]);
        }
        va1 = (1 / (float)cp) * va1; va2 = (1 / (float)cp) * va2;   // :52-55
        vb1 = (1 / (float)cp) * vb1; vb2 = (1 / (float)cp) * vb2;
        float bracket = (va1 * vb1 + va2 * vb2) /
                        (std::sqrt(std::pow(va1, 2) + std::pow(va2, 2)) * std::sqrt(std::pow(vb1, 2) + std::pow(vb2, 2)));   // :57
        if (bracket < -1) bracket = -1; else if (bracket > 1) bracket = 1;
        float alpha = std::acos(bracket) * 180 / M_PI;             // :63
        if (alpha <= prm.angleFilter2 &&
            (max1 - std::abs(g.z[j]) >= prm.curbHeight || max2 - std::abs(g.z[j]) >= prm.curbHeight) &&
            std::abs(max1 - max2) >= 0.05) {                       // :66-69
          g.label[j] = 2;
        }
      }
    }
  }
}

// blind_spots.cpp:7-283. Bounded-loop form of the reference's `for (j = 0; alpha[j] <= hi && j < n; j++)` scans: the
// reference reads alpha one element past the ring before testing j (zero-initialised storage, no effect on results).
void blind_spots(const P& prm, std::vector<Ring>& rings, const std::vector<float>& maxDistance, const urf_oracle_debug* dbg) {
  const int index = (int)rings.size();
  float q1 = 0, q2 = 180, q3 = 180, q4 = 360;                     // :13
  if (prm.blind && index > 1) {                                    // :17-57 (ring index 1; empty when index < 2)
    const Ring& g = rings[1];
    for (int i = 0; i < g.n(); i++) {
      if (g.label[i] == 2) {
        float a = g.alpha[i];
        if (a >= 0 && a < 90) { if (a > q1) q1 = a; }
        else if (a >= 90 && a < 180) { if (a < q2) q2 = a; }
        else if (a >= 180 && a < 270) { if (a > q3) q3 = a; }
        else { if (a < q4) q4 = a; }
      }
    }
  }
  float arcDistance = ((maxDistance[0] * M_PI) / 180) * prm.beamZone;   // :65
  int* reach = dbg ? dbg->reach : nullptr;
  if (dbg && dbg->q) { dbg->q[0] = q1; dbg->q[1] = q2; dbg->q[2] = q3; dbg->q[3] = q4; }
  if (dbg && dbg->A) for (int k = 1; k < index; k++) dbg->A[k] = arcDistance / ((maxDistance[k] * M_PI) / 180);   // :142
  if (reach) for (int t = 0; t < 2 * 361; t++) reach[t] = -1;
  auto is_blind = [&](int i) {                                     // :72-99 / :181-208
    if (!prm.blind) return false;
    if (prm.xDirection == 0)
      return (q1 != 0 && q4 != 360 && (i <= q1 || i >= q4)) || (q2 != 180 && q3 != 180 && i >= q2 && i <= q3);
    if (prm.xDirection == 1)
      return (q2 != 180 && i >= q2 && i <= 270) || (q1 != 0 && (i <= q1 || i >= 270));
    return (q4 != 360 && (i >= q4 || i <= 90)) || (q3 != 180 && i <= q3 && i >= 90);
  };
  // forward, :68-174
  for (int i = 0; i <= 360 - prm.beamZone; i++) {
    if (is_blind(i)) continue;
    int notRoad = 0;
    Ring& g0 = rings[0];
    for (int j = 0; j < g0.n() && g0.alpha[j] <= i + prm.beamZone; j++)            // :107
      if (g0.alpha[j] >= i && g0.label[j] == 2) { notRoad = 1; break; }
    if (reach) reach[i] = 0;
    if (notRoad) continue;
    for (int j = 0; j < g0.n() && g0.alpha[j] <= i + prm.beamZone; j++)            // :124
      if (g0.alpha[j] >= i) g0.label[j] = 1;
    if (reach) reach[i] = index;
    for (int k = 1; k < index; k++) {                                              // :133
      float currentDegree;
      if (i == 360 - prm.beamZone) currentDegree = 360;                            // :136-139
      else currentDegree = i + arcDistance / ((maxDistance[k] * M_PI) / 180);      // :142
      Ring& g = rings[k];
      for (int l = 0; l < g.n() && g.alpha[l] <= currentDegree; l++)               // :146
        if (g.alpha[l] >= i && g.label[l] == 2) { notRoad = 1; break; }
      if (notRoad) { if (reach) reach[i] = k; break; }                             // :160
      for (int l = 0; l < g.n() && g.alpha[l] <= currentDegree; l++)               // :164
        if (g.alpha[l] >= i) g.label[l] = 1;
    }
  }
  // backward, :177-283
  for (int i = 360; i >= 0 + prm.beamZone; --i) {
    if (is_blind(i)) continue;
    int notRoad = 0;
    Ring& g0 = rings[0];
    for (int j = g0.n() - 1; j >= 0 && g0.alpha[j] >= i - prm.beamZone; --j)       // :216
      if (g0.alpha[j] <= i && g0.label[j] == 2) { notRoad = 1; break; }
    if (reach) reach[361 + i] = 0;
    if (notRoad) continue;
    for (int j = g0.n() - 1; j >= 0 && g0.alpha[j] >= i - prm.beamZone; --j)       // :233
      if (g0.alpha[j] <= i) g0.label[j] = 1;
    if (reach) reach[361 + i] = index;
    for (int k = 1; k < index; k++) {                                              // :242
      float currentDegree;
      if (i == 0 + prm.beamZone) currentDegree = 0;                                // :245-248
      else currentDegree = i - arcDistance / ((maxDistance[k] * M_PI) / 180);      // :251
      Ring& g = rings[k];
      for (int l = g.n() - 1; l >= 0 && g.alpha[l] >= currentDegree; --l)          // :255
        if (g.alpha[l] <= i && g.label[l] == 2) { notRoad = 1; break; }
      if (notRoad) { if (reach) reach[361 + i] = k; break; }
      for (int l = g.n() - 1; l >= 0 && g.alpha[l] >= currentDegree; --l)          // :273
        if (g.alpha[l] <= i) g.label[l] = 1;
    }
  }
}

int run(const float* xyzi, int n_in, const urf_params* up, urf_result* out, const urf_oracle_debug* dbg = nullptr) {
  const P prm = narrow(up);
  if (prm.channels < 1 || prm.channels > URF_MAX_CHANNELS) return URF_ERR_INVALID;
  out->status = URF_OK; out->n_in = n_in; out->n_roi = 0; out->n_rings = 0; out->n_order = 0;
  out->n_road = 0; out->n_curb = 0; out->n_vert = 0; out->flags = 0; out->reserved = 0;
  if (out->label) for (int i = 0; i < n_in; i++) out->label[i] = URF_LABEL_OUTSIDE;
  if (out->ring) for (int i = 0; i < n_in; i++) out->ring[i] = -1;

  // ---- ROI crop, lidar_segmentation.cpp:100-120 (+ PCL ConditionalRemoval: drops non-finite, keeps order) ----------
  std::vector<int> rid;            // input index of each ROI point
  std::vector<float> X, Y, Z;
  for (int i = 0; i < n_in; i++) {
    float x = xyzi[4 * i], y = xyzi[4 * i + 1], z = xyzi[4 * i + 2];
    if (!std::isfinite(x) || !std::isfinite(y) || !std::isfinite(z)) continue;
    if (x >= prm.min_X && x <= prm.max_X && y >= prm.min_Y && y <= prm.max_Y && z >= prm.min_Z && z <= prm.max_Z &&
        x + y + z != 0) {                                                           // :108-111
      rid.push_back(i); X.push_back(x); Y.push_back(y); Z.push_back(z);
    }
  }
  const int piece = (int)rid.size();                                               // :120
  out->n_roi = piece;
  if (piece < 30) { out->status = URF_TOO_FEW_POINTS; return 0; }                  // :124-126: nothing is published

  // ---- loop A: range, elevation angle, greedy ring registration, :128-197 -------------------------------------------
  const int channels = prm.channels;
  std::vector<float> alphaV(piece);
  std::vector<float> angle(channels, 0.0f);                                        // :136
  int index = 0;
  for (int i = 0; i < piece; i++) {
    float d = std::sqrt(std::pow(X[i], 2) + std::pow(Y[i], 2) + std::pow(Z[i], 2));   // :148 (double math, narrowed)
    float bracket = std::abs(Z[i]) / d;                                            // :151
    if (bracket < -1) bracket = -1; else if (bracket > 1) bracket = 1;
    if (Z[i] < 0) alphaV[i] = std::acos(bracket) * 180 / M_PI;                     // :162
    else alphaV[i] = (std::asin(bracket) * 180 / M_PI) + 90;                       // :165
    int newCircle = 1;
    for (int j = 0; j < channels; j++) {                                           // :174-184
      if (angle[j] == 0) break;
      if (std::abs(angle[j] - alphaV[i]) <= prm.interval) { newCircle = 0; break; }
    }
    if (newCircle == 1 && index < channels) { angle[index] = alphaV[i]; index++; } // :187-196
  }

  // ---- star shaped search on ROI order, :199-200 ---------------------------------------------------------------------
  std::vector<short> mark2D(piece, 0);
  if (prm.star) {
    std::vector<short> sector(dbg && dbg->sector ? piece : 0);
    int ties = star_shaped(prm, X, Y, Z, mark2D, dbg && dbg->sector ? &sector : nullptr);
    if (ties) out->flags |= 2;
    if (dbg && dbg->sector) for (int i = 0; i < piece; i++) dbg->sector[rid[i]] = sector[i];
  }

  std::sort(angle.begin(), angle.begin() + index);                                 // :205
  if (dbg) {
    for (int i = 0; i < piece; i++) {
      if (dbg->alpha_v) dbg->alpha_v[rid[i]] = alphaV[i];
      if (dbg->star_mark) dbg->star_mark[rid[i]] = (int8_t)mark2D[i];
    }
    if (dbg->ring_angle) for (int j = 0; j < index; j++) dbg->ring_angle[j] = angle[j];
  }

  // ---- loop B: ring buckets in input order, planar range, azimuth, :207-278 ------------------------------------------
  std::vector<Ring> rings(index);
  std::vector<float> maxDistance(std::max(index, 1), 0.0f);
  for (int i = 0; i < piece; i++) {
    int j, results = 0;
    for (j = 0; j < index; j++) {                                                  // :226-233
      if (std::abs(angle[j] - alphaV[i]) <= prm.interval) { results = 1; break; }
    }
    if (results == 1) {
      Ring& g = rings[j];
      float d = std::sqrt(std::pow(X[i], 2) + std::pow(Y[i], 2));                  // :245
      float bracket = std::abs(X[i]) / d;                                          // :248
      if (bracket < -1) bracket = -1; else if (bracket > 1) bracket = 1;
      float a;
      if (X[i] >= 0 && Y[i] <= 0) a = std::asin(bracket) * 180 / M_PI;             // :254-257
      else if (X[i] >= 0 && Y[i] > 0) a = 180 - (std::asin(bracket) * 180 / M_PI); // :258-261
      else if (X[i] < 0 && Y[i] >= 0) a = 180 + (std::asin(bracket) * 180 / M_PI); // :262-265
      else a = 360 - (std::asin(bracket) * 180 / M_PI);                            // :266-269
      g.x.push_back(X[i]); g.y.push_back(Y[i]); g.z.push_back(Z[i]); g.d.push_back(d); g.alpha.push_back(a);
      g.label.push_back(prm.star ? mark2D[i] : (short)0);                          // :241-242
      g.id.push_back(rid[i]);
      if (d > maxDistance[j]) maxDistance[j] = d;                                  // :271-274
      if (out->ring) out->ring[rid[i]] = j;
    }
  }

  if (prm.x_zero) x_zero(prm, rings);                                              // :280-281
  if (prm.z_zero) z_zero(prm, rings);                                              // :282-283

  if (dbg) {
    for (int j = 0; j < index; j++) {
      const Ring& g = rings[j];
      if (dbg->max_dist) dbg->max_dist[j] = maxDistance[j];
      for (int t = 0; t < g.n(); t++) {
        if (dbg->az) dbg->az[g.id[t]] = g.alpha[t];
        if (dbg->d2) dbg->d2[g.id[t]] = g.d[t];
        if (dbg->det_label) dbg->det_label[g.id[t]] = (int8_t)g.label[t];
      }
    }
  }

  // ---- per-ring azimuth sort, :289-291 -------------------------------------------------------------------------------
  for (Ring& g : rings) {
    const int n = g.n();
    std::vector<int> perm(n);
    for (int i = 0; i < n; i++) perm[i] = i;
    bool weird = false;
    for (int i = 0; i < n; i++) if (std::isnan(g.alpha[i])) weird = true;
    if (!weird) {
      std::stable_sort(perm.begin(), perm.end(), [&](int a, int b) { return g.alpha[a] < g.alpha[b]; });
      for (int i = 1; i < n; i++) if (g.alpha[perm[i]] == g.alpha[perm[i - 1]]) weird = true;
    }
    if (weird) {   // ties (or NaN): only the reference's own unstable Lomuto order is "the" answer
      out->flags |= 4;
      for (int i = 0; i < n; i++) perm[i] = i;
      lomuto_sort(g.alpha, perm);
    }
    apply_perm(g.x, perm); apply_perm(g.y, perm); apply_perm(g.z, perm); apply_perm(g.d, perm);
    apply_perm(g.alpha, perm); apply_perm(g.label, perm); apply_perm(g.id, perm);
  }

  blind_spots(prm, rings, maxDistance, dbg);                                       // :293

  // ---- marker candidate vertices, :298-351 ---------------------------------------------------------------------------
  int cM = 0;
  for (int i = 0; i <= 360; i++) {
    int ID1 = -1, ID2 = -1, redPoints = 0;
    float maxDistanceRoad = 0;
    for (int j = 0; j < index; j++) {
      const Ring& g = rings[j];
      for (int k = 0; k < g.n(); k++) {
        if (g.label[k] != 1 && g.alpha[k] >= i && g.alpha[k] < i + 1) { redPoints = 1; break; }   // :318-322
        if (g.label[k] == 1 && g.alpha[k] >= i && g.alpha[k] < i + 1) {                           // :325
          float d = std::sqrt(std::pow(0 - g.x[k], 2) + std::pow(0 - g.y[k], 2));                // :327 (float d, :285)
          if (d > maxDistanceRoad) { maxDistanceRoad = d; ID1 = j; ID2 = k; }
        }
      }
      if (redPoints == 1) break;                                                    // :338
    }
    if (ID1 != -1 && ID2 != -1) {                                                   // :343-350
      out->vert[cM][0] = rings[ID1].x[ID2]; out->vert[cM][1] = rings[ID1].y[ID2];
      out->vert[cM][2] = rings[ID1].z[ID2]; out->vert[cM][3] = (float)redPoints;
      cM++;
    }
  }
  out->n_vert = cM;

  // ---- outputs: labels in input order, emission order (:354-367), counts ---------------------------------------------
  out->n_rings = index;
  if (out->label) for (int i = 0; i < piece; i++) out->label[rid[i]] = URF_LABEL_NONE;
  int k = 0;
  for (int j = 0; j < index; j++) {
    if (out->ring_start) out->ring_start[j] = k;
    const Ring& g = rings[j];
    for (int t = 0; t < g.n(); t++) {
      if (out->label) out->label[g.id[t]] = g.label[t];
      if (out->order) out->order[k] = g.id[t];
      if (g.label[t] == 1) out->n_road++;
      else if (g.label[t] == 2) out->n_curb++;
      k++;
    }
  }
  if (out->ring_start) out->ring_start[index] = k;
  out->n_order = k;
  return 0;
}

}  // namespace

extern "C" {

int urf_oracle_run(const float* xyzi, int n, const urf_params* prm, urf_result* out) {
  if (!xyzi || !prm || !out || n < 0) return URF_ERR_INVALID;
  return run(xyzi, n, prm, out);
}

int urf_oracle_run_debug(const float* xyzi, int n, const urf_params* prm, urf_result* out, const urf_oracle_debug* dbg) {
  if (!xyzi || !prm || !out || n < 0) return URF_ERR_INVALID;
  return run(xyzi, n, prm, out, dbg);
}

// seconds for `repeat` full passes over one cloud (labels/order buffers allocated once, outside the timed region)
double urf_oracle_time(const float* xyzi, int n, const urf_params* prm, int repeat) {
  std::vector<int32_t> label(n > 0 ? n : 1), order(n > 0 ? n : 1);
  urf_result r;
  std::memset(&r, 0, sizeof(r));
  r.label = label.data(); r.order = order.data();
  auto t0 = std::chrono::steady_clock::now();
  for (int i = 0; i < repeat; i++) run(xyzi, n, prm, &r);
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

}  // extern "C"
