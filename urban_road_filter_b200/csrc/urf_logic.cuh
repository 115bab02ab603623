// urf_logic.cuh — the per-element logic of the path as host+device functions.
//
// Everything that decides a label lives here, written with the URF_F*/URF_D* round-to-nearest macros of urf_math.cuh in
// exactly the operation order of the reference (file:line cited; paths relative to the reference repo). The CUDA kernels
// (urf_kernels.cuh) only add indexing, staging and synchronisation around these functions. Because the same functions
// also compile for the host (g++ -ffp-contract=off), tests/kat/model_check.cpp runs them sequentially on the CPU and
// diffs every stage against the oracle without needing a GPU.
#pragma once
#include <math.h>

#include "urf_device.cuh"
#include "urf_math.cuh"

#if defined(__CUDA_ARCH__)
#define URF_D2F(x) __double2float_rn((x))
#define URF_F2I_RZ(x) __float2int_rz((x))
#else
#define URF_D2F(x) ((float)(x))
#define URF_F2I_RZ(x) ((int)(x))
#endif

#define URF_TWO_PI_D 6.283185307179586476925286766559

namespace urf {

URF_HD unsigned fbits(float f) { return (unsigned)URF_F2I(f); }
URF_HD float bitsf(unsigned u) { return URF_I2F((int32_t)u); }
URF_HD double dsq(float a) { return URF_DMUL((double)a, (double)a); }      // pow(float, 2): exact in double

// tail of every `acos(..) * 180 / M_PI` of the reference: float multiply, then double divide (urfm::div_pi: the same
// correctly rounded quotient from two FMAs)
// (every caller passes rad >= +0: acosf(.) or asinf(b) with b >= 0)
URF_HD double deg_d(float rad) { return urfm::div_pi_nonneg((double)URF_FMUL(rad, 180.0f)); }

URF_HD float clamp_unit(float b) {   // lidar_segmentation.cpp:154-157 (NaN passes through)
  if (b < -1.0f) return -1.0f;
  if (b > 1.0f) return 1.0f;
  return b;
}

// ROI crop predicate, lidar_segmentation.cpp:106-113 (+ PCL ConditionalRemoval drops non-finite xyz)
// The six bounds are finite (validate_params), so a coordinate that passes its two compares is finite itself: NaN fails
// every compare, an infinity lies outside any finite interval — PCL's non-finite test needs no instructions of its own.
URF_HD bool roi_keep(const DevParams& prm, float x, float y, float z) {
  return x >= prm.min_X && x <= prm.max_X && y >= prm.min_Y && y <= prm.max_Y && z >= prm.min_Z && z <= prm.max_Z &&
         URF_FADD(URF_FADD(x, y), z) != 0.0f;
}

// elevation angle in degrees, lidar_segmentation.cpp:148-166
URF_HD float elev_alpha(float x, float y, float z) {
  const float d = URF_D2F(URF_DSQRT(URF_DADD(URF_DADD(dsq(x), dsq(y)), dsq(z))));     // :148
  const float br = clamp_unit(URF_FDIV(fabsf(z), d));                                  // :151-157
  if (z < 0.0f) return URF_D2F(deg_d(urfm::acosf_glibc(br)));                          // :162
  return URF_D2F(URF_DADD(deg_d(urfm::asinf_glibc(br)), 90.0));                        // :165
}

// planar range and azimuth, lidar_segmentation.cpp:245-269; sxy = (double)x*x + (double)y*y (the caller may share it)
URF_HD void planar_az_from(float x, float y, double sxy, float* d_out, float* az_out) {
  const float d = URF_D2F(URF_DSQRT(sxy));
  const float br = clamp_unit(URF_FDIV(fabsf(x), d));
  const double t = deg_d(urfm::asinf_glibc(br));
  // the four quadrant cases t, 180 - t, 180 + t, 360 - t (:257-268) as c + s * t: negating t is exact, and 0 + t is t
  // itself for t >= +0, so one double addition serves all four (NaN coordinates cannot reach this point)
  const bool xp = x >= 0.f;
  const double c = xp ? (y <= 0.f ? 0.0 : 180.0) : (y >= 0.f ? 180.0 : 360.0);
  const bool neg = xp ? !(y <= 0.f) : !(y >= 0.f);
  *d_out = d;
  *az_out = URF_D2F(URF_DADD(c, neg ? -t : t));
}
URF_HD void planar_az(float x, float y, float* d_out, float* az_out) { planar_az_from(x, y, URF_DADD(dsq(x), dsq(y)), d_out, az_out); }

// everything k_points derives from one point: elevation angle (:148-166) and planar range / azimuth (:245-269), with the
// squares shared: (x*x + y*y) + z*z is the reference's left-to-right sum, x*x + y*y its planar one
URF_HD void point_angles(float x, float y, float z, float* alpha, float* d2, float* az) {
  const double sxy = URF_DADD(dsq(x), dsq(y));
  const float d = URF_D2F(URF_DSQRT(URF_DADD(sxy, dsq(z))));                           // :148
  const float br = clamp_unit(URF_FDIV(fabsf(z), d));                                  // :151-157
  *alpha = z < 0.0f ? URF_D2F(deg_d(urfm::acosf_glibc(br)))                            // :162
                    : URF_D2F(URF_DADD(deg_d(urfm::asinf_glibc(br)), 90.0));           // :165
  planar_az_from(x, y, sxy, d2, az);
}

// maxDistance[k] (lidar_segmentation.cpp:271-274) is the largest (float)sqrt((double)x*x + y*y) of the ring. Square root
// and narrowing are both monotone, so it equals (float)sqrt(max of the double sums): the kernels keep the maximum of the
// sums (non-negative doubles order like their bit patterns) and take one square root per ring.
URF_HD unsigned long long planar_sum_bits(float x, float y) {
#if defined(__CUDA_ARCH__)
  return (unsigned long long)__double_as_longlong(URF_DADD(dsq(x), dsq(y)));
#else
  const double s = URF_DADD(dsq(x), dsq(y)); unsigned long long u; memcpy(&u, &s, 8); return u;
#endif
}
URF_HD float maxdist_from_bits(unsigned long long u) {
#if defined(__CUDA_ARCH__)
  return URF_D2F(URF_DSQRT(__longlong_as_double((long long)u)));
#else
  double s; memcpy(&s, &u, 8); return URF_D2F(URF_DSQRT(s));
#endif
}

// star-shaped sector of a point, star_shaped_search.cpp:164-173: f = (int)(fi * Kfi) with fi = atan2f(y, x), wrapped into
// [0, 2 pi). The exact index needs glibc's atan2f bit for bit:
URF_HD int star_sector_exact(const DevParams& prm, float x, float y) {
  float fi = urfm::atan2f_glibc(y, x);                                       // :166
  if (fi < 0.0f) fi = URF_D2F(URF_DADD((double)fi, URF_TWO_PI_D));           // :168-169
  int f = URF_F2I_RZ(URF_FMUL(fi, prm.Kfi));                                 // :171
  if (f >= kSectKeys || f < 0) f = 0;   // reference: null-pointer dereference for f == 360 (UB, SURVEY.md H5); we wrap
  return f;
}
// ... but only the INTEGER part of fi * Kfi is used, so a cheap angle decides almost every point: a degree-13 odd polynomial
// for atan on [0, 1] (|error| < 3.5e-7 rad), octant fix-ups, degrees = angle * 57.29578. The value the reference computes
// lies within 6e-5 degrees of the true angle in degrees (atan2f < 1 ulp, the float rounding of fi + 2 pi, of the product and
// of Kfi), the cheap one within 3e-5; when the cheap value is at least 1e-3 degrees away from both neighbouring integers
// the two truncate to the same sector. Everything else (boundaries, the 0/360 wrap, zero / non-finite input) returns -1
// and takes the exact path. tests/kat/math_sweep.cpp checks "fast < 0 or fast == exact" on random and on near-boundary
// points; the arithmetic is the same on host and device (single roundings, fmaf).
URF_HD int star_sector_fast(float x, float y) {
  const float ax = fabsf(x), ay = fabsf(y);
  const bool steep = ay > ax;
  // tan of the angle to the nearer axis, in [0, 1]. The device may take the 2-ulp fast division here: it moves the angle by
  // < 3e-7 rad, far inside the 1e-3 degree margin below, and either way a decided sector is the reference's sector
#if defined(__CUDA_ARCH__)
  const float t = __fdividef(steep ? ax : ay, steep ? ay : ax);
#else
  const float t = URF_FDIV(steep ? ax : ay, steep ? ay : ax);
#endif
  const float s = URF_FMUL(t, t);
  float p = 0.006811792496591806f;
  p = URF_FFMA(p, s, -0.0336042195558548f);
  p = URF_FFMA(p, s, 0.07962366938591003f);
  p = URF_FFMA(p, s, -0.1323334276676178f);
  p = URF_FFMA(p, s, 0.19807815551757812f);
  p = URF_FFMA(p, s, -0.3331736922264099f);
  p = URF_FFMA(p, s, 0.9999961256980896f);
  float a = URF_FMUL(t, p);                                                   // atan(t) in [0, pi / 4]
  if (steep) a = URF_FSUB(1.57079637f, a);
  if (x < 0.0f) a = URF_FSUB(3.14159274f, a);
  if (y < 0.0f) a = URF_FSUB(6.28318548f, a);
  const float u = URF_FMUL(a, 57.2957802f);                                   // degrees in [0, 360]
  const int f = URF_F2I_RZ(u);
  const float fr = URF_FSUB(u, (float)f);
  return (fr > 1e-3f && fr < 0.999f && f >= 0 && f < kSectKeys) ? f : -1;     // NaN / inf fail the compares
}
// sector or -1 (outside the rectangular beam filter :73-107)
URF_HD int star_sector(const DevParams& prm, float x, float y, const float* beam_d, const float* beam_o,
                       const unsigned char* beam_yx) {
  int f = star_sector_fast(x, y);
  if (f < 0) f = star_sector_exact(prm, x, y);
  if (prm.starbeam) {                                                        // :73-107
    const float bd = beam_d[f], bo = beam_o[f];
    if (beam_yx[f]) { const float c = URF_FMUL(bd, y); if (!(URF_FSUB(c, bo) < x && x < URF_FADD(c, bo))) return -1; }
    else            { const float c = URF_FMUL(bd, x); if (!(URF_FSUB(c, bo) < y && y < URF_FADD(c, bo))) return -1; }
  }
  return f;
}
URF_HD float star_radius(float x, float y) { return URF_FSQRT(URF_FADD(URF_FMUL(x, x), URF_FMUL(y, y))); }   // :164

// ring of an elevation angle: first sorted registered angle within `interval` (lidar_segmentation.cpp:226-233).
// *lo_out = first j with angle[j] - a >= -interval (float subtraction is monotone in angle[j]).
URF_HD int assign_ring(const float* angle, int R, float a, float interval, int* lo_out) {
  int lo = 0, hi = R;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (URF_FSUB(angle[mid], a) >= -interval) hi = mid; else lo = mid + 1;
  }
  *lo_out = lo;
  return (lo < R && fabsf(URF_FSUB(angle[lo], a)) <= interval) ? lo : -1;    // :228
}

// Fine elevation bin of an angle (speculation bins of k_points and the ring-search lookup table); monotone in a.
URF_HD int elev_bin(float a) {
  int bin = (int)(a * (kElevBins / 180.0f));
  return bin < 0 ? 0 : (bin > kElevBins ? kElevBins : bin);
}
// Lookup table entry for elevation bin e: the ring search start for an angle one whole bin below e, which is <= the
// search start of every angle that falls into bin e (assign_ring's `lo` is non-decreasing in the angle).
URF_HD int ring_lut_entry(const float* angle, int R, float interval, int e) {
  int lo;
  assign_ring(angle, R, (float)(e - 1) * (180.0f / kElevBins), interval, &lo);
  return lo;
}
// assign_ring with the binary search replaced by a short linear walk from a lookup-table start (start <= lo)
URF_HD int assign_ring_from(const float* angle, int R, float a, float interval, int start, int* lo_out) {
  int lo = start;
  while (lo < R && !(URF_FSUB(angle[lo], a) >= -interval)) lo++;
  *lo_out = lo;
  return (lo < R && fabsf(URF_FSUB(angle[lo], a)) <= interval) ? lo : -1;    // :228
}

// Verification of a speculated registration for input point i (see k_register): true = the sequential algorithm of
// lidar_segmentation.cpp:170-196 would have behaved differently at this point, i.e. the speculation is wrong.
URF_HD bool registration_violation(const float* angle, const int* regidx, const int* regorder, int R, int channels,
                                   float interval, float a, int i, int lo) {
  // common case first: the first covering angle was itself registered at or before point i
  if (lo < R && regidx[lo] <= i && fabsf(URF_FSUB(angle[lo], a)) <= interval) return false;
  int minreg = 0x7fffffff;
  for (int j = lo; j < R && fabsf(URF_FSUB(angle[j], a)) <= interval; j++) minreg = regidx[j] < minreg ? regidx[j] : minreg;
  if (minreg <= i) return false;           // covered by an angle registered at or before i (== i: i is the registrant)
  int l2 = 0, h2 = R;                      // registrants with input index < i
  while (l2 < h2) { const int mid = (l2 + h2) >> 1; if (regorder[mid] < i) l2 = mid + 1; else h2 = mid; }
  return l2 < channels;                    // uncovered and room left: it would have registered
}

// A ring's points in ring order, as the two detectors read them: array-of-float4 (global memory, host model) or three
// separate coordinate arrays (the shared-memory tiles of the ring detectors). q = local index inside the ring.
struct RingAoS {
  const float4* p;
  URF_HDM float x(int q) const { return p[q].x; }
  URF_HDM float y(int q) const { return p[q].y; }
  URF_HDM float z(int q) const { return p[q].z; }
};
struct RingSoA {
  const float *px, *py, *pz;
  URF_HDM float x(int q) const { return px[q]; }
  URF_HDM float y(int q) const { return py[q]; }
  URF_HDM float z(int q) const { return pz[q]; }
};

// x-zero test with local index m as the middle point p2 = j + cp/2 (x_zero_method.cpp:30-67), split in two: the index
// range + height gate (cheap, float only; false for most points) and the triangle-angle test behind it. The kernel runs
// the second half only for the points that pass the first (compacted per CTA); xzero_mark_t is both, for the host model.
// CP > 0: curb_points known at compile time; CP == 0: taken from the parameters. Same arithmetic either way.
template <int CP, class RV>
URF_HD bool xzero_pre_t(const DevParams& prm, const RV& ring, int n, int m) {
  const int cp = CP > 0 ? CP : prm.curbPoints;
  const int j = m - cp / 2;
  if (!(j >= cp && j <= (n - 1) - cp)) return false;
  const float az = ring.z(j), cz = ring.z(j + cp), z = ring.z(m);
  return (fabsf(URF_FSUB(az, z)) >= prm.curbHeight || fabsf(URF_FSUB(cz, z)) >= prm.curbHeight) &&
         (double)fabsf(URF_FSUB(az, cz)) >= 0.05;                                                             // :62-64
}
template <class RV>
URF_HD bool xzero_post(const DevParams& prm, const RV& ring, int m, const float* newY) {
  const int cp = prm.curbPoints;
  const int j = m - cp / 2, p3 = j + cp;
  const float az = ring.z(j), cz = ring.z(p3), z = ring.z(m);
  const float dd = URF_D2F(URF_DSQRT(URF_DADD(dsq(URF_FSUB(ring.x(p3), ring.x(j))), dsq(URF_FSUB(ring.y(p3), ring.y(j))))));   // :35-37
  if (!((double)dd < 5.0)) return false;                                                                      // :40
  const float yj = newY[j], y2 = newY[m], y3 = newY[p3];
  const float x1 = URF_D2F(URF_DSQRT(URF_DADD(dsq(URF_FSUB(y2, yj)), dsq(URF_FSUB(z, az)))));                // :42-44
  const float x2 = URF_D2F(URF_DSQRT(URF_DADD(dsq(URF_FSUB(y3, y2)), dsq(URF_FSUB(cz, z)))));                // :45-47
  const float x3 = URF_D2F(URF_DSQRT(URF_DADD(dsq(URF_FSUB(y3, yj)), dsq(URF_FSUB(cz, az)))));               // :48-50
  const double num = URF_DSUB(URF_DSUB(dsq(x3), dsq(x1)), dsq(x2));
  const float den = URF_FMUL(URF_FMUL(-2.0f, x1), x2);
  const float bk = clamp_unit(URF_D2F(URF_DDIV(num, (double)den)));                                           // :52-56
  const float al = URF_D2F(deg_d(urfm::acosf_glibc(bk)));                                                     // :58
  return al <= prm.angleFilter1;                                                                              // :61
}
template <int CP>
URF_HD bool xzero_mark_t(const DevParams& prm, const float4* ring, int n, int m, const float* newY) {
  const RingAoS rv{ring};
  return xzero_pre_t<CP>(prm, rv, n, m) && xzero_post(prm, rv, m, newY);
}

// z-zero test centred on local index m (z_zero_method.cpp:21-72), split the same way, with the same CP convention (loops
// unroll when CP > 0).
template <int CP, class RV>
URF_HD bool zzero_pre_t(const DevParams& prm, const RV& ring, int n, int m) {
  const int cp = CP > 0 ? CP : prm.curbPoints;
  if (!(m >= cp && m <= (n - 1) - cp)) return false;
  const float az0 = fabsf(ring.z(m));
  float max1 = az0, max2 = az0;
#pragma unroll
  for (int u = 1; u <= cp; u++) { const float v = fabsf(ring.z(m - u)); if (v > max1) max1 = v; }            // :38-40 (k = j-1 .. j-cp)
#pragma unroll
  for (int u = 1; u <= cp; u++) { const float v = fabsf(ring.z(m + u)); if (v > max2) max2 = v; }            // :47-49 (k = j+1 .. j+cp)
  return (URF_FSUB(max1, az0) >= prm.curbHeight || URF_FSUB(max2, az0) >= prm.curbHeight) &&
         (double)fabsf(URF_FSUB(max1, max2)) >= 0.05;                                                         // :67-69
}
template <int CP, class RV>
URF_HD bool zzero_post_t(const DevParams& prm, const RV& ring, int m) {
  const int cp = CP > 0 ? CP : prm.curbPoints;
  const float dd = URF_D2F(URF_DSQRT(URF_DADD(dsq(URF_FSUB(ring.x(m + cp), ring.x(m - cp))), dsq(URF_FSUB(ring.y(m + cp), ring.y(m - cp))))));   // :23-25
  if (!((double)dd < 5.0)) return false;                                                                      // :28
  const float mx = ring.x(m), my = ring.y(m);
  float va1 = 0.f, va2 = 0.f, vb1 = 0.f, vb2 = 0.f;
#pragma unroll
  for (int u = 1; u <= cp; u++) { va1 = URF_FADD(va1, URF_FSUB(ring.x(m - u), mx)); va2 = URF_FADD(va2, URF_FSUB(ring.y(m - u), my)); }   // :35-37, same order
#pragma unroll
  for (int u = 1; u <= cp; u++) { vb1 = URF_FADD(vb1, URF_FSUB(ring.x(m + u), mx)); vb2 = URF_FADD(vb2, URF_FSUB(ring.y(m + u), my)); }   // :44-46
  const float sc = URF_FDIV(1.0f, (float)cp);
  va1 = URF_FMUL(sc, va1); va2 = URF_FMUL(sc, va2); vb1 = URF_FMUL(sc, vb1); vb2 = URF_FMUL(sc, vb2);        // :52-55
  const float dot = URF_FADD(URF_FMUL(va1, vb1), URF_FMUL(va2, vb2));
  const double nrm = URF_DMUL(URF_DSQRT(URF_DADD(dsq(va1), dsq(va2))), URF_DSQRT(URF_DADD(dsq(vb1), dsq(vb2))));
  const float bk = clamp_unit(URF_D2F(URF_DDIV((double)dot, nrm)));                                           // :57-61
  const float al = URF_D2F(deg_d(urfm::acosf_glibc(bk)));                                                     // :63
  return al <= prm.angleFilter2;                                                                              // :66
}
template <int CP>
URF_HD bool zzero_mark_t(const DevParams& prm, const float4* ring, int n, int m) {
  const RingAoS rv{ring};
  return zzero_pre_t<CP>(prm, rv, n, m) && zzero_post_t<CP>(prm, rv, m);
}

// Edge search along one radius-sorted sector (star_shaped_search.cpp:112-150) as a step function: state after point
// i-1, fed point i (planar radius r, height z); returns true when point i gets marked (the scan then stops).
struct StarState { float avg, dev, nan, bx, by; };
URF_HD void star_init(StarState& s, float r0, float z0) { s.avg = 0.f; s.dev = 0.f; s.nan = 0.f; s.bx = r0; s.by = z0; }   // :118-121
// slope between consecutive radius-sorted points (:27-30,125-129); *dx = r - r_prev
URF_HD float star_slope(float r_prev, float z_prev, float r, float z, float* dx) {
  *dx = URF_FSUB(r, r_prev);
  return URF_FDIV(URF_FSUB(z, z_prev), *dx);
}
URF_HD float star_inv(int i) { return URF_FDIV(1.0f, (float)i); }       // 1 / (i - nan) while nan == 0
// running mean / average absolute deviation update and edge test for point i (:131-148); inv_i = star_inv(i)
URF_HD bool star_update(const DevParams& prm, StarState& s, int i, float slp, float dxk /* (bx - ax) * kdist */, float inv_i) {
  if (isnan(slp)) s.nan = URF_FADD(s.nan, 1.0f);                        // :131-132
  else {
    const float im = URF_FSUB((float)i, s.nan);                         // i - nan
    const float c1 = URF_FSUB(im, 1.0f);                                // i - nan - 1
    const float c2 = s.nan == 0.0f ? inv_i : URF_FDIV(1.0f, im);        // 1 / (i - nan)
    s.avg = URF_FMUL(s.avg, c1); s.avg = URF_FADD(s.avg, slp); s.avg = URF_FMUL(s.avg, c2);                    // :135-137
    s.dev = URF_FMUL(s.dev, c1); s.dev = URF_FADD(s.dev, fabsf(URF_FSUB(slp, s.avg))); s.dev = URF_FMUL(s.dev, c2);   // :138-140
  }
  const float lhs = URF_FMUL(URF_FMUL(URF_FSUB(URF_FMUL(slp, slp), URF_FMUL(s.avg, s.avg)), prm.kdev), dxk);   // :143
  return slp > prm.slope_param || (i > prm.dmin && lhs > s.dev);        // :142-143
}
URF_HD bool star_step(const DevParams& prm, StarState& s, int i, float r, float z) {
  float dx;
  const float slp = star_slope(s.bx, s.by, r, z, &dx);
  s.bx = r; s.by = z;
  return star_update(prm, s, i, slp, URF_FMUL(dx, prm.kdist), star_inv(i));
}
// whole sector at once: pts[i] = (r, z, -, -); returns the local index of the marked point or -1
URF_HD int star_scan_sector(const DevParams& prm, const float4* pts, int n) {
  if (n <= 1) return -1;                                                // :112
  StarState st;
  star_init(st, pts[0].x, pts[0].y);
  for (int i = 1; i < n; i++)                                           // :123
    if (star_step(prm, st, i, pts[i].x, pts[i].y)) return i;            // :146
  return -1;
}

// ---------------------------------------------------------------------------------------------------------------------
// blindSpots as tables (blind_spots.cpp:7-283). The curb set is fixed while blindSpots runs (it only ever writes 1, and
// never into a window that holds a 2), so a point ends as road iff some non-blind window start i of either direction
// accepts the point's ring (no curb in rings 0..k inside the window) and the point's azimuth lies in the window.
// Curb points are summarised per (ring, integer-degree bin): min and max curb azimuth and a prefix count of non-empty bins.
struct CurbView {
  const unsigned* cmin; const unsigned* cmax; const unsigned short* ne;   // tables of one scan
  URF_HDM float mn(int k, int bin) const { return bitsf(cmin[(size_t)k * kDegBins + bin]); }   // +inf when empty
  URF_HDM float mx(int k, int bin) const { return bitsf(cmax[(size_t)k * kDegBins + bin]); }   // 0 when empty
  URF_HDM int cnt(int k, int b0, int b1) const {                          // non-empty bins in [b0, b1)
    if (b1 <= b0) return 0;
    return (int)ne[(size_t)k * (kDegBins + 1) + b1] - (int)ne[(size_t)k * (kDegBins + 1) + b0];
  }
  // any curb point of ring k with (float)i <= azimuth <= hi   (blind_spots.cpp:107-117,146-157)
  URF_HDM bool fwd(int k, int i, float hi) const {
    if (!(hi >= (float)i)) return false;
    const int fb = hi >= 361.0f ? 361 : (int)hi;
    if (cnt(k, i, fb) > 0) return true;
    return fb <= 360 && mn(k, fb) <= hi;
  }
  // any curb point of ring k with lo <= azimuth <= (float)i   (blind_spots.cpp:216-227,255-266)
  URF_HDM bool bwd(int k, int i, float lo) const {
    if (!(lo <= (float)i)) return false;
    if (mn(k, i) <= (float)i) return true;                               // azimuth == i exactly
    if (lo <= 0.0f) return cnt(k, 0, i) > 0;
    const int lb = (int)lo;
    if (lb >= i) return false;
    if (mx(k, lb) >= lo) return true;
    return cnt(k, lb + 1, i) > 0;
  }
};

URF_HD float fwd_hi(const DevParams& prm, int k, int i, double A) {
  if (k == 0) return URF_FADD((float)i, prm.beamZone);                                     // blind_spots.cpp:107
  if (i == prm.fwd_special) return 360.0f;                                                 // :136-139
  return URF_D2F(URF_DADD((double)i, A));                                                  // :142
}
URF_HD float bwd_lo(const DevParams& prm, int k, int i, double A) {
  if (k == 0) return URF_FSUB((float)i, prm.beamZone);                                     // :216
  if (i == prm.bwd_special) return 0.0f;                                                   // :245-248
  return URF_D2F(URF_DSUB((double)i, A));                                                  // :251
}

// arcDistance (blind_spots.cpp:65) and the per-ring width arcDistance / ((maxDistance[k] * M_PI) / 180) (:142)
URF_HD float arc_distance(const DevParams& prm, float maxdist0) {
  return URF_D2F(URF_DMUL(URF_DDIV(URF_DMUL((double)maxdist0, URF_PI_D), 180.0), (double)prm.beamZone));
}
URF_HD double ring_width(float arc, float maxdist_k) {
  return URF_DDIV((double)arc, URF_DDIV(URF_DMUL((double)maxdist_k, URF_PI_D), 180.0));
}

URF_HD bool is_blind(const DevParams& prm, const float* q, int i) {                        // blind_spots.cpp:72-99,181-208
  if (!prm.blind) return false;
  const float fi = (float)i, q1 = q[0], q2 = q[1], q3 = q[2], q4 = q[3];
  if (prm.xDirection == 0)
    return (q1 != 0.f && q4 != 360.f && (fi <= q1 || fi >= q4)) || (q2 != 180.f && q3 != 180.f && fi >= q2 && fi <= q3);
  if (prm.xDirection == 1)
    return (q2 != 180.f && fi >= q2 && i <= 270) || (q1 != 0.f && (fi <= q1 || i >= 270));
  return (q4 != 360.f && (fi >= q4 || i <= 90)) || (q3 != 180.f && fi <= q3 && i >= 90);
}

// q1..q4 from the curb bins of ring index 1 (blind_spots.cpp:13-57); which = 0..3
URF_HD float blind_quarter(const DevParams& prm, const CurbView& cv, int R, int which) {
  float q = which == 0 ? 0.f : which == 3 ? 360.f : 180.f;
  if (prm.blind && R > 1) {
    const int b0 = which * 90, b1 = which == 3 ? 361 : b0 + 90;
    for (int bin = b0; bin < b1; bin++) {
      if (cv.cmin[(size_t)kDegBins + bin] == 0x7f800000u) continue;
      if (which == 0 || which == 2) { const float v = cv.mx(1, bin); if (v > q) q = v; }
      else { const float v = cv.mn(1, bin); if (v < q) q = v; }
    }
  }
  return q;
}

// number of rings window start i accepts: forward (blind_spots.cpp:68-174) dir = 0, backward (:177-283) dir = 1
URF_HD int window_reach(const DevParams& prm, const CurbView& cv, const double* A, const float* q, int R, int dir, int i) {
  const bool in_loop = dir == 0 ? (i <= prm.fwd_last) : (i >= prm.bwd_first);
  if (!in_loop || is_blind(prm, q, i)) return 0;
  int k = 0;
  for (; k < R; k++) {
    const bool curb = dir == 0 ? cv.fwd(k, i, fwd_hi(prm, k, i, A[k])) : cv.bwd(k, i, bwd_lo(prm, k, i, A[k]));
    if (curb) break;
  }
  return k;
}

// Reference formulation of the per-point window test (search for the window start range + range-max over reach); kept
// for the CPU model, which checks that the threshold tables above give the same answer for every point.
struct SparseMax { unsigned short st[2][kStLevels][kDegBins]; };
URF_HD int st_max(const SparseMax& tab, int dir, int lo, int hi) {                           // max reach over [lo, hi]
  if (hi < lo) return 0;
  int l = 0;
  while ((2 << l) <= hi - lo + 1) l++;
  const unsigned short a = tab.st[dir][l][lo], c = tab.st[dir][l][hi - (1 << l) + 1];
  return a > c ? a : c;
}

// road iff a forward or backward window start accepts ring k and contains azimuth a
URF_HD bool covered_by_window(const DevParams& prm, const SparseMax& tab, double A, int k, float a) {
  if (!(a >= 0.0f)) return false;
  const double w = k == 0 ? (double)prm.beamZone : A;
  {  // forward: (float)i <= a and a <= hi(i); hi(i) >= a is monotone (false..false,true..true) in i
    int imax = (int)a; if (imax > prm.fwd_last) imax = prm.fwd_last;
    if (imax >= 0) {
      const double e = ceil((double)a - w);
      int est = !(e >= 0.0) ? 0 : (e > (double)(imax + 1) ? imax + 1 : (int)e);
      while (est > 0 && fwd_hi(prm, k, est - 1, A) >= a) est--;
      while (est <= imax && !(fwd_hi(prm, k, est, A) >= a)) est++;
      if (est <= imax && st_max(tab, 0, est, imax) > k) return true;
    }
  }
  {  // backward: a <= (float)i and lo(i) <= a; lo(i) <= a is monotone (true..true,false..false) in i
    int imin = (int)a; if ((float)imin < a) imin++;
    if (imin < prm.bwd_first) imin = prm.bwd_first;
    if (imin <= 360) {
      const double e = floor((double)a + w);
      int est = !(e <= 360.0) ? 360 : (e < (double)(imin - 1) ? imin - 1 : (int)e);
      while (est < 360 && bwd_lo(prm, k, est + 1, A) <= a) est++;
      while (est >= imin && !(bwd_lo(prm, k, est, A) <= a)) est--;
      if (est >= imin && st_max(tab, 1, imin, est) > k) return true;
    }
  }
  return false;
}

// Threshold tables: for ring k and integer degree j, Tf[k][j] = hi_k(i*) with i* the LARGEST accepted window start
// i <= j (forward), Tb[k][j] = lo_k(i*) with i* the SMALLEST accepted start i >= j (backward). hi_k and lo_k are
// non-decreasing in i, so a point of ring k with azimuth a is covered iff a <= Tf[k][floor(a)] or Tb[k][ceil(a)] <= a.
// `accepted`: i inside the loop range, not blind, and reach[dir][i] > k. Row stride kTStride.
constexpr int kTStride = kDegBins + 3;
URF_HD bool accepted_fwd(const DevParams& prm, const int* reach_f, const float* q, int k, int j) {
  return j <= prm.fwd_last && reach_f[j] > k && !is_blind(prm, q, j);
}
URF_HD bool accepted_bwd(const DevParams& prm, const int* reach_b, const float* q, int k, int j) {
  return j >= prm.bwd_first && reach_b[j] > k && !is_blind(prm, q, j);
}
URF_HD float T_fwd_value(const DevParams& prm, int k, int last, double A) { return last >= 0 ? fwd_hi(prm, k, last, A) : -INFINITY; }
URF_HD float T_bwd_value(const DevParams& prm, int k, int nxt, double A) { return nxt <= 360 ? bwd_lo(prm, k, nxt, A) : INFINITY; }
URF_HD void build_T_row(const DevParams& prm, const int* reach_f, const int* reach_b, const float* q, int k, double A,
                        float* Tf, float* Tb) {
  int last = -1;
  for (int j = 0; j < kDegBins; j++) {
    if (accepted_fwd(prm, reach_f, q, k, j)) last = j;
    Tf[j] = T_fwd_value(prm, k, last, A);
  }
  int nxt = 361;
  for (int j = kDegBins - 1; j >= 0; j--) {
    if (accepted_bwd(prm, reach_b, q, k, j)) nxt = j;
    Tb[j] = T_bwd_value(prm, k, nxt, A);
  }
}
// table columns an azimuth a in [0, 360] looks at: j = floor(a) (also its degree bin), jc = ceil(a)
URF_HD void T_indices(float a, int* j_out, int* jc_out) {
  int j = (int)a; if (j > 360) j = 360;
  int jc = j; if ((float)jc < a) jc++; if (jc > 360) jc = 360;
  *j_out = j; *jc_out = jc;
}
URF_HD bool covered_from(float a, float tf, float tb) { return a <= tf || tb <= a; }
URF_HD bool covered_T(const float* Tf, const float* Tb, int k, float a) {
  if (!(a >= 0.0f)) return false;
  int j, jc;
  T_indices(a, &j, &jc);
  return covered_from(a, Tf[(size_t)k * kTStride + j], Tb[(size_t)k * kTStride + jc]);
}
// first ring with a curb point inside window start i of direction dir, given the per-cell test (k_reach evaluates the
// cells in parallel and keeps the minimum): true when ring k blocks window i
URF_HD bool window_blocked(const DevParams& prm, const CurbView& cv, double A, int dir, int i, int k) {
  return dir == 0 ? cv.fwd(k, i, fwd_hi(prm, k, i, A)) : cv.bwd(k, i, bwd_lo(prm, k, i, A));
}

// integer-degree bin of an azimuth (lidar_segmentation.cpp:318: `alpha >= i && alpha < i + 1`), a >= 0
URF_HD int deg_bin(float a) { int bin = (int)a; return bin > 360 ? 360 : bin; }

// Marker candidate vertices (lidar_segmentation.cpp:305-351): keys that order points inside the reference's scan order
URF_HD unsigned long long cut_key(unsigned az_bits, int p) { return ((unsigned long long)az_bits << 32) | (unsigned)p; }
URF_HD unsigned long long best_key(int k, unsigned az_bits, int p) {
  return ((unsigned long long)k << 56) | ((unsigned long long)az_bits << 24) | (unsigned)p;
}
// road point of ring k scanned before the first non-road point of its bin? cutbest = min best_key over the bin's
// non-road points (~0 if none): (ring, azimuth, position) order is the reference's scan order (:313-316)
URF_HD bool marker_candidate(unsigned long long cutbest, int k, unsigned az_bits, int p) {
  return best_key(k, az_bits, p) < cutbest;
}

}  // namespace urf
