// ros/urf_glue_common.hpp — what the two glue nodes share: the dynamic_reconfigure callback (src/main.cpp:4-34) and the
// road_marker MarkerArray built from urf_build_markers' strips (lidar_segmentation.cpp:417-601).
#pragma once
#include <cstdio>
#include <string>

#include <ros/ros.h>
#include <visualization_msgs/Marker.h>
#include <visualization_msgs/MarkerArray.h>
#include <dynamic_reconfigure/server.h>
#include <urban_road_filter/LidarFiltersConfig.h>

#include "urf.h"

namespace urf_glue {

inline urf_params g_params;          // what paramsCallback last received (the reference keeps them in params:: globals)
inline bool g_params_dirty = true;

// node parameter ~reference_tie_order (default false): equal azimuths inside a ring in the order the reference's Lomuto
// quicksort leaves them (its clouds and marker vertices bit for bit) instead of input order; see urf_set_tie_order
inline void set_tie_order(urf_ctx* ctx, bool reference) {
  const int rc = urf_set_tie_order(ctx, reference ? URF_TIES_REFERENCE : URF_TIES_INPUT_ORDER);
  if (rc != URF_OK) {
    ROS_FATAL("urf_set_tie_order: %s (%s)", urf_strerror(rc), urf_last_cuda_error(ctx));
    throw std::runtime_error(std::string("urf_set_tie_order: ") + urf_strerror(rc));
  }
}

// paramsCallback, src/main.cpp:4-34: same fields, same order; narrowing to float happens inside urf_set_params
inline void paramsCallback(urban_road_filter::LidarFiltersConfig& config, uint32_t /*level*/) {
  urf_params& p = g_params;
  std::snprintf(p.fixed_frame, sizeof(p.fixed_frame), "%s", config.fixed_frame.c_str());
  std::snprintf(p.topic_name, sizeof(p.topic_name), "%s", config.topic_name.c_str());
  p.x_zero_method = config.x_zero_method;
  p.z_zero_method = config.z_zero_method;
  p.star_shaped_method = config.star_shaped_method;
  p.blind_spots = config.blind_spots;
  p.xDirection = config.xDirection;
  p.interval = config.interval;
  p.curb_height = config.curb_height;
  p.curb_points = config.curb_points;
  p.beamZone = config.beamZone;
  p.cylinder_deg_x = config.cylinder_deg_x;
  p.cylinder_deg_z = config.cylinder_deg_z;
  p.curb_slope_deg = config.curb_slope_deg;
  p.min_x = config.min_x; p.max_x = config.max_x;
  p.min_y = config.min_y; p.max_y = config.max_y;
  p.min_z = config.min_z; p.max_z = config.max_z;
  p.kdev_param = config.kdev_param;
  p.kdist_param = config.kdist_param;
  p.starbeam_filter = config.starbeam_filter;
  p.dmin_param = config.dmin_param;
  p.simple_poly_allow = config.simple_poly_allow;
  p.poly_s_param = config.poly_s_param;
  p.poly_z_avg_allow = config.poly_z_avg_allow;
  p.poly_z_manual = config.poly_z_manual;
  g_params_dirty = true;
  ROS_INFO("Updated params %s", ros::this_node::getName().c_str());
}

// road_marker, lidar_segmentation.cpp:369-602: strips from the candidate vertices, then one Marker per strip. Returns false
// when nothing is to be published (fewer than three vertices, :371) or the marker tail failed (logged).
inline bool build_marker_array(const urf_result& res, int* ghostcount, visualization_msgs::MarkerArray* ma) {
  if (!(res.n_vert > 2)) return false;
  static urf_strip strips[URF_MAX_VERTS * 2 + 64];
  static double pts[3 * 4 * URF_MAX_VERTS];
  int npts = 0;
  const int ns = urf_build_markers(&g_params, res.vert, res.n_vert, ghostcount, strips, URF_MAX_VERTS * 2 + 64, pts, 4 * URF_MAX_VERTS, &npts);
  if (ns < 0) { ROS_ERROR("urf_build_markers: %s", urf_strerror(ns)); return false; }
  for (int s = 0; s < ns; s++) {
    visualization_msgs::Marker m;
    m.header.frame_id = g_params.fixed_frame;                                               // :424-427
    m.header.stamp = ros::Time();
    m.type = visualization_msgs::Marker::LINE_STRIP;
    m.action = strips[s].action == 2 ? visualization_msgs::Marker::DELETE : visualization_msgs::Marker::ADD;
    m.id = strips[s].id;
    m.pose.orientation.w = 1.0;                                                              // marker_init, :25-39
    m.scale.x = m.scale.y = m.scale.z = 0.5;
    m.color.r = strips[s].red ? 1.0f : 0.0f; m.color.g = strips[s].red ? 0.0f : 1.0f; m.color.b = 0.0f; m.color.a = 1.0f;
    m.lifetime = ros::Duration(0);
    for (int k = 0; k < strips[s].count; k++) {
      geometry_msgs::Point q;
      q.x = pts[3 * (strips[s].first + k)]; q.y = pts[3 * (strips[s].first + k) + 1]; q.z = pts[3 * (strips[s].first + k) + 2];
      m.points.push_back(q);
    }
    ma->markers.push_back(m);
  }
  return true;
}

}  // namespace urf_glue
