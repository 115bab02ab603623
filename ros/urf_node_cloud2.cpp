// ros/urf_node_cloud2.cpp — the same drop-in node as ros/urf_node.cpp, but without PCL on either side of the GPU call:
// it subscribes to the raw sensor_msgs/PointCloud2 message (what the reference's subscriber receives before pcl_ros
// deserialises it, src/lidar_segmentation.cpp:53,95), hands the message's `data` bytes to urf_process_cloud2_packed —
// records are unpacked on the device, the four output clouds are packed there in the reference's emission order — and
// wraps the returned 32-byte pcl::PointXYZI records into PointCloud2 messages with the field layout pcl_ros produces for
// the reference's `pcl::PointCloud<pcl::PointXYZI>` publishers (x, y, z FLOAT32 at 0 / 4 / 8, intensity at 16, point_step
// 32, src/lidar_segmentation.cpp:55-59,618-621). Same node name, topics and LidarFilters.cfg surface as the reference.
// Run against the shim headers of oracle/shim by tests/test_glue.py; builds unchanged in a catkin workspace (ros/CMakeLists.txt).
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include <ros/ros.h>
#include <sensor_msgs/PointCloud2.h>

#include "urf_glue_common.hpp"

namespace urf_glue {

class DetectorCloud2 {
 public:
  DetectorCloud2(ros::NodeHandle* nh, int device = 0, int max_points = 1 << 20, int channels = 64, bool reference_tie_order = false) : max_points_(max_points), channels_(channels) {
    const int rc = urf_create(&ctx_, device, max_points, 1);
    if (rc != URF_OK) {
      ROS_FATAL("urf_create(device %d, %d points): %s (%s)", device, max_points, urf_strerror(rc), urf_last_cuda_error(nullptr));
      throw std::runtime_error(std::string("urf_create: ") + urf_strerror(rc));
    }
    set_tie_order(ctx_, reference_tie_order);
    for (urf_point_xyzi** c : {&clouds_.road, &clouds_.curb, &clouds_.roi, &clouds_.road_probably}) {
      *c = static_cast<urf_point_xyzi*>(urf_pinned_alloc(sizeof(urf_point_xyzi) * (size_t)max_points));   // D2H at full PCIe rate
      if (!*c) throw std::runtime_error("urf_pinned_alloc failed");
    }
    sub_ = nh->subscribe(std::string(g_params.topic_name), 1, &DetectorCloud2::filtered, this);      // lidar_segmentation.cpp:53
    pub_road_ = nh->advertise<sensor_msgs::PointCloud2>("road", 1);                                    // :55-59
    pub_high_ = nh->advertise<sensor_msgs::PointCloud2>("curb", 1);
    pub_box_ = nh->advertise<sensor_msgs::PointCloud2>("roi", 1);
    pub_pobroad_ = nh->advertise<sensor_msgs::PointCloud2>("road_probably", 1);
    pub_marker_ = nh->advertise<visualization_msgs::MarkerArray>("road_marker", 1);
    ROS_INFO("Ready");
  }
  ~DetectorCloud2() {
    urf_destroy(ctx_);
    for (urf_point_xyzi* c : {clouds_.road, clouds_.curb, clouds_.roi, clouds_.road_probably}) urf_pinned_free(c);
  }
  void set_ghostcount(int g) { ghostcount_ = g; }
  int ghostcount() const { return ghostcount_; }

  // scan callback, replaces Detector::filtered (lidar_segmentation.cpp:95-622)
  void filtered(const sensor_msgs::PointCloud2& msg) {
    if (g_params_dirty) {
      g_params.channels = channels_;
      const int prc = urf_set_params(ctx_, &g_params);
      if (prc != URF_OK) { ROS_ERROR_THROTTLE(5.0, "urf_set_params rejected the configuration (%s): scans are dropped until it is valid", urf_strerror(prc)); return; }
      g_params_dirty = false;
    }
    int off[4] = {-1, -1, -1, -1};                      // x, y, z, intensity (FLOAT32 fields of the message)
    for (const sensor_msgs::PointField& f : msg.fields) {
      if (f.datatype != sensor_msgs::PointField::FLOAT32) continue;
      if (f.name == "x") off[0] = (int)f.offset; else if (f.name == "y") off[1] = (int)f.offset;
      else if (f.name == "z") off[2] = (int)f.offset; else if (f.name == "intensity") off[3] = (int)f.offset;
    }
    const long long n = (long long)msg.width * msg.height;
    if (off[0] < 0 || off[1] < 0 || off[2] < 0 || msg.is_bigendian || msg.point_step > URF_MAX_POINT_STEP || n > max_points_ ||
        msg.data.size() < (size_t)n * msg.point_step || (msg.height > 1 && msg.row_step != msg.width * msg.point_step)) {
      ROS_ERROR_THROTTLE(5.0, "unsupported PointCloud2 (%lld points of %u bytes; needs little-endian FLOAT32 x/y/z, point_step <= %d, at most %d points)",
                         n, msg.point_step, URF_MAX_POINT_STEP, max_points_);
      return;
    }
    urf_result res;
    std::memset(&res, 0, sizeof(res));
    const int rc = urf_process_cloud2_packed(ctx_, msg.data.data(), (int)n, (int)msg.point_step, off[0], off[1], off[2], off[3], &res, &clouds_);
    if (rc != URF_OK) { ROS_ERROR_THROTTLE(5.0, "urf_process_cloud2_packed(%lld points): %s (%s)", n, urf_strerror(rc), urf_last_cuda_error(ctx_)); return; }
    if (res.status == URF_TOO_FEW_POINTS) return;       // lidar_segmentation.cpp:124-126: nothing is published
    visualization_msgs::MarkerArray ma;                 // road_marker, :369-602
    if (build_marker_array(res, &ghostcount_, &ma)) pub_marker_.publish(ma);                       // :601
    pub_road_.publish(wrap(msg, clouds_.road, clouds_.n_road));                                    // :618-621
    pub_high_.publish(wrap(msg, clouds_.curb, clouds_.n_curb));
    pub_box_.publish(wrap(msg, clouds_.roi, clouds_.n_roi));
    pub_pobroad_.publish(wrap(msg, clouds_.road_probably, clouds_.n_road_probably));
  }

 private:
  // `count` pcl::PointXYZI records as the PointCloud2 pcl_ros serialises for a pcl::PointCloud<pcl::PointXYZI> (header of the
  // input message, :612-615)
  static sensor_msgs::PointCloud2 wrap(const sensor_msgs::PointCloud2& in, const urf_point_xyzi* rec, int count) {
    sensor_msgs::PointCloud2 out;
    out.header = in.header;
    out.height = 1; out.width = (uint32_t)count;
    const char* names[4] = {"x", "y", "z", "intensity"};
    const uint32_t offs[4] = {0, 4, 8, 16};
    for (int k = 0; k < 4; k++) {
      sensor_msgs::PointField f;
      f.name = names[k]; f.offset = offs[k]; f.datatype = sensor_msgs::PointField::FLOAT32; f.count = 1;
      out.fields.push_back(f);
    }
    out.is_bigendian = false; out.is_dense = true;
    out.point_step = sizeof(urf_point_xyzi); out.row_step = out.point_step * out.width;
    out.data.resize((size_t)out.row_step);
    if (count > 0) std::memcpy(out.data.data(), rec, out.data.size());
    return out;
  }

  urf_ctx* ctx_ = nullptr;
  int max_points_, channels_;
  int ghostcount_ = 0;                                  // lidar_segmentation.cpp:23
  urf_clouds clouds_{};
  ros::Publisher pub_road_, pub_high_, pub_box_, pub_pobroad_, pub_marker_;
  ros::Subscriber sub_;
};

}  // namespace urf_glue

#ifndef URF_GLUE_NO_MAIN
int main(int argc, char** argv) {                        // src/main.cpp:37-56
  ros::init(argc, argv, "urban_road_filt");
  ROS_INFO("Initializing %s", ros::this_node::getName().c_str());
  urf_default_params(&urf_glue::g_params);
  dynamic_reconfigure::Server<urban_road_filter::LidarFiltersConfig> server;
  dynamic_reconfigure::Server<urban_road_filter::LidarFiltersConfig>::CallbackType f = &urf_glue::paramsCallback;
  server.setCallback(f);
  ros::NodeHandle nh;
  ros::NodeHandle pnh("~");
  int device = 0, max_points = 1 << 20, channels = 64;
  pnh.param("device", device, 0);
  pnh.param("max_points", max_points, 1 << 20);
  pnh.param("channels", channels, 64);                   // the reference's global `int channels = 64` (lidar_segmentation.cpp:4)
  bool reference_tie_order = false;
  pnh.param("reference_tie_order", reference_tie_order, false);
  urf_glue::DetectorCloud2 detector(&nh, device, max_points, channels, reference_tie_order);
  ros::spin();
  return 0;
}
#endif
