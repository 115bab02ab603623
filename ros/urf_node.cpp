// ros/urf_node.cpp — thin ROS1 glue that drops liburf_b200 into the existing urban_road_filter graph.
//
// Same node name, same subscribed topic, same five published topics and the same LidarFilters.cfg dynamic_reconfigure
// surface as the reference node (src/main.cpp:1-56, src/lidar_segmentation.cpp:51-65,601-621): only the body of the
// scan callback changes — it hands the cloud to urf_process() (include/urf.h) instead of running the CPU detectors, then
// rebuilds the reference's four clouds and its road_marker MarkerArray from the labels, the emission order and the marker
// vertices. ROS / PCL are not available in the build container: this file is compile- and run-checked against the shim
// headers of oracle/shim by tests/test_glue.py (on the GPU box its published output is compared with the fixtures the
// unmodified reference produced); in a catkin workspace it builds unchanged against the real headers (INTEGRATION.md).
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include <ros/ros.h>
#include <pcl_conversions/pcl_conversions.h>
#include <pcl/point_cloud.h>
#include <pcl_ros/point_cloud.h>
#include <pcl/point_types.h>

#include "urf_glue_common.hpp"

namespace urf_glue {

class Detector {
 public:
  // device: CUDA device index; max_points: largest scan the sensor can produce; channels: ring count (reference constant 64)
  Detector(ros::NodeHandle* nh, int device = 0, int max_points = 1 << 20, int channels = 64, bool reference_tie_order = false) : channels_(channels) {
    const int rc = urf_create(&ctx_, device, max_points, 1);
    if (rc != URF_OK) {                                   // no GPU, no node: the reference never runs silently without output
      ROS_FATAL("urf_create(device %d, %d points): %s (%s)", device, max_points, urf_strerror(rc), urf_last_cuda_error(nullptr));
      throw std::runtime_error(std::string("urf_create: ") + urf_strerror(rc));
    }
    set_tie_order(ctx_, reference_tie_order);
    sub_ = nh->subscribe(std::string(g_params.topic_name), 1, &Detector::filtered, this);        // lidar_segmentation.cpp:53
    pub_road_ = nh->advertise<pcl::PCLPointCloud2>("road", 1);                                     // :55-59
    pub_high_ = nh->advertise<pcl::PCLPointCloud2>("curb", 1);
    pub_box_ = nh->advertise<pcl::PCLPointCloud2>("roi", 1);
    pub_pobroad_ = nh->advertise<pcl::PCLPointCloud2>("road_probably", 1);
    pub_marker_ = nh->advertise<visualization_msgs::MarkerArray>("road_marker", 1);
    ROS_INFO("Ready");
  }
  ~Detector() { urf_destroy(ctx_); }

  void set_ghostcount(int g) { ghostcount_ = g; }
  int ghostcount() const { return ghostcount_; }

  // scan callback, replaces Detector::filtered (lidar_segmentation.cpp:95-622)
  void filtered(const pcl::PointCloud<pcl::PointXYZI>& cloud) {
    if (!ctx_) return;
    if (g_params_dirty) {
      g_params.channels = channels_;
      const int prc = urf_set_params(ctx_, &g_params);
      if (prc != URF_OK) { ROS_ERROR_THROTTLE(5.0, "urf_set_params rejected the configuration (%s): scans are dropped until it is valid", urf_strerror(prc)); return; }
      g_params_dirty = false;
    }
    const int n = (int)cloud.points.size();
    xyzi_.resize((size_t)4 * (n > 0 ? n : 1));
    for (int i = 0; i < n; i++) {                      // first 16 bytes of the 32-byte PointXYZI record, intensity in w
      const pcl::PointXYZI& p = cloud.points[i];
      xyzi_[4 * i] = p.x; xyzi_[4 * i + 1] = p.y; xyzi_[4 * i + 2] = p.z; xyzi_[4 * i + 3] = p.intensity;
    }
    label_.resize(n > 0 ? n : 1); order_.resize(n > 0 ? n : 1);
    ring_start_.resize(URF_MAX_CHANNELS + 1);
    urf_result res;
    std::memset(&res, 0, sizeof(res));
    res.label = label_.data(); res.order = order_.data(); res.ring_start = ring_start_.data();
    const int rc = urf_process(ctx_, xyzi_.data(), n, &res);
    if (rc != URF_OK) {                                 // e.g. a scan larger than max_points: say so instead of a dead topic
      ROS_ERROR_THROTTLE(5.0, "urf_process(%d points): %s (%s)", n, urf_strerror(rc), urf_last_cuda_error(ctx_));
      return;
    }
    if (res.status == URF_TOO_FEW_POINTS) return;      // lidar_segmentation.cpp:124-126: nothing is published

    pcl::PointCloud<pcl::PointXYZI> road, high, probably;
    auto box = boost::make_shared<pcl::PointCloud<pcl::PointXYZI>>();
    for (int i = 0; i < n; i++) if (label_[i] >= 0) box->push_back(cloud.points[i]);               // roi cloud, input order
    for (int k = 0; k < res.n_order; k++) {                                                        // :354-367
      const int i = order_[k];
      if (label_[i] == URF_LABEL_ROAD) road.push_back(cloud.points[i]);
      else if (label_[i] == URF_LABEL_CURB) high.push_back(cloud.points[i]);
    }
    if (res.n_rings > 10)                                                                          // :605-608
      for (int k = ring_start_[10]; k < ring_start_[11]; k++) probably.push_back(cloud.points[order_[k]]);

    visualization_msgs::MarkerArray ma;                                                            // road_marker, :369-602
    if (build_marker_array(res, &ghostcount_, &ma)) pub_marker_.publish(ma);                       // :601
    road.header = cloud.header; probably.header = cloud.header; high.header = cloud.header; box->header = cloud.header;   // :612-615
    pub_road_.publish(road);                                                                       // :618-621
    pub_high_.publish(high);
    pub_box_.publish(box);
    pub_pobroad_.publish(probably);
  }

 private:
  urf_ctx* ctx_ = nullptr;
  int channels_;
  int ghostcount_ = 0;                                 // lidar_segmentation.cpp:23
  std::vector<float> xyzi_;
  std::vector<int32_t> label_, order_, ring_start_;
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
  urf_glue::Detector detector(&nh, device, max_points, channels, reference_tie_order);
  ros::spin();
  return 0;
}
#endif
