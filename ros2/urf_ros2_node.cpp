// ros2/urf_ros2_node.cpp — the drop-in road filter for ROS 2: the rclcpp component urf_b200::RoadFilterNode (executable
// lidar_road_b200), with the reference's node name, topics and LidarFilters parameters. It makes the same GPU call as
// ros/urf_node_cloud2.cpp: the `data` bytes of each sensor_msgs/msg/PointCloud2 go to urf_process_cloud2_packed as they
// are, the records are unpacked on the device, and the four output clouds come back packed in the reference's emission
// order as 32-byte pcl::PointXYZI records (x, y, z FLOAT32 at 0 / 4 / 8, intensity at 16), published with the input's
// header.
//
// The reference's dynamic_reconfigure parameters (cfg/LidarFilters.cfg there) are ROS 2 parameters that the node declares
// from one table, kParams: name, type, default, range and description. Two things differ from the ROS1 node:
//   - a value outside its range is refused, where dynamic_reconfigure clamps it to the range;
//   - a refused update leaves the running set in force, where the ROS1 node drops scans until urf_set_params accepts
//     its configuration.
// topic_name and the node parameters device, max_points, channels and reference_tie_order are read-only: they are set
// when the node starts. Only rclcpp calls that exist in both Humble and Jazzy are used.
// tests/test_ros2_glue.py runs this file against the shim headers of tests/ros2_shim (ros2/CMakeLists.txt builds it).
#include <cstddef>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include <rcl_interfaces/msg/parameter_descriptor.hpp>
#include <rcl_interfaces/msg/set_parameters_result.hpp>
#include <rclcpp/rclcpp.hpp>
#include <rclcpp_components/register_node_macro.hpp>
#include <sensor_msgs/msg/point_cloud2.hpp>
#include <sensor_msgs/msg/point_field.hpp>
#include <visualization_msgs/msg/marker_array.hpp>

#include "urf.h"

namespace urf_b200 {

// One parameter of the node. A bool or integer value goes to an int field of urf_params, a double to a double field and
// a string to a char[128] field.
struct ParamSpec {
  const char* name;
  rclcpp::ParameterType type;
  double def;                // default of a bool, integer or double parameter
  const char* def_str;       // default of a string parameter
  double lo, hi;             // range of an integer or double parameter
  bool read_only;
  long field;                // offsetof(urf_params, ...), or -1 for a node parameter that urf_params does not hold
  const char* description;
};

constexpr rclcpp::ParameterType kBool = rclcpp::PARAMETER_BOOL, kInt = rclcpp::PARAMETER_INTEGER,
                                kDouble = rclcpp::PARAMETER_DOUBLE, kString = rclcpp::PARAMETER_STRING;
#define URF_FIELD(f) static_cast<long>(offsetof(urf_params, f))

// The LidarFilters parameters with the reference's names, types, defaults and ranges, then the node parameters of the
// ROS1 nodes' private namespace.
inline const ParamSpec kParams[] = {
    {"fixed_frame", kString, 0, "left_os1/os1_lidar", 0, 0, false, URF_FIELD(fixed_frame), "Frame of the road_marker markers"},
    {"topic_name", kString, 0, "/left_os1/os1_cloud_node/points", 0, 0, true, URF_FIELD(topic_name), "PointCloud2 topic the node subscribes to"},
    {"x_zero_method", kBool, 1, nullptr, 0, 0, false, URF_FIELD(x_zero_method), "Run the X-zero curb detector"},
    {"z_zero_method", kBool, 1, nullptr, 0, 0, false, URF_FIELD(z_zero_method), "Run the Z-zero curb detector"},
    {"star_shaped_method", kBool, 1, nullptr, 0, 0, false, URF_FIELD(star_shaped_method), "Run the star-shaped curb search"},
    {"blind_spots", kBool, 1, nullptr, 0, 0, false, URF_FIELD(blind_spots), "Filter the road behind obstacles (blind spots)"},
    {"xDirection", kInt, 0, nullptr, 0, 2, false, URF_FIELD(xDirection), "Blind-spot filtering along X: 0 both directions, 1 only +X, 2 only -X"},
    {"interval", kDouble, 0.18, nullptr, 0.01, 10, false, URF_FIELD(interval), "Elevation tolerance that groups points into one ring [deg]"},
    {"curb_height", kDouble, 0.05, nullptr, 0.01, 0.5, false, URF_FIELD(curb_height), "Smallest curb height [m]"},
    {"curb_points", kInt, 5, nullptr, 1, 30, false, URF_FIELD(curb_points), "Expected number of points on a curb"},
    {"beamZone", kDouble, 30, nullptr, 10, 100, false, URF_FIELD(beamZone), "Width of the blind-spot beam zone [deg]"},
    {"min_x", kDouble, 0, nullptr, -200, 200, false, URF_FIELD(min_x), "Region of interest: smallest x [m]"},
    {"max_x", kDouble, 30, nullptr, -200, 200, false, URF_FIELD(max_x), "Region of interest: largest x [m]"},
    {"min_y", kDouble, -10, nullptr, -200, 200, false, URF_FIELD(min_y), "Region of interest: smallest y [m]"},
    {"max_y", kDouble, 10, nullptr, -200, 200, false, URF_FIELD(max_y), "Region of interest: largest y [m]"},
    {"min_z", kDouble, -3, nullptr, -200, 200, false, URF_FIELD(min_z), "Region of interest: smallest z [m]"},
    {"max_z", kDouble, -1, nullptr, -200, 200, false, URF_FIELD(max_z), "Region of interest: largest z [m]"},
    {"cylinder_deg_x", kDouble, 150, nullptr, 0, 180, false, URF_FIELD(cylinder_deg_x), "X-zero detector: angle threshold of three points [deg]"},
    {"cylinder_deg_z", kDouble, 140, nullptr, 0, 180, false, URF_FIELD(cylinder_deg_z), "Z-zero detector: angle threshold of two vectors [deg]"},
    {"curb_slope_deg", kDouble, 50, nullptr, 0, 180, false, URF_FIELD(curb_slope_deg), "Star-shaped search: radial slope threshold [deg]"},
    {"kdev_param", kDouble, 1.225, nullptr, 0.5, 5, false, URF_FIELD(kdev_param), "Star-shaped search: dispersion coefficient"},
    {"kdist_param", kDouble, 2, nullptr, 0.4, 10, false, URF_FIELD(kdist_param), "Star-shaped search: distance coefficient"},
    {"starbeam_filter", kBool, 0, nullptr, 0, 0, false, URF_FIELD(starbeam_filter), "Star-shaped search: rectangular beams instead of whole sectors"},
    {"dmin_param", kInt, 10, nullptr, 3, 30, false, URF_FIELD(dmin_param), "Star-shaped search: fewest points for a dispersion"},
    {"simple_poly_allow", kBool, 1, nullptr, 0, 0, false, URF_FIELD(simple_poly_allow), "Simplify the road_marker polygon (drops its heights)"},
    {"poly_s_param", kDouble, 0.7, nullptr, 0, 1, false, URF_FIELD(poly_s_param), "Polygon simplification coefficient"},
    {"poly_z_manual", kDouble, -1.5, nullptr, -5, 5, false, URF_FIELD(poly_z_manual), "Constant polygon height [m]"},
    {"poly_z_avg_allow", kBool, 1, nullptr, 0, 0, false, URF_FIELD(poly_z_avg_allow), "Set the polygon height to the average height"},
    {"channels", kInt, 64, nullptr, 1, URF_MAX_CHANNELS, true, URF_FIELD(channels), "Largest number of rings in a scan"},
    {"device", kInt, 0, nullptr, 0, 255, true, -1, "CUDA device the node runs on"},
    {"max_points", kInt, 1 << 20, nullptr, 1, 1 << 24, true, -1, "Largest scan in points; larger scans are refused"},
    {"reference_tie_order", kBool, 0, nullptr, 0, 0, true, -1,
     "Order equal azimuths in a ring as the reference's quicksort leaves them, instead of in input order"},
};
#undef URF_FIELD

inline const ParamSpec* find_param(const std::string& name) {
  for (const ParamSpec& s : kParams) if (name == s.name) return &s;
  return nullptr;
}

inline rclcpp::ParameterValue default_value(const ParamSpec& s) {
  switch (s.type) {
    case kBool: return rclcpp::ParameterValue(s.def != 0);
    case kInt: return rclcpp::ParameterValue(static_cast<int64_t>(s.def));
    case kDouble: return rclcpp::ParameterValue(s.def);
    default: return rclcpp::ParameterValue(std::string(s.def_str));
  }
}

inline rcl_interfaces::msg::ParameterDescriptor describe(const ParamSpec& s) {
  rcl_interfaces::msg::ParameterDescriptor d;
  d.name = s.name;
  d.type = s.type;
  d.description = s.description;
  d.read_only = s.read_only;
  if (s.type == kDouble) {
    rcl_interfaces::msg::FloatingPointRange r;
    r.from_value = s.lo; r.to_value = s.hi; r.step = 0.0;
    d.floating_point_range.push_back(r);
  } else if (s.type == kInt) {
    rcl_interfaces::msg::IntegerRange r;
    r.from_value = static_cast<int64_t>(s.lo); r.to_value = static_cast<int64_t>(s.hi); r.step = 1;
    d.integer_range.push_back(r);
  }
  return d;
}

// The type and range of one value: "" when it fits its table row, otherwise the reason it does not. The range test is
// rclcpp's own: the bounds are inside, and NaN is not refused here (urf_set_params refuses a non-finite value of the
// parameters the pipeline uses).
inline std::string check_value(const ParamSpec& s, const rclcpp::Parameter& p) {
  const std::string name = s.name;
  if (p.get_type() != s.type)
    return name + ": expected a " + rclcpp::to_string(s.type) + " value, got " + rclcpp::to_string(p.get_type());
  const double v = s.type == kInt ? static_cast<double>(p.as_int()) : s.type == kDouble ? p.as_double() : 0.0;
  if ((s.type == kInt || s.type == kDouble) && (v < s.lo || v > s.hi)) {
    char buf[160];
    std::snprintf(buf, sizeof(buf), ": %.17g is outside [%.17g, %.17g]", v, s.lo, s.hi);
    return name + buf;
  }
  if (s.type == kString && p.as_string().size() >= sizeof(urf_params::fixed_frame))
    return name + ": longer than " + std::to_string(sizeof(urf_params::fixed_frame) - 1) + " bytes";
  return "";
}

// Writes a value that passed check_value into its urf_params field.
inline void store(const ParamSpec& s, const rclcpp::Parameter& p, urf_params* out) {
  if (s.field < 0) return;
  char* f = reinterpret_cast<char*>(out) + s.field;
  if (s.type == kDouble) {
    const double v = p.as_double();
    std::memcpy(f, &v, sizeof(v));
  } else if (s.type == kString) {
    std::snprintf(f, sizeof(urf_params::fixed_frame), "%s", p.as_string().c_str());
  } else {
    const int v = s.type == kBool ? static_cast<int>(p.as_bool()) : static_cast<int>(p.as_int());
    std::memcpy(f, &v, sizeof(v));
  }
}

// The set `cur` with `changes` applied, in *out: "" when every change is acceptable, otherwise the reason the whole
// request is refused (an unknown or read-only name, a wrong type, a value outside its range). The caller then asks
// urf_set_params, which has the last word.
inline std::string candidate(const urf_params& cur, const std::vector<rclcpp::Parameter>& changes, urf_params* out) {
  *out = cur;
  for (const rclcpp::Parameter& p : changes) {
    const ParamSpec* s = find_param(p.get_name());
    if (!s) return p.get_name() + ": no such parameter";
    if (s->read_only) return p.get_name() + ": read-only, set it when the node starts";
    const std::string why = check_value(*s, p);
    if (!why.empty()) return why;
    store(*s, p, out);
  }
  return "";
}

class RoadFilterNode : public rclcpp::Node {
 public:
  using PointCloud2 = sensor_msgs::msg::PointCloud2;
  using MarkerArray = visualization_msgs::msg::MarkerArray;

  explicit RoadFilterNode(const rclcpp::NodeOptions& options) : rclcpp::Node("urban_road_filt", options) {
    for (const ParamSpec& s : kParams) {
      const rclcpp::Parameter p(s.name, declare_parameter(s.name, default_value(s), describe(s)));
      const std::string why = check_value(s, p);
      if (!why.empty()) throw std::invalid_argument(why);
      store(s, p, &params_);
    }
    max_points_ = static_cast<int>(get_parameter("max_points").as_int());
    const int device = static_cast<int>(get_parameter("device").as_int());
    urf_ctx* ctx = nullptr;
    int rc = urf_create(&ctx, device, max_points_, 1);
    if (rc != URF_OK) fail("urf_create(device " + std::to_string(device) + ", " + std::to_string(max_points_) + " points)", rc, nullptr);
    ctx_.reset(ctx);
    rc = urf_set_tie_order(ctx, get_parameter("reference_tie_order").as_bool() ? URF_TIES_REFERENCE : URF_TIES_INPUT_ORDER);
    if (rc != URF_OK) fail("urf_set_tie_order", rc, ctx);
    rc = urf_set_params(ctx, &params_);
    if (rc != URF_OK) fail("urf_set_params refused the parameters", rc, ctx);
    urf_point_xyzi** dst[4] = {&clouds_.road, &clouds_.curb, &clouds_.roi, &clouds_.road_probably};
    for (int k = 0; k < 4; k++) {     // pinned, so that the clouds come back at full PCIe rate
      bufs_[k].reset(static_cast<urf_point_xyzi*>(urf_pinned_alloc(sizeof(urf_point_xyzi) * static_cast<size_t>(max_points_))));
      if (!bufs_[k]) fail("urf_pinned_alloc", URF_ERR_NOMEM, ctx);
      *dst[k] = bufs_[k].get();
    }
    strips_.resize(URF_MAX_VERTS * 2 + 64);
    strip_points_.resize(3 * 4 * URF_MAX_VERTS);

    on_set_ = add_on_set_parameters_callback([this](const std::vector<rclcpp::Parameter>& ps) { return update(ps); });
    // KeepLast(1) is the reference's queue of 1. Best effort also matches the SensorDataQoS publishers of the LiDAR drivers.
    sub_ = create_subscription<PointCloud2>(params_.topic_name, rclcpp::QoS(rclcpp::KeepLast(1)).best_effort(),
                                            [this](PointCloud2::ConstSharedPtr msg) { filtered(*msg); });
    const rclcpp::QoS out = rclcpp::QoS(rclcpp::KeepLast(1)).reliable();
    pub_road_ = create_publisher<PointCloud2>("road", out);
    pub_curb_ = create_publisher<PointCloud2>("curb", out);
    pub_roi_ = create_publisher<PointCloud2>("roi", out);
    pub_road_probably_ = create_publisher<PointCloud2>("road_probably", out);
    pub_marker_ = create_publisher<MarkerArray>("road_marker", out);
    RCLCPP_INFO(get_logger(), "Ready");
  }

  // ghostcount carries the strip count of the last published road_marker from scan to scan (per node here, per process
  // in the reference)
  int ghostcount() const { return ghostcount_; }
  void set_ghostcount(int g) { ghostcount_ = g; }

 private:
  [[noreturn]] void fail(const std::string& what, int rc, const urf_ctx* ctx) {
    RCLCPP_FATAL(get_logger(), "%s: %s (%s)", what.c_str(), urf_strerror(rc), urf_last_cuda_error(ctx));
    throw std::runtime_error(what + ": " + urf_strerror(rc));
  }

  // The on-set callback: a refused request changes nothing; an accepted one runs from the next scan on. It shares the
  // node's default mutually exclusive callback group with the subscription; the mutex also orders it against a
  // set_parameters call from another thread of the process.
  rcl_interfaces::msg::SetParametersResult update(const std::vector<rclcpp::Parameter>& changes) {
    std::lock_guard<std::mutex> lock(mu_);
    rcl_interfaces::msg::SetParametersResult r;
    urf_params cand;
    r.reason = candidate(params_, changes, &cand);
    if (r.reason.empty()) {
      const int rc = urf_set_params(ctx_.get(), &cand);
      if (rc != URF_OK) r.reason = std::string("urf_set_params refused the parameters: ") + urf_strerror(rc);
    }
    r.successful = r.reason.empty();
    if (r.successful) params_ = cand;
    return r;
  }

  // the scan callback, as DetectorCloud2::filtered in ros/urf_node_cloud2.cpp
  void filtered(const PointCloud2& msg) {
    std::lock_guard<std::mutex> lock(mu_);
    int off[4] = {-1, -1, -1, -1};                      // x, y, z, intensity (FLOAT32 fields of the message)
    for (const sensor_msgs::msg::PointField& f : msg.fields) {
      if (f.datatype != sensor_msgs::msg::PointField::FLOAT32) continue;
      if (f.name == "x") off[0] = static_cast<int>(f.offset);
      else if (f.name == "y") off[1] = static_cast<int>(f.offset);
      else if (f.name == "z") off[2] = static_cast<int>(f.offset);
      else if (f.name == "intensity") off[3] = static_cast<int>(f.offset);
    }
    const long long n = static_cast<long long>(msg.width) * msg.height;
    if (off[0] < 0 || off[1] < 0 || off[2] < 0 || msg.is_bigendian || msg.point_step > URF_MAX_POINT_STEP || n > max_points_ ||
        msg.data.size() < static_cast<size_t>(n) * msg.point_step || (msg.height > 1 && msg.row_step != msg.width * msg.point_step)) {
      RCLCPP_ERROR_THROTTLE(get_logger(), *get_clock(), 5000,
                            "unsupported PointCloud2 (%lld points of %u bytes; needs little-endian FLOAT32 x/y/z, point_step <= %d, "
                            "unpadded rows, at most %d points)", n, msg.point_step, URF_MAX_POINT_STEP, max_points_);
      return;
    }
    urf_result res;
    std::memset(&res, 0, sizeof(res));
    const int rc = urf_process_cloud2_packed(ctx_.get(), msg.data.data(), static_cast<int>(n), static_cast<int>(msg.point_step),
                                             off[0], off[1], off[2], off[3], &res, &clouds_);
    if (rc != URF_OK) {
      RCLCPP_ERROR_THROTTLE(get_logger(), *get_clock(), 5000, "urf_process_cloud2_packed(%lld points): %s (%s)", n, urf_strerror(rc),
                            urf_last_cuda_error(ctx_.get()));
      return;
    }
    if (res.status == URF_TOO_FEW_POINTS) return;       // the reference publishes nothing for such a scan
    if (auto ma = markers(res)) pub_marker_->publish(std::move(ma));
    pub_road_->publish(wrap(msg, clouds_.road, clouds_.n_road));
    pub_curb_->publish(wrap(msg, clouds_.curb, clouds_.n_curb));
    pub_roi_->publish(wrap(msg, clouds_.roi, clouds_.n_roi));
    pub_road_probably_->publish(wrap(msg, clouds_.road_probably, clouds_.n_road_probably));
  }

  // `count` pcl::PointXYZI records as pcl_conversions lays out a pcl::PointCloud<pcl::PointXYZI>, with the input's header
  static std::unique_ptr<PointCloud2> wrap(const PointCloud2& in, const urf_point_xyzi* rec, int count) {
    auto out = std::make_unique<PointCloud2>();
    out->header = in.header;
    out->height = 1;
    out->width = static_cast<uint32_t>(count);
    const char* names[4] = {"x", "y", "z", "intensity"};
    const uint32_t offs[4] = {0, 4, 8, 16};
    for (int k = 0; k < 4; k++) {
      sensor_msgs::msg::PointField f;
      f.name = names[k]; f.offset = offs[k]; f.datatype = sensor_msgs::msg::PointField::FLOAT32; f.count = 1;
      out->fields.push_back(f);
    }
    out->is_bigendian = false;
    out->is_dense = true;
    out->point_step = sizeof(urf_point_xyzi);
    out->row_step = out->point_step * out->width;
    out->data.resize(out->row_step);
    if (count > 0) std::memcpy(out->data.data(), rec, out->data.size());
    return out;
  }

  // road_marker: one LINE_STRIP per strip of urf_build_markers, as build_marker_array in ros/urf_glue_common.hpp. Null
  // when nothing is to be published (fewer than three vertices) or the marker tail failed (logged).
  std::unique_ptr<MarkerArray> markers(const urf_result& res) {
    if (!(res.n_vert > 2)) return nullptr;
    int npts = 0;
    const int ns = urf_build_markers(&params_, res.vert, res.n_vert, &ghostcount_, strips_.data(), static_cast<int>(strips_.size()),
                                     strip_points_.data(), static_cast<int>(strip_points_.size() / 3), &npts);
    if (ns < 0) {
      RCLCPP_ERROR(get_logger(), "urf_build_markers: %s", urf_strerror(ns));
      return nullptr;
    }
    auto ma = std::make_unique<MarkerArray>();
    for (int s = 0; s < ns; s++) {
      const urf_strip& st = strips_[s];
      visualization_msgs::msg::Marker m;
      m.header.frame_id = params_.fixed_frame;          // zero stamp, as the reference's ros::Time()
      m.type = visualization_msgs::msg::Marker::LINE_STRIP;
      m.action = st.action == 2 ? visualization_msgs::msg::Marker::DELETE : visualization_msgs::msg::Marker::ADD;
      m.id = st.id;
      m.pose.orientation.w = 1.0;
      m.scale.x = m.scale.y = m.scale.z = 0.5;
      m.color.r = st.red ? 1.0f : 0.0f; m.color.g = st.red ? 0.0f : 1.0f; m.color.b = 0.0f; m.color.a = 1.0f;
      for (int k = 0; k < st.count; k++) {
        const double* q = &strip_points_[3 * static_cast<size_t>(st.first + k)];
        geometry_msgs::msg::Point p;
        p.x = q[0]; p.y = q[1]; p.z = q[2];
        m.points.push_back(p);
      }
      ma->markers.push_back(std::move(m));
    }
    return ma;
  }

  struct CtxDestroy { void operator()(urf_ctx* c) const { urf_destroy(c); } };
  struct PinnedFree { void operator()(urf_point_xyzi* p) const { urf_pinned_free(p); } };

  std::mutex mu_;
  urf_params params_{};                                 // the running set
  int max_points_ = 0;
  int ghostcount_ = 0;
  std::unique_ptr<urf_ctx, CtxDestroy> ctx_;
  std::unique_ptr<urf_point_xyzi, PinnedFree> bufs_[4];
  urf_clouds clouds_{};
  std::vector<urf_strip> strips_;
  std::vector<double> strip_points_;
  OnSetParametersCallbackHandle::SharedPtr on_set_;
  rclcpp::Subscription<PointCloud2>::SharedPtr sub_;
  rclcpp::Publisher<PointCloud2>::SharedPtr pub_road_, pub_curb_, pub_roi_, pub_road_probably_;
  rclcpp::Publisher<MarkerArray>::SharedPtr pub_marker_;
};

}  // namespace urf_b200

RCLCPP_COMPONENTS_REGISTER_NODE(urf_b200::RoadFilterNode)
