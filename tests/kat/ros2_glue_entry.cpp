// tests/kat/ros2_glue_entry.cpp — TEST CODE. Builds ros2/urf_ros2_node.cpp (the product's ROS 2 node) against the shim
// headers of tests/ros2_shim and exports C entries for tests/test_ros2_glue.py: create the component with parameter
// overrides, deliver a PointCloud2 to its subscription, read back what it published and logged (as JSON, records as
// bytes), set parameters through its on-set callback, and read the parameter table and candidate check without a GPU.
#include "../../ros2/urf_ros2_node.cpp"

#include <cmath>

namespace {

using urf_b200::RoadFilterNode;
using sensor_msgs::msg::PointCloud2;
using visualization_msgs::msg::MarkerArray;

// Parameters from C arrays; types are rclcpp::ParameterType values (1 bool, 2 integer, 3 double, 4 string; 0 not set).
std::vector<rclcpp::Parameter> params_of(int n, const char* const* names, const int* types, const double* nums, const char* const* strs) {
  std::vector<rclcpp::Parameter> out;
  for (int i = 0; i < n; i++) {
    switch (types[i]) {
      case rclcpp::PARAMETER_BOOL: out.emplace_back(names[i], nums[i] != 0); break;
      case rclcpp::PARAMETER_INTEGER: out.emplace_back(names[i], static_cast<int64_t>(nums[i])); break;
      case rclcpp::PARAMETER_DOUBLE: out.emplace_back(names[i], nums[i]); break;
      case rclcpp::PARAMETER_STRING: out.emplace_back(names[i], std::string(strs[i])); break;
      default: out.emplace_back(names[i], rclcpp::ParameterValue()); break;
    }
  }
  return out;
}

int put(const std::string& s, char* buf, int len) {
  if (buf && len > 0) std::snprintf(buf, static_cast<size_t>(len), "%s", s.c_str());
  return static_cast<int>(s.size());
}

std::string jstr(const std::string& s) {
  std::string o = "\"";
  for (char c : s) {
    if (c == '"' || c == '\\') { o += '\\'; o += c; }
    else if (static_cast<unsigned char>(c) < 0x20) { char b[8]; std::snprintf(b, sizeof(b), "\\u%04x", c); o += b; }
    else o += c;
  }
  return o + "\"";
}
std::string jnum(double v) {
  if (std::isnan(v)) return "NaN";
  char b[40];
  std::snprintf(b, sizeof(b), "%.17g", v);
  std::string o = b;
  if (std::isfinite(v) && o.find_first_of(".e") == std::string::npos) o += ".0";   // JSON readers keep it a float
  return o == "inf" ? "Infinity" : o == "-inf" ? "-Infinity" : o;
}
std::string jval(const rclcpp::ParameterValue& v) {
  switch (v.get_type()) {
    case rclcpp::PARAMETER_BOOL: return v.as_bool() ? "true" : "false";
    case rclcpp::PARAMETER_INTEGER: return std::to_string(v.as_int());
    case rclcpp::PARAMETER_DOUBLE: return jnum(v.as_double());
    case rclcpp::PARAMETER_STRING: return jstr(v.as_string());
    default: return "null";
  }
}
std::string jdesc(const rcl_interfaces::msg::ParameterDescriptor& d) {
  std::string o = "{\"name\": " + jstr(d.name) + ", \"type\": " + std::to_string(d.type) + ", \"description\": " + jstr(d.description) +
                  ", \"read_only\": " + (d.read_only ? "true" : "false") + ", \"floating_point_range\": [";
  for (size_t k = 0; k < d.floating_point_range.size(); k++)
    o += std::string(k ? ", " : "") + "[" + jnum(d.floating_point_range[k].from_value) + ", " + jnum(d.floating_point_range[k].to_value) +
         ", " + jnum(d.floating_point_range[k].step) + "]";
  o += "], \"integer_range\": [";
  for (size_t k = 0; k < d.integer_range.size(); k++)
    o += std::string(k ? ", " : "") + "[" + std::to_string(d.integer_range[k].from_value) + ", " + std::to_string(d.integer_range[k].to_value) +
         ", " + std::to_string(d.integer_range[k].step) + "]";
  return o + "]}";
}
std::string jqos(const rclcpp::QoS& q) {
  return std::string("{\"reliability\": ") + (q.reliability() == rclcpp::ReliabilityPolicy::BestEffort ? "\"best_effort\"" : "\"reliable\"") +
         ", \"depth\": " + std::to_string(q.depth()) + "}";
}

struct Handle {
  std::shared_ptr<rclcpp::Node> node;
  RoadFilterNode* filter;
};

template <class M>
rclcpp::Publisher<M>* publisher(Handle* h, const std::string& topic) {
  auto it = h->node->shim_publishers.find(topic);
  return it == h->node->shim_publishers.end() ? nullptr : dynamic_cast<rclcpp::Publisher<M>*>(it->second.get());
}

}  // namespace

extern "C" {

// The component, created through its registration as the component container does; NULL with the reason in err when
// its constructor throws.
void* urf_ros2_create(int n, const char* const* names, const int* types, const double* nums, const char* const* strs, char* err, int err_len) {
  rclcpp::shim_logs().clear();
  try {
    rclcpp::NodeOptions opts;
    opts.parameter_overrides(params_of(n, names, types, nums, strs));
    std::shared_ptr<rclcpp::Node> node = rclcpp_components_shim::registry().at("urf_b200::RoadFilterNode")(opts);
    RoadFilterNode* f = dynamic_cast<RoadFilterNode*>(node.get());
    put("", err, err_len);
    return new Handle{node, f};
  } catch (const std::exception& e) {
    put(e.what(), err, err_len);
    return nullptr;
  }
}

void urf_ros2_destroy(void* h) { delete static_cast<Handle*>(h); }

// One PointCloud2 through the node's subscription. What the node published and logged before is cleared first.
int urf_ros2_feed(void* hv, uint32_t width, uint32_t height, uint32_t point_step, uint32_t row_step, int is_bigendian, int n_fields,
                  const char* const* fnames, const int* foffs, const int* ftypes, const uint8_t* data, size_t data_len, int32_t sec,
                  uint32_t nanosec, const char* frame_id) {
  Handle* h = static_cast<Handle*>(hv);
  for (auto& kv : h->node->shim_publishers) {
    if (auto* p = dynamic_cast<rclcpp::Publisher<PointCloud2>*>(kv.second.get())) p->shim_sent.clear();
    if (auto* p = dynamic_cast<rclcpp::Publisher<MarkerArray>*>(kv.second.get())) p->shim_sent.clear();
  }
  rclcpp::shim_logs().clear();
  auto msg = std::make_shared<PointCloud2>();
  msg->header.stamp.sec = sec; msg->header.stamp.nanosec = nanosec; msg->header.frame_id = frame_id;
  msg->width = width; msg->height = height; msg->point_step = point_step; msg->row_step = row_step;
  msg->is_bigendian = is_bigendian != 0;
  for (int k = 0; k < n_fields; k++) {
    sensor_msgs::msg::PointField f;
    f.name = fnames[k]; f.offset = static_cast<uint32_t>(foffs[k]); f.datatype = static_cast<uint8_t>(ftypes[k]); f.count = 1;
    msg->fields.push_back(f);
  }
  msg->data.assign(data, data + data_len);
  if (h->node->shim_subscriptions.size() != 1) return -1;
  auto* sub = dynamic_cast<rclcpp::Subscription<PointCloud2>*>(h->node->shim_subscriptions.begin()->second.get());
  if (!sub) return -1;
  sub->shim_deliver(msg);
  return 0;
}

// The clouds published on `topic` by the last feed: returns how many; the last one's layout and header go to json, its
// records to data (cap bytes at most).
int urf_ros2_cloud(void* hv, const char* topic, char* json, int json_len, uint8_t* data, size_t cap) {
  rclcpp::Publisher<PointCloud2>* p = publisher<PointCloud2>(static_cast<Handle*>(hv), topic);
  if (!p) return -1;
  if (p->shim_sent.empty()) { put("null", json, json_len); return 0; }
  const PointCloud2& m = *p->shim_sent.back();
  std::string o = "{\"frame_id\": " + jstr(m.header.frame_id) + ", \"sec\": " + std::to_string(m.header.stamp.sec) +
                  ", \"nanosec\": " + std::to_string(m.header.stamp.nanosec) + ", \"height\": " + std::to_string(m.height) +
                  ", \"width\": " + std::to_string(m.width) + ", \"point_step\": " + std::to_string(m.point_step) +
                  ", \"row_step\": " + std::to_string(m.row_step) + ", \"is_bigendian\": " + (m.is_bigendian ? "true" : "false") +
                  ", \"is_dense\": " + (m.is_dense ? "true" : "false") + ", \"size\": " + std::to_string(m.data.size()) + ", \"fields\": [";
  for (size_t k = 0; k < m.fields.size(); k++)
    o += std::string(k ? ", " : "") + "[" + jstr(m.fields[k].name) + ", " + std::to_string(m.fields[k].offset) + ", " +
         std::to_string(m.fields[k].datatype) + ", " + std::to_string(m.fields[k].count) + "]";
  put(o + "]}", json, json_len);
  if (data) std::memcpy(data, m.data.data(), std::min(cap, m.data.size()));
  return static_cast<int>(p->shim_sent.size());
}

// The MarkerArrays published by the last feed: returns how many; the last one goes to json.
int urf_ros2_markers(void* hv, char* json, int json_len) {
  rclcpp::Publisher<MarkerArray>* p = publisher<MarkerArray>(static_cast<Handle*>(hv), "road_marker");
  if (!p) return -1;
  std::string o = "[";
  if (!p->shim_sent.empty()) {
    const MarkerArray& ma = *p->shim_sent.back();
    for (size_t s = 0; s < ma.markers.size(); s++) {
      const visualization_msgs::msg::Marker& m = ma.markers[s];
      o += std::string(s ? ", " : "") + "{\"frame_id\": " + jstr(m.header.frame_id) + ", \"sec\": " + std::to_string(m.header.stamp.sec) +
           ", \"nanosec\": " + std::to_string(m.header.stamp.nanosec) + ", \"ns\": " + jstr(m.ns) + ", \"id\": " + std::to_string(m.id) +
           ", \"type\": " + std::to_string(m.type) + ", \"action\": " + std::to_string(m.action) +
           ", \"orientation\": [" + jnum(m.pose.orientation.x) + ", " + jnum(m.pose.orientation.y) + ", " + jnum(m.pose.orientation.z) +
           ", " + jnum(m.pose.orientation.w) + "], \"scale\": [" + jnum(m.scale.x) + ", " + jnum(m.scale.y) + ", " + jnum(m.scale.z) +
           "], \"color\": [" + jnum(m.color.r) + ", " + jnum(m.color.g) + ", " + jnum(m.color.b) + ", " + jnum(m.color.a) +
           "], \"lifetime\": [" + std::to_string(m.lifetime.sec) + ", " + std::to_string(m.lifetime.nanosec) + "], \"points\": [";
      for (size_t k = 0; k < m.points.size(); k++)
        o += std::string(k ? ", " : "") + "[" + jnum(m.points[k].x) + ", " + jnum(m.points[k].y) + ", " + jnum(m.points[k].z) + "]";
      o += "]}";
    }
  }
  put(o + "]", json, json_len);
  return static_cast<int>(p->shim_sent.size());
}

// What the last feed, creation or parameter request logged: [[level, text], ...]
int urf_ros2_logs(char* json, int json_len) {
  std::string o = "[";
  for (size_t k = 0; k < rclcpp::shim_logs().size(); k++)
    o += std::string(k ? ", " : "") + "[" + jstr(std::string(1, rclcpp::shim_logs()[k].level)) + ", " + jstr(rclcpp::shim_logs()[k].text) + "]";
  return put(o + "]", json, json_len);
}

// set_parameters_atomically (atomic) or set_parameters: returns the number of accepted requests (0 or 1 when atomic);
// the reasons of the refused ones, joined by " | ", go to reason.
int urf_ros2_set(void* hv, int atomic, int n, const char* const* names, const int* types, const double* nums, const char* const* strs,
                 char* reason, int reason_len) {
  Handle* h = static_cast<Handle*>(hv);
  const std::vector<rclcpp::Parameter> ps = params_of(n, names, types, nums, strs);
  std::vector<rcl_interfaces::msg::SetParametersResult> rs;
  if (atomic) rs.push_back(h->node->set_parameters_atomically(ps));
  else rs = h->node->set_parameters(ps);
  int ok = 0;
  std::string why;
  for (const auto& r : rs) {
    if (r.successful) ok++;
    else why += (why.empty() ? "" : " | ") + r.reason;
  }
  put(why, reason, reason_len);
  return ok;
}

// The node's ghostcount; set >= 0 replaces it first.
int urf_ros2_ghostcount(void* hv, int set) {
  Handle* h = static_cast<Handle*>(hv);
  if (set >= 0) h->filter->set_ghostcount(set);
  return h->filter->ghostcount();
}

// Name, topics with their QoS, on-set callbacks, and every declared parameter with its descriptor and current value.
int urf_ros2_info(void* hv, char* json, int json_len) {
  rclcpp::Node& node = *static_cast<Handle*>(hv)->node;
  std::string o = "{\"name\": " + jstr(node.get_name()) + ", \"callbacks\": " + std::to_string(node.shim_callback_count()) + ", \"subscriptions\": {";
  bool first = true;
  for (const auto& kv : node.shim_subscriptions) {
    auto* s = dynamic_cast<rclcpp::Subscription<PointCloud2>*>(kv.second.get());
    o += std::string(first ? "" : ", ") + jstr(kv.first) + ": " + (s ? jqos(s->shim_qos()) : "null");
    first = false;
  }
  o += "}, \"publishers\": {";
  first = true;
  for (const auto& kv : node.shim_publishers) {
    std::string q = "null";
    if (auto* p = dynamic_cast<rclcpp::Publisher<PointCloud2>*>(kv.second.get())) q = "[\"PointCloud2\", " + jqos(p->shim_qos()) + "]";
    if (auto* p = dynamic_cast<rclcpp::Publisher<MarkerArray>*>(kv.second.get())) q = "[\"MarkerArray\", " + jqos(p->shim_qos()) + "]";
    o += std::string(first ? "" : ", ") + jstr(kv.first) + ": " + q;
    first = false;
  }
  o += "}, \"parameters\": {";
  first = true;
  for (const auto& kv : node.shim_descriptors) {
    o += std::string(first ? "" : ", ") + jstr(kv.first) + ": {\"value\": " + jval(node.get_parameter(kv.first).get_parameter_value()) +
         ", \"descriptor\": " + jdesc(kv.second) + "}";
    first = false;
  }
  return put(o + "}}", json, json_len);
}

// Without a GPU: the node's parameter table, each row as the node declares it (descriptor and default).
int urf_ros2_table(char* json, int json_len) {
  std::string o = "[";
  bool first = true;
  for (const urf_b200::ParamSpec& s : urf_b200::kParams) {
    o += std::string(first ? "" : ", ") + "{\"default\": " + jval(urf_b200::default_value(s)) + ", \"cfg_field\": " +
         (s.field >= 0 ? "true" : "false") + ", \"descriptor\": " + jdesc(urf_b200::describe(s)) + "}";
    first = false;
  }
  return put(o + "]", json, json_len);
}

// Without a GPU: the node's table checks of one request against the default set. 1 when the request passes them (the
// node would then ask urf_set_params), 0 with the reason otherwise.
int urf_ros2_check(int n, const char* const* names, const int* types, const double* nums, const char* const* strs, char* reason, int reason_len) {
  urf_params defaults{};
  for (const urf_b200::ParamSpec& s : urf_b200::kParams) urf_b200::store(s, rclcpp::Parameter(s.name, urf_b200::default_value(s)), &defaults);
  urf_params cand;
  const std::string why = urf_b200::candidate(defaults, params_of(n, names, types, nums, strs), &cand);
  put(why, reason, reason_len);
  return why.empty() ? 1 : 0;
}

}  // extern "C"
