// ROS 2 shim (test code only): RCLCPP_COMPONENTS_REGISTER_NODE records a factory of the component under its class name,
// which is the PLUGIN name rclcpp_components_register_node is given, so the test entry creates the node the way the
// component container and the generated executable do.
#pragma once
#include <functional>
#include <map>
#include <memory>
#include <string>

#include <rclcpp/rclcpp.hpp>

namespace rclcpp_components_shim {
using Factory = std::function<std::shared_ptr<rclcpp::Node>(const rclcpp::NodeOptions&)>;
inline std::map<std::string, Factory>& registry() { static std::map<std::string, Factory> r; return r; }
struct Registrar {
  Registrar(const char* name, Factory f) { registry()[name] = std::move(f); }
};
}  // namespace rclcpp_components_shim

#define URF_SHIM_CAT2(a, b) a##b
#define URF_SHIM_CAT(a, b) URF_SHIM_CAT2(a, b)
#define RCLCPP_COMPONENTS_REGISTER_NODE(NodeClass)                                                       \
  static ::rclcpp_components_shim::Registrar URF_SHIM_CAT(urf_shim_component_, __LINE__)(              \
      #NodeClass, [](const rclcpp::NodeOptions& o) { return std::shared_ptr<rclcpp::Node>(std::make_shared<NodeClass>(o)); });
