// ROS 2 shim (test code only): rcl_interfaces/msg/SetParametersResult.
#pragma once
#include <string>

namespace rcl_interfaces::msg {
struct SetParametersResult {
  bool successful = false;
  std::string reason;
};
}  // namespace rcl_interfaces::msg
