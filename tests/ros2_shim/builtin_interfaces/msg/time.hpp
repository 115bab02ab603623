// ROS 2 shim (test code only): builtin_interfaces/msg/Time.
#pragma once
#include <cstdint>

namespace builtin_interfaces::msg {
struct Time {
  int32_t sec = 0;
  uint32_t nanosec = 0;
};
}  // namespace builtin_interfaces::msg
