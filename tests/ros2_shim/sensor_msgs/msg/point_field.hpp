// ROS 2 shim (test code only): sensor_msgs/msg/PointField.
#pragma once
#include <cstdint>
#include <string>

namespace sensor_msgs::msg {
struct PointField {
  static constexpr uint8_t INT8 = 1u, UINT8 = 2u, INT16 = 3u, UINT16 = 4u, INT32 = 5u, UINT32 = 6u, FLOAT32 = 7u, FLOAT64 = 8u;
  std::string name;
  uint32_t offset = 0;
  uint8_t datatype = 0;
  uint32_t count = 0;
};
}  // namespace sensor_msgs::msg
