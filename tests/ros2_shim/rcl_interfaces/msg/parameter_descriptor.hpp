// ROS 2 shim (test code only): rcl_interfaces/msg/ParameterDescriptor with its FloatingPointRange and IntegerRange.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace rcl_interfaces::msg {
struct FloatingPointRange {
  double from_value = 0.0;
  double to_value = 0.0;
  double step = 0.0;
};
struct IntegerRange {
  int64_t from_value = 0;
  int64_t to_value = 0;
  uint64_t step = 0;
};
struct ParameterDescriptor {
  std::string name;
  uint8_t type = 0;
  std::string description;
  std::string additional_constraints;
  bool read_only = false;
  bool dynamic_typing = false;
  std::vector<FloatingPointRange> floating_point_range;
  std::vector<IntegerRange> integer_range;
};
}  // namespace rcl_interfaces::msg
