// ROS 2 shim (test code only): visualization_msgs/msg/Marker and MarkerArray, the fields ros2/urf_ros2_node.cpp uses.
#pragma once
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include <builtin_interfaces/msg/duration.hpp>
#include <geometry_msgs/msg/point.hpp>
#include <std_msgs/msg/color_rgba.hpp>
#include <std_msgs/msg/header.hpp>

namespace visualization_msgs::msg {
struct Marker {
  static constexpr int32_t LINE_STRIP = 4;
  static constexpr int32_t ADD = 0, DELETE = 2;
  std_msgs::msg::Header header;
  std::string ns;
  int32_t id = 0;
  int32_t type = 0;
  int32_t action = 0;
  geometry_msgs::msg::Pose pose;
  geometry_msgs::msg::Vector3 scale;
  std_msgs::msg::ColorRGBA color;
  builtin_interfaces::msg::Duration lifetime;
  bool frame_locked = false;
  std::vector<geometry_msgs::msg::Point> points;
};
struct MarkerArray {
  using SharedPtr = std::shared_ptr<MarkerArray>;
  using ConstSharedPtr = std::shared_ptr<const MarkerArray>;
  using UniquePtr = std::unique_ptr<MarkerArray>;
  std::vector<Marker> markers;
};
}  // namespace visualization_msgs::msg
