// ROS 2 shim (test code only): std_msgs/msg/Header.
#pragma once
#include <string>

#include <builtin_interfaces/msg/time.hpp>

namespace std_msgs::msg {
struct Header {
  builtin_interfaces::msg::Time stamp;
  std::string frame_id;
};
}  // namespace std_msgs::msg
