// ROS 2 shim (test code only): std_msgs/msg/ColorRGBA.
#pragma once

namespace std_msgs::msg {
struct ColorRGBA {
  float r = 0.0f, g = 0.0f, b = 0.0f, a = 0.0f;
};
}  // namespace std_msgs::msg
