// ROS 2 shim (test code only): geometry_msgs/msg/Point, Vector3, Quaternion and Pose, with the IDL defaults (w = 1).
#pragma once

namespace geometry_msgs::msg {
struct Point {
  double x = 0.0, y = 0.0, z = 0.0;
};
struct Vector3 {
  double x = 0.0, y = 0.0, z = 0.0;
};
struct Quaternion {
  double x = 0.0, y = 0.0, z = 0.0, w = 1.0;
};
struct Pose {
  Point position;
  Quaternion orientation;
};
}  // namespace geometry_msgs::msg
