"""The road filter node of the reference's launch/demo1.launch for ROS 2: namespace urban_road_filter, node name
urban_road_filt, with the GPU node parameters as launch arguments. rviz and rqt_reconfigure are left out: the reference's
configurations for them are ROS1 files.

    ros2 launch urban_road_filter_b200 demo1_b200.launch.py device:=0 max_points:=1048576 channels:=64
"""
from launch import LaunchDescription
from launch.actions import DeclareLaunchArgument
from launch.substitutions import LaunchConfiguration
from launch_ros.actions import Node
from launch_ros.parameter_descriptions import ParameterValue


def generate_launch_description():
    return LaunchDescription([
        DeclareLaunchArgument("device", default_value="0", description="CUDA device the node runs on"),
        DeclareLaunchArgument("max_points", default_value="1048576", description="largest scan in points"),
        DeclareLaunchArgument("channels", default_value="64", description="largest number of rings in a scan"),
        Node(
            package="urban_road_filter_b200",
            executable="lidar_road_b200",
            namespace="urban_road_filter",
            name="urban_road_filt",
            output="screen",
            parameters=[{
                "device": ParameterValue(LaunchConfiguration("device"), value_type=int),
                "max_points": ParameterValue(LaunchConfiguration("max_points"), value_type=int),
                "channels": ParameterValue(LaunchConfiguration("channels"), value_type=int),
            }],
        ),
    ])
