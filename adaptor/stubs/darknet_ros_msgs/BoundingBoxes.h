// Minimal stand-in for the message headers darknet_ros generates from darknet_ros_msgs/msg/BoundingBox.msg and
// BoundingBoxes.msg: the fields, with the types the .msg files give them.  Only used where the ROS-generated headers are
// absent (this image); in the reference's catkin workspace the generated header is found first and this directory is not on
// the include path.
#pragma once
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

namespace std_msgs {
struct Header {            // std_msgs/Header (stamp as seconds here; ros::Time in ROS)
    uint32_t seq = 0;
    double stamp = 0;
    std::string frame_id;
};
}  // namespace std_msgs

namespace darknet_ros_msgs {
struct BoundingBox {
    double probability = 0;
    int64_t xmin = 0, ymin = 0, xmax = 0, ymax = 0;
    int16_t id = 0;
    std::string Class;
};
struct BoundingBoxes {
    std_msgs::Header header;
    std_msgs::Header image_header;
    std::vector<BoundingBox> bounding_boxes;
};
typedef std::shared_ptr<BoundingBoxes> BoundingBoxesPtr;
typedef std::shared_ptr<const BoundingBoxes> BoundingBoxesConstPtr;   // boost::shared_ptr in ROS 1
}  // namespace darknet_ros_msgs
