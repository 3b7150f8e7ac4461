// yolo_check: YoloObjectDetector on one raw BGR8 frame, for the tests (tests/test_detector_tf32_gpu.py).
//   yolo_check cfg weights thresh precision frame.bgr width height
// precision: GF_DETECTOR_EXACT (0) or GF_DETECTOR_TF32 (1), applied by setPrecision.  Prints one line per published box:
// class id, probability (%.9g) and xmin ymin xmax ymax.
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iterator>
#include <vector>

#include "yolo_object_detector.h"

int main(int argc, char** argv)
{
    if (argc != 8) {
        fprintf(stderr, "usage: yolo_check cfg weights thresh precision frame.bgr width height\n");
        return 2;
    }
    const int w = atoi(argv[6]), h = atoi(argv[7]);
    std::ifstream f(argv[5], std::ios::binary);
    std::vector<unsigned char> bgr((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    if ((long)bgr.size() != 3l * w * h) {
        fprintf(stderr, "frame size mismatch\n");
        return 2;
    }
    try {
        YoloObjectDetector det(argv[1], argv[2], (float)atof(argv[3]));
        det.setPrecision(atoi(argv[4]));
        cv::Mat m(h, w, CV_8UC3, bgr.data());
        const darknet_ros_msgs::BoundingBoxes boxes = det.detect(m);
        for (const auto& b : boxes.bounding_boxes)
            printf("%d %.9g %lld %lld %lld %lld\n", (int)b.id, (double)b.probability, (long long)b.xmin, (long long)b.ymin,
                   (long long)b.xmax, (long long)b.ymax);
    } catch (const std::exception& e) {
        fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    return 0;
}
