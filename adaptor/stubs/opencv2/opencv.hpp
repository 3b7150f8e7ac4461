// Minimal stand-in for the slice of <opencv2/opencv.hpp> the adaptor touches (cv::Mat as a non-owning or owning 2-D byte
// buffer, cv::Point2f).  Only used when the real OpenCV headers are absent (this image); in the reference's catkin
// workspace the real header is found first and this directory is not on the include path.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <memory>
#define CV_8UC1 0
#define CV_16UC1 2
#define CV_8UC3 16
namespace cv {
struct Point2f { float x = 0, y = 0; Point2f() {} Point2f(float a, float b) : x(a), y(b) {} };
class Mat {
public:
    int rows = 0, cols = 0;
    size_t step = 0;
    unsigned char *data = nullptr;
    Mat() {}
    Mat(int r, int c, int type) : rows(r), cols(c), type_(type) { step = (size_t)c * esz(); own_.reset(new unsigned char[step * r]); data = own_.get(); }
    Mat(int r, int c, int type, void *d, size_t s = 0) : rows(r), cols(c), type_(type) { data = (unsigned char *)d; step = s ? s : (size_t)c * esz(); }
    bool empty() const { return data == nullptr || rows == 0 || cols == 0; }
    int type() const { return type_; }
    template <class T> T *ptr(int r = 0) { return (T *)(data + step * r); }
    template <class T> const T *ptr(int r = 0) const { return (const T *)(data + step * r); }
private:
    size_t esz() const { return type_ == CV_16UC1 ? 2 : type_ == CV_8UC3 ? 3 : 1; }
    int type_ = CV_8UC1;
    std::shared_ptr<unsigned char[]> own_;
};
}  // namespace cv
