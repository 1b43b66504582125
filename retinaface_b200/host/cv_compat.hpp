// cv_compat.hpp -- the slice of OpenCV's C++ surface the RetinaFace class shell needs.
// With OpenCV headers installed the real ones are used (so reference callers compile unchanged);
// otherwise a minimal cv::Mat (8UC3 images and 8UC1 YUV 4:2:0 frames, row pointer + step) stands in.  No image processing
// lives here: resizing / letter-boxing / colour conversion happens on the GPU inside librf_b200.
#pragma once
#if defined(RF_USE_OPENCV) || (defined(__has_include) && __has_include(<opencv2/core.hpp>))
#include <opencv2/core.hpp>
#else
#include <cstddef>
#include <cstring>
#include <memory>
#ifndef CV_8UC1
#define CV_8UC1 0
#endif
#ifndef CV_8UC3
#define CV_8UC3 16
#endif
namespace cv {
class Mat {
   public:
    int rows = 0, cols = 0;
    unsigned char *data = nullptr;
    size_t step = 0;  // bytes per row
    Mat() {}
    // wraps caller memory (like cv::Mat(rows, cols, CV_8UC3, data, step))
    Mat(int r, int c, int type, void *d, size_t s = 0)
        : rows(r), cols(c), data((unsigned char *)d), step(s ? s : (size_t)c * cn(type)), cn_(cn(type)) {}
    Mat(int r, int c, int type) : rows(r), cols(c), step((size_t)c * cn(type)), cn_(cn(type)) {
        own_.reset(new unsigned char[(size_t)r * step](), std::default_delete<unsigned char[]>());
        data = own_.get();
    }
    bool empty() const { return data == nullptr || rows == 0 || cols == 0; }
    bool isContinuous() const { return step == (size_t)cols * cn_; }
    Mat clone() const {
        Mat m(rows, cols, cn_ == 1 ? CV_8UC1 : CV_8UC3);
        for (int y = 0; y < rows; y++) std::memcpy(m.data + (size_t)y * m.step, data + (size_t)y * step, (size_t)cols * cn_);
        return m;
    }
   private:
    static int cn(int type) { return type == CV_8UC1 ? 1 : 3; }
    int cn_ = 3;
    std::shared_ptr<unsigned char> own_;
};
}  // namespace cv
#endif
