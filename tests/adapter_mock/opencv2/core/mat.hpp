// mock of the OpenCV declarations the adapter uses from opencv2/core/mat.hpp (cv::_InputArray, core/mat.hpp) and
// opencv2/core/hal/interface.h (CV_8UC1), which the real mat.hpp includes
#pragma once
#include "../core.hpp"
#define CV_8UC1 0
namespace cv {
struct _InputArray {
    _InputArray(const Mat &m) { (void)m; }
    int type(int i = -1) const { (void)i; return CV_8UC1; }
};
}  // namespace cv
