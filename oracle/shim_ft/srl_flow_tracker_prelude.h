// TEST INFRASTRUCTURE (oracle/): force-included after shim/srl_prelude.h in front of the reference's src/opticalFlowTracker.cpp
// only (oracle/flow_tracker.mk).  The OpenCV calls that file makes, beyond the shared declaration-only stand-ins of shim/:
//   * cv::Point_'s `-` and `/ double`, restated from OpenCV 4's core/types.hpp (operator -, operator /, operator /=): a
//     difference saturate_cast to the element type, and a quotient x / b in double saturate_cast to it (for float: a plain
//     conversion).  Parity of these two against a real OpenCV is not pinned (DESIGN.md section 2).
//   * cv::findFundamentalMat, cv::solvePnPRansac and cv::cvtColor, defined by the harness (srl_flow_tracker_harness.cpp): the
//     two RANSACs return the test's mask and inliers (or throw), cvtColor does nothing (its output feeds no decision).
//   * eigen2cv and initUndistortRectifyMap (setIntrinsic, which the harness never calls): bodies that throw.
#pragma once
#include <stdexcept>
#include <string>
#include <vector>

#define CV_16SC2 11
namespace cv {
enum { COLOR_BGR2GRAY = 6 };
enum { FM_RANSAC = 8 };
struct Exception : std::exception {
    std::string msg;
    explicit Exception(const std::string& m = "") : msg(m) {}
    const char* what() const noexcept override { return msg.c_str(); }
};
template <class T> struct Point3_ { T x = 0, y = 0, z = 0; Point3_() {} Point3_(T a, T b, T c) : x(a), y(b), z(c) {} };
typedef Point3_<float> Point3f;

template <class T> inline Point_<T> operator-(const Point_<T>& a, const Point_<T>& b) {
    return Point_<T>(saturate_cast<T>(a.x - b.x), saturate_cast<T>(a.y - b.y));
}
template <class T> inline Point_<T>& operator/=(Point_<T>& a, double b) {
    a.x = saturate_cast<T>(a.x / b);
    a.y = saturate_cast<T>(a.y / b);
    return a;
}
template <class T> inline Point_<T> operator/(const Point_<T>& a, double b) {
    Point_<T> tmp(a);
    tmp /= b;
    return tmp;
}

void cvtColor(const Mat& src, Mat& dst, int code);
Mat findFundamentalMat(const std::vector<Point2f>& p1, const std::vector<Point2f>& p2, int method, double thr, double conf,
                       std::vector<uchar>& mask);
bool solvePnPRansac(const std::vector<Point3f>& p3, const std::vector<Point2f>& p2, const Mat& k, const Mat& dist, Mat& rvec, Mat& tvec,
                    bool guess, int iterations, float err, double conf, std::vector<int>& inliers);
[[noreturn]] inline void srl_ft_not_in_harness() { throw std::logic_error("opticalFlowTracker::setIntrinsic is not part of the harness"); }
template <class... A> void eigen2cv(A&&...) { srl_ft_not_in_harness(); }
template <class... A> void initUndistortRectifyMap(A&&...) { srl_ft_not_in_harness(); }
}  // namespace cv
