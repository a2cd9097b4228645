// TEST INFRASTRUCTURE (oracle/): force-included after shim/srl_prelude.h in front of the reference's src/imageProcessing.cpp
// only (oracle/vio.mk).  That file also holds the image steps of process (:91-200), which the camera-update tests never run:
// the OpenCV calls only they make are declared here with bodies that throw.  The shared stand-in headers under shim/ stay as
// they are, so every other library built from them is unchanged.
#pragma once
#include <stdexcept>
#include <vector>

#define CV_16SC2 11
namespace cv {
enum { INTER_LINEAR = 1 };
enum { COLOR_RGB2GRAY = 7, COLOR_BGR2YCrCb = 36, COLOR_YCrCb2BGR = 38 };
[[noreturn]] inline void srl_vio_image_step() { throw std::logic_error("imageProcessing's image steps are not part of the camera-update harness"); }
template <class... A> void eigen2cv(A&&...) { srl_vio_image_step(); }
template <class... A> void initUndistortRectifyMap(A&&...) { srl_vio_image_step(); }
template <class... A> void resize(A&&...) { srl_vio_image_step(); }
template <class... A> void remap(A&&...) { srl_vio_image_step(); }
template <class... A> void cvtColor(A&&...) { srl_vio_image_step(); }
template <class... A> void split(A&&...) { srl_vio_image_step(); }
template <class... A> void merge(A&&...) { srl_vio_image_step(); }
struct CLAHE { template <class... A> void apply(A&&...) { srl_vio_image_step(); } };
template <class T> struct Ptr;
template <class... A> Ptr<CLAHE> createCLAHE(A&&...) { srl_vio_image_step(); }
}  // namespace cv

// `double += rowvector * matrix * vector` (:497): real Eigen converts the 1 x 1 product to its scalar.  The stand-in evaluates
// the product as Eigen 3.3.7 does for these fixed sizes (the 1 x 3 row vector first, then its dot product with the vector,
// each a 3-term reduction c0 + (c1 + c2)); this adds the conversion.
inline double& operator+=(double& a, const Eigen::Matrix<double, 1, 1>& m) { return a += m(0, 0); }
