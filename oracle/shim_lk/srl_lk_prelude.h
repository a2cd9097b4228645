// TEST INFRASTRUCTURE (oracle/): force-included (-include) in front of src/lkpyramid.cpp and oracle/srl_lk_harness.cpp.
// The harness reads LKOpticalFlowKernel's private pyramids and derivative buffers: every standard header and the OpenCV
// stand-in come first, then `private` is opened up for the reference's own header (as shim/srl_prelude.h does).
#pragma once
#include <omp.h>

#include <cfloat>
#include <cstdint>
#include <cstdio>
#include <future>
#include <iostream>
#include <math.h>
#include <numeric>
#include <vector>

#include "srl_lk_cv.h"
#define private public
#define protected public
