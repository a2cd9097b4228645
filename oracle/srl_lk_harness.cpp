// TEST INFRASTRUCTURE (oracle/): C entry points of _ref/libsrl_lk_ref.so (oracle/lk.mk) over the reference's own
// LKOpticalFlowKernel (src/lkpyramid.cpp, compiled unmodified over the OpenCV stand-in in shim_lk/).  Bound by tests/lk_ref.py.
//
//   lk_create / lk_destroy   an LKOpticalFlowKernel(Size(win_w, win_h), max_level, TermCriteria(type, count, eps), flags, min_eig)
//   lk_track                 trackImage(curr_img, last_pts, curr_pts, status): the image is a header over the caller's bytes;
//                            status is copied in first, so what trackImage leaves untouched reads back unchanged
//   lk_info                  getMaxLevel() (trackImage overwrites it with the level count the pyramid build returns) and the window
//   lk_level                 level `level` of prev_img_pyr (which 0: the last image's, after trackImage's swap) or curr_img_pyr
//                            (which 1: the image before it), padding included, and its derivative buffer
//   lk_pyr_down, lk_copy_make_border   the stand-in's pyrDown and copyMakeBorder alone (tests/test_lk_pin.py)
#include "lkpyramid.h"

#include <cstring>

extern "C" {

void* lk_create(int win_w, int win_h, int max_level, int crit_type, int max_count, double epsilon, int flags, double min_eig) {
    return new LKOpticalFlowKernel(cv::Size(win_w, win_h), max_level, cv::TermCriteria(crit_type, max_count, epsilon), flags, min_eig);
}

void lk_destroy(void* h) { delete static_cast<LKOpticalFlowKernel*>(h); }

int lk_track(void* h, const uint8_t* img, int cols, int rows, size_t pitch, const float* last_pts, int64_t n, float* curr_pts, uint8_t* status) {
    auto* k = static_cast<LKOpticalFlowKernel*>(h);
    cv::Mat image(rows, cols, CV_8UC1, const_cast<uint8_t*>(img), pitch);
    std::vector<cv::Point2f> last((size_t)n), curr;
    if (n) std::memcpy(last.data(), last_pts, (size_t)n * sizeof(cv::Point2f));
    std::vector<uchar> st(status, status + n);
    const int ret = k->trackImage(image, last, curr, st);
    if (curr.size() != (size_t)n || st.size() != (size_t)n) return -1;
    if (n) {
        std::memcpy(curr_pts, curr.data(), (size_t)n * sizeof(cv::Point2f));
        std::memcpy(status, st.data(), (size_t)n);
    }
    return ret;
}

void lk_info(void* h, int* max_level, int* win_w, int* win_h, int* max_count, double* epsilon) {
    auto* k = static_cast<LKOpticalFlowKernel*>(h);
    *max_level = k->maxLevel;
    *win_w = k->lk_win_size.width;
    *win_h = k->lk_win_size.height;
    *max_count = k->terminate_criteria.maxCount;
    *epsilon = k->terminate_criteria.epsilon;
}

// level sizes: cols/rows of the level's image (without padding).  img: (rows + 2 win_h) x (cols + 2 win_w) bytes; deriv: the
// same count of (Ix, Iy) short pairs.  Either may be null.  Returns 0, or -1 when the level does not exist.
int lk_level(void* h, int which, int level, int* cols, int* rows, uint8_t* img, int16_t* deriv) {
    auto* k = static_cast<LKOpticalFlowKernel*>(h);
    const std::vector<cv::Mat>& pyr = which == 0 ? k->prev_img_pyr : k->curr_img_pyr;
    const std::vector<cv::Mat>& buf = which == 0 ? k->prev_img_deriv_I_buff : k->curr_img_deriv_I_buff;
    if (level < 0 || level >= (int)pyr.size() || pyr[level].empty()) return -1;
    const int ww = k->lk_win_size.width, wh = k->lk_win_size.height;
    cv::Mat m = pyr[level];
    *cols = m.cols;
    *rows = m.rows;
    m.adjustROI(wh, wh, ww, ww);
    if (m.cols != *cols + 2 * ww || m.rows != *rows + 2 * wh) return -1;
    if (img)
        for (int y = 0; y < m.rows; ++y) std::memcpy(img + (size_t)y * m.cols, m.ptr(y), (size_t)m.cols);
    if (deriv) {
        if (level >= (int)buf.size()) return -1;
        const cv::Mat& d = buf[level];
        if (d.cols != m.cols || d.rows != m.rows) return -1;
        for (int y = 0; y < d.rows; ++y) std::memcpy(deriv + (size_t)y * d.cols * 2, d.ptr(y), (size_t)d.cols * 4);
    }
    return 0;
}

// pyrDown of a continuous cols x rows 8-bit image into dst ((cols + 1) / 2 x (rows + 1) / 2)
void lk_pyr_down(const uint8_t* src, int cols, int rows, uint8_t* dst) {
    cv::Mat s(rows, cols, CV_8UC1, const_cast<uint8_t*>(src));
    cv::Mat d((rows + 1) / 2, (cols + 1) / 2, CV_8UC1, dst);
    cv::pyrDown(s, d, d.size());
}

// copyMakeBorder of the ROI (rx, ry, rcols, rrows) of a continuous wcols x wrows matrix of `elem`-byte elements (1: 8U, 4: 16SC2).
// inplace = 0: into a new matrix, copied to dst; its size goes to *dcols, *drows.  inplace = 1: the whole matrix is the
// destination (OpenCV's ROI-of-the-destination case); the result is copied to dst.
int lk_copy_make_border(const uint8_t* whole, int wcols, int wrows, int elem, int rx, int ry, int rcols, int rrows, int top, int bottom,
                        int left, int right, int border, int inplace, uint8_t* dst, int* dcols, int* drows) {
    const int type = elem == 1 ? CV_8UC1 : CV_MAKETYPE(CV_16S, 2);
    cv::Mat w;
    w.create(wrows, wcols, type);
    std::memcpy(w.ptr(), whole, (size_t)wrows * wcols * elem);
    cv::Mat roi = w(cv::Rect(rx, ry, rcols, rrows));
    cv::Mat out;
    if (inplace) {
        if (rcols + left + right != wcols || rrows + top + bottom != wrows) return -1;
        cv::copyMakeBorder(roi, w, top, bottom, left, right, border);
        out = w;
    } else {
        cv::copyMakeBorder(roi, out, top, bottom, left, right, border);
    }
    *dcols = out.cols;
    *drows = out.rows;
    if (dst)
        for (int y = 0; y < out.rows; ++y) std::memcpy(dst + (size_t)y * out.cols * elem, out.ptr(y), (size_t)out.cols * elem);
    return 0;
}

}  // extern "C"
