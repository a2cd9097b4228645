// TEST INFRASTRUCTURE (oracle/): the OpenCV stand-in of the reference's pyramidal Lucas-Kanade (src/lkpyramid.cpp,
// include/lkpyramid.h), which is compiled unmodified over it into _ref/libsrl_lk_ref.so (oracle/lk.mk).  OpenCV is not in
// this image.  Only what lkpyramid.{h,cpp} touch is here:
//   - cv::Mat with OpenCV's header semantics: shared storage, step, ROIs that remember their parent (adjustROI, locateROI,
//     isSubmatrix), create() that keeps a buffer of the right size and type, headers over external data;
//   - Size, Rect, Range, Point_ arithmetic and ddot, TermCriteria, AutoBuffer, alignSize / alignPtr, DataType, CV_MAKETYPE;
//   - cvRound / cvFloor as OpenCV 4 has them on x86-64 (cvRound = cvtss2si, round half to even; cvFloor = (int)v - (i > v));
//   - the v_int16x8 subset of the universal intrinsics used by calcSharrDeriv, on SSE2 with OpenCV's wrap-around semantics;
//   - _InputArray / _OutputArray over Mat, std::vector<Mat>, std::vector<Point2f>, std::vector<uchar>, std::vector<float>;
//   - a sequential parallel_for_;
//   - pyrDown and copyMakeBorder, restated from OpenCV 4's published imgproc/src/pyramids.cpp and core/src/copy.cpp
//     (copyMakeBorder_8u, copyMakeConstBorder_8u).  These two are NOT pinned against OpenCV itself (DESIGN.md section 2);
//     tests/test_lk_pin.py checks them against an independent numpy restatement.
// The _mm_* code inside calculateLKOpticalFlow is the real SSE2 of the compiler and is not touched.
#pragma once
#include <emmintrin.h>

#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <vector>

#define CV_MAJOR_VERSION 4
#define CV_SSE2 1
#define CV_DECL_ALIGNED(x) __attribute__((aligned(x)))
#define CV_Assert(expr)                                                                                   \
    do {                                                                                                  \
        if (!(expr)) { std::fprintf(stderr, "CV_Assert failed: %s (%s:%d)\n", #expr, __FILE__, __LINE__); std::abort(); } \
    } while (0)

#define CV_8U 0
#define CV_8S 1
#define CV_16U 2
#define CV_16S 3
#define CV_32S 4
#define CV_32F 5
#define CV_64F 6
#define CV_CN_SHIFT 3
#define CV_MAT_DEPTH(t) ((t) & 7)
#define CV_MAT_CN(t) ((((t) >> CV_CN_SHIFT) & 511) + 1)
#define CV_MAKETYPE(depth, cn) (CV_MAT_DEPTH(depth) + (((cn) - 1) << CV_CN_SHIFT))
#define CV_8UC1 CV_MAKETYPE(CV_8U, 1)
#define CV_32FC2 CV_MAKETYPE(CV_32F, 2)
#define CV_CPU_SSE2 3
#define CV_CPU_NEON 100

typedef unsigned char uchar;

inline int cvRound(double v) { return _mm_cvtsd_si32(_mm_set_sd(v)); }
inline int cvRound(float v) { return _mm_cvtss_si32(_mm_set_ss(v)); }
inline int cvFloor(double v) { int i = (int)v; return i - (i > v); }
inline int cvFloor(float v) { int i = (int)v; return i - (i > v); }

namespace cv {

enum BorderTypes {
    BORDER_CONSTANT = 0, BORDER_REPLICATE = 1, BORDER_REFLECT = 2, BORDER_WRAP = 3, BORDER_REFLECT_101 = 4,
    BORDER_TRANSPARENT = 5, BORDER_REFLECT101 = BORDER_REFLECT_101, BORDER_DEFAULT = BORDER_REFLECT_101, BORDER_ISOLATED = 16
};
enum { OPTFLOW_USE_INITIAL_FLOW = 4, OPTFLOW_LK_GET_MIN_EIGENVALS = 8, OPTFLOW_FARNEBACK_GAUSSIAN = 256 };

inline bool checkHardwareSupport(int feature) { return feature == CV_CPU_SSE2; }

template <typename T> struct DataType;
template <> struct DataType<uchar> { enum { depth = CV_8U }; };
template <> struct DataType<short> { enum { depth = CV_16S }; };
template <> struct DataType<int> { enum { depth = CV_32S }; };
template <> struct DataType<float> { enum { depth = CV_32F }; };

inline size_t alignSize(size_t sz, int n) { return (sz + n - 1) & -n; }
template <typename T> inline T* alignPtr(T* p, int n = (int)sizeof(T)) { return (T*)(((size_t)p + n - 1) & -n); }

template <typename T> class AutoBuffer {
public:
    explicit AutoBuffer(size_t n) : buf_(n ? n : 1) {}
    T* data() { return buf_.data(); }
    operator T*() { return buf_.data(); }
    operator const T*() const { return buf_.data(); }
private:
    std::vector<T> buf_;
};

template <typename T> struct Point_ {
    T x, y;
    Point_() : x(0), y(0) {}
    Point_(T x_, T y_) : x(x_), y(y_) {}
    template <typename U> operator Point_<U>() const { return Point_<U>((U)x, (U)y); }
    double ddot(const Point_& p) const { return (double)x * p.x + (double)y * p.y; }
};
template <typename T> inline Point_<T>& operator+=(Point_<T>& a, const Point_<T>& b) { a.x = a.x + b.x; a.y = a.y + b.y; return a; }
template <typename T> inline Point_<T>& operator-=(Point_<T>& a, const Point_<T>& b) { a.x = a.x - b.x; a.y = a.y - b.y; return a; }
template <typename T> inline Point_<T> operator+(const Point_<T>& a, const Point_<T>& b) { return Point_<T>(a.x + b.x, a.y + b.y); }
template <typename T> inline Point_<T> operator-(const Point_<T>& a, const Point_<T>& b) { return Point_<T>(a.x - b.x, a.y - b.y); }
template <typename T> inline Point_<T> operator*(const Point_<T>& a, float s) { return Point_<T>((T)(a.x * s), (T)(a.y * s)); }
template <typename T> inline Point_<T> operator*(const Point_<T>& a, double s) { return Point_<T>((T)(a.x * s), (T)(a.y * s)); }
template <typename T> inline bool operator==(const Point_<T>& a, const Point_<T>& b) { return a.x == b.x && a.y == b.y; }
typedef Point_<int> Point2i;
typedef Point_<float> Point2f;
typedef Point_<double> Point2d;
typedef Point2i Point;

struct Size {
    int width = 0, height = 0;
    Size() {}
    Size(int w, int h) : width(w), height(h) {}
    int area() const { return width * height; }
    bool operator==(const Size& o) const { return width == o.width && height == o.height; }
    bool operator!=(const Size& o) const { return !(*this == o); }
};
struct Rect {
    int x = 0, y = 0, width = 0, height = 0;
    Rect() {}
    Rect(int x_, int y_, int w, int h) : x(x_), y(y_), width(w), height(h) {}
};
struct Range {
    int start = 0, end = 0;
    Range() {}
    Range(int s, int e) : start(s), end(e) {}
};
struct TermCriteria {
    enum Type { COUNT = 1, MAX_ITER = COUNT, EPS = 2 };
    int type = 0, maxCount = 0;
    double epsilon = 0;
    TermCriteria() {}
    TermCriteria(int t, int c, double e) : type(t), maxCount(c), epsilon(e) {}
};

template <typename T> using Ptr = std::shared_ptr<T>;
template <typename T, typename... A> Ptr<T> makePtr(A&&... a) { return std::make_shared<T>(std::forward<A>(a)...); }

inline int elem_size1(int type) {
    static const int sz[8] = {1, 1, 2, 2, 4, 4, 8, 0};
    return sz[CV_MAT_DEPTH(type)];
}

class Mat {
public:
    int rows = 0, cols = 0;
    size_t step = 0;
    uchar* data = nullptr;
    const uchar* datastart = nullptr;
    const uchar* dataend = nullptr;

    Mat() {}
    Mat(int r, int c, int type) { create(r, c, type); }
    Mat(Size s, int type) { create(s.height, s.width, type); }
    Mat(int r, int c, int type, void* d, size_t st = 0) : rows(r), cols(c), type_(type) {
        step = st ? st : (size_t)c * elemSize();
        data = (uchar*)d;
        datastart = data;
        dataend = data + step * (r - 1) + (size_t)c * elemSize();
    }
    Mat(Size s, int type, void* d, size_t st = 0) : Mat(s.height, s.width, type, d, st) {}

    int type() const { return type_; }
    int depth() const { return CV_MAT_DEPTH(type_); }
    int channels() const { return CV_MAT_CN(type_); }
    size_t elemSize1() const { return (size_t)elem_size1(type_); }
    size_t elemSize() const { return elemSize1() * channels(); }
    bool empty() const { return data == nullptr || rows == 0 || cols == 0; }
    Size size() const { return Size(cols, rows); }
    bool isContinuous() const { return rows == 1 || step == (size_t)cols * elemSize(); }
    bool isSubmatrix() const { return submatrix_; }
    size_t total() const { return (size_t)rows * cols; }

    void create(int r, int c, int type) {
        if (data && r == rows && c == cols && type == type_) return;
        type_ = type;
        rows = r;
        cols = c;
        step = (size_t)c * elemSize();
        const size_t bytes = std::max<size_t>(step * r, 1);
        void* q = nullptr;
        CV_Assert(posix_memalign(&q, 64, alignSize(bytes, 64)) == 0);
        uchar* p = static_cast<uchar*>(q);
        store_.reset(p, [](uchar* q) { std::free(q); });
        data = p;
        datastart = p;
        dataend = p + step * r;
        submatrix_ = false;
    }
    void create(Size s, int type) { create(s.height, s.width, type); }
    void release() { *this = Mat(); }

    uchar* ptr(int y = 0) { return data + step * y; }
    const uchar* ptr(int y = 0) const { return data + step * y; }
    template <typename T> T* ptr(int y = 0) { return (T*)(data + step * y); }
    template <typename T> const T* ptr(int y = 0) const { return (const T*)(data + step * y); }

    Mat operator()(const Rect& r) const {
        CV_Assert(r.x >= 0 && r.y >= 0 && r.width >= 0 && r.height >= 0 && r.x + r.width <= cols && r.y + r.height <= rows);
        Mat m = *this;
        m.data = data + step * r.y + elemSize() * r.x;
        m.rows = r.height;
        m.cols = r.width;
        if (r.width < cols || r.height < rows) m.submatrix_ = true;
        return m;
    }

    void locateROI(Size& wholeSize, Point& ofs) const {
        const size_t esz = elemSize();
        const ptrdiff_t delta1 = data - datastart, delta2 = dataend - datastart;
        if (delta1 == 0) {
            ofs.x = ofs.y = 0;
        } else {
            ofs.y = (int)(delta1 / step);
            ofs.x = (int)((delta1 - step * ofs.y) / esz);
        }
        const size_t minstep = (ofs.x + cols) * esz;
        wholeSize.height = (int)((delta2 - minstep) / step + 1);
        wholeSize.height = std::max(wholeSize.height, ofs.y + rows);
        wholeSize.width = (int)((delta2 - step * (wholeSize.height - 1)) / esz);
        wholeSize.width = std::max(wholeSize.width, ofs.x + cols);
    }

    Mat& adjustROI(int dtop, int dbottom, int dleft, int dright) {
        Size wholeSize;
        Point ofs;
        const size_t esz = elemSize();
        locateROI(wholeSize, ofs);
        int row1 = std::min(std::max(ofs.y - dtop, 0), wholeSize.height), row2 = std::max(0, std::min(ofs.y + rows + dbottom, wholeSize.height));
        int col1 = std::min(std::max(ofs.x - dleft, 0), wholeSize.width), col2 = std::max(0, std::min(ofs.x + cols + dright, wholeSize.width));
        if (row1 > row2) std::swap(row1, row2);
        if (col1 > col2) std::swap(col1, col2);
        data += (row1 - ofs.y) * (ptrdiff_t)step + (col1 - ofs.x) * (ptrdiff_t)esz;
        rows = row2 - row1;
        cols = col2 - col1;
        submatrix_ = !(rows == wholeSize.height && cols == wholeSize.width);
        return *this;
    }

    void copyTo(Mat& dst) const {
        dst.create(rows, cols, type_);
        for (int y = 0; y < rows; ++y) std::memcpy(dst.ptr(y), ptr(y), (size_t)cols * elemSize());
    }
    void copyTo(Mat&& dst) const { Mat d = dst; copyTo(d); }   // into a ROI header of the right size

    int checkVector(int elemChannels, int depth_ = -1, bool requireContinuous = true) const {
        if (data == nullptr) return 0;
        if (depth_ >= 0 && depth() != depth_) return -1;
        if (requireContinuous && !isContinuous()) return -1;
        if (channels() == elemChannels && (cols == 1 || rows == 1)) return rows * cols;
        if (channels() == 1 && cols == elemChannels) return rows;
        return -1;
    }

private:
    int type_ = 0;
    bool submatrix_ = false;
    std::shared_ptr<uchar> store_;
};

// ---- _InputArray / _OutputArray over the kinds lkpyramid.cpp hands them -------------------------------------------------
class _InputArray {
public:
    enum Kind { NONE, MAT, STD_VECTOR_MAT, STD_VECTOR_POINT2F, STD_VECTOR_UCHAR, STD_VECTOR_FLOAT };
    _InputArray() {}
    _InputArray(const Mat& m) : kind_(MAT), obj_((void*)&m) {}
    _InputArray(const std::vector<Mat>& v) : kind_(STD_VECTOR_MAT), obj_((void*)&v) {}
    _InputArray(const std::vector<Point2f>& v) : kind_(STD_VECTOR_POINT2F), obj_((void*)&v) {}
    _InputArray(const std::vector<uchar>& v) : kind_(STD_VECTOR_UCHAR), obj_((void*)&v) {}
    _InputArray(const std::vector<float>& v) : kind_(STD_VECTOR_FLOAT), obj_((void*)&v) {}

    Mat getMat(int i = -1) const {
        switch (kind_) {
        case MAT: return *(Mat*)obj_;
        case STD_VECTOR_MAT: return (*(std::vector<Mat>*)obj_)[i < 0 ? 0 : i];
        case STD_VECTOR_POINT2F: { auto& v = *(std::vector<Point2f>*)obj_; return v.empty() ? Mat() : Mat((int)v.size(), 1, CV_32FC2, v.data()); }
        case STD_VECTOR_UCHAR: { auto& v = *(std::vector<uchar>*)obj_; return v.empty() ? Mat() : Mat((int)v.size(), 1, CV_8UC1, v.data()); }
        case STD_VECTOR_FLOAT: { auto& v = *(std::vector<float>*)obj_; return v.empty() ? Mat() : Mat((int)v.size(), 1, CV_32F, v.data()); }
        default: return Mat();
        }
    }
    bool needed() const { return kind_ != NONE; }

protected:
    Kind kind_ = NONE;
    void* obj_ = nullptr;
};

class _OutputArray : public _InputArray {
public:
    _OutputArray() {}
    _OutputArray(Mat& m) : _InputArray(m) {}
    _OutputArray(std::vector<Mat>& v) : _InputArray(v) {}
    _OutputArray(std::vector<Point2f>& v) : _InputArray(v) {}
    _OutputArray(std::vector<uchar>& v) : _InputArray(v) {}
    _OutputArray(std::vector<float>& v) : _InputArray(v) {}

    // i < 0 on a vector kind: resize the vector to rows * cols elements (rows or cols is 1), as OpenCV does
    void create(int r, int c, int mtype, int i = -1, bool allowTransposed = false, int fixedDepthMask = 0) const {
        (void)allowTransposed; (void)fixedDepthMask;
        const size_t len = (size_t)r * c > 0 ? (size_t)r + c - 1 : 0;
        switch (kind_) {
        case MAT: ((Mat*)obj_)->create(r, c, mtype); break;
        case STD_VECTOR_MAT:
            if (i < 0) ((std::vector<Mat>*)obj_)->resize(len);
            else (*(std::vector<Mat>*)obj_)[i].create(r, c, mtype);
            break;
        case STD_VECTOR_POINT2F: ((std::vector<Point2f>*)obj_)->resize(len); break;
        case STD_VECTOR_UCHAR: ((std::vector<uchar>*)obj_)->resize(len); break;
        case STD_VECTOR_FLOAT: ((std::vector<float>*)obj_)->resize(len); break;
        default: CV_Assert(!"create() on an empty _OutputArray");
        }
    }
    void create(Size sz, int mtype, int i = -1, bool allowTransposed = false, int fixedDepthMask = 0) const {
        create(sz.height, sz.width, mtype, i, allowTransposed, fixedDepthMask);
    }
    Mat& getMatRef(int i = -1) const {
        if (kind_ == MAT) return *(Mat*)obj_;
        CV_Assert(kind_ == STD_VECTOR_MAT && i >= 0);
        return (*(std::vector<Mat>*)obj_)[i];
    }
    void release() const {
        switch (kind_) {
        case MAT: ((Mat*)obj_)->release(); break;
        case STD_VECTOR_MAT: ((std::vector<Mat>*)obj_)->clear(); break;
        case STD_VECTOR_POINT2F: ((std::vector<Point2f>*)obj_)->clear(); break;
        case STD_VECTOR_UCHAR: ((std::vector<uchar>*)obj_)->clear(); break;
        case STD_VECTOR_FLOAT: ((std::vector<float>*)obj_)->clear(); break;
        default: break;
        }
    }
};
typedef _OutputArray _InputOutputArray;
typedef const _InputArray& InputArray;
typedef InputArray InputArrayOfArrays;
typedef const _OutputArray& OutputArray;
typedef OutputArray OutputArrayOfArrays;
typedef OutputArray InputOutputArray;
inline _InputOutputArray& noArray() { static _InputOutputArray none; return none; }

// ---- parallel_for_: sequential ---------------------------------------------------------------------------------------------
class ParallelLoopBody {
public:
    virtual ~ParallelLoopBody() {}
    virtual void operator()(const Range& range) const = 0;
};
inline void parallel_for_(const Range& range, const ParallelLoopBody& body, double nstripes = -1.) { (void)nstripes; body(range); }
inline void parallel_for_(const Range& range, std::function<void(const Range&)> functor, double nstripes = -1.) { (void)nstripes; functor(range); }

// ---- the v_int16x8 subset of the universal intrinsics (SSE2; add, sub and mul wrap around as in OpenCV) ---------------------
struct v_uint16x8 { __m128i val; };
struct v_int16x8 { __m128i val; };
inline v_int16x8 v_setall_s16(short v) { return v_int16x8{_mm_set1_epi16(v)}; }
inline v_int16x8 v_reinterpret_as_s16(const v_uint16x8& a) { return v_int16x8{a.val}; }
inline v_uint16x8 v_load_expand(const uchar* p) { return v_uint16x8{_mm_unpacklo_epi8(_mm_loadl_epi64((const __m128i*)p), _mm_setzero_si128())}; }
inline v_int16x8 v_load(const short* p) { return v_int16x8{_mm_loadu_si128((const __m128i*)p)}; }
inline void v_store(short* p, const v_int16x8& a) { _mm_storeu_si128((__m128i*)p, a.val); }
inline v_int16x8 operator+(const v_int16x8& a, const v_int16x8& b) { return v_int16x8{_mm_add_epi16(a.val, b.val)}; }
inline v_int16x8 operator-(const v_int16x8& a, const v_int16x8& b) { return v_int16x8{_mm_sub_epi16(a.val, b.val)}; }
inline v_int16x8 operator*(const v_int16x8& a, const v_int16x8& b) { return v_int16x8{_mm_mullo_epi16(a.val, b.val)}; }
// (a0 b0 a1 b1 ... a7 b7)
inline void v_store_interleave(short* p, const v_int16x8& a, const v_int16x8& b) {
    _mm_storeu_si128((__m128i*)p, _mm_unpacklo_epi16(a.val, b.val));
    _mm_storeu_si128((__m128i*)(p + 8), _mm_unpackhi_epi16(a.val, b.val));
}

// ---- borderInterpolate, copyMakeBorder, pyrDown (OpenCV 4, restated; parity unpinned) ---------------------------------------
inline int borderInterpolate(int p, int len, int borderType) {
    if ((unsigned)p < (unsigned)len) return p;
    if (borderType == BORDER_REPLICATE) return p < 0 ? 0 : len - 1;
    if (borderType == BORDER_REFLECT || borderType == BORDER_REFLECT_101) {
        const int delta = borderType == BORDER_REFLECT_101;
        if (len == 1) return 0;
        do {
            if (p < 0) p = -p - 1 + delta;
            else p = len - 1 - (p - len) - delta;
        } while ((unsigned)p >= (unsigned)len);
        return p;
    }
    if (borderType == BORDER_WRAP) {
        if (p < 0) p -= ((p - len + 1) / len) * len;
        if (p >= len) p %= len;
        return p;
    }
    return -1;   // BORDER_CONSTANT
}

// dst (dstroi) already holds, or receives, src (srcroi) at (top, left); the border is filled from the copied interior.
// src may lie inside dst (the in-place case of a ROI of dst): then the interior is not copied.
inline void copyMakeBorder_8u(const uchar* src, size_t srcstep, Size srcroi, uchar* dst, size_t dststep, Size dstroi, int top, int left, int cn,
                              int borderType) {
    std::vector<int> tab((size_t)std::max(dstroi.width - srcroi.width, 0) * cn + 1);
    const int right = dstroi.width - srcroi.width - left;
    const int bottom = dstroi.height - srcroi.height - top;
    for (int i = 0; i < left; i++) {
        const int j = borderInterpolate(i - left, srcroi.width, borderType) * cn;
        for (int k = 0; k < cn; k++) tab[i * cn + k] = j + k;
    }
    for (int i = 0; i < right; i++) {
        const int j = borderInterpolate(srcroi.width + i, srcroi.width, borderType) * cn;
        for (int k = 0; k < cn; k++) tab[(i + left) * cn + k] = j + k;
    }
    const int sw = srcroi.width * cn, dw = dstroi.width * cn, l = left * cn, r = right * cn;
    uchar* dstInner = dst + dststep * top + l;
    for (int i = 0; i < srcroi.height; i++, dstInner += dststep, src += srcstep) {
        if (dstInner != src) std::memcpy(dstInner, src, sw);
        for (int j = 0; j < l; j++) dstInner[j - l] = src[tab[j]];
        for (int j = 0; j < r; j++) dstInner[j + sw] = src[tab[j + l]];
    }
    dst += dststep * top;
    for (int i = 0; i < top; i++) {
        const int j = borderInterpolate(i - top, srcroi.height, borderType);
        std::memcpy(dst + (i - top) * (ptrdiff_t)dststep, dst + j * (ptrdiff_t)dststep, dw);
    }
    for (int i = 0; i < bottom; i++) {
        const int j = borderInterpolate(i + srcroi.height, srcroi.height, borderType);
        std::memcpy(dst + (i + srcroi.height) * (ptrdiff_t)dststep, dst + j * (ptrdiff_t)dststep, dw);
    }
}

// constant border of zero bytes (the only value lkpyramid.cpp asks for)
inline void copyMakeConstBorder_8u(const uchar* src, size_t srcstep, Size srcroi, uchar* dst, size_t dststep, Size dstroi, int top, int left, int cn) {
    const int right = dstroi.width - srcroi.width - left;
    const int bottom = dstroi.height - srcroi.height - top;
    const int sw = srcroi.width * cn, dw = dstroi.width * cn, l = left * cn, r = right * cn;
    uchar* dstInner = dst + dststep * top + l;
    for (int i = 0; i < srcroi.height; i++, dstInner += dststep, src += srcstep) {
        if (dstInner != src) std::memcpy(dstInner, src, sw);
        std::memset(dstInner - l, 0, l);
        std::memset(dstInner + sw, 0, r);
    }
    for (int i = 0; i < top; i++) std::memset(dst + i * dststep, 0, dw);
    dst += dststep * (top + srcroi.height);
    for (int i = 0; i < bottom; i++) std::memset(dst + i * dststep, 0, dw);
}

inline void copyMakeBorder(InputArray _src, OutputArray _dst, int top, int bottom, int left, int right, int borderType) {
    CV_Assert(top >= 0 && bottom >= 0 && left >= 0 && right >= 0);
    Mat src = _src.getMat();
    const int type = src.type();
    if (src.isSubmatrix() && (borderType & BORDER_ISOLATED) == 0) {
        Size wholeSize;
        Point ofs;
        src.locateROI(wholeSize, ofs);
        const int dtop = std::min(ofs.y, top);
        const int dbottom = std::min(wholeSize.height - src.rows - ofs.y, bottom);
        const int dleft = std::min(ofs.x, left);
        const int dright = std::min(wholeSize.width - src.cols - ofs.x, right);
        src.adjustROI(dtop, dbottom, dleft, dright);
        top -= dtop;
        left -= dleft;
        bottom -= dbottom;
        right -= dright;
    }
    _dst.create(src.rows + top + bottom, src.cols + left + right, type);
    Mat dst = _dst.getMat();
    if (top == 0 && left == 0 && bottom == 0 && right == 0) {
        if (src.data != dst.data || src.step != dst.step) src.copyTo(dst);
        return;
    }
    borderType &= ~BORDER_ISOLATED;
    if (borderType != BORDER_CONSTANT)
        copyMakeBorder_8u(src.ptr(), src.step, src.size(), dst.ptr(), dst.step, dst.size(), top, left, (int)src.elemSize(), borderType);
    else
        copyMakeConstBorder_8u(src.ptr(), src.step, src.size(), dst.ptr(), dst.step, dst.size(), top, left, (int)src.elemSize());
}

// 5x5 Gaussian [1 4 6 4 1]^2 / 256 at (2x, 2y), integer rows then columns, (s + 128) >> 8; 8-bit, one channel
inline void pyrDown(InputArray _src, OutputArray _dst, const Size& dstsize = Size(), int borderType = BORDER_DEFAULT) {
    Mat src = _src.getMat();
    CV_Assert(src.type() == CV_8UC1 && borderType != BORDER_CONSTANT);
    const Size ssize = src.size();
    const Size dsize = dstsize.width <= 0 ? Size((ssize.width + 1) / 2, (ssize.height + 1) / 2) : dstsize;
    CV_Assert(std::abs(dsize.width * 2 - ssize.width) <= 2 && std::abs(dsize.height * 2 - ssize.height) <= 2);
    _dst.create(dsize, src.type());
    Mat dst = _dst.getMat();
    std::vector<int> rowbuf((size_t)5 * dsize.width);
    for (int y = 0; y < dsize.height; y++) {
        for (int k = 0; k < 5; k++) {
            const uchar* s = src.ptr(borderInterpolate(2 * y - 2 + k, ssize.height, borderType));
            int* row = rowbuf.data() + (size_t)k * dsize.width;
            for (int x = 0; x < dsize.width; x++) {
                const int x0 = borderInterpolate(2 * x - 2, ssize.width, borderType), x1 = borderInterpolate(2 * x - 1, ssize.width, borderType);
                const int x3 = borderInterpolate(2 * x + 1, ssize.width, borderType), x4 = borderInterpolate(2 * x + 2, ssize.width, borderType);
                row[x] = s[2 * x] * 6 + (s[x1] + s[x3]) * 4 + s[x0] + s[x4];
            }
        }
        uchar* d = dst.ptr(y);
        const int *r0 = rowbuf.data(), *r1 = r0 + dsize.width, *r2 = r1 + dsize.width, *r3 = r2 + dsize.width, *r4 = r3 + dsize.width;
        for (int x = 0; x < dsize.width; x++) d[x] = (uchar)((r2[x] * 6 + (r1[x] + r3[x]) * 4 + r0[x] + r4[x] + 128) >> 8);
    }
}

}  // namespace cv
