// Stand-in for the OpenCV C++ headers, ONLY so that the reference's own first-party sources
//     /root/reference/src/mdBRIEFextractorOct.cpp, src/cam_model_omni.cpp, src/misc.cpp
// compile WHERE THEY LIE in a container that has no OpenCV C++ (oracle/Makefile target `ref`).   TEST INFRASTRUCTURE.
//
// What is ours here and what is the reference's: every line of reference logic (constructor tables, pyramid driver, cell
// loop, DistributeOctTree incl. its std::list / pointer-sort behaviour, IC_Angle, pattern rotation + distortion,
// ORB/dBRIEF/mdBRIEF bit tests, output assembly, the camera model) runs from the reference's unmodified sources.  This header
// supplies the un-vendored third-party layer underneath: cv::Mat (ref-counted, ROI views with parent tracking), the small
// geometric types, and the six image primitives the path calls -- resize (INTER_LINEAR / INTER_NEAREST), copyMakeBorder,
// boxFilter, FAST-9/16 + NMS + mask filter, fastAtan2, cvRound/cvFloor/cvCeil -- written from OpenCV's published algorithms
// and pinned bit for bit against the real cv2 4.13 by tests/test_ref_stub_cv2.py (run where cv2 is importable) and
// oracle/pin_ref.py.  Anything the path does not touch is absent on purpose.
#pragma once
#include <algorithm>
#include <cassert>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <limits>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#define CV_8U 0
#define CV_8S 1
#define CV_16U 2
#define CV_16S 3
#define CV_32S 4
#define CV_32F 5
#define CV_64F 6
#define CV_MAKETYPE(depth, cn) ((depth) + (((cn) - 1) << 3))
#define CV_8UC1 CV_MAKETYPE(CV_8U, 1)
#define CV_32FC1 CV_MAKETYPE(CV_32F, 1)
#define CV_64FC1 CV_MAKETYPE(CV_64F, 1)
#define CV_PI 3.1415926535897932384626433832795
#define CV_Assert(expr) do { if (!(expr)) throw cv::Exception(#expr); } while (0)

// OpenCV core/fast_math.hpp: cvRound = round-half-to-even (lrint), cvFloor / cvCeil by truncation + correction.  cvRound(double)
// on x86-64 is cvtsd2si: NaN and values outside int give INT_MIN (a plain (int)lrint would wrap 2^32 + 5 to 5)
inline int cvRound(double v) { const double r = nearbyint(v); return (r >= -2147483648.0 && r < 2147483648.0) ? (int)r : (-2147483647 - 1); }
inline int cvRound(float v) { return (int)lrintf(v); }
inline int cvRound(int v) { return v; }
inline int cvFloor(double v) { int i = (int)v; return i - (i > v); }
inline int cvFloor(float v) { int i = (int)v; return i - (i > v); }
inline int cvCeil(double v) { int i = (int)v; return i + (i < v); }
inline int cvCeil(float v) { int i = (int)v; return i + (i < v); }

namespace cv {

typedef unsigned char uchar;

struct Exception : public std::runtime_error {
    explicit Exception(const char* what) : std::runtime_error(what) {}
};

template <class T> inline T saturate_cast(double v) { return (T)v; }
template <> inline uchar saturate_cast<uchar>(double v) { int i = cvRound(v); return (uchar)(i < 0 ? 0 : (i > 255 ? 255 : i)); }
template <> inline int saturate_cast<int>(double v) { return cvRound(v); }

// ---------------------------------------------------------------------------------------------- small geometric types
template <class T, int N> struct Vec;
template <class T> struct Point_ {
    T x, y;
    Point_() : x(0), y(0) {}
    Point_(T x_, T y_) : x(x_), y(y_) {}
    Point_(const Vec<T, 2>& v);                      // cv::Point_(const Vec<_Tp, 2>&): used at src/mdBRIEFextractorOct.cpp:369,429
    template <class U> Point_(const Point_<U>& o) : x((T)o.x), y((T)o.y) {}
};
template <class T> inline Point_<T>& operator*=(Point_<T>& a, float b) { a.x = (T)(a.x * b); a.y = (T)(a.y * b); return a; }
template <class T> inline Point_<T>& operator*=(Point_<T>& a, double b) { a.x = (T)(a.x * b); a.y = (T)(a.y * b); return a; }
template <class T> inline Point_<T>& operator*=(Point_<T>& a, int b) { a.x = (T)(a.x * b); a.y = (T)(a.y * b); return a; }
template <class T> inline Point_<T> operator+(const Point_<T>& a, const Point_<T>& b) { return Point_<T>(a.x + b.x, a.y + b.y); }
template <class T> inline Point_<T> operator-(const Point_<T>& a, const Point_<T>& b) { return Point_<T>(a.x - b.x, a.y - b.y); }
typedef Point_<int> Point2i;
typedef Point_<int> Point;
typedef Point_<float> Point2f;
typedef Point_<double> Point2d;

template <class T> struct Point3_ {
    T x, y, z;
    Point3_() : x(0), y(0), z(0) {}
    Point3_(T x_, T y_, T z_) : x(x_), y(y_), z(z_) {}
};
typedef Point3_<double> Point3d;
typedef Point3_<float> Point3f;

template <class T> struct Size_ {
    T width, height;
    Size_() : width(0), height(0) {}
    Size_(T w, T h) : width(w), height(h) {}
};
typedef Size_<int> Size;

template <class T> struct Rect_ {
    T x, y, width, height;
    Rect_() : x(0), y(0), width(0), height(0) {}
    Rect_(T x_, T y_, T w, T h) : x(x_), y(y_), width(w), height(h) {}
};
typedef Rect_<int> Rect;

struct Scalar {
    double val[4];
    Scalar(double a = 0, double b = 0, double c = 0, double d = 0) { val[0] = a; val[1] = b; val[2] = c; val[3] = d; }
};

// fixed-size matrices: enough of cv::Matx / cv::Vec for include/misc.h and src/misc.cpp
template <class T, int M, int N> struct Matx {
    T val[M * N];
    Matx() { for (int i = 0; i < M * N; ++i) val[i] = T(0); }
    template <class... A, class = typename std::enable_if<(sizeof...(A) == M * N) && (M * N > 1)>::type>
    Matx(A... a) { const T v[] = {(T)a...}; for (int i = 0; i < M * N; ++i) val[i] = v[i]; }
    explicit Matx(T v0) { for (int i = 0; i < M * N; ++i) val[i] = T(0); val[0] = v0; }
    static Matx eye() { Matx m; for (int i = 0; i < (M < N ? M : N); ++i) m(i, i) = T(1); return m; }
    static Matx zeros() { return Matx(); }
    T& operator()(int r, int c) { return val[r * N + c]; }
    const T& operator()(int r, int c) const { return val[r * N + c]; }
    T& operator()(int i) { return val[i]; }
    const T& operator()(int i) const { return val[i]; }
    Matx<T, N, M> t() const { Matx<T, N, M> r; for (int i = 0; i < M; ++i) for (int j = 0; j < N; ++j) r(j, i) = (*this)(i, j); return r; }
    T dot(const Matx& o) const { T s = T(0); for (int i = 0; i < M * N; ++i) s += val[i] * o.val[i]; return s; }
    template <int M1, int N1> Matx<T, M1, N1> get_minor(int r0, int c0) const {
        Matx<T, M1, N1> r; for (int i = 0; i < M1; ++i) for (int j = 0; j < N1; ++j) r(i, j) = (*this)(r0 + i, c0 + j); return r;
    }
    Matx<T, N, M> inv() const {                      // Gauss-Jordan with partial pivoting (square matrices only are used)
        static_assert(M == N, "inv(): square matrix");
        Matx a = *this; Matx r = Matx::eye();
        for (int c = 0; c < N; ++c) {
            int p = c;
            for (int i = c + 1; i < N; ++i) if (std::abs(a(i, c)) > std::abs(a(p, c))) p = i;
            if (a(p, c) == T(0)) return Matx<T, N, M>();
            for (int j = 0; j < N; ++j) { std::swap(a(c, j), a(p, j)); std::swap(r(c, j), r(p, j)); }
            const T d = a(c, c);
            for (int j = 0; j < N; ++j) { a(c, j) /= d; r(c, j) /= d; }
            for (int i = 0; i < N; ++i) if (i != c) { const T f = a(i, c); for (int j = 0; j < N; ++j) { a(i, j) -= f * a(c, j); r(i, j) -= f * r(c, j); } }
        }
        return r;
    }
};
template <class T, int N> struct Vec : public Matx<T, N, 1> {
    Vec() {}
    template <class... A, class = typename std::enable_if<(sizeof...(A) == N) && (N > 1)>::type>
    Vec(A... a) : Matx<T, N, 1>(a...) {}
    Vec(T v0) : Matx<T, N, 1>(v0) {}                 // cv::Vec(_Tp v0) is implicit: `pt2 = 0.0;` (src/cam_system_omni.cpp:56)
    Vec(const Matx<T, N, 1>& m) : Matx<T, N, 1>(m) {}
    T& operator[](int i) { return this->val[i]; }
    const T& operator[](int i) const { return this->val[i]; }
    T& operator()(int i) { return this->val[i]; }
    const T& operator()(int i) const { return this->val[i]; }
    T dot(const Vec& o) const { T s = T(0); for (int i = 0; i < N; ++i) s += this->val[i] * o.val[i]; return s; }
};
template <class T> inline Point_<T>::Point_(const Vec<T, 2>& v) : x(v.val[0]), y(v.val[1]) {}
template <class T, int M, int N> inline Matx<T, M, N> operator+(const Matx<T, M, N>& a, const Matx<T, M, N>& b) { Matx<T, M, N> r; for (int i = 0; i < M * N; ++i) r.val[i] = a.val[i] + b.val[i]; return r; }
template <class T, int M, int N> inline Matx<T, M, N> operator-(const Matx<T, M, N>& a, const Matx<T, M, N>& b) { Matx<T, M, N> r; for (int i = 0; i < M * N; ++i) r.val[i] = a.val[i] - b.val[i]; return r; }
template <class T, int M, int N> inline Matx<T, M, N> operator-(const Matx<T, M, N>& a) { Matx<T, M, N> r; for (int i = 0; i < M * N; ++i) r.val[i] = -a.val[i]; return r; }
template <class T, int M, int N> inline Matx<T, M, N> operator*(const Matx<T, M, N>& a, double s) { Matx<T, M, N> r; for (int i = 0; i < M * N; ++i) r.val[i] = (T)(a.val[i] * s); return r; }
template <class T, int M, int N> inline Matx<T, M, N> operator*(double s, const Matx<T, M, N>& a) { return a * s; }
template <class T, int M, int L, int N> inline Matx<T, M, N> operator*(const Matx<T, M, L>& a, const Matx<T, L, N>& b) {
    Matx<T, M, N> r;
    for (int i = 0; i < M; ++i) for (int j = 0; j < N; ++j) { T s = T(0); for (int k = 0; k < L; ++k) s += a(i, k) * b(k, j); r(i, j) = s; }
    return r;
}
template <class T, int M, int N> inline Vec<T, M> operator*(const Matx<T, M, N>& a, const Vec<T, N>& b) {
    Vec<T, M> r;
    for (int i = 0; i < M; ++i) { T s = T(0); for (int k = 0; k < N; ++k) s += a(i, k) * b.val[k]; r.val[i] = s; }
    return r;
}
template <class T, int N> inline Vec<T, N> operator+(const Vec<T, N>& a, const Vec<T, N>& b) { Vec<T, N> r; for (int i = 0; i < N; ++i) r.val[i] = a.val[i] + b.val[i]; return r; }
template <class T, int N> inline Vec<T, N> operator-(const Vec<T, N>& a, const Vec<T, N>& b) { Vec<T, N> r; for (int i = 0; i < N; ++i) r.val[i] = a.val[i] - b.val[i]; return r; }
template <class T, int N> inline Vec<T, N> operator-(const Vec<T, N>& a) { Vec<T, N> r; for (int i = 0; i < N; ++i) r.val[i] = -a.val[i]; return r; }
template <class T, int N> inline Vec<T, N> operator*(const Vec<T, N>& a, double s) { Vec<T, N> r; for (int i = 0; i < N; ++i) r.val[i] = (T)(a.val[i] * s); return r; }
template <class T, int N> inline Vec<T, N> operator*(double s, const Vec<T, N>& a) { return a * s; }
template <class T, int N> inline Vec<T, N>& operator/=(Vec<T, N>& a, double s) { for (int i = 0; i < N; ++i) a.val[i] = (T)(a.val[i] / s); return a; }
template <class T, int M, int N> inline double norm(const Matx<T, M, N>& a) { double s = 0; for (int i = 0; i < M * N; ++i) s += (double)a.val[i] * a.val[i]; return std::sqrt(s); }
typedef Matx<double, 2, 2> Matx22d;
typedef Matx<double, 3, 3> Matx33d;
typedef Matx<double, 4, 4> Matx44d;
typedef Matx<double, 3, 1> Matx31d;
typedef Matx<double, 6, 1> Matx61d;
typedef Matx<double, 1, 3> Matx13d;
typedef Matx<double, 3, 4> Matx34d;
typedef Matx<double, 4, 1> Matx41d;
typedef Vec<double, 2> Vec2d;
typedef Vec<double, 3> Vec3d;
typedef Vec<double, 4> Vec4d;
typedef Vec<float, 2> Vec2f;
typedef Vec<float, 3> Vec3f;

using std::sqrt;      // cv::sqrt(double) is called qualified by src/cam_model_omni.cpp; same entity as std::sqrt, so the
                      // reference's `using namespace cv; using namespace std;` stays unambiguous

struct KeyPoint {
    Point2f pt;
    float size, angle, response;
    int octave, class_id;
    KeyPoint() : pt(0, 0), size(0), angle(-1), response(0), octave(0), class_id(-1) {}
    KeyPoint(float x, float y, float size_, float angle_ = -1, float response_ = 0, int octave_ = 0, int class_id_ = -1)
        : pt(x, y), size(size_), angle(angle_), response(response_), octave(octave_), class_id(class_id_) {}
};

template <class T> class AutoBuffer {
public:
    explicit AutoBuffer(size_t n) : v_(n) {}
    operator T*() { return v_.data(); }
private:
    std::vector<T> v_;
};

template <class T> using Ptr = std::shared_ptr<T>;

// ---------------------------------------------------------------------------------------------- cv::Mat
class Mat;
// result of Mat::zeros / Mat::ones: assigning it to an existing Mat goes through Mat::create (a no-op for an equally sized
// and typed view) and then fills -- the MatExpr semantics the reference relies on at src/mdBRIEFextractorOct.cpp:1215-1216
struct MatFillExpr { int rows, cols, type; double value; };

class Mat {
public:
    int rows, cols;
    uchar* data;
    size_t step;          // bytes per row
    Mat() : rows(0), cols(0), data(nullptr), step(0), type_(0), wrows_(0), wcols_(0), ox_(0), oy_(0) {}
    Mat(int r, int c, int type) : Mat() { create(r, c, type); }
    Mat(Size s, int type) : Mat() { create(s.height, s.width, type); }
    Mat(int r, int c, int type, void* ext, size_t step_ = 0) : Mat() {        // view on caller-owned memory
        rows = r; cols = c; type_ = type; data = (uchar*)ext; step = step_ ? step_ : (size_t)c * elemSize();
        wrows_ = r; wcols_ = c; base_ = data;
    }
    Mat(const MatFillExpr& e) : Mat() { *this = e; }
    template <class T, int M, int N> Mat(const Matx<T, M, N>& mx);            // copies (cv::Mat(const Matx&, copyData = true))
    Mat& operator=(const MatFillExpr& e) { create(e.rows, e.cols, e.type); setTo(e.value); return *this; }

    static MatFillExpr zeros(int r, int c, int type) { return MatFillExpr{r, c, type, 0.0}; }
    static MatFillExpr zeros(Size s, int type) { return MatFillExpr{s.height, s.width, type, 0.0}; }
    static MatFillExpr ones(int r, int c, int type) { return MatFillExpr{r, c, type, 1.0}; }
    static MatFillExpr ones(Size s, int type) { return MatFillExpr{s.height, s.width, type, 1.0}; }

    // cv::Mat::create: keeps the current buffer (also of a view) when size and type already match
    void create(int r, int c, int type) {
        if (data && rows == r && cols == c && type_ == type) return;
        type_ = type; rows = r; cols = c;
        step = (size_t)c * elemSize();
        buf_ = std::shared_ptr<uchar>(new uchar[(size_t)r * step + 64](), std::default_delete<uchar[]>());
        data = base_ = buf_.get();
        wrows_ = r; wcols_ = c; ox_ = oy_ = 0;
    }
    void create(Size s, int type) { create(s.height, s.width, type); }
    void release() { buf_.reset(); data = base_ = nullptr; rows = cols = 0; step = 0; wrows_ = wcols_ = ox_ = oy_ = 0; }
    bool empty() const { return data == nullptr || rows == 0 || cols == 0; }
    int type() const { return type_; }
    int depth() const { return type_ & 7; }
    int channels() const { return (type_ >> 3) + 1; }
    size_t elemSize1() const { static const int s[7] = {1, 1, 2, 2, 4, 4, 8}; return (size_t)s[depth()]; }
    size_t elemSize() const { return elemSize1() * channels(); }
    size_t step1() const { return step / elemSize1(); }
    Size size() const { return Size(cols, rows); }
    bool isContinuous() const { return step == (size_t)cols * elemSize(); }
    bool isSubmatrix() const { return rows != wrows_ || cols != wcols_; }
    void locateROI(Size& whole, Point& ofs) const { whole = Size(wcols_, wrows_); ofs = Point(ox_, oy_); }
    // pointer to pixel (x, y) given in ROI coordinates, which may lie outside the ROI but inside the parent buffer
    const uchar* parentPtr(int y, int x) const { return base_ + (size_t)(oy_ + y) * step + (size_t)(ox_ + x) * elemSize(); }

    Mat operator()(const Rect& r) const {
        Mat m(*this);
        m.data = data + (size_t)r.y * step + (size_t)r.x * elemSize();
        m.rows = r.height; m.cols = r.width; m.ox_ = ox_ + r.x; m.oy_ = oy_ + r.y;
        return m;
    }
    Mat rowRange(int a, int b) const { return (*this)(Rect(0, a, cols, b - a)); }
    Mat colRange(int a, int b) const { return (*this)(Rect(a, 0, b - a, rows)); }
    Mat row(int r) const { return rowRange(r, r + 1); }
    Mat clone() const {
        Mat m;
        if (!empty()) { m.create(rows, cols, type_); for (int y = 0; y < rows; ++y) std::memcpy(m.data + (size_t)y * m.step, data + (size_t)y * step, (size_t)cols * elemSize()); }
        return m;
    }
    void copyTo(Mat& dst) const {
        dst.create(rows, cols, type_);
        for (int y = 0; y < rows; ++y) std::memmove(dst.data + (size_t)y * dst.step, data + (size_t)y * step, (size_t)cols * elemSize());
    }
    void setTo(double v) {
        for (int y = 0; y < rows; ++y) {
            uchar* p = data + (size_t)y * step;
            if (depth() == CV_8U) std::memset(p, (int)v, (size_t)cols);
            else if (depth() == CV_64F) for (int x = 0; x < cols; ++x) ((double*)p)[x] = v;
            else if (depth() == CV_32F) for (int x = 0; x < cols; ++x) ((float*)p)[x] = (float)v;
            else throw Exception("setTo: depth");
        }
    }
    template <class T> T* ptr(int r = 0) { return (T*)(data + (size_t)r * step); }
    template <class T> const T* ptr(int r = 0) const { return (const T*)(data + (size_t)r * step); }
    template <class T> T& at(int r, int c) { return ((T*)(data + (size_t)r * step))[c]; }
    template <class T> const T& at(int r, int c) const { return ((const T*)(data + (size_t)r * step))[c]; }
    template <class T> T& at(int i) { return rows == 1 ? at<T>(0, i) : (cols == 1 ? at<T>(i, 0) : at<T>(i / cols, i % cols)); }
    template <class T> const T& at(int i) const { return rows == 1 ? at<T>(0, i) : (cols == 1 ? at<T>(i, 0) : at<T>(i / cols, i % cols)); }
    // the reference takes cv::InputArray / cv::OutputArray and calls getMat() on them
    Mat getMat() const { return *this; }

protected:
    int type_;
    std::shared_ptr<uchar> buf_;
    uchar* base_ = nullptr;       // first byte of the parent (whole) matrix
    int wrows_, wcols_, ox_, oy_;
};
typedef const Mat& InputArray;
typedef Mat& OutputArray;

template <class T> struct DepthOf;
template <> struct DepthOf<double> { enum { value = CV_64F }; };
template <> struct DepthOf<float> { enum { value = CV_32F }; };
template <> struct DepthOf<uchar> { enum { value = CV_8U }; };
template <> struct DepthOf<int> { enum { value = CV_32S }; };

template <class T, int M, int N> inline Mat::Mat(const Matx<T, M, N>& mx) : Mat() {
    create(M, N, DepthOf<T>::value);
    for (int i = 0; i < M; ++i) for (int j = 0; j < N; ++j) at<T>(i, j) = mx(i, j);
}

template <class T> class Mat_;
template <class T> struct MatCommaInitializer_ {
    Mat_<T>* m; int idx;
    MatCommaInitializer_(Mat_<T>* m_) : m(m_), idx(0) {}
    template <class U> MatCommaInitializer_& operator,(U v);
};
template <class T> class Mat_ : public Mat {
public:
    Mat_() : Mat() {}
    Mat_(int r, int c) : Mat(r, c, DepthOf<T>::value) {}
    Mat_(const Mat& m) : Mat(m) { if (!m.empty() && m.type() != (int)DepthOf<T>::value) throw Exception("Mat_: type"); }
    Mat_(const MatFillExpr& e) : Mat(e) {}
    Mat_(const MatCommaInitializer_<T>& ci) : Mat(*ci.m) {}
    T& operator()(int r, int c) { return this->template at<T>(r, c); }
    const T& operator()(int r, int c) const { return this->template at<T>(r, c); }
};
template <class T> template <class U> inline MatCommaInitializer_<T>& MatCommaInitializer_<T>::operator,(U v) {
    m->template at<T>(idx / m->cols, idx % m->cols) = (T)v; ++idx; return *this;
}
template <class T, class U> inline MatCommaInitializer_<T> operator<<(const Mat_<T>& m, U v) {
    MatCommaInitializer_<T> ci(const_cast<Mat_<T>*>(&m));       // the temporary's buffer is shared with the copy made from ci
    return (ci, v);
}

// ---------------------------------------------------------------------------------------------- image primitives
enum { INTER_NEAREST = 0, INTER_LINEAR = 1 };
enum { BORDER_CONSTANT = 0, BORDER_REPLICATE = 1, BORDER_REFLECT = 2, BORDER_WRAP = 3, BORDER_REFLECT_101 = 4,
       BORDER_REFLECT101 = 4, BORDER_DEFAULT = 4, BORDER_ISOLATED = 16 };
enum { NORM_HAMMING = 6 };

// cv::borderInterpolate for the two modes the path uses
inline int borderInterpolate(int p, int len, int borderType) {
    if ((unsigned)p < (unsigned)len) return p;
    if (borderType == BORDER_REFLECT_101) {
        if (len == 1) return 0;
        do { if (p < 0) p = -p; else p = 2 * (len - 1) - p; } while ((unsigned)p >= (unsigned)len);
        return p;
    }
    if (borderType == BORDER_CONSTANT) return -1;
    throw Exception("borderInterpolate: mode");
}

// cv::resize for CV_8UC1, INTER_LINEAR (imgproc/resize.cpp: HResizeLinear<uchar,int,short,2048> + VResizeLinear with
// FixedPtCast<int,uchar,22>) and INTER_NEAREST (resizeNN).  dst keeps its buffer when it already has size dsize.
inline void resize(InputArray src, OutputArray dst, Size dsize, double fx = 0, double fy = 0, int interpolation = INTER_LINEAR) {
    (void)fx; (void)fy;
    CV_Assert(src.type() == CV_8UC1 && !src.empty() && dsize.width > 0 && dsize.height > 0);
    dst.create(dsize, src.type());
    const int sw = src.cols, sh = src.rows, dw = dsize.width, dh = dsize.height;
    const double inv_scale_x = (double)dw / sw, inv_scale_y = (double)dh / sh;
    const double scale_x = 1. / inv_scale_x, scale_y = 1. / inv_scale_y;
    if (interpolation == INTER_NEAREST) {
        std::vector<int> x_ofs(dw);
        for (int x = 0; x < dw; ++x) x_ofs[x] = std::min(cvFloor(x * scale_x), sw - 1);
        for (int y = 0; y < dh; ++y) {
            const uchar* S = src.ptr<uchar>(std::min(cvFloor(y * scale_y), sh - 1));
            uchar* D = dst.ptr<uchar>(y);
            for (int x = 0; x < dw; ++x) D[x] = S[x_ofs[x]];
        }
        return;
    }
    CV_Assert(interpolation == INTER_LINEAR);
    auto coeff = [](float v) { int i = (int)lrintf(v); return (short)(i < -32768 ? -32768 : (i > 32767 ? 32767 : i)); };
    std::vector<int> xofs(dw), yofs(dh);
    std::vector<short> alpha(2 * dw), beta(2 * dh);
    for (int dx = 0; dx < dw; ++dx) {
        float f = (float)((dx + 0.5) * scale_x - 0.5);
        int s = cvFloor(f);
        f -= s;
        if (s < 0) { f = 0; s = 0; }
        if (s >= sw - 1) { f = 0; s = sw - 1; }
        xofs[dx] = s; alpha[2 * dx] = coeff((1.f - f) * 2048.f); alpha[2 * dx + 1] = coeff(f * 2048.f);
    }
    for (int dy = 0; dy < dh; ++dy) {
        float f = (float)((dy + 0.5) * scale_y - 0.5);
        int s = cvFloor(f);
        f -= s;
        yofs[dy] = s; beta[2 * dy] = coeff((1.f - f) * 2048.f); beta[2 * dy + 1] = coeff(f * 2048.f);
    }
    std::vector<int> h0(dw), h1(dw);
    for (int dy = 0; dy < dh; ++dy) {
        const int y0 = std::min(std::max(yofs[dy], 0), sh - 1), y1 = std::min(std::max(yofs[dy] + 1, 0), sh - 1);
        const uchar* S0 = src.ptr<uchar>(y0);
        const uchar* S1 = src.ptr<uchar>(y1);
        for (int dx = 0; dx < dw; ++dx) {
            const int s = xofs[dx], s1 = std::min(s + 1, sw - 1);
            h0[dx] = S0[s] * alpha[2 * dx] + S0[s1] * alpha[2 * dx + 1];
            h1[dx] = S1[s] * alpha[2 * dx] + S1[s1] * alpha[2 * dx + 1];
        }
        const int b0 = beta[2 * dy], b1 = beta[2 * dy + 1];
        uchar* D = dst.ptr<uchar>(dy);
        for (int dx = 0; dx < dw; ++dx) {
            const int v = (((b0 * (h0[dx] >> 4)) >> 16) + ((b1 * (h1[dx] >> 4)) >> 16) + 2) >> 2;
            D[dx] = (uchar)(v < 0 ? 0 : (v > 255 ? 255 : v));
        }
    }
}

// cv::copyMakeBorder (core/copy.cpp) for CV_8UC1, REFLECT_101 or CONSTANT, with the BORDER_ISOLATED handling of a
// sub-matrix source: without the flag the pixels that exist around the ROI in the parent are used first.
inline void copyMakeBorder(InputArray src_, OutputArray dst, int top, int bottom, int left, int right, int borderType,
                           const Scalar& value = Scalar()) {
    CV_Assert(src_.type() == CV_8UC1 && top >= 0 && bottom >= 0 && left >= 0 && right >= 0);
    Mat src = src_;
    if (src.isSubmatrix() && (borderType & BORDER_ISOLATED) == 0) {
        Size wholeSize; Point ofs;
        src.locateROI(wholeSize, ofs);
        const int dtop = std::min(ofs.y, top), dbottom = std::min(wholeSize.height - src.rows - ofs.y, bottom);
        const int dleft = std::min(ofs.x, left), dright = std::min(wholeSize.width - src.cols - ofs.x, right);
        Mat whole = src;                                           // widen the view inside the parent (Mat::adjustROI)
        src = Mat(src.rows + dtop + dbottom, src.cols + dleft + dright, src.type(), (void*)src.parentPtr(-dtop, -dleft), src.step);
        (void)whole;
        top -= dtop; left -= dleft; bottom -= dbottom; right -= dright;
    }
    borderType &= ~BORDER_ISOLATED;
    const int sw = src.cols, sh = src.rows, dw = sw + left + right, dh = sh + top + bottom;
    // the source may be a view into dst itself (reference :1185-1189): read it completely before dst is touched
    std::vector<uchar> s((size_t)sw * sh);
    for (int y = 0; y < sh; ++y) std::memcpy(s.data() + (size_t)y * sw, src.ptr<uchar>(y), (size_t)sw);
    dst.create(dh, dw, src.type());
    const int cval = (int)value.val[0];
    for (int y = 0; y < dh; ++y) {
        const int sy = borderInterpolate(y - top, sh, borderType);
        uchar* D = dst.ptr<uchar>(y);
        for (int x = 0; x < dw; ++x) {
            const int sx = borderInterpolate(x - left, sw, borderType);
            D[x] = (sy < 0 || sx < 0) ? (uchar)cval : s[(size_t)sy * sw + sx];
        }
    }
}

// cv::boxFilter for CV_8UC1, normalized, anchor at the centre (imgproc/box_filter: RowSum<uchar,int> + ColumnSum<int,uchar>
// with scale 1/(kw*kh), saturate_cast<uchar>(sum * scale)).  Without BORDER_ISOLATED a sub-matrix is filtered with the
// pixels that surround it in its parent; only beyond the parent does the border mode extrapolate (FilterEngine::apply with
// wholeSize / ofs).  Works in place (all taps are read before anything is written).
inline void boxFilter(InputArray src, OutputArray dst, int ddepth, Size ksize, Point anchor = Point(-1, -1), bool normalize = true,
                      int borderType = BORDER_DEFAULT) {
    CV_Assert(src.type() == CV_8UC1 && (ddepth == CV_8U || ddepth < 0) && normalize && anchor.x == -1 && anchor.y == -1);
    const int kw = ksize.width, kh = ksize.height, ax = kw / 2, ay = kh / 2;
    Size whole(src.cols, src.rows); Point ofs(0, 0);
    const bool isolated = (borderType & BORDER_ISOLATED) != 0;
    if (!isolated) src.locateROI(whole, ofs);
    borderType &= ~BORDER_ISOLATED;
    const int w = src.cols, h = src.rows;
    std::vector<int> colsum((size_t)(h + kh - 1) * w);            // horizontal sums for rows -ay .. h-1+ay
    for (int yy = 0; yy < h + kh - 1; ++yy) {
        const int wy = borderInterpolate(ofs.y + yy - ay, whole.height, borderType);       // row in whole-image coordinates
        for (int x = 0; x < w; ++x) {
            int sacc = 0;
            for (int k = 0; k < kw; ++k) {
                const int wx = borderInterpolate(ofs.x + x + k - ax, whole.width, borderType);
                sacc += *src.parentPtr(wy - ofs.y, wx - ofs.x);
            }
            colsum[(size_t)yy * w + x] = sacc;
        }
    }
    const double scale = 1. / (kw * kh);
    std::vector<uchar> out((size_t)w * h);
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            int sacc = 0;
            for (int k = 0; k < kh; ++k) sacc += colsum[(size_t)(y + k) * w + x];
            out[(size_t)y * w + x] = saturate_cast<uchar>(sacc * scale);
        }
    dst.create(h, w, src.type());
    for (int y = 0; y < h; ++y) std::memcpy(dst.ptr<uchar>(y), out.data() + (size_t)y * w, (size_t)w);
}

// cv::buildPyramid: level i+1 = pyrDown(level i), size ((w+1)/2, (h+1)/2).  The path only reads the level SIZES
// (src/cam_model_omni.cpp:189-199, on an all-zero image), so the levels are produced as zero images of the right size.
inline void buildPyramid(InputArray src, std::vector<Mat>& dst, int maxlevel) {
    dst.resize(maxlevel + 1);
    dst[0] = src;
    for (int i = 1; i <= maxlevel; ++i) dst[i] = Mat::zeros((dst[i - 1].rows + 1) / 2, (dst[i - 1].cols + 1) / 2, src.type());
}

// cv::fastAtan2 (core/mathfuncs_core.simd.hpp atan_f32 / fastAtan32f scalar path): degrees, fp32, evaluated WITHOUT fused
// multiply-add (volatile temporaries keep the compiler from contracting)
inline float fastAtan2(float y, float x) {
    const float scale = (float)(180.0 / CV_PI);
    const float p1 = 0.9997878412794807f * scale, p3 = -0.3258083974640975f * scale;
    const float p5 = 0.1555786518463281f * scale, p7 = -0.04432655554792128f * scale;
    volatile float ax = std::abs(x), ay = std::abs(y);
    volatile float a, c, c2, t;
    if (ax >= ay) {
        c = ay / (ax + (float)DBL_EPSILON); c2 = c * c;
        t = p7 * c2; t = t + p5; t = t * c2; t = t + p3; t = t * c2; t = t + p1; a = t * c;
    } else {
        c = ax / (ay + (float)DBL_EPSILON); c2 = c * c;
        t = p7 * c2; t = t + p5; t = t * c2; t = t + p3; t = t * c2; t = t + p1; a = 90.f - t * c;
    }
    if (x < 0) a = 180.f - a;
    if (y < 0) a = 360.f - a;
    return a;
}

// ---------------------------------------------------------------------------------------------- FAST
namespace stub_detail {
// ring of the 9_16 detector in OpenCV's order (features2d/fast_score.cpp makeOffsets, patternSize 16)
static const int kRing16[16][2] = {{0, 3}, {1, 3}, {2, 2}, {3, 1}, {3, 0}, {3, -1}, {2, -2}, {1, -3},
                                   {0, -3}, {-1, -3}, {-2, -2}, {-3, -1}, {-3, 0}, {-3, 1}, {-2, 2}, {-1, 3}};
// cornerScore<16> (features2d/fast_score.cpp)
inline int cornerScore16(const uchar* ptr, const int pixel[25], int threshold) {
    const int K = 8, N = K * 3 + 1;
    int k, v = ptr[0];
    short d[N];
    for (k = 0; k < N; k++) d[k] = (short)(v - ptr[pixel[k]]);
    int a0 = threshold;
    for (k = 0; k < 16; k += 2) {
        int a = std::min((int)d[k + 1], (int)d[k + 2]);
        a = std::min(a, (int)d[k + 3]);
        if (a <= a0) continue;
        a = std::min(a, (int)d[k + 4]); a = std::min(a, (int)d[k + 5]); a = std::min(a, (int)d[k + 6]);
        a = std::min(a, (int)d[k + 7]); a = std::min(a, (int)d[k + 8]);
        a0 = std::max(a0, std::min(a, (int)d[k]));
        a0 = std::max(a0, std::min(a, (int)d[k + 9]));
    }
    int b0 = -a0;
    for (k = 0; k < 16; k += 2) {
        int b = std::max((int)d[k + 1], (int)d[k + 2]);
        b = std::max(b, (int)d[k + 3]); b = std::max(b, (int)d[k + 4]); b = std::max(b, (int)d[k + 5]);
        if (b >= b0) continue;
        b = std::max(b, (int)d[k + 6]); b = std::max(b, (int)d[k + 7]); b = std::max(b, (int)d[k + 8]);
        b0 = std::min(b0, std::max(b, (int)d[k]));
        b0 = std::min(b0, std::max(b, (int)d[k + 9]));
    }
    return -b0 - 1;
}
// FAST_t<16> (features2d/fast.cpp): segment test with the threshold table, score buffer of three rows, strict 8-neighbour
// non-maximum suppression one row behind; keypoints come out row-major with size 7, angle -1, response = score.
inline void FAST9_16(const Mat& img, std::vector<KeyPoint>& keypoints, int threshold, bool nonmax) {
    const int K = 8, N = 25;
    int pixel[25];
    for (int k = 0; k < 16; ++k) pixel[k] = kRing16[k][0] + kRing16[k][1] * (int)img.step;
    for (int k = 16; k < 25; ++k) pixel[k] = pixel[k - 16];
    keypoints.clear();
    threshold = std::min(std::max(threshold, 0), 255);
    uchar threshold_tab[512];
    for (int i = -255; i <= 255; i++) threshold_tab[i + 255] = (uchar)(i < -threshold ? 1 : i > threshold ? 2 : 0);
    const int cols = img.cols, rows = img.rows;
    if (cols < 7 || rows < 7) return;
    std::vector<uchar> bufmem((size_t)cols * 3, 0);
    uchar* buf[3] = {bufmem.data(), bufmem.data() + cols, bufmem.data() + 2 * cols};
    std::vector<int> cpmem((size_t)(cols + 1) * 3, 0);
    int* cpbuf[3] = {cpmem.data() + 1, cpmem.data() + (cols + 1) + 1, cpmem.data() + 2 * (cols + 1) + 1};   // cpbuf[k][-1] = count
    for (int i = 3; i < rows - 2; i++) {
        const uchar* ptr = img.ptr<uchar>(i) + 3;
        uchar* curr = buf[(i - 3) % 3];
        int* cornerpos = cpbuf[(i - 3) % 3];
        std::memset(curr, 0, (size_t)cols);
        int ncorners = 0;
        if (i < rows - 3) {
            for (int j = 3; j < cols - 3; j++, ptr++) {
                const int v = ptr[0];
                const uchar* tab = &threshold_tab[0] - v + 255;
                int d = tab[ptr[pixel[0]]] | tab[ptr[pixel[8]]];
                if (d == 0) continue;
                d &= tab[ptr[pixel[2]]] | tab[ptr[pixel[10]]];
                d &= tab[ptr[pixel[4]]] | tab[ptr[pixel[12]]];
                d &= tab[ptr[pixel[6]]] | tab[ptr[pixel[14]]];
                if (d == 0) continue;
                d &= tab[ptr[pixel[1]]] | tab[ptr[pixel[9]]];
                d &= tab[ptr[pixel[3]]] | tab[ptr[pixel[11]]];
                d &= tab[ptr[pixel[5]]] | tab[ptr[pixel[13]]];
                d &= tab[ptr[pixel[7]]] | tab[ptr[pixel[15]]];
                if (d & 1) {
                    const int vt = v - threshold; int count = 0;
                    for (int k = 0; k < N; k++) {
                        const int x = ptr[pixel[k]];
                        if (x < vt) { if (++count > K) { cornerpos[ncorners++] = j; if (nonmax) curr[j] = (uchar)cornerScore16(ptr, pixel, threshold); break; } }
                        else count = 0;
                    }
                }
                if (d & 2) {
                    const int vt = v + threshold; int count = 0;
                    for (int k = 0; k < N; k++) {
                        const int x = ptr[pixel[k]];
                        if (x > vt) { if (++count > K) { cornerpos[ncorners++] = j; if (nonmax) curr[j] = (uchar)cornerScore16(ptr, pixel, threshold); break; } }
                        else count = 0;
                    }
                }
            }
        }
        cornerpos[-1] = ncorners;
        if (i == 3) continue;
        const uchar* prev = buf[(i - 4 + 3) % 3];
        const uchar* pprev = buf[(i - 5 + 3) % 3];
        cornerpos = cpbuf[(i - 4 + 3) % 3];
        ncorners = cornerpos[-1];
        for (int k = 0; k < ncorners; k++) {
            const int j = cornerpos[k];
            const int score = prev[j];
            if (!nonmax || (score > prev[j + 1] && score > prev[j - 1] && score > pprev[j - 1] && score > pprev[j] && score > pprev[j + 1] &&
                            score > curr[j - 1] && score > curr[j] && score > curr[j + 1]))
                keypoints.push_back(KeyPoint((float)j, (float)(i - 1), 7.f, -1, (float)score));
        }
    }
}
// KeyPointsFilter::runByPixelsMask (features2d/keypoint.cpp MaskPredicate)
inline void runByPixelsMask(std::vector<KeyPoint>& keypoints, const Mat& mask) {
    if (mask.empty()) return;
    size_t n = 0;
    for (size_t i = 0; i < keypoints.size(); ++i) {
        const KeyPoint& kp = keypoints[i];
        if (mask.at<uchar>((int)(kp.pt.y + 0.5f), (int)(kp.pt.x + 0.5f)) != 0) keypoints[n++] = kp;
    }
    keypoints.resize(n);
}
}  // namespace stub_detail

inline void FAST(InputArray image, std::vector<KeyPoint>& keypoints, int threshold, bool nonmaxSuppression = true) {
    stub_detail::FAST9_16(image, keypoints, threshold, nonmaxSuppression);
}

class FastFeatureDetector {
public:
    enum { TYPE_5_8 = 0, TYPE_7_12 = 1, TYPE_9_16 = 2 };
    static Ptr<FastFeatureDetector> create(int threshold = 10, bool nonmaxSuppression = true, int type = TYPE_9_16) {
        Ptr<FastFeatureDetector> p(new FastFeatureDetector);
        p->threshold_ = threshold; p->nonmax_ = nonmaxSuppression; p->type_ = type;
        return p;
    }
    // Feature2D::detect -> FastFeatureDetector_Impl::detect: FAST(...) then KeyPointsFilter::runByPixelsMask
    void detect(InputArray image, std::vector<KeyPoint>& keypoints, InputArray mask = Mat()) {
        if (image.empty()) { keypoints.clear(); return; }
        if (type_ != TYPE_9_16) throw Exception("stand-in FastFeatureDetector: only TYPE_9_16 is provided");
        stub_detail::FAST9_16(image, keypoints, threshold_, nonmax_);
        stub_detail::runByPixelsMask(keypoints, mask);
    }
    void setThreshold(int t) { threshold_ = t; }
private:
    int threshold_ = 10, type_ = TYPE_9_16; bool nonmax_ = true;
};

class AgastFeatureDetector {       // constructed unconditionally by the reference (:869-870), used only when useAgast is set
public:
    static Ptr<AgastFeatureDetector> create(int = 10, bool = true, int = 3) { return Ptr<AgastFeatureDetector>(new AgastFeatureDetector); }
    void detect(InputArray, std::vector<KeyPoint>&, InputArray = Mat()) { throw Exception("stand-in AgastFeatureDetector: AGAST is not provided"); }
    void setThreshold(int) {}
};

struct KeyPointsFilter {           // only reached from ComputeKeyPointsOld, which operator() never calls
    static void retainBest(std::vector<KeyPoint>& keypoints, int npoints) {
        if (npoints >= 0 && keypoints.size() > (size_t)npoints) {
            std::stable_sort(keypoints.begin(), keypoints.end(), [](const KeyPoint& a, const KeyPoint& b) { return a.response > b.response; });
            keypoints.resize((size_t)npoints);
        }
    }
};

}  // namespace cv
