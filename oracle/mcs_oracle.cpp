/*
 * mcs_oracle.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Scalar CPU restatement of the MultiCol-SLAM feature hot path, used only as the parity checker
 * by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
 * Nothing under multicol_slam_b200/ may call into this file.
 *
 * Each function cites the reference file:line it restates (paths relative to /root/reference).
 * PINNED BY REFERENCE-RUN OUTPUTS.  The reference's own sources -- src/mdBRIEFextractorOct.cpp, src/cORBmatcher.cpp,
 * src/cam_model_omni.cpp, src/cam_system_omni.cpp, src/misc.cpp, src/cConverter.cpp and the vendored DBoW2 -- are compiled where
 * they lie (oracle/Makefile target `ref` -> oracle/_ref/libmcs_ref.so, libdbow2_ref.so) against a stand-in OpenCV header
 * (oracle/ref_mcs/stub: cv::Mat + the six image primitives the extractor calls, themselves pinned bit for bit against cv2 4.13.0
 * by oracle/pin_cv2.py / pin_ref.py) and data-only stand-ins of the three SLAM container classes the matcher reads
 * (oracle/ref_mcs/stub_slam.h).  Every function of this file is checked against that library:
 *   extractor (all stages, ORB / dBRIEF / mdBRIEF, 19 configurations)  tests/test_ref_pin_cpu.py, tests/golden/ref_extract_*.npz
 *   every cORBmatcher entry point of the path                         tests/test_ref_match_cpu.py
 *   bag of words                                                       tests/test_bow_cpu.py
 * and the GPU path against the same outputs (tests/test_ref_pin_gpu.py, tests/test_ref_match_gpu.py, tests/golden/).
 * One tie-break of the reference depends on heap addresses (sort of pair<int, ExtractorNode*>, src/mdBRIEFextractorOct.cpp:782);
 * the reference library is run under a monotonic allocator so that "larger address" = "created later", which is the order
 * this file (and the GPU kernel) implement by a creation counter.
 *
 * Build: g++ -O2 -std=c++17 -ffp-contract=off -fPIC -shared (oracle/Makefile).
 * -ffp-contract=off: double expressions are evaluated without FMA contraction (ISO semantics).
 */
#include "../include/mcs_b200.h"

#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <list>
#include <map>
#include <atomic>
#include <malloc.h>
#include <thread>
#include <utility>
#include <vector>

namespace {

constexpr int EDGE = 25;          // EDGE_THRESHOLD   src/mdBRIEFextractorOct.cpp:85
constexpr int HALF_PATCH = 16;    // HALF_PATCH_SIZE  :84
constexpr int PATCH = 32;         // PATCH_SIZE       :83

static const signed char kPairs[2048] = {
#include "../multicol_slam_b200/csrc/brief_pairs_64.inc"
};

// cvRound: round half to even; as OpenCV's x86-64 path (cvtsd2si), NaN and values outside int give INT_MIN rather than wrapping
inline int cv_round(double v) { const double r = std::nearbyint(v); return (r >= -2147483648.0 && r < 2147483648.0) ? (int)r : INT_MIN; }
inline int cv_floor(double v) { int i = (int)v; return i - (i > v); }
inline int cv_ceil(double v) { int i = (int)v; return i + (i < v); }

// ------------------------------------------------------------------------------------------
// camera model  (src/cam_model_omni.cpp, include/misc.h:115-122)
// ------------------------------------------------------------------------------------------
inline double horner(const double* c, int n, double x) {
    double r = 0.0;
    for (int i = n - 1; i >= 0; --i) r = r * x + c[i];
    return r;
}

// src/cam_model_omni.cpp:146-161
void world_to_img(const mcs_ocam& cam, double x, double y, double z, double& u, double& v) {
    double norm = std::sqrt(x * x + y * y);
    if (norm == 0.0) norm = 1e-14;
    const double theta = std::atan(-z / norm);
    const double rho = horner(cam.inv_pol, 12, theta);
    const double uu = x / norm * rho;
    const double vv = y / norm * rho;
    u = uu * cam.c + vv * cam.d + cam.u0;
    v = uu * cam.e + vv + cam.v0;
}

// src/cam_model_omni.cpp:49-67
void img_to_world(const mcs_ocam& cam, double u, double v, double& x, double& y, double& z) {
    const double inv_affine = cam.c - cam.d * cam.e;
    const double u_t = u - cam.u0;
    const double v_t = v - cam.v0;
    x = (u_t - cam.d * v_t) / inv_affine;
    y = (-cam.e * u_t + cam.c * v_t) / inv_affine;
    const double X2 = x * x, Y2 = y * y;
    z = -horner(cam.pol, 5, std::sqrt(X2 + Y2));
    const double norm = std::sqrt(X2 + Y2 + z * z);
    x /= norm; y /= norm; z /= norm;
}

// include/cam_model_omni.h:127-138
void undistort_ocam(const mcs_ocam& cam, double px, double py, double s, double& ox, double& oy) {
    double x, y, z;
    img_to_world(cam, px, py, x, y, z);
    ox = -x / z * s;
    oy = -y / z * s;
}

// ------------------------------------------------------------------------------------------
// OpenCV primitives (restated; pinned against cv2 4.13 by oracle/pin_cv2.py)
// ------------------------------------------------------------------------------------------
struct Img {
    int w = 0, h = 0;
    std::vector<uint8_t> d;
    Img() {}
    Img(int w_, int h_) : w(w_), h(h_), d((size_t)w_ * h_) {}
    uint8_t* row(int y) { return d.data() + (size_t)y * w; }
    const uint8_t* row(int y) const { return d.data() + (size_t)y * w; }
};

inline short sat_short_round(float v) {
    int i = (int)lrintf(v);
    return (short)std::min(std::max(i, -32768), 32767);
}

// cv::resize(..., INTER_LINEAR) for CV_8UC1 (SURVEY Appendix A.1; OpenCV imgproc/resize.cpp,
// HResizeLinear + VResizeLinear<uchar,int,short,FixedPtCast<int,uchar,22>>)
void resize_linear(const Img& s, Img& dst, int dw, int dh) {
    dst = Img(dw, dh);
    const int sw = s.w, sh = s.h;
    const double scale_x = 1.0 / ((double)dw / sw), scale_y = 1.0 / ((double)dh / sh);
    std::vector<int> xofs(dw), yofs(dh);
    std::vector<short> alpha(2 * dw), beta(2 * dh);
    for (int dx = 0; dx < dw; ++dx) {
        float fx = (float)((dx + 0.5) * scale_x - 0.5);
        int sx = cv_floor(fx);
        fx -= sx;
        if (sx < 0) { fx = 0; sx = 0; }
        if (sx >= sw - 1) { fx = 0; sx = sw - 1; }
        xofs[dx] = sx;
        alpha[2 * dx] = sat_short_round((1.f - fx) * 2048.f);
        alpha[2 * dx + 1] = sat_short_round(fx * 2048.f);
    }
    for (int dy = 0; dy < dh; ++dy) {
        float fy = (float)((dy + 0.5) * scale_y - 0.5);
        int sy = cv_floor(fy);
        fy -= sy;
        yofs[dy] = sy;
        beta[2 * dy] = sat_short_round((1.f - fy) * 2048.f);
        beta[2 * dy + 1] = sat_short_round(fy * 2048.f);
    }
    auto clip = [](int x, int a, int b) { return x >= a ? (x < b ? x : b - 1) : a; };
    std::vector<int> r0(dw), r1(dw);
    for (int dy = 0; dy < dh; ++dy) {
        const int sy0 = clip(yofs[dy], 0, sh), sy1 = clip(yofs[dy] + 1, 0, sh);
        const uint8_t* S0 = s.row(sy0);
        const uint8_t* S1 = s.row(sy1);
        for (int dx = 0; dx < dw; ++dx) {
            const int sx = xofs[dx], sx1 = std::min(sx + 1, sw - 1);
            const int a0 = alpha[2 * dx], a1 = alpha[2 * dx + 1];
            r0[dx] = S0[sx] * a0 + S0[sx1] * a1;
            r1[dx] = S1[sx] * a0 + S1[sx1] * a1;
        }
        const int b0 = beta[2 * dy], b1 = beta[2 * dy + 1];
        uint8_t* D = dst.row(dy);
        for (int dx = 0; dx < dw; ++dx) {
            int v = (((b0 * (r0[dx] >> 4)) >> 16) + ((b1 * (r1[dx] >> 4)) >> 16) + 2) >> 2;
            D[dx] = (uint8_t)std::min(std::max(v, 0), 255);
        }
    }
}

// cv::resize(..., INTER_NEAREST) (Appendix A.1, resizeNN)
void resize_nearest(const Img& s, Img& dst, int dw, int dh) {
    dst = Img(dw, dh);
    const double ifx = 1.0 / ((double)dw / s.w), ify = 1.0 / ((double)dh / s.h);
    std::vector<int> xo(dw);
    for (int x = 0; x < dw; ++x) xo[x] = std::min(cv_floor(x * ifx), s.w - 1);
    for (int y = 0; y < dh; ++y) {
        const uint8_t* S = s.row(std::min(cv_floor(y * ify), s.h - 1));
        uint8_t* D = dst.row(y);
        for (int x = 0; x < dw; ++x) D[x] = S[xo[x]];
    }
}

inline int reflect101(int p, int n) {
    if (n == 1) return 0;
    while (p < 0 || p >= n) {
        if (p < 0) p = -p;
        else p = 2 * (n - 1) - p;
    }
    return p;
}

// cv::copyMakeBorder with BORDER_REFLECT_101 / BORDER_CONSTANT(0)
void make_border(const Img& s, Img& dst, int b, bool reflect) {
    dst = Img(s.w + 2 * b, s.h + 2 * b);
    for (int y = 0; y < dst.h; ++y) {
        int sy = y - b;
        uint8_t* D = dst.row(y);
        if (!reflect && (sy < 0 || sy >= s.h)) { std::memset(D, 0, dst.w); continue; }
        const uint8_t* S = s.row(reflect ? reflect101(sy, s.h) : sy);
        for (int x = 0; x < dst.w; ++x) {
            int sx = x - b;
            if (reflect) D[x] = S[reflect101(sx, s.w)];
            else D[x] = (sx < 0 || sx >= s.w) ? 0 : S[sx];
        }
    }
}

// cv::boxFilter 5x5 normalized, BORDER_REFLECT_101, on the ROI of a bordered buffer, in place
// (Appendix A.3): dst = (S + 12) / 25; pixels outside the ROI are the (unblurred) ring.
void box5_inplace_roi(Img& buf, int b, int w, int h) {
    std::vector<uint8_t> out((size_t)w * h);
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            int s = 0;
            for (int dy = -2; dy <= 2; ++dy) {
                const uint8_t* R = buf.row(y + b + dy);
                for (int dx = -2; dx <= 2; ++dx) s += R[x + b + dx];
            }
            out[(size_t)y * w + x] = (uint8_t)((s + 12) / 25);
        }
    for (int y = 0; y < h; ++y) std::memcpy(buf.row(y + b) + b, out.data() + (size_t)y * w, w);
}

// cv::fastAtan2 (Appendix A.4, OpenCV core/mathfuncs_core: atan_f32, no FMA)
float fast_atan2(float y, float x) {
    const float s = (float)(180.0 / 3.14159265358979323846);
    const float p1 = 0.9997878412794807f * s, p3 = -0.3258083974640975f * s;
    const float p5 = 0.1555786518463281f * s, p7 = -0.04432655554792128f * s;
    volatile float ax = std::fabs(x), ay = std::fabs(y);
    volatile float a, c, c2, t;
    if (ax >= ay) {
        c = ay / (ax + (float)DBL_EPSILON);
        c2 = c * c;
        t = p7 * c2; t = t + p5; t = t * c2; t = t + p3; t = t * c2; t = t + p1;
        a = t * c;
    } else {
        c = ax / (ay + (float)DBL_EPSILON);
        c2 = c * c;
        t = p7 * c2; t = t + p5; t = t * c2; t = t + p3; t = t * c2; t = t + p1;
        a = 90.f - t * c;
    }
    if (x < 0) a = 180.f - a;
    if (y < 0) a = 360.f - a;
    return a;
}

// FAST-9/16 score (OpenCV features2d/fast_score.cpp cornerScore<16>; Appendix A.5)
static const int kRing[16][2] = {{0, 3},  {1, 3},   {2, 2},   {3, 1},  {3, 0},  {3, -1}, {2, -2}, {1, -3},
                                 {0, -3}, {-1, -3}, {-2, -2}, {-3, -1}, {-3, 0}, {-3, 1}, {-2, 2}, {-1, 3}};

inline int corner_score16(const uint8_t* p, int stride, int threshold) {
    int d[25];
    const int v = p[0];
    for (int k = 0; k < 25; ++k) d[k] = v - p[kRing[k & 15][1] * stride + kRing[k & 15][0]];
    int a0 = threshold;
    for (int k = 0; k < 16; k += 2) {
        int a = std::min(d[k + 1], d[k + 2]);
        a = std::min(a, d[k + 3]);
        if (a <= a0) continue;
        a = std::min(a, d[k + 4]); a = std::min(a, d[k + 5]); a = std::min(a, d[k + 6]);
        a = std::min(a, d[k + 7]); a = std::min(a, d[k + 8]);
        a0 = std::max(a0, std::min(a, d[k]));
        a0 = std::max(a0, std::min(a, d[k + 9]));
    }
    int b0 = -a0;
    for (int k = 0; k < 16; k += 2) {
        int b = std::max(d[k + 1], d[k + 2]);
        b = std::max(b, d[k + 3]); b = std::max(b, d[k + 4]); b = std::max(b, d[k + 5]);
        if (b >= b0) continue;
        b = std::max(b, d[k + 6]); b = std::max(b, d[k + 7]); b = std::max(b, d[k + 8]);
        b0 = std::min(b0, std::max(b, d[k]));
        b0 = std::min(b0, std::max(b, d[k + 9]));
    }
    return -b0 - 1;
}

struct RawKp { float x, y, response; };

// cv::FAST(img, kps, threshold, nonmax=true, TYPE_9_16) on a sub-image given by pointer/stride
// (OpenCV features2d/fast.cpp FAST_t<16>), followed by KeyPointsFilter::runByPixelsMask.
void fast9_cell(const uint8_t* img, int stride, const uint8_t* mask, int mstride, int cols, int rows,
                int threshold, std::vector<RawKp>& out) {
    out.clear();
    if (cols < 7 || rows < 7) return;
    std::vector<int> score((size_t)cols * rows, 0);
    for (int i = 3; i < rows - 3; ++i) {
        const uint8_t* ptr = img + (size_t)i * stride;
        for (int j = 3; j < cols - 3; ++j) {
            const int v = ptr[j];
            // segment test: >= 9 contiguous ring pixels all < v-t or all > v+t
            bool corner = false;
            for (int pass = 0; pass < 2 && !corner; ++pass) {
                int count = 0;
                for (int k = 0; k < 25; ++k) {
                    const int x = ptr[j + kRing[k & 15][1] * stride + kRing[k & 15][0]];
                    const bool hit = pass == 0 ? (x < v - threshold) : (x > v + threshold);
                    if (hit) { if (++count > 8) { corner = true; break; } }
                    else count = 0;
                }
            }
            if (corner) score[(size_t)i * cols + j] = corner_score16(ptr + j, stride, threshold);
        }
    }
    for (int i = 3; i < rows - 3; ++i)
        for (int j = 3; j < cols - 3; ++j) {
            const int s = score[(size_t)i * cols + j];
            if (s == 0) continue;   // a corner always scores >= threshold >= 1 ... see note below
            bool keep = true;
            for (int dy = -1; dy <= 1 && keep; ++dy)
                for (int dx = -1; dx <= 1; ++dx) {
                    if (!dx && !dy) continue;
                    if (s <= score[(size_t)(i + dy) * cols + j + dx]) { keep = false; break; }
                }
            if (!keep) continue;
            if (mask && mask[(size_t)((int)(i + 0.5f)) * mstride + (int)(j + 0.5f)] == 0) continue;
            out.push_back({(float)j, (float)i, (float)s});
        }
}

// ------------------------------------------------------------------------------------------
// extractor
// ------------------------------------------------------------------------------------------
struct Extractor {
    mcs_extractor_params p;
    int nlevels;
    double scale_factor;                       // (double)(float)1.2f
    std::vector<double> sf, isf;               // mvScaleFactor / mvInvScaleFactor
    std::vector<int> quota;                    // mnFeaturesPerLevel
    std::vector<int> umax;
    std::vector<std::pair<int, int>> pattern;  // first 16*descSize points
    // last-call intermediates (bordered buffers)
    std::vector<Img> pyr, pyr_blur, mpyr;
    std::vector<int> lw, lh;
    std::vector<std::vector<RawKp>> raw;       // per level, cell-grid coordinates (origin minBorder)
};

// src/mdBRIEFextractorOct.cpp:134-203
Extractor* make_extractor(const mcs_extractor_params& p) {
    Extractor* e = new Extractor;
    e->p = p;
    e->nlevels = p.nlevels;
    e->scale_factor = (double)p.scale_factor;
    e->sf.resize(p.nlevels); e->isf.resize(p.nlevels);
    e->sf[0] = 1;
    for (int i = 1; i < p.nlevels; ++i) e->sf[i] = e->sf[i - 1] * e->scale_factor;
    const double inv = 1.0 / e->scale_factor;
    e->isf[0] = 1;
    for (int i = 1; i < p.nlevels; ++i) e->isf[i] = e->isf[i - 1] * inv;
    e->quota.resize(p.nlevels);
    const double factor = 1.0 / e->scale_factor;
    double nd = p.nfeatures * (1 - factor) / (1 - std::pow(factor, p.nlevels));
    int sum = 0;
    for (int l = 0; l < p.nlevels - 1; ++l) {
        e->quota[l] = cv_round(nd);
        sum += e->quota[l];
        nd *= factor;
    }
    e->quota[p.nlevels - 1] = std::max(p.nfeatures - sum, 0);
    const int npoints = 2 * 8 * p.desc_size;
    for (int i = 0; i < npoints; ++i) e->pattern.push_back({kPairs[2 * i], kPairs[2 * i + 1]});
    e->umax.assign(HALF_PATCH + 1, 0);
    int v, v0;
    const int vmax = cv_floor(HALF_PATCH * std::sqrt(2.f) / 2 + 1);
    const int vmin = cv_ceil(HALF_PATCH * std::sqrt(2.f) / 2);
    const double hp2 = HALF_PATCH * HALF_PATCH;
    for (v = 0; v <= vmax; ++v) e->umax[v] = cv_round(std::sqrt(hp2 - v * v));
    for (v = HALF_PATCH, v0 = 0; v >= vmin; --v) {
        while (e->umax[v0] == e->umax[v0 + 1]) ++v0;
        e->umax[v] = v0;
        ++v0;
    }
    return e;
}

// src/mdBRIEFextractorOct.cpp:1158-1201
void compute_pyramid(Extractor& e, const Img& image, const Img& mask) {
    const int L = e.nlevels;
    e.pyr.assign(L, Img()); e.mpyr.assign(L, Img()); e.pyr_blur.assign(L, Img());
    e.lw.assign(L, 0); e.lh.assign(L, 0);
    Img prev = image, prevm = mask;
    for (int l = 0; l < L; ++l) {
        const double scale = e.isf[l];
        const int w = cv_round((double)image.w * scale), h = cv_round((double)image.h * scale);
        e.lw[l] = w; e.lh[l] = h;
        Img cur, curm;
        if (l != 0) {
            resize_linear(prev, cur, w, h);
            resize_nearest(prevm, curm, w, h);
        } else {
            cur = image; curm = mask;
        }
        make_border(cur, e.pyr[l], EDGE, true);
        make_border(curm, e.mpyr[l], EDGE, false);
        prev = cur; prevm = curm;
    }
}

// ---- octree (src/mdBRIEFextractorOct.cpp:569-861) ----
struct Node {
    std::vector<RawKp> keys;
    int ULx, ULy, URx, URy, BLx, BLy, BRx, BRy;
    bool no_more = false;
    long seq = 0;                       // creation sequence number: deterministic stand-in for the
                                        // heap address the reference sorts on (:782) -- later == larger
    std::list<Node>::iterator lit;
};

void divide_node(const Node& n, Node& n1, Node& n2, Node& n3, Node& n4) {   // :569-629
    const int halfX = (int)std::ceil((double)(n.URx - n.ULx) / 2.0);
    const int halfY = (int)std::ceil((double)(n.BRy - n.ULy) / 2.0);
    n1.ULx = n.ULx; n1.ULy = n.ULy; n1.URx = n.ULx + halfX; n1.URy = n.ULy;
    n1.BLx = n.ULx; n1.BLy = n.ULy + halfY; n1.BRx = n.ULx + halfX; n1.BRy = n.ULy + halfY;
    n2.ULx = n1.URx; n2.ULy = n1.URy; n2.URx = n.URx; n2.URy = n.URy;
    n2.BLx = n1.BRx; n2.BLy = n1.BRy; n2.BRx = n.URx; n2.BRy = n.ULy + halfY;
    n3.ULx = n1.BLx; n3.ULy = n1.BLy; n3.URx = n1.BRx; n3.URy = n1.BRy;
    n3.BLx = n.BLx; n3.BLy = n.BLy; n3.BRx = n1.BRx; n3.BRy = n.BLy;
    n4.ULx = n3.URx; n4.ULy = n3.URy; n4.URx = n2.BRx; n4.URy = n2.BRy;
    n4.BLx = n3.BRx; n4.BLy = n3.BRy; n4.BRx = n.BRx; n4.BRy = n.BRy;
    for (const RawKp& kp : n.keys) {
        if (kp.x < n1.URx) {
            if (kp.y < n1.BRy) n1.keys.push_back(kp); else n3.keys.push_back(kp);
        } else if (kp.y < n1.BRy) n2.keys.push_back(kp);
        else n4.keys.push_back(kp);
    }
    if (n1.keys.size() == 1) n1.no_more = true;
    if (n2.keys.size() == 1) n2.no_more = true;
    if (n3.keys.size() == 1) n3.no_more = true;
    if (n4.keys.size() == 1) n4.no_more = true;
}

std::vector<RawKp> distribute_octree(const std::vector<RawKp>& keys, int minX, int maxX, int minY, int maxY,
                                     int N) {   // :631-861
    std::vector<RawKp> result;
    const int nIni = cv_round((double)(maxX - minX) / (maxY - minY));
    const double hX = (double)(maxX - minX) / nIni;
    std::list<Node> nodes;
    std::vector<Node*> ini(nIni);
    long seq = 0;
    for (int i = 0; i < nIni; ++i) {
        Node ni;
        ni.ULx = (int)(hX * (double)i); ni.ULy = 0;
        ni.URx = (int)(hX * (double)(i + 1)); ni.URy = 0;
        ni.BLx = ni.ULx; ni.BLy = maxY - minY;
        ni.BRx = ni.URx; ni.BRy = maxY - minY;
        ni.seq = seq++;
        nodes.push_back(ni);
        ini[i] = &nodes.back();
    }
    for (const RawKp& kp : keys) ini[(int)(kp.x / hX)]->keys.push_back(kp);
    for (auto it = nodes.begin(); it != nodes.end();) {
        if (it->keys.size() == 1) { it->no_more = true; ++it; }
        else if (it->keys.empty()) it = nodes.erase(it);
        else ++it;
    }
    bool finish = false;
    typedef std::pair<int, Node*> SP;
    auto by_size_then_seq = [](const SP& a, const SP& b) {
        if (a.first != b.first) return a.first < b.first;
        return a.second->seq < b.second->seq;
    };
    std::vector<SP> size_ptr;
    auto push_child = [&](Node& c, int& nToExpand) {
        if (c.keys.empty()) return;
        c.seq = seq++;
        nodes.push_front(c);
        if (c.keys.size() > 1) {
            ++nToExpand;
            size_ptr.push_back({(int)c.keys.size(), &nodes.front()});
            nodes.front().lit = nodes.begin();
        }
    };
    while (!finish) {
        int prevSize = (int)nodes.size();
        auto it = nodes.begin();
        int nToExpand = 0;
        size_ptr.clear();
        while (it != nodes.end()) {
            if (it->no_more) { ++it; continue; }
            Node n1, n2, n3, n4;
            divide_node(*it, n1, n2, n3, n4);
            push_child(n1, nToExpand); push_child(n2, nToExpand);
            push_child(n3, nToExpand); push_child(n4, nToExpand);
            it = nodes.erase(it);
        }
        if ((int)nodes.size() >= N || (int)nodes.size() == prevSize) {
            finish = true;
        } else if (((int)nodes.size() + nToExpand * 3) > N) {
            while (!finish) {
                prevSize = (int)nodes.size();
                std::vector<SP> prev = size_ptr;
                size_ptr.clear();
                std::sort(prev.begin(), prev.end(), by_size_then_seq);
                for (int j = (int)prev.size() - 1; j >= 0; --j) {
                    Node n1, n2, n3, n4;
                    divide_node(*prev[j].second, n1, n2, n3, n4);
                    int dummy = 0;
                    push_child(n1, dummy); push_child(n2, dummy);
                    push_child(n3, dummy); push_child(n4, dummy);
                    nodes.erase(prev[j].second->lit);
                    if ((int)nodes.size() >= N) break;
                }
                if ((int)nodes.size() >= N || (int)nodes.size() == prevSize) finish = true;
            }
        }
    }
    for (auto& n : nodes) {
        const RawKp* best = &n.keys[0];
        float maxr = best->response;
        for (size_t k = 1; k < n.keys.size(); ++k)
            if (n.keys[k].response > maxr) { best = &n.keys[k]; maxr = n.keys[k].response; }
        result.push_back(*best);
    }
    return result;
}

// src/mdBRIEFextractorOct.cpp:221-248 ; image = bordered buffer, (x,y) in ROI coordinates
float ic_angle(const Img& buf, float ptx, float pty, const std::vector<int>& umax) {
    int m01 = 0, m10 = 0;
    const int step = buf.w;
    const uint8_t* center = buf.row(cv_round(pty) + EDGE) + cv_round(ptx) + EDGE;
    for (int u = -HALF_PATCH; u <= HALF_PATCH; ++u) m10 += u * center[u];
    for (int v = 1; v <= HALF_PATCH; ++v) {
        int v_sum = 0;
        const int d = umax[v];
        for (int u = -d; u <= d; ++u) {
            const int vp = center[u + v * step], vm = center[u - v * step];
            v_sum += (vp - vm);
            m10 += u * (vp + vm);
        }
        m01 += v * v_sum;
    }
    return fast_atan2((float)m01, (float)m10);
}

typedef std::pair<int, int> Pt;

// :285-301
void rotate_pattern(const std::vector<Pt>& in, std::vector<Pt>& out, double ax, double ay) {
    out.resize(in.size());
    for (size_t p = 0; p < in.size(); ++p) {
        out[p].first = cv_round(in[p].first * ax - in[p].second * ay);
        out[p].second = cv_round(in[p].first * ay + in[p].second * ax);
    }
}

// :250-283
void rotate_distort_pattern(double ukx, double uky, const std::vector<Pt>& in, std::vector<Pt>& out,
                            const mcs_ocam& cam, double ax, double ay) {
    const size_t n = in.size();
    out.resize(n);
    std::vector<double> xs(n), ys(n);
    double sumX = 0.0, sumY = 0.0;
    for (size_t p = 0; p < n; ++p) {
        const double xr = in[p].first * ax - in[p].second * ay + ukx;
        const double yr = in[p].first * ay + in[p].second * ax + uky;
        world_to_img(cam, xr, yr, -cam.pol[0], xs[p], ys[p]);   // distortPointsOcam, cam_model_omni.h:140-145
        sumX += xs[p];
        sumY += ys[p];
    }
    const double meanX = sumX / (double)n, meanY = sumY / (double)n;
    for (size_t p = 0; p < n; ++p) {
        out[p].first = cv_round(xs[p] - meanX);
        out[p].second = cv_round(ys[p] - meanY);
    }
}

inline int sample(const Img& buf, int row, int col, const Pt& p) {
    return buf.row(row + p.second + EDGE)[col + p.first + EDGE];
}

const float DEG2RADf = (float)(3.14159265358979323846) / 180.f;   // :82 static_cast<float>(CV_PI)/180.f
const double RHOd = 180.0 / 3.1415926535897932384626433832795028841971693993;   // misc.h:40
const float RHOf = 180.0f / 3.1415926535897932384626f;                          // misc.h:41

// :303-554 ; blurred = bordered, blurred-ROI buffer
void describe(const Extractor& e, const Img& blurred, const mcs_keypoint& kp, double ukx, double uky,
              const mcs_ocam& cam, uint8_t* desc, uint8_t* dmask) {
    const int ds = e.p.desc_size;
    std::vector<Pt> pat, m1, m2;
    const int row = cv_round(kp.y), col = cv_round(kp.x);
    if (e.p.learn_masks) {
        const double rot = 20.0 / RHOd;
        const double angle = (double)(kp.angle / RHOf);
        rotate_distort_pattern(ukx, uky, e.pattern, pat, cam, std::cos(angle), std::sin(angle));
        rotate_distort_pattern(ukx, uky, e.pattern, m1, cam, std::cos(angle + rot), std::sin(angle + rot));
        rotate_distort_pattern(ukx, uky, e.pattern, m2, cam, std::cos(angle - rot), std::sin(angle - rot));
    } else {
        const double angle = (double)(kp.angle * DEG2RADf);
        if (e.p.do_dbrief) rotate_distort_pattern(ukx, uky, e.pattern, pat, cam, std::cos(angle), std::sin(angle));
        else rotate_pattern(e.pattern, pat, std::cos(angle), std::sin(angle));
    }
    for (int i = 0; i < ds; ++i) {
        int val = 0, mval = 0;
        for (int b = 0; b < 8; ++b) {
            const int k = 16 * i + 2 * b;
            const int t = sample(blurred, row, col, pat[k]) < sample(blurred, row, col, pat[k + 1]);
            val |= t << b;
            if (e.p.learn_masks) {
                const int s1 = (sample(blurred, row, col, m1[k]) < sample(blurred, row, col, m1[k + 1])) ^ t;
                const int s2 = (sample(blurred, row, col, m2[k]) < sample(blurred, row, col, m2[k + 1])) ^ t;
                mval |= ((s1 + s2) == 0) << b;
            }
        }
        desc[i] = (uint8_t)val;
        if (dmask) dmask[i] = (uint8_t)mval;
    }
}

// cell loop of ComputeKeyPointsOctTree  :863-949 ; fills e.raw[level] in cell-grid coordinates
void detect_level(Extractor& e, int level) {
    const int w = e.lw[level], h = e.lh[level];
    const Img& img = e.pyr[level];
    const Img& msk = e.mpyr[level];
    std::vector<RawKp>& out = e.raw[level];
    out.clear();
    const int minBX = EDGE - 3, minBY = minBX, maxBX = w - EDGE + 3, maxBY = h - EDGE + 3;
    const double width = (maxBX - minBX), height = (maxBY - minBY);
    const int nCols = (int)(width / 30.0), nRows = (int)(height / 30.0);
    if (nCols <= 0 || nRows <= 0) return;
    const int wCell = (int)std::ceil(width / nCols), hCell = (int)std::ceil(height / nRows);
    std::vector<RawKp> cell;
    for (int i = 0; i < nRows; ++i) {
        const double iniY = minBY + i * hCell;
        double maxY = iniY + hCell + 6;
        if (iniY >= maxBY - 3) continue;
        if (maxY > maxBY) maxY = maxBY;
        for (int j = 0; j < nCols; ++j) {
            const double iniX = minBX + j * wCell;
            double maxX = iniX + wCell + 6;
            if (iniX >= maxBX - 6) continue;
            if (maxX > maxBX) maxX = maxBX;
            const int x0 = (int)iniX, y0 = (int)iniY, cw = (int)maxX - x0, ch = (int)maxY - y0;
            fast9_cell(img.row(y0 + EDGE) + x0 + EDGE, img.w, msk.row(y0 + EDGE) + x0 + EDGE, msk.w, cw, ch,
                       e.p.fast_threshold, cell);
            for (RawKp& k : cell) {
                k.x += j * wCell;
                k.y += i * hCell;
                out.push_back(k);
            }
        }
    }
}

// Output slots per image: sum over the levels of max(N + 2, 16), fixed before the image size is known (the extractor's rule)
int out_capacity(const Extractor& e) {
    int cap = 0;
    for (int l = 0; l < e.nlevels; ++l) cap += std::max(e.quota[l] + 2, 16);
    return cap;
}

// The most keypoints DistributeOctTree returns for w x h images: its first pass divides every one of the nIni roots (:640)
// whatever the quota N, and every later pass starts below N and adds at most 3 nodes per division (:693-854)
int octree_bound(const Extractor& e, int w, int h) {
    int most = 0;
    for (int l = 0; l < e.nlevels; ++l) {
        const int lw = cv_round((double)w * e.isf[l]), lh = cv_round((double)h * e.isf[l]);
        const int nIni = cv_round((double)(lw - 2 * (EDGE - 3)) / (lh - 2 * (EDGE - 3)));
        most += std::max(e.quota[l] + 2, 4 * nIni);
    }
    return most;
}

// operator()  :1244-1337
int extract(Extractor& e, const Img& image, const Img& mask, const mcs_ocam& cam, mcs_keypoint* kps,
            uint8_t* desc, uint8_t* dmask, int capacity) {
    const int L = e.nlevels, ds = e.p.desc_size;
    compute_pyramid(e, image, mask);
    e.raw.assign(L, {});
    std::vector<std::vector<mcs_keypoint>> all(L);
    for (int l = 0; l < L; ++l) {
        detect_level(e, l);
        const int minB = EDGE - 3, maxBX = e.lw[l] - EDGE + 3, maxBY = e.lh[l] - EDGE + 3;
        std::vector<RawKp> sel;
        if (!e.raw[l].empty()) sel = distribute_octree(e.raw[l], minB, maxBX, minB, maxBY, e.quota[l]);
        const int scaledPatch = (int)(PATCH * e.sf[l]);
        for (const RawKp& r : sel) {
            mcs_keypoint k;
            k.x = r.x + minB; k.y = r.y + minB;
            k.size = (float)scaledPatch; k.angle = -1.f; k.response = r.response;
            k.octave = l; k.class_id = -1;
            all[l].push_back(k);
        }
    }
    for (int l = 0; l < L; ++l)
        for (mcs_keypoint& k : all[l]) k.angle = ic_angle(e.pyr[l], k.x, k.y, e.umax);
    int n = 0;
    for (int l = 0; l < L; ++l) n += (int)all[l].size();
    if (n > capacity) return -1;
    const double scaleF = cam.pol[0];
    int off = 0;
    for (int l = 0; l < L; ++l) {
        e.pyr_blur[l] = e.pyr[l];
        if (all[l].empty()) continue;
        box5_inplace_roi(e.pyr_blur[l], EDGE, e.lw[l], e.lh[l]);
        const float scale = (float)e.sf[l];
        for (mcs_keypoint& k : all[l]) {
            double ux = 0, uy = 0;
            if (e.p.do_dbrief)
                undistort_ocam(cam, (double)(k.x * scale), (double)(k.y * scale), scaleF, ux, uy);
            uint8_t* dm = dmask ? dmask + (size_t)off * ds : nullptr;
            if (dm) std::memset(dm, 0, ds);
            describe(e, e.pyr_blur[l], k, ux, uy, cam, desc + (size_t)off * ds, dm);
            mcs_keypoint o = k;
            if (l != 0) { o.x = k.x * scale; o.y = k.y * scale; }
            kps[off] = o;
            ++off;
        }
    }
    return n;
}

// ------------------------------------------------------------------------------------------
// matching
// ------------------------------------------------------------------------------------------
int dist64(const uint64_t* a, const uint64_t* b, int dim) {   // src/cORBmatcher.cpp:2438-2450
    uint64_t d = 0;
    for (int i = 0; i < dim / 8; ++i) d += __builtin_popcountll(a[i] ^ b[i]);
    return (int)d;
}
int dist64m(const uint64_t* a, const uint64_t* b, const uint64_t* ma, const uint64_t* mb, int dim) {   // :2452-2474
    uint64_t d = 0;
    for (int i = 0; i < dim / 8; ++i) {
        const uint64_t x = a[i] ^ b[i];
        d += __builtin_popcountll(x & ma[i]);
        d += __builtin_popcountll(x & mb[i]);
    }
    return (int)(d / 2);
}
inline const uint64_t* row64(const uint8_t* base, int idx, int dim) {
    return (const uint64_t*)(base + (size_t)idx * dim);
}

struct Grid {   // src/cMultiFrame.cpp:128-184, :342-353
    int n_cams;
    std::vector<double> winv, hinv;
    std::vector<std::vector<int>> cells;   // [cam*64*48 + ix*48 + iy]
};

void build_grid(const mcs_frame_view& f, Grid& g) {
    g.n_cams = f.n_cams;
    g.winv.resize(f.n_cams); g.hinv.resize(f.n_cams);
    for (int c = 0; c < f.n_cams; ++c) {
        g.winv[c] = (double)MCS_FRAME_GRID_COLS / (double)f.cam_width[c];
        g.hinv[c] = (double)MCS_FRAME_GRID_ROWS / (double)f.cam_height[c];
    }
    g.cells.assign((size_t)f.n_cams * MCS_FRAME_GRID_COLS * MCS_FRAME_GRID_ROWS, {});
    for (int i = 0; i < f.n_keys; ++i) {
        const int c = f.key_cam[i];
        const int px = cv_round((f.keys[i].x - 0) * g.winv[c]);   // float - int -> float, * double
        const int py = cv_round((f.keys[i].y - 0) * g.hinv[c]);
        if (px < 0 || px >= MCS_FRAME_GRID_COLS || py < 0 || py >= MCS_FRAME_GRID_ROWS) continue;
        g.cells[((size_t)c * MCS_FRAME_GRID_COLS + px) * MCS_FRAME_GRID_ROWS + py].push_back(i);
    }
}

// src/cMultiFrame.cpp:272-340
void features_in_area(const mcs_frame_view& f, const Grid& g, int cam, double x, double y, double r, int minLevel,
                      int maxLevel, std::vector<int>& out) {
    out.clear();
    int nMinCellX = (int)std::floor((x - 0 - r) * g.winv[cam]);
    nMinCellX = std::max(0, nMinCellX);
    if (nMinCellX >= MCS_FRAME_GRID_COLS) return;
    int nMaxCellX = (int)std::ceil((x - 0 + r) * g.winv[cam]);
    nMaxCellX = std::min(MCS_FRAME_GRID_COLS - 1, nMaxCellX);
    if (nMaxCellX < 0) return;
    int nMinCellY = (int)std::floor((y - 0 - r) * g.hinv[cam]);
    nMinCellY = std::max(0, nMinCellY);
    if (nMinCellY >= MCS_FRAME_GRID_ROWS) return;
    int nMaxCellY = (int)std::ceil((y - 0 + r) * g.hinv[cam]);
    nMaxCellY = std::min(MCS_FRAME_GRID_ROWS - 1, nMaxCellY);
    if (nMaxCellY < 0) return;
    bool check = true, same = false;
    if (minLevel == -1 && maxLevel == -1) check = false;
    else if (minLevel == maxLevel) same = true;
    for (int ix = nMinCellX; ix <= nMaxCellX; ++ix)
        for (int iy = nMinCellY; iy <= nMaxCellY; ++iy) {
            const std::vector<int>& cell = g.cells[((size_t)cam * MCS_FRAME_GRID_COLS + ix) * MCS_FRAME_GRID_ROWS + iy];
            for (int idx : cell) {
                const mcs_keypoint& kp = f.keys[idx];
                if (check && !same) {
                    if (kp.octave < minLevel || kp.octave > maxLevel) continue;
                } else if (same) {
                    if (kp.octave != minLevel) continue;
                }
                if (std::abs(kp.x - x) > r || std::abs(kp.y - y) > r) continue;   // float - double
                out.push_back(idx);
            }
        }
}

}  // namespace

// ==========================================================================================
// C entry points used by the tests (ctypes) -- prefix mcso_
// ==========================================================================================
extern "C" {

struct mcso_extractor { Extractor* e; };

mcso_extractor* mcso_extractor_create(const mcs_extractor_params* p) {
    if (!p || p->use_agast || p->fast_agast_type != 2) return nullptr;
    mcso_extractor* h = new mcso_extractor;
    h->e = make_extractor(*p);
    return h;
}
void mcso_extractor_destroy(mcso_extractor* h) {
    if (h) { delete h->e; delete h; }
}
int mcso_extractor_get_info(const mcso_extractor* h, mcs_extractor_info* info) {
    const Extractor& e = *h->e;
    std::memset(info, 0, sizeof(*info));
    info->nlevels = e.nlevels;
    info->capacity = out_capacity(e);
    info->desc_size = e.p.desc_size;
    for (int l = 0; l < e.nlevels; ++l) {
        info->features_per_level[l] = e.quota[l];
        info->scale_factor[l] = e.sf[l];
        info->inv_scale_factor[l] = e.isf[l];
    }
    return 0;
}
int mcso_extractor_umax(const mcso_extractor* h, int* out17) {
    for (int i = 0; i <= HALF_PATCH; ++i) out17[i] = h->e->umax[i];
    return 0;
}

int mcso_extract(mcso_extractor* h, const uint8_t* image, int w, int hgt, int stride, const uint8_t* mask,
                 int mstride, const mcs_ocam* cam, mcs_keypoint* kps, uint8_t* desc, uint8_t* dmask, int capacity,
                 int* n_out) {
    // the extractor refuses such images up front rather than drop keypoints
    if (octree_bound(*h->e, w, hgt) > out_capacity(*h->e)) return MCS_ERR_UNSUPPORTED;
    Img im(w, hgt), mk(w, hgt);
    for (int y = 0; y < hgt; ++y) {
        std::memcpy(im.row(y), image + (size_t)y * stride, w);
        std::memcpy(mk.row(y), mask + (size_t)y * mstride, w);
    }
    const int n = extract(*h->e, im, mk, *cam, kps, desc, dmask, capacity);
    if (n < 0) return MCS_ERR_CAPACITY;
    *n_out = n;
    return 0;
}

// what: 0 unblurred ROI, 1 blurred ROI, 2 mask ROI, 3 raw corners (x,y,score int32 triples, cell-grid
// coordinates + minBorder, i.e. ROI coordinates, reference order)
int mcso_debug_read(mcso_extractor* h, int level, int what, void* out, size_t out_bytes, int* w_out, int* h_out) {
    Extractor& e = *h->e;
    if (level < 0 || level >= e.nlevels || e.lw.empty()) return MCS_ERR_INVALID;
    const int w = e.lw[level], hh = e.lh[level];
    if (what == 3) {
        const std::vector<RawKp>& r = e.raw[level];
        *w_out = (int)r.size(); *h_out = 3;
        if (out_bytes < r.size() * 12) return MCS_ERR_CAPACITY;
        int32_t* o = (int32_t*)out;
        for (size_t i = 0; i < r.size(); ++i) {
            o[3 * i] = (int)r[i].x + EDGE - 3; o[3 * i + 1] = (int)r[i].y + EDGE - 3; o[3 * i + 2] = (int)r[i].response;
        }
        return 0;
    }
    *w_out = w; *h_out = hh;
    if (out_bytes < (size_t)w * hh) return MCS_ERR_CAPACITY;
    const Img& src = what == 0 ? e.pyr[level] : what == 1 ? e.pyr_blur[level] : e.mpyr[level];
    for (int y = 0; y < hh; ++y) std::memcpy((uint8_t*)out + (size_t)y * w, src.row(y + EDGE) + EDGE, w);
    return 0;
}

// stand-alone primitives for pinning against cv2
void mcso_resize_linear(const uint8_t* src, int sw, int sh, uint8_t* dst, int dw, int dh) {
    Img s(sw, sh); std::memcpy(s.d.data(), src, (size_t)sw * sh);
    Img d; resize_linear(s, d, dw, dh);
    std::memcpy(dst, d.d.data(), (size_t)dw * dh);
}
void mcso_resize_nearest(const uint8_t* src, int sw, int sh, uint8_t* dst, int dw, int dh) {
    Img s(sw, sh); std::memcpy(s.d.data(), src, (size_t)sw * sh);
    Img d; resize_nearest(s, d, dw, dh);
    std::memcpy(dst, d.d.data(), (size_t)dw * dh);
}
void mcso_box5_reflect101(const uint8_t* src, int w, int h, uint8_t* dst) {
    Img s(w, h); std::memcpy(s.d.data(), src, (size_t)w * h);
    Img b; make_border(s, b, EDGE, true);
    box5_inplace_roi(b, EDGE, w, h);
    for (int y = 0; y < h; ++y) std::memcpy(dst + (size_t)y * w, b.row(y + EDGE) + EDGE, w);
}
float mcso_fast_atan2(float y, float x) { return fast_atan2(y, x); }
// FAST on one sub-image; out = (x,y,score) int32 triples; returns count
int mcso_fast9(const uint8_t* img, int w, int h, int stride, const uint8_t* mask, int mstride, int threshold,
               int32_t* out, int cap) {
    std::vector<RawKp> r;
    fast9_cell(img, stride, mask, mstride, w, h, threshold, r);
    const int n = std::min((int)r.size(), cap);
    for (int i = 0; i < n; ++i) { out[3 * i] = (int)r[i].x; out[3 * i + 1] = (int)r[i].y; out[3 * i + 2] = (int)r[i].response; }
    return (int)r.size();
}
// octree on an explicit corner list (x,y in cell-grid coords, response); out = selected (x,y,response)
int mcso_octree(const float* xyr, int n, int minX, int maxX, int minY, int maxY, int N, float* out, int cap) {
    std::vector<RawKp> k(n);
    for (int i = 0; i < n; ++i) k[i] = {xyr[3 * i], xyr[3 * i + 1], xyr[3 * i + 2]};
    std::vector<RawKp> r = n ? distribute_octree(k, minX, maxX, minY, maxY, N) : std::vector<RawKp>();
    const int m = std::min((int)r.size(), cap);
    for (int i = 0; i < m; ++i) { out[3 * i] = r[i].x; out[3 * i + 1] = r[i].y; out[3 * i + 2] = r[i].response; }
    return (int)r.size();
}

void mcso_cam_world_to_img(const mcs_ocam* cam, double x, double y, double z, double* u, double* v) {
    world_to_img(*cam, x, y, z, *u, *v);
}
void mcso_cam_img_to_world(const mcs_ocam* cam, double u, double v, double* x, double* y, double* z) {
    img_to_world(*cam, u, v, *x, *y, *z);
}
// src/cam_model_omni.cpp:181-220, level 0 only (Appendix C.9: u0/v0 names swapped on purpose)
int mcso_cam_mirror_mask(const mcs_ocam* cam, uint8_t* out) {
    const int w = cam->width, h = cam->height;
    if (cam->mirror_mask != 1) { std::memset(out, 1, (size_t)w * h); return 0; }
    const float u0 = (float)cam->v0, v0 = (float)cam->u0;
    for (int i = 0; i < h; ++i)
        for (int j = 0; j < w; ++j) {
            const float ans = std::sqrt((float)std::pow(i - u0, 2) + (float)std::pow(j - v0, 2));
            out[(size_t)i * w + j] = ans < (u0 + 22.0f) ? 255 : 0;
        }
    return 0;
}

int mcso_descriptor_distance64(const uint64_t* a, const uint64_t* b, int dim) { return dist64(a, b, dim); }
int mcso_descriptor_distance64_masked(const uint64_t* a, const uint64_t* b, const uint64_t* ma, const uint64_t* mb,
                                      int dim) { return dist64m(a, b, ma, mb, dim); }

// cORBmatcher::SearchByBoW(KF1,KF2) src/cORBmatcher.cpp:885-966
int mcso_match_bruteforce(const uint8_t* q, const uint8_t* qmask, const uint8_t* valid1, int nq, const uint8_t* d,
                          const uint8_t* dmask, const uint8_t* valid2, int nd, int dim, int th_low, double nnratio,
                          int* matches12, int* nmatches) {
    const bool masks = qmask && dmask;
    std::vector<uint8_t> matched2(nd, 0);
    int nm = 0;
    for (int i1 = 0; i1 < nq; ++i1) {
        matches12[i1] = -1;
        if (valid1 && !valid1[i1]) continue;
        int best1 = INT_MAX, best2 = INT_MAX, bestIdx = -1;
        for (int i2 = 0; i2 < nd; ++i2) {
            if (matched2[i2] || (valid2 && !valid2[i2])) continue;
            const int dist = masks ? dist64m(row64(q, i1, dim), row64(d, i2, dim), row64(qmask, i1, dim),
                                             row64(dmask, i2, dim), dim)
                                   : dist64(row64(q, i1, dim), row64(d, i2, dim), dim);
            if (dist < best1) { best2 = best1; best1 = dist; bestIdx = i2; }
            else if (dist < best2) best2 = dist;
        }
        if (best1 < th_low && (double)best1 < nnratio * (double)best2) {
            matches12[i1] = bestIdx;
            matched2[bestIdx] = 1;
            ++nm;
        }
    }
    *nmatches = nm;
    return 0;
}

// CheckDistEpipolarLine  src/misc.cpp:53-69
static bool check_epipolar(const double* r1, const double* r2, const double* E, double thresh) {
    double t[3];
    for (int j = 0; j < 3; ++j) { double s = 0; for (int i = 0; i < 3; ++i) s += r2[i] * E[3 * i + j]; t[j] = s; }
    double nom = 0; for (int j = 0; j < 3; ++j) nom += t[j] * r1[j];
    double ex1[3], etx2[3];
    for (int i = 0; i < 3; ++i) { double s = 0; for (int k = 0; k < 3; ++k) s += E[3 * i + k] * r1[k]; ex1[i] = s; }
    for (int i = 0; i < 3; ++i) { double s = 0; for (int k = 0; k < 3; ++k) s += E[3 * k + i] * r2[k]; etx2[i] = s; }
    const double den = ex1[0] * ex1[0] + ex1[1] * ex1[1] + ex1[2] * ex1[2] + etx2[0] * etx2[0] + etx2[1] * etx2[1] + etx2[2] * etx2[2];
    if (den == 0.0) return false;
    return (nom * nom) / den < thresh;
}

// cORBmatcher::SearchForTriangulationRaw  src/cORBmatcher.cpp:968-1156 (mbCheckOrientation == false)
// exported for tests/test_ref_pin_cpu.py (compared with the reference's own CheckDistEpipolarLine, src/misc.cpp:53-69)
int mcso_check_epipolar(const double* r1, const double* r2, const double* E, double thresh) { return check_epipolar(r1, r2, E, thresh) ? 1 : 0; }

int mcso_search_for_triangulation(const uint8_t* desc1, const uint8_t* mask1, const int* cam1, const uint8_t* free1, const double* rays1,
                                  int n1, const uint8_t* desc2, const uint8_t* mask2, const int* cam2, const uint8_t* free2,
                                  const double* rays2, int n2, int dim, int th_low, const double* E, int n_cams, double epi_thresh,
                                  int* matches12, int* nmatches) {
    const bool masks = mask1 && mask2;
    std::vector<uint8_t> matched2(n2, 0);
    int nm = 0;
    for (int i1 = 0; i1 < n1; ++i1) {
        matches12[i1] = -1;
        if (!free1[i1]) continue;
        std::vector<std::pair<int, size_t>> cand;
        for (int i2 = 0; i2 < n2; ++i2) {
            if (matched2[i2] || !free2[i2]) continue;
            if (cam1[i1] != cam2[i2]) continue;
            const int dist = masks ? dist64m(row64(desc1, i1, dim), row64(desc2, i2, dim), row64(mask1, i1, dim), row64(mask2, i2, dim), dim)
                                   : dist64(row64(desc1, i1, dim), row64(desc2, i2, dim), dim);
            if (dist > th_low) continue;
            cand.push_back({dist, (size_t)i2});
        }
        if (cand.empty()) continue;
        std::sort(cand.begin(), cand.end());
        const int dist_th = cv_round(2 * cand.front().first);
        for (auto& c : cand) {
            if (c.first > dist_th) break;
            if (check_epipolar(rays1 + 3 * (size_t)i1, rays2 + 3 * c.second, E + ((size_t)cam1[i1] * n_cams + cam2[c.second]) * 9, epi_thresh)) {
                matched2[c.second] = 1; matches12[i1] = (int)c.second; ++nm;
                break;
            }
        }
    }
    *nmatches = nm;
    return 0;
}

// candidate lists: GetFeaturesInArea + distances, reference visiting order
int mcso_window_search(const mcs_frame_view* f, const mcs_window_query* qs, int nq, const uint8_t* qdesc,
                       const uint8_t* qmask, int max_cand, int* cand_idx, int* cand_dist, int* cand_count) {
    Grid g; build_grid(*f, g);
    std::vector<int> idx;
    const bool masks = qmask && f->dmask;
    int status = 0;
    for (int i = 0; i < nq; ++i) {
        const mcs_window_query& q = qs[i];
        features_in_area(*f, g, q.cam, q.x, q.y, q.r, q.min_level, q.max_level, idx);
        cand_count[i] = (int)idx.size();
        if ((int)idx.size() > max_cand) status = MCS_ERR_CAPACITY;
        for (int k = 0; k < (int)idx.size() && k < max_cand; ++k) {
            cand_idx[(size_t)i * max_cand + k] = idx[k];
            cand_dist[(size_t)i * max_cand + k] =
                masks ? dist64m(row64(qdesc, q.desc_index, f->dim), row64(f->desc, idx[k], f->dim),
                                row64(qmask, q.desc_index, f->dim), row64(f->dmask, idx[k], f->dim), f->dim)
                      : dist64(row64(qdesc, q.desc_index, f->dim), row64(f->desc, idx[k], f->dim), f->dim);
        }
    }
    return status;
}

// cORBmatcher::SearchByProjection(F, vpMapPoints, th)  src/cORBmatcher.cpp:67-166
int mcso_search_by_projection(const mcs_frame_view* f, const mcs_mappoint_view* mps, double th, double nnratio,
                              int th_high, int having_masks, int* frame_mp, int* nmatches) {
    Grid g; build_grid(*f, g);
    int nm = 0;
    const bool bFactor = th != 1.0;
    std::vector<int> near;
    for (int i = 0; i < mps->n_points; ++i) {
        if (mps->bad && mps->bad[i]) continue;
        for (int cam = 0; cam < f->n_cams; ++cam) {
            const size_t k = (size_t)i * f->n_cams + cam;
            if (!mps->in_view[k]) continue;
            const int lvl = mps->level[k];
            double r = mps->view_cos[k] > 0.998 ? 2.5 : 4.0;   // RadiusByViewingCos :169-175
            if (bFactor) r *= th;
            features_in_area(*f, g, cam, mps->proj_x[k], mps->proj_y[k], r * f->scale_factors[lvl], lvl - 1, lvl, near);
            if (near.empty()) continue;
            const uint64_t* dmp = row64(mps->desc, i, f->dim);
            const uint64_t* mmp = having_masks ? row64(mps->dmask, i, f->dim) : nullptr;
            int bestDist = INT_MAX, bestLevel = -1, bestDist2 = INT_MAX, bestLevel2 = -1, bestIdx = -1;
            for (int idx : near) {
                if (frame_mp[idx] >= 0) continue;
                const int dist = having_masks ? dist64m(dmp, row64(f->desc, idx, f->dim), mmp, row64(f->dmask, idx, f->dim), f->dim)
                                              : dist64(dmp, row64(f->desc, idx, f->dim), f->dim);
                if (dist < bestDist) {
                    bestDist2 = bestDist; bestDist = dist; bestLevel2 = bestLevel;
                    bestLevel = f->keys[idx].octave; bestIdx = idx;
                } else if (dist < bestDist2) {
                    bestLevel2 = f->keys[idx].octave; bestDist2 = dist;
                }
            }
            if (bestDist <= th_high) {
                if (bestLevel == bestLevel2 && bestDist > nnratio * bestDist2) continue;
                frame_mp[bestIdx] = i;
                ++nm;
            }
        }
    }
    *nmatches = nm;
    return 0;
}

// bearing rays + grid of the cMultiFrame constructor  src/cMultiFrame.cpp:143-184, :342-353
int mcso_frame_prepare(const mcs_keypoint* keys, const int* key_cam, int n_keys, const mcs_ocam* cams, int n_cams, double* rays,
                       int* cell_start, int* cell_items, int* n_in_grid) {
    std::vector<int> cw(n_cams), ch(n_cams);
    for (int c = 0; c < n_cams; ++c) { cw[c] = cams[c].width; ch[c] = cams[c].height; }
    mcs_frame_view f{};
    f.n_cams = n_cams; f.n_keys = n_keys; f.keys = keys; f.key_cam = key_cam; f.cam_width = cw.data(); f.cam_height = ch.data();
    Grid g; build_grid(f, g);
    int pos = 0;
    for (size_t c = 0; c < g.cells.size(); ++c) {
        cell_start[c] = pos;
        for (int i : g.cells[c]) cell_items[pos++] = i;
    }
    cell_start[g.cells.size()] = pos;
    *n_in_grid = pos;
    for (int i = 0; i < n_keys; ++i)
        img_to_world(cams[key_cam[i]], (double)keys[i].x, (double)keys[i].y, rays[3 * i], rays[3 * i + 1], rays[3 * i + 2]);
    return 0;
}

// cMultiFrame::isInFrustum for every (map point, camera)  src/cMultiFrame.cpp:218-270, with
// cMultiCamSys_::WorldToCamHom_fast src/cam_system_omni.cpp:92-112 and isPointInMirrorMask src/cam_model_omni.cpp:163-178
int mcso_project_mappoints(int n_cams, const double* mtmc_inv, const double* mtmc, const mcs_ocam* cams, const uint8_t* masks,
                           int n_points, const double* pos, const double* nrm, const double* dmin, const double* dmax,
                           const double* sf, int n_levels, uint8_t* in_view, int* level, double* px, double* py, double* vcos) {
    for (int i = 0; i < n_points; ++i)
        for (int c = 0; c < n_cams; ++c) {
            const size_t t = (size_t)i * n_cams + c;
            in_view[t] = 0; level[t] = 0; px[t] = py[t] = vcos[t] = 0.0;
            const double* M = mtmc_inv + 16 * c;
            double r[3];
            for (int k = 0; k < 3; ++k) {        // cv::Matx product: s = 0; s += a(i,k) b(k) for k = 0..3
                double s = 0;
                s += M[4 * k] * pos[3 * i]; s += M[4 * k + 1] * pos[3 * i + 1]; s += M[4 * k + 2] * pos[3 * i + 2]; s += M[4 * k + 3] * 1.0;
                r[k] = s;
            }
            double u, v;
            world_to_img(cams[c], r[0], r[1], r[2], u, v);
            const int ur = cv_round(u), vr = cv_round(v);
            const int w = cams[c].width, h = cams[c].height;
            if (ur >= w || ur <= 0 || vr >= h || vr <= 0) continue;
            if (masks[(size_t)c * w * h + (size_t)vr * w + ur] == 0) continue;
            const double* T = mtmc + 16 * c;
            const double o[3] = {pos[3 * i] - T[3], pos[3 * i + 1] - T[7], pos[3 * i + 2] - T[11]};
            double s2 = 0; for (int k = 0; k < 3; ++k) s2 += o[k] * o[k];
            const double dist = std::sqrt(s2);
            if (dist < dmin[i] || dist > dmax[i]) continue;
            double dot = 0; for (int k = 0; k < 3; ++k) dot += o[k] * nrm[3 * i + k];
            const double ratio = dist / dmin[i];
            int lv = (int)(std::lower_bound(sf, sf + n_levels, ratio) - sf);
            if (lv >= n_levels) lv = n_levels - 1;
            in_view[t] = 1; px[t] = u; py[t] = v; level[t] = lv; vcos[t] = dot / dist;
        }
    return 0;
}

// Generic window search with the acceptance rules of WindowSearch (src/cORBmatcher.cpp:326-474, rule 0),
// SearchByProjection(Current, Last, th) (:1990-2118, rule 1) and SearchByProjection(F, MapPoints, th) (:67-166, rule 2);
// the per-candidate loop is the one those functions share (:385-418, :2046-2068, :115-148).
int mcso_search_windows(const mcs_frame_view* f, const mcs_window_query* qs, int nq, const uint8_t* qdesc, const uint8_t* qmask,
                        const int* query_tag, int rule, double nnratio, int threshold, int* assigned, int* nmatches) {
    Grid g; build_grid(*f, g);
    std::vector<int> near;
    const bool masks = qmask && f->dmask;
    int nm = 0;
    for (int i = 0; i < nq; ++i) {
        const mcs_window_query& q = qs[i];
        features_in_area(*f, g, q.cam, q.x, q.y, q.r, q.min_level, q.max_level, near);
        const bool stateless = rule == 3 || rule == 4;
        if (near.empty()) { if (stateless) assigned[i] = -1; continue; }
        if (rule == 4) {   // Fuse(pKF, vpMapPoints, th) :1420-1568: the distance is computed and discarded (:1506-1514), dist stays 0
            assigned[i] = 0 <= threshold ? near[0] : -1;
            nm += assigned[i] >= 0;
            continue;
        }
        int cam_first = 0, cam_end = f->n_keys;          // rule 5: rows of camera q.cam in the contiguous order
        if (rule == 5) {
            cam_first = 0;
            while (cam_first < f->n_keys && f->key_cam[cam_first] != q.cam) ++cam_first;
            cam_end = cam_first;
            while (cam_end < f->n_keys && f->key_cam[cam_end] == q.cam) ++cam_end;
        }
        int bestDist = INT_MAX, bestLevel = -1, bestDist2 = INT_MAX, bestLevel2 = -1, bestIdx = -1;
        for (int idx : near) {
            if (!stateless && assigned[idx] >= 0) continue;
            int row = idx;
            if (rule == 5) {   // SearchByProjection(pKF, Scw, ...) :2367,2372: GetDescriptorRowPtr(camIdx, idx) with the CONTIGUOUS idx
                row = cam_first + idx;
                if (row >= cam_end) continue;            // the reference reads past camera camIdx's matrix here (undefined): dropped
            }
            const int dist = masks ? dist64m(row64(qdesc, q.desc_index, f->dim), row64(f->desc, row, f->dim),
                                             row64(qmask, q.desc_index, f->dim), row64(f->dmask, row, f->dim), f->dim)
                                   : dist64(row64(qdesc, q.desc_index, f->dim), row64(f->desc, row, f->dim), f->dim);
            if (dist < bestDist) {
                bestDist2 = bestDist; bestDist = dist; bestLevel2 = bestLevel; bestLevel = f->keys[idx].octave; bestIdx = idx;
            } else if (dist < bestDist2) {
                bestLevel2 = f->keys[idx].octave; bestDist2 = dist;
            }
        }
        if (rule == 3) {   // Fuse / SearchBySim3 core (src/cORBmatcher.cpp:1326-1366): best only, nothing skipped or marked
            const bool hit = bestIdx >= 0 && bestDist <= threshold;
            assigned[i] = hit ? bestIdx : -1;
            nm += hit;
            continue;
        }
        bool ok;
        if (rule == 0) ok = bestDist <= bestDist2 * nnratio && bestDist <= threshold;
        else if (rule == 1) ok = bestDist <= threshold;
        else if (rule == 5) ok = bestDist <= threshold && bestIdx > 0;      // :2385
        else ok = bestDist <= threshold && !(bestLevel == bestLevel2 && bestDist > nnratio * bestDist2);
        if (ok && bestIdx >= 0) { assigned[bestIdx] = query_tag[i]; ++nm; }
    }
    *nmatches = nm;
    return 0;
}

// cORBmatcher::SearchForInitialization  src/cORBmatcher.cpp:579-726 (mbCheckOrientation == false)
int mcso_search_for_initialization(const mcs_frame_view* f1, const mcs_frame_view* f2, double* prev_matched,
                                   int window_size, double nnratio, int th_low, int having_masks, int* matches12,
                                   int* nmatches) {
    Grid g; build_grid(*f2, g);
    int nm = 0;
    for (int i = 0; i < f1->n_keys; ++i) matches12[i] = -1;
    std::vector<int> matchedDist(f2->n_keys, INT_MAX), matches21(f2->n_keys, -1), cand;
    for (int i1 = 0; i1 < f1->n_keys; ++i1) {
        const int level1 = f1->keys[i1].octave;
        const int cam1 = f1->key_cam[i1];
        features_in_area(*f2, g, cam1, prev_matched[2 * i1], prev_matched[2 * i1 + 1], window_size, level1, level1, cand);
        if (cand.empty()) continue;
        const uint64_t* d1 = row64(f1->desc, i1, f1->dim);
        const uint64_t* m1 = having_masks ? row64(f1->dmask, i1, f1->dim) : nullptr;
        int bestDist = INT_MAX, bestDist2 = INT_MAX, bestIdx2 = -1;
        for (int i2 : cand) {
            const int dist = having_masks ? dist64m(d1, row64(f2->desc, i2, f2->dim), m1, row64(f2->dmask, i2, f2->dim), f1->dim)
                                          : dist64(d1, row64(f2->desc, i2, f2->dim), f1->dim);
            if (matchedDist[i2] <= dist) continue;
            if (dist < bestDist) { bestDist2 = bestDist; bestDist = dist; bestIdx2 = i2; }
            else if (dist < bestDist2) bestDist2 = dist;
        }
        if (bestDist <= th_low) {
            if (bestDist < (double)bestDist2 * nnratio) {
                if (matches21[bestIdx2] >= 0) { matches12[matches21[bestIdx2]] = -1; nm--; }
                matches12[i1] = bestIdx2;
                matches21[bestIdx2] = i1;
                matchedDist[bestIdx2] = bestDist;
                nm++;
            }
        }
    }
    for (int i1 = 0; i1 < f1->n_keys; ++i1)
        if (matches12[i1] >= 0) {
            prev_matched[2 * i1] = f2->keys[matches12[i1]].x;
            prev_matched[2 * i1 + 1] = f2->keys[matches12[i1]].y;
        }
    *nmatches = nm;
    return 0;
}

// Multi-threaded driver for the CPU baseline of bench.py: n_frames x n_cams images (frame-major), one oracle extractor per
// worker thread (the reference runs one thread per camera, src/cMultiFrame.cpp:128), then SearchByBoW-style brute force
// of every (frame, camera) against (frame-1, camera).  Returns the number of features; *n_matches gets the match count.
long mcso_stream_mt(const mcs_extractor_params* p, int n_threads, int n_frames, int n_cams, const uint8_t* images, int w, int h,
                    const uint8_t* masks, const mcs_ocam* cams, int th_low, double nnratio, long* n_matches) {
    // keep freed blocks in the per-thread arenas instead of mmap/munmap-ing every large temporary: with many worker
    // threads the page-fault / mmap_sem traffic otherwise dominates and the baseline stops scaling with the core count
    mallopt(M_MMAP_THRESHOLD, 1 << 30);
    mallopt(M_TRIM_THRESHOLD, 1 << 30);
    const int n_img = n_frames * n_cams, ds = p->desc_size;
    const int cap = p->nfeatures + 16 * p->nlevels;
    std::vector<std::vector<mcs_keypoint>> kps(n_img);
    std::vector<std::vector<uint8_t>> desc(n_img), dmask(n_img);
    std::vector<int> counts(n_img, 0);
    std::atomic<int> next(0), nextm(n_cams);
    std::atomic<long> matches(0);
    auto work = [&]() {
        Extractor* e = make_extractor(*p);
        std::vector<mcs_keypoint> k(cap);
        std::vector<uint8_t> d((size_t)cap * ds), m((size_t)cap * ds);
        for (int i; (i = next.fetch_add(1)) < n_img;) {
            const int c = i % n_cams;
            Img im(w, h), mk(w, h);
            std::memcpy(im.d.data(), images + (size_t)i * w * h, (size_t)w * h);
            std::memcpy(mk.d.data(), masks + (size_t)c * w * h, (size_t)w * h);
            const int n = extract(*e, im, mk, cams[c], k.data(), d.data(), m.data(), cap);
            counts[i] = std::max(n, 0);
            kps[i].assign(k.begin(), k.begin() + counts[i]);
            desc[i].assign(d.begin(), d.begin() + (size_t)counts[i] * ds);
            dmask[i].assign(m.begin(), m.begin() + (size_t)counts[i] * ds);
        }
        delete e;
    };
    std::vector<std::thread> th;
    for (int t = 0; t < n_threads; ++t) th.emplace_back(work);
    for (auto& t : th) t.join();
    auto matchwork = [&]() {
        std::vector<int> m12;
        for (int i; (i = nextm.fetch_add(1)) < n_img;) {
            m12.assign(counts[i], -1);
            int nm = 0;
            mcso_match_bruteforce(desc[i].data(), p->learn_masks ? dmask[i].data() : nullptr, nullptr, counts[i], desc[i - n_cams].data(),
                                  p->learn_masks ? dmask[i - n_cams].data() : nullptr, nullptr, counts[i - n_cams], ds, th_low, nnratio,
                                  m12.data(), &nm);
            matches += nm;
        }
    };
    th.clear();
    for (int t = 0; t < n_threads; ++t) th.emplace_back(matchwork);
    for (auto& t : th) t.join();
    long total = 0;
    for (int c : counts) total += c;
    if (n_matches) *n_matches = matches.load();
    return total;
}

// ------------------------------------------------------------------------------------------------
// Bag of words: DBoW2::TemplatedVocabulary<FORB::TDescriptor, FORB> as the reference uses it
// (include/cORBVocabulary.h:34; ThirdParty/DBoW2/DBoW2/TemplatedVocabulary.h, FORB.cpp, BowVector.cpp,
//  FeatureVector.cpp, ScoringObject.cpp).  Pinned against the reference's own DBoW2 compiled in place
//  (oracle/_ref/libdbow2_ref.so, tests/test_bow_cpu.py) and tests/golden/bow_small_voc.npz.
// ------------------------------------------------------------------------------------------------
struct mcso_voc {
    int k, L, scoring, weighting;
    std::vector<std::vector<int>> children;      // in the order load() appended them
    std::vector<double> weight;
    std::vector<uint8_t> desc;                   // n_nodes x 32
    std::vector<int> word_of_node;
};

mcso_voc* mcso_voc_create(int k, int L, int scoring, int weighting, int n_nodes, const int* parent, const double* weight,
                          const uint8_t* desc, const int* node_order, int n_words, const int* word_node) {
    mcso_voc* v = new mcso_voc();
    v->k = k; v->L = L; v->scoring = scoring; v->weighting = weighting;
    v->children.resize(n_nodes);
    for (int i = 0; i + 1 < n_nodes; ++i) {       // TemplatedVocabulary.h:1596-1608: m_nodes[pid].children.push_back(nid) in file order
        const int nid = node_order ? node_order[i] : i + 1;
        v->children[parent[nid]].push_back(nid);
    }
    v->weight.assign(weight, weight + n_nodes);
    v->desc.assign(desc, desc + (size_t)n_nodes * 32);
    v->word_of_node.assign(n_nodes, -1);
    for (int w = 0; w < n_words; ++w) v->word_of_node[word_node[w]] = w;     // :1615-1622
    return v;
}
void mcso_voc_destroy(mcso_voc* v) { delete v; }

// FORB::distance  FORB.cpp:84-104: 8 x 32-bit words, bit count (the parallel bit trick there == popcount)
static int forb_distance(const uint8_t* a, const uint8_t* b) {
    int d = 0;
    for (int i = 0; i < 8; ++i) {
        uint32_t x, y;
        std::memcpy(&x, a + 4 * i, 4); std::memcpy(&y, b + 4 * i, 4);
        d += __builtin_popcount(x ^ y);
    }
    return d;
}

// transform(feature, word_id, weight, nid, levelsup)  TemplatedVocabulary.h:1218-1261.
// nid: the reference only assigns it when the descent passes level L - levelsup (or that level is <= 0 -> root);
// a shallower leaf leaves the caller's variable indeterminate.  Restated as "the leaf itself" (documented in DESIGN.md).
static void voc_descend(const mcso_voc* v, const uint8_t* f, int levelsup, int* word, double* weight, int* nid) {
    const int nid_level = v->L - levelsup;
    int node = 0, level = 0, at_level = nid_level <= 0 ? 0 : -1;
    do {
        ++level;
        const std::vector<int>& ch = v->children[node];
        node = ch[0];
        double best = (double)forb_distance(f, &v->desc[(size_t)node * 32]);
        for (size_t c = 1; c < ch.size(); ++c) {
            const double d = (double)forb_distance(f, &v->desc[(size_t)ch[c] * 32]);
            if (d < best) { best = d; node = ch[c]; }
        }
        if (level == nid_level) at_level = node;
    } while (!v->children[node].empty());
    *word = v->word_of_node[node];
    *weight = v->weight[node];
    *nid = at_level >= 0 ? at_level : node;
}

int mcso_bow_transform(const mcso_voc* v, const uint8_t* desc, int n, int levelsup, int* word, double* weight, int* node) {
    for (int i = 0; i < n; ++i) {
        int w, nd; double wt;
        voc_descend(v, desc + (size_t)i * 32, levelsup, &w, &wt, &nd);
        if (word) word[i] = w;
        if (weight) weight[i] = wt;
        if (node) node[i] = nd;
    }
    return 0;
}

// transform(features, BowVector, FeatureVector, levelsup)  TemplatedVocabulary.h:1126-1194 with
// BowVector::addWeight / addIfNotExist / normalize (BowVector.cpp:34-95) and FeatureVector::addFeature (FeatureVector.cpp:28-42)
int mcso_bow_vectors(const mcso_voc* v, const uint8_t* desc, int n, int levelsup, int* bow_words, double* bow_values, int* n_bow,
                     int* fv_nodes, int* fv_off, int* n_fv, int* fv_feat) {
    std::map<unsigned, double> bow;
    std::map<unsigned, std::vector<unsigned>> fv;
    // scoring objects: mustNormalize (ScoringObject.h:74-89): all but DOT_PRODUCT; L2 norm only for L2_NORM
    const bool must = v->scoring != 5;
    const bool l2 = v->scoring == 1;
    const bool accumulate = v->weighting == 0 || v->weighting == 1;          // TF_IDF, TF
    if (!v->children.empty() && !v->children[0].empty())
        for (int i = 0; i < n; ++i) {
            int w, nd; double wt;
            voc_descend(v, desc + (size_t)i * 32, levelsup, &w, &wt, &nd);
            if (!(wt > 0)) continue;                                         // stopped word
            auto it = bow.find((unsigned)w);
            if (it == bow.end()) bow[(unsigned)w] = wt;
            else if (accumulate) it->second += wt;
            fv[(unsigned)nd].push_back((unsigned)i);
        }
    if (accumulate && !bow.empty() && !must) {
        const double nd = (double)bow.size();
        for (auto& e : bow) e.second /= nd;
    }
    if (must) {
        double norm = 0.0;
        if (!l2) for (auto& e : bow) norm += std::fabs(e.second);
        else { for (auto& e : bow) norm += e.second * e.second; norm = std::sqrt(norm); }
        if (norm > 0.0) for (auto& e : bow) e.second /= norm;
    }
    int k = 0;
    for (auto& e : bow) { bow_words[k] = (int)e.first; bow_values[k] = e.second; ++k; }
    *n_bow = k;
    int f = 0, o = 0;
    for (auto& e : fv) {
        fv_nodes[f] = (int)e.first; fv_off[f] = o;
        for (unsigned i : e.second) fv_feat[o++] = (int)i;
        ++f;
    }
    fv_off[f] = o; *n_fv = f;
    return 0;
}

// GeneralScoring::score flavours  ScoringObject.cpp:23-313 (the lower_bound skips there are a plain sorted merge)
double mcso_bow_score(int scoring, const int* w1, const double* v1, int n1, const int* w2, const double* v2, int n2) {
    const double LOG_EPS = std::log(DBL_EPSILON);                            // ScoringObject.cpp:18
    double score = 0;
    int i = 0, j = 0;
    while (i < n1 && j < n2) {
        const double vi = v1[i], wi = v2[j];
        if (w1[i] == w2[j]) {
            switch (scoring) {
                case 0: score += std::fabs(vi - wi) - std::fabs(vi) - std::fabs(wi); break;
                case 1: case 5: score += vi * wi; break;
                case 2: if (vi + wi != 0.0) score += vi * wi / (vi + wi); break;
                case 3: if (vi != 0 && wi != 0) score += vi * std::log(vi / wi); break;
                case 4: score += std::sqrt(vi * wi); break;
            }
            ++i; ++j;
        } else if (w1[i] < w2[j]) {
            if (scoring == 3) score += vi * (std::log(vi) - LOG_EPS);        // KL also charges words only v1 has (:196-200)
            ++i;
        } else {
            ++j;
        }
    }
    switch (scoring) {
        case 0: return -score / 2.0;
        case 1: return score >= 1 ? 1.0 : 1.0 - std::sqrt(1.0 - score);
        case 2: return 2. * score;
        case 3:
            for (; i < n1; ++i) if (v1[i] != 0) score += v1[i] * (std::log(v1[i]) - LOG_EPS);
            return score;
        default: return score;
    }
}

// cORBmatcher::SearchByBoW(cMultiKeyFrame*, cMultiFrame&, vpMapPointMatches)  src/cORBmatcher.cpp:179-324
// (mbCheckOrientation == false).  Feature vectors as CSR (nodes ascending).
int mcso_search_by_bow(const uint8_t* desc1, const uint8_t* mask1, const uint8_t* valid1, int n1, const int* fv1_nodes,
                       const int* fv1_off, int n_fv1, const int* fv1_feat, const uint8_t* desc2, const uint8_t* mask2, int n2,
                       const int* fv2_nodes, const int* fv2_off, int n_fv2, const int* fv2_feat, int dim, int th_low,
                       double nnratio, int* match_of_2, int* nmatches) {
    const bool masks = mask1 && mask2;
    for (int i = 0; i < n2; ++i) match_of_2[i] = -1;
    int nm = 0, a = 0, b = 0;
    while (a < n_fv1 && b < n_fv2) {
        if (fv1_nodes[a] == fv2_nodes[b]) {
            for (int ia = fv1_off[a]; ia < fv1_off[a + 1]; ++ia) {
                const int i1 = fv1_feat[ia];
                if (valid1 && !valid1[i1]) continue;
                int best1 = INT_MAX, best2 = INT_MAX, bestIdx = -1;
                for (int ib = fv2_off[b]; ib < fv2_off[b + 1]; ++ib) {
                    const int i2 = fv2_feat[ib];
                    if (match_of_2[i2] >= 0) continue;
                    const int dist = masks ? dist64m(row64(desc1, i1, dim), row64(desc2, i2, dim), row64(mask1, i1, dim),
                                                     row64(mask2, i2, dim), dim)
                                           : dist64(row64(desc1, i1, dim), row64(desc2, i2, dim), dim);
                    if (dist < best1) { best2 = best1; best1 = dist; bestIdx = i2; }
                    else if (dist < best2) best2 = dist;
                }
                if (best1 <= th_low && (double)best1 < nnratio * (double)best2) {
                    match_of_2[bestIdx] = i1;
                    ++nm;
                }
            }
            ++a; ++b;
        } else if (fv1_nodes[a] < fv2_nodes[b]) ++a;
        else ++b;
    }
    *nmatches = nm;
    return 0;
}

}  // extern "C"
