// stub_mappoint.h -- stand-ins for what the reference's own src/cMapPoint.cpp needs from the rest of the system, so that it compiles
// WHERE IT LIES into its own library (oracle/_ref/libmappoint_ref.so, ref_mappoint/Makefile).   TEST INFRASTRUCTURE.
//
// Force-included (-include) ahead of the reference's include/cMapPoint.h: it pre-defines the include guards of cMultiKeyFrame.h,
// cMap.h, cMultiFrame.h and cORBmatcher.h, so the real cMapPoint class (include/cMapPoint.h) meets only the data-only key frame and
// map below.  This library never links the stand-in cMapPoint of ref_mcs/stub_slam.h (libmcs_ref.so): the two cMapPoint classes
// stay in separate links.
//
// Besides the stand-in OpenCV of ref_mcs/stub, cMapPoint.cpp needs cv::DataType<int> and Vec / scalar, added here; the division
// has OpenCV's semantics: core/matx.hpp (3.x and 4.x) defines operator/(const Vec&, double) and operator/(const Vec&, int) as
// Vec(a, 1./alpha, Matx_ScaleOp()), i.e. every element times the rounded reciprocal (saturate_cast<double> is the identity).
#pragma once
#define MULTIKEYFRAME_H
#define MAP_H
#define MULTIFRAME_H
#define ORBMATCHER_H

#include <opencv2/opencv.hpp>
#include <cstdint>
#include <map>
#include <unordered_map>
#include <vector>

#include "misc.h"            // the reference's median() (include/misc.h:96-104), which cMultiKeyFrame.h would bring

namespace cv {
template <class T> struct DataType;
// cMapPoint.cpp only makes Mat::zeros(N, N, DataType<int>::type) and reads it through ptr<int>: any 4-byte type whose zero is all
// zero bits serves, and the stand-in Mat's setTo fills CV_32F (not CV_32S)
template <> struct DataType<int> { enum { type = CV_32F }; };
template <class T, int N> inline Vec<T, N> operator/(const Vec<T, N>& a, double alpha) {
    const double s = 1. / alpha;
    Vec<T, N> r;
    for (int i = 0; i < N; ++i) r.val[i] = (T)(a.val[i] * s);
    return r;
}
template <class T, int N> inline Vec<T, N> operator/(const Vec<T, N>& a, int alpha) {
    const double s = 1. / alpha;
    Vec<T, N> r;
    for (int i = 0; i < N; ++i) r.val[i] = (T)(a.val[i] * s);
    return r;
}
}  // namespace cv

namespace MultiColSLAM
{
class cMapPoint;

// include/cORBmatcher.h:43-53; defined by the reference's src/cORBmatcher.cpp, reached at run time (wrap_mappoint.cpp)
int DescriptorDistance64(const uint64_t* descr_i, const uint64_t* descr_j, const int& dim);
int DescriptorDistance64Masked(const uint64_t* descr_i, const uint64_t* descr_j, const uint64_t* mask_i, const uint64_t* mask_j,
                               const int& dim);

struct StubCamSystem { int nCams = 1; int GetNrCams() const { return nCams; } };

class cMultiKeyFrame      // include/cMultiKeyFrame.h: the members src/cMapPoint.cpp reads, filled by wrap_mappoint.cpp
{
public:
	long unsigned int mnId = 0;
	StubCamSystem camSystem;
	bool bad = false, masksLearned = false;
	cv::Vec3d ow;
	int dim = 32;
	std::vector<cv::Mat> desc, dmask;          // per camera [capacity x dim]
	std::vector<int> octave;                   // per contiguous index
	std::vector<double> mvScaleFactors;
	int mnScaleLevels = 1;
	std::unordered_map<size_t, int> keypoint_to_cam;            // include/cMultiKeyFrame.h:222
	std::unordered_map<size_t, int> cont_idx_to_local_cam_idx;  // include/cMultiKeyFrame.h:227

	bool isBad() { return bad; }
	bool HavingMasks() { return masksLearned; }
	cv::Vec3d GetCameraCenter() { return ow; }
	int GetKeyPointScaleLevel(const size_t& idx) const { return octave[idx]; }                         // src/cMultiKeyFrame.cpp:341-344
	cv::Mat GetDescriptor(const int& cam, const size_t& idx) const { return desc[cam].row((int)idx).clone(); }       // :346-349
	cv::Mat GetDescriptorMask(const int& cam, const size_t& idx) const { return dmask[cam].row((int)idx).clone(); }  // :351-354
	double GetScaleFactor(int nLevel = 1) const { return mvScaleFactors[nLevel]; }                     // include/cMultiKeyFrame.h:153
	int GetScaleLevels() const { return mnScaleLevels; }                                                // :168
	void EraseMapPointMatch(const size_t&) {}
	void ReplaceMapPointMatch(const size_t&, cMapPoint*) {}
};

class cMap
{
public:
	void EraseMapPoint(cMapPoint*) {}
};
}  // namespace MultiColSLAM
