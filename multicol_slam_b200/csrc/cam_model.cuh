// cam_model.cuh -- Scaramuzza/OCam projection, the exact double arithmetic of the reference
// (ref src/cam_model_omni.cpp:49-67, :146-161; include/cam_model_omni.h:127-145; include/misc.h:115-122).
// Host and device share this code; build with -fmad=false / -ffp-contract=off.
#pragma once
#include <math.h>
#include "../../include/mcs_b200.h"

#ifdef __CUDACC__
#define MCS_HD __host__ __device__ __forceinline__
#else
#define MCS_HD inline
#endif

namespace mcs {

MCS_HD double cam_horner(const double* c, int n, double x) {
    double r = 0.0;
    for (int i = n - 1; i >= 0; --i) r = r * x + c[i];
    return r;
}

MCS_HD void cam_world_to_img(const mcs_ocam& cam, double x, double y, double z, double& u, double& v) {
    double norm = sqrt(x * x + y * y);
    if (norm == 0.0) norm = 1e-14;
    const double theta = atan(-z / norm);
    const double rho = cam_horner(cam.inv_pol, 12, theta);
    const double uu = x / norm * rho;
    const double vv = y / norm * rho;
    u = uu * cam.c + vv * cam.d + cam.u0;
    v = uu * cam.e + vv + cam.v0;
}

#ifdef __CUDACC__
// WorldToCamHom_fast (ref src/cam_system_omni.cpp:92-133) then isPointInMirrorMask(u, v, 0) (ref src/cam_model_omni.cpp:163-178).
// M: the camera's MtMc_inv (row-major 4x4), mask: its level-0 mirror mask.  ptRot = M * (P, 1) is the cv::Matx product,
// s = 0 + a0 b0 + a1 b1 + a2 b2 + a3 b3 in this order, no FMA.  Returns whether (u, v) lies in the mask.
__device__ __forceinline__ bool cam_project_in_mask(const double* M, const mcs_ocam& cam, const uint8_t* mask, double P0, double P1,
                                                    double P2, double& u, double& v) {
    double r[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) r[k] = ((M[4 * k] * P0 + M[4 * k + 1] * P1) + M[4 * k + 2] * P2) + M[4 * k + 3] * 1.0;
    cam_world_to_img(cam, r[0], r[1], r[2], u, v);
    const int ur = __double2int_rn(u), vr = __double2int_rn(v);
    if (ur >= cam.width || ur <= 0 || vr >= cam.height || vr <= 0) return false;
    return mask[(size_t)vr * cam.width + ur] != 0;
}
#endif

MCS_HD void cam_img_to_world(const mcs_ocam& cam, double u, double v, double& x, double& y, double& z) {
    const double inv_affine = cam.c - cam.d * cam.e;
    const double u_t = u - cam.u0;
    const double v_t = v - cam.v0;
    x = (u_t - cam.d * v_t) / inv_affine;
    y = (-cam.e * u_t + cam.c * v_t) / inv_affine;
    const double X2 = x * x, Y2 = y * y;
    z = -cam_horner(cam.pol, 5, sqrt(X2 + Y2));
    const double norm = sqrt(X2 + Y2 + z * z);
    x /= norm; y /= norm; z /= norm;
}

MCS_HD void cam_undistort(const mcs_ocam& cam, double px, double py, double s, double& ox, double& oy) {
    double x, y, z;
    cam_img_to_world(cam, px, py, x, y, z);
    ox = -x / z * s;
    oy = -y / z * s;
}

// CheckDistEpipolarLine(ray1, ray2, E12, thresh) (ref src/misc.cpp:53-69).  The cv::Matx products accumulate s = 0; s += a * b in
// index order; the host search (mcs_search_for_triangulation) and the device one (tr_epi_kernel, tr_walk_kernel) both call this.
MCS_HD bool cam_epipolar_ok(const double* r1, const double* r2, const double* E, double thresh) {
    double t[3];                                       // ray2^T * E  (1x3)
    for (int j = 0; j < 3; ++j) { double s = 0; for (int i = 0; i < 3; ++i) s += r2[i] * E[3 * i + j]; t[j] = s; }
    double nom = 0; for (int j = 0; j < 3; ++j) nom += t[j] * r1[j];
    double ex1[3], etx2[3];
    for (int i = 0; i < 3; ++i) { double s = 0; for (int k = 0; k < 3; ++k) s += E[3 * i + k] * r1[k]; ex1[i] = s; }
    for (int i = 0; i < 3; ++i) { double s = 0; for (int k = 0; k < 3; ++k) s += E[3 * k + i] * r2[k]; etx2[i] = s; }
    const double den = ex1[0] * ex1[0] + ex1[1] * ex1[1] + ex1[2] * ex1[2] + etx2[0] * etx2[0] + etx2[1] * etx2[1] + etx2[2] * etx2[2];
    if (den == 0.0) return false;
    return (nom * nom) / den < thresh;
}

}  // namespace mcs
