// describe_kernel.cu -- K3: orientation + descriptor, one warp per selected keypoint.
//
//   IC_Angle            ref src/mdBRIEFextractorOct.cpp:221-248   integer moments over the 845-px disc, fastAtan2
//   undistortPointsOcam ref :1306-1317, include/cam_model_omni.h:127-138
//   rotate[AndDistort]Pattern  ref :250-301
//   compute_ORB / compute_dBRIEF / compute_mdBRIEF   ref :303-554
//   output assembly     ref :1327-1335  (pt *= scale for levels > 0)
//
// Layout of the work: lane b of the warp owns descriptor byte b, i.e. the 16 pattern points 16b..16b+15 (8 test
// pairs).  For the distorted variants the lane parks the 16 projected points of one pattern in its own shared-memory
// slots, the warp reduces their sum (the reference subtracts the mean of all 512 projected points, :262-281), then every
// lane rounds and samples its own points: no shuffles, no second projection pass.  Warp-uniform state that is only needed
// again in the rare paths or at the end lives in a per-warp context in shared memory (WarpCtx), not in registers.
//
// Fisheye projection cost.  cCamModelGeneral_::WorldToImg evaluates, per pattern point, sqrt + 3 divisions +
// atan + a 12-term Horner in double (~250 FP64 instructions; 1536 points per mdBRIEF keypoint).  Because the
// third coordinate is the per-camera constant z = -a0, u = x*g(r)*c + y*g(r)*d + u0 with
//     g(r) = R(r) / r,   R(r) = rho(atan(-z / r)),      r = sqrt(x^2 + y^2),
// and R is a smooth 1-D function of r ("the distortion baked into a LUT" of the north star).  Only
// cvRound(u - mean(u)) has to agree with the reference, so a pattern is evaluated by the cheapest of three tiers
// whose error bound still decides every rounding:
//   tier 1 (fp32, ~96 % of the patterns): everything RELATIVE to the keypoint.  With X_k the undistorted keypoint, r_k its
//     radius and d the rotated pattern offset (|d| <= 21.3), n = r^2 - r_k^2 = 2 X_k.d + |d|^2 and delta = n / (r + r_k) carry
//     the radius change without cancellation; the host tabulates, per camera and integer radius i, a degree-6 polynomial
//     of R(i + s) - R(i) (double constant + float coefficients), from which g(r) - g(r_k) = (R(r) - R(r_k) - g_k delta) / r;
//     then u - u_k = A [ g(r) d + (g(r) - g(r_k)) X_k ] with the affine part A.  All quantities are O(20 px), so fp32
//     (ulp 1.9e-6 at 16..32) is enough: measured worst error 5e-6 px (tools/k3_fp32_model.py, numpy without FMA).  A pattern
//     with any coordinate closer than kT1Guard = 2.5e-5 px to a rounding tie (or a sample outside the staged patch) falls
//     through to tier 2;
//     m-form of tier 1 (centres >= ~64 px, 94 % of the Lafida keypoints): g itself is a smooth function of m = r^2 away from the
//     centre, and n = m - m_k comes without a square root: with c_i, hw_i centre and half-width of centre i's window in m and
//     t = (m - c_i) / hw_i in [-1, 1], the host tabulates g - G(c_i) = t P(t) (P of degree 7: 8 float coefficients, fit error
//     below 1e-6 px in terms of the displacement it multiplies), so that g(r) - g(r_k) = t P(t) - t_k P(t_k) needs no rsqrt, no
//     reciprocal and no Newton steps: 28 instead of 39 instructions per point.  Same measured error as the s-form (4.7e-6 px,
//     tools/k3_fp32_model.py MFORM=1); nearer the centre the window is too wide in m (sqrt singularity of the odd part of R at
//     m = 0) and the s-form above serves;
//   tier 2 (FP64, degree-9 polynomial of R around the keypoint's radius, |error| < 2e-8 px, two rolled passes: sum, then
//     recompute + round): decides everything farther than 5e-7 px from a tie; also serves keypoints closer than
//     kT1MinRadius px to the distortion centre, where g has a pole;
//   tier 3 (exact): the reference's own operation sequence (cam_model.cuh), p ~ 2e-4 per pattern.
#include <cstdlib>
#include <cstring>
#include <vector>

#include "cam_model.cuh"
#include "kernels.h"
#include "mcs_common.cuh"

namespace mcs {

__constant__ signed char c_pairs[2048];          // learned_pattern_64_ORB (ref include/mdBRIEFextractorOct.h:44-47)
// the same pattern as floats in the kernel's [j][lane] order (point 16*byte + k, byte = lane + 32*(j/16), k = j%16): the CTAs copy it
// to shared memory with four 8-byte loads per thread instead of rebuilding it from bytes (constant-bank loads + I2F on the XU pipe)
__device__ float2 g_patf[1024];
__constant__ signed char c_disc_u[848], c_disc_v[848];   // c_disc_u[0..16] = umax[] of the IC_Angle disc (ref :187-202); rest unused

// cv::fastAtan2 (SURVEY Appendix A.4), evaluated without FMA
__device__ __forceinline__ float fast_atan2_deg(float y, float x) {
    const float s = (float)(180.0 / 3.14159265358979323846);
    const float p1 = 0.9997878412794807f * s, p3 = -0.3258083974640975f * s;
    const float p5 = 0.1555786518463281f * s, p7 = -0.04432655554792128f * s;
    const float ax = fabsf(x), ay = fabsf(y);
    float a, c, c2;
    if (ax >= ay) {
        c = __fdiv_rn(ay, __fadd_rn(ax, (float)2.2204460492503131e-16));
        c2 = __fmul_rn(c, c);
        a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
    } else {
        c = __fdiv_rn(ax, __fadd_rn(ay, (float)2.2204460492503131e-16));
        c2 = __fmul_rn(c, c);
        a = __fsub_rn(90.f, __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c));
    }
    if (x < 0) a = __fsub_rn(180.f, a);
    if (y < 0) a = __fsub_rn(360.f, a);
    return a;
}

__device__ __forceinline__ int sample_px(const uint8_t* bimg, const uint8_t* uimg, const LevelGeom& g, int row, int col) {
    // blurred ROI; outside the ROI the reference reads the un-blurred REFLECT_101 ring of its buffer
    if ((unsigned)row < (unsigned)g.h && (unsigned)col < (unsigned)g.w) return bimg[(size_t)row * g.pitch + col];
    row = min(max(row, -kEdge), g.h - 1 + kEdge); col = min(max(col, -kEdge), g.w - 1 + kEdge);   // memory-safety clamp
    return uimg[(size_t)reflect101(row, g.h) * g.pitch + reflect101(col, g.w)];
}

constexpr int kDescWarps = 4;
constexpr int kPatchR = 25;                       // staged patch: rows/cols ky/kx -25 .. +25 (keypoints are >= 25 px inside the ROI)
constexpr int kPatchS = 64;                       // bytes per staged patch row (4-byte aligned start + 51 columns)
constexpr int kLutDeg = 9;                        // degree of the per-centre polynomial of R(r)  (kernels.h: DistortLut)
#ifndef MCS_K3_T1
#define MCS_K3_T1 1                  // 0: tier 1 off (A/B builds: everything goes through tier 2)
#endif
#ifndef MCS_K3_REPAIR
#define MCS_K3_REPAIR 1              // 0: flagged tier-1 patterns go straight to tier 2 (A/B builds)
#endif
#ifndef MCS_K3_V3
#define MCS_K3_V3 1                  // round-2 instruction diet (0 restores the previous forms for A/B builds): IC-angle disc read from a
#endif                               // shared-memory copy, warp mean by one integer REDUX, tie / range test as running maxima
#ifndef MCS_K3_MINB
#define MCS_K3_MINB 5                // resident CTAs per SM the register budget is cut for.  sm_90a, H100 80GB HBM3, 400 W limit, bench.py config 2, 2 alternating runs,
                                     // K3 ms per 384 images: 4 -> 126-128 registers, no spills: 5.49 / 5.90; 5 -> 96 registers,
                                     // 80-144 B spilled: 5.39 / 5.51; 6 -> 80 registers: 5.81 / 5.85
#endif
#ifndef MCS_K3_U1
#define MCS_K3_U1 4                  // unroll of tier-1 pass 1 (m-form), points per iteration   (A/B builds)
#endif
#ifndef MCS_K3_U2
#define MCS_K3_U2 2                  // unroll of tier-1 pass 2, point PAIRS per iteration        (A/B builds)
#endif
constexpr int kT1Unroll1 = MCS_K3_U1, kT1Unroll2 = MCS_K3_U2;
constexpr int kT1Coef = 6;                        // tier 1: q(s') of degree 5, R(i + s) - R(i) = s' q(s'), s' = s / kT1Scale
constexpr float kT1Scale = 32.f;
constexpr double kT1MinRadius = 40.0;             // tier 1 needs r >= r_k - 21.3 well away from the pole of g at r = 0
constexpr float kT1Guard = 2.5e-5f;               // px; 5x the worst tier-1 error measured by tools/k3_fp32_model.py
// doubles per centre: [0] tau offset, [1] tau scale, [2..11] kLutDeg + 1 coefficients (tier 2);
// [12] R(i), [13] q0 (double), [14..16] q1..q5 as floats (+ one pad float), [17] 1.0 when the tier-1 entry is usable
constexpr double kLutReach = 22.5;                // half-width of a centre's interval: pattern radius 15*sqrt(2) + 0.5 + margin
// [18] G(c_i) (double), [19..22] a0..a7 of the m-form as floats, [23] 1.0 when the m-form entry is usable  (MCS_K3_MFORM)
constexpr int kLutStride = 24;
#ifndef MCS_K3_MFORM
#define MCS_K3_MFORM 1               // tier 1 in the variable m = r^2 where the centre's table allows it (0: always the s-form; A/B builds)
#endif
constexpr int kT1MCoef = 8;                       // m-form: g(r) - G(c_i) = t P(t), P of degree 7, t = (r^2 - c_i) / hw_i
// centre and half-width of centre i's window in m = r^2: r in [i - reach, i + reach]  (i >= reach, checked where the entry is built)
__host__ __device__ inline double t1m_centre(int i) { return (double)i * (double)i + kLutReach * kLutReach; }
__host__ __device__ inline double t1m_halfwidth(int i) { return 2.0 * kLutReach * (double)i; }

// Rare path: one pattern of one keypoint with the reference's exact operation sequence (two projection passes;
// per-lane partial sums + butterfly: within ~1e-13 of the reference's sequential sum; the tier-1 guard band below keeps every
// pattern whose rounding that difference could change on this path, see DESIGN.md "K3 tiers").
// Returns the descriptor byte(s) of this lane for that pattern, byte bb in bits [8bb, 8bb+8).
template <int PPL>
__device__ __noinline__ unsigned exact_pattern(const mcs_ocam* cam, const float2* s_pat, double angle, double ukx,
                                               double uky, int lane, int ds, const uint8_t* bimg, const uint8_t* uimg,
                                               const LevelGeom* g, int kx, int ky) {
    const double ca = cos(angle), sa = sin(angle);      // the reference's own cos(angle) / sin(angle) (ref :430-436)
    const double z = -cam->pol[0];
    double su = 0.0, sv = 0.0;
    for (int j = 0; j < PPL; ++j) {
        const float2 pp = s_pat[j * 32 + lane];
        const double px = (double)pp.x, py = (double)pp.y;
        const double xr = px * ca - py * sa + ukx;
        const double yr = px * sa + py * ca + uky;
        double u, v;
        cam_world_to_img(*cam, xr, yr, z, u, v);
        if (lane + 32 * (j >> 4) < ds) { su += u; sv += v; }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        su += __shfl_xor_sync(0xffffffffu, su, o);
        sv += __shfl_xor_sync(0xffffffffu, sv, o);
    }
    const double mu = su / (double)(16 * ds), mv = sv / (double)(16 * ds);
    unsigned out = 0;
    for (int j = 0; j < PPL; j += 2) {
        int smp[2];
        for (int e = 0; e < 2; ++e) {
            const float2 pp = s_pat[(j + e) * 32 + lane];
            const double px = (double)pp.x, py = (double)pp.y;
            const double xr = px * ca - py * sa + ukx;
            const double yr = px * sa + py * ca + uky;
            double u, v;
            cam_world_to_img(*cam, xr, yr, z, u, v);
            smp[e] = sample_px(bimg, uimg, *g, ky + __double2int_rn(v - mv), kx + __double2int_rn(u - mu));
        }
        out |= (unsigned)(smp[0] < smp[1]) << (j >> 1);
    }
    return out;
}

// ORB rotation (ref :285-301) and generic sampling straight from global memory; used for ORB when an offset leaves
// the staged patch (never for sane inputs) -- keeps the reference's read semantics (blurred ROI / reflected ring).
template <int PPL>
__device__ __noinline__ unsigned orb_pattern_global(const float2* s_pat, double ca, double sa, int lane, const uint8_t* bimg,
                                                    const uint8_t* uimg, const LevelGeom* g, int kx, int ky) {
    unsigned out = 0;
    for (int j = 0; j < PPL; j += 2) {
        int smp[2];
        for (int e = 0; e < 2; ++e) {
            const float2 pp = s_pat[(j + e) * 32 + lane];
            const double px = (double)pp.x, py = (double)pp.y;
            smp[e] = sample_px(bimg, uimg, *g, ky + __double2int_rn(px * sa + py * ca), kx + __double2int_rn(px * ca - py * sa));
        }
        out |= (unsigned)(smp[0] < smp[1]) << (j >> 1);
    }
    return out;
}

// Tier 2: one pattern through the per-keypoint degree-9 polynomial of R(r) in double (error < 2e-8 px).  Two rolled passes --
// sum of the projected coordinates, then recompute + subtract the mean + round + sample -- so that the live set stays small;
// the recomputation is the same instruction sequence, hence the same values.  Sets *need_exact when a coordinate lies within
// 5e-7 px of a rounding tie, outside the fitted interval or outside the staged patch (tier 3 then decides).
struct Tier2Poly { double t_off, t_scale, P[kLutDeg + 1]; };
__device__ __forceinline__ void tier2_point(const Tier2Poly& L, const mcs_ocam& cam, const double2 pp, double ca, double sa, double ukx,
                                            double uky, double& u, double& v, int& worst_tau) {
    const double xr = fma(pp.x, ca, fma(-pp.y, sa, ukx));
    const double yr = fma(pp.x, sa, fma(pp.y, ca, uky));
    const double s2 = fma(xr, xr, yr * yr);
    // 1/sqrt(s2): hardware approximation (~1e-7) + one third-order step -> < 1e-16 relative
    double y0;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y0) : "d"(s2));
    const double e = fma(-(s2 * y0), y0, 1.0);
    const double rinv = fma(y0 * e, fma(0.375, e, 0.5), y0), r = s2 * rinv;
    // R(r) by Horner; |tau| > 1 (a point outside the fitted interval, or NaN from s2 == 0) is caught by the caller
    const double tau = fma(r, L.t_scale, L.t_off);
    double gg = L.P[kLutDeg];
#pragma unroll
    for (int k = kLutDeg - 1; k >= 0; --k) gg = fma(gg, tau, L.P[k]);
    worst_tau = max(worst_tau, __double2hiint(tau) & 0x7fffffff);
    gg *= rinv;
    const double uu = xr * gg, vv = yr * gg;
    u = fma(uu, cam.c, fma(vv, cam.d, cam.u0));
    v = fma(uu, cam.e, vv + cam.v0);
}
template <int PPL>
__device__ __noinline__ unsigned tier2_pattern(const mcs_ocam* camp, const float2* s_patf, const double* __restrict__ row, double ca,
                                               double sa, double ukx, double uky, int lane, int ds, const uint8_t* patch, int pofs,
                                               int* need_exact) {
    const mcs_ocam& cam = *camp;
    Tier2Poly L;
    {
        const double2* cp = (const double2*)row;
        const double2 h = __ldg(cp);
        L.t_off = h.x; L.t_scale = h.y;
#pragma unroll
        for (int k = 0; k < (kLutDeg + 1) / 2; ++k) {
            const double2 cc = __ldg(cp + 1 + k);
            L.P[2 * k] = cc.x; L.P[2 * k + 1] = cc.y;
        }
    }
    const bool lane_valid = (PPL == 32) || (lane < ds);      // descSize 16: lanes 16..31 own no byte
    double su = 0.0, sv = 0.0;
    int worst_tau = 0;
#pragma unroll 2
    for (int j = 0; j < PPL; ++j) {
        double u, v;
        { const float2 pf = s_patf[j * 32 + lane]; tier2_point(L, cam, make_double2((double)pf.x, (double)pf.y), ca, sa, ukx, uky, u, v, worst_tau); }
        if (lane_valid) { su += u; sv += v; }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        su += __shfl_xor_sync(0xffffffffu, su, o);
        sv += __shfl_xor_sync(0xffffffffu, sv, o);
    }
    const double inv_n = 1.0 / (double)(16 * ds);
    const double mu = su * inv_n, mv = sv * inv_n;
    // round-to-nearest-even through the 1.5*2^52 trick: no F2I/I2F (XU pipe), same result as lrint
    constexpr double kMagic = 6755399441055744.0;
    int worst_frac = 0;
    unsigned worst_ofs = 0, out = 0;
#pragma unroll 1
    for (int j = 0; j < PPL; j += 2) {
        int smp[2];
#pragma unroll
        for (int e2 = 0; e2 < 2; ++e2) {
            double u, v;
            { const float2 pf = s_patf[(j + e2) * 32 + lane]; tier2_point(L, cam, make_double2((double)pf.x, (double)pf.y), ca, sa, ukx, uky, u, v, worst_tau); }
            const double du = u - mu, dv = v - mv;
            const double tu = du + kMagic, tv = dv + kMagic;
            int ix = __double2loint(tu), iy = __double2loint(tv);
            // closeness to a rounding tie as integer maxima: the high word of |frac| orders like the double itself
            const int hu = __double2hiint(du - (tu - kMagic)) & 0x7fffffff, hv = __double2hiint(dv - (tv - kMagic)) & 0x7fffffff;
            worst_frac = max(worst_frac, max(hu, hv));
            worst_ofs = max(worst_ofs, max((unsigned)(ix + kPatchR), (unsigned)(iy + kPatchR)));
            ix = min(max(ix, -kPatchR), kPatchR); iy = min(max(iy, -kPatchR), kPatchR);      // stay inside the patch; redone if it mattered
            smp[e2] = patch[pofs + iy * kPatchS + ix];
        }
        out |= (unsigned)(smp[0] < smp[1]) << (j >> 1);
    }
    // closer than ~7e-7 px to a rounding tie (high word of 0.5 - 5e-7), outside the fitted interval (|tau| >= 1; a NaN has a
    // huge high word) or outside the staged patch -> exact path
    if (lane_valid && (worst_frac >= __double2hiint(0.5 - 5e-7) || worst_ofs > 2u * kPatchR || worst_tau >= __double2hiint(1.0)))
        *need_exact = 1;
    return out;
}

// Tier 1 repair: a tier-1 pattern in which a few coordinates came out closer than kT1Guard to a rounding tie.  The mean of the
// parked fp32 values is re-summed in double (its error against the exact mean is the SYSTEMATIC part of the tier-1 error only:
// <= 1.5e-7 px, tools/k3_fp32_model.py "mean err", plus the <= 1e-6 px fit error build_distort_lut accepts), and just the flagged points are recomputed through the tier-2 polynomial
// (|error| < 2e-8 px) relative to the keypoint's own image.  A recomputed coordinate still within kT1RepairGuard of a tie, or
// outside the patch / fitted interval, sets *fail (the whole pattern then goes to tier 2).
constexpr double kT1RepairGuard = 4e-6;
template <int PPL>
__device__ __noinline__ unsigned tier1_repair(const mcs_ocam* camp, const float2* s_patf, const float2* park, const double* __restrict__ row,
                                              double ca, double sa, double ukx, double uky, int lane, int ds, const uint8_t* patch, int pofs,
                                              int* fail) {
    const mcs_ocam& cam = *camp;
    Tier2Poly L;
    {
        const double2* cp = (const double2*)row;
        const double2 h = __ldg(cp);
        L.t_off = h.x; L.t_scale = h.y;
#pragma unroll
        for (int k = 0; k < (kLutDeg + 1) / 2; ++k) {
            const double2 cc = __ldg(cp + 1 + k);
            L.P[2 * k] = cc.x; L.P[2 * k + 1] = cc.y;
        }
    }
    const bool lane_valid = (PPL == 32) || (lane < ds);
    double su = 0.0, sv = 0.0;
#pragma unroll 4
    for (int j = 0; j < PPL; ++j) {
        const float2 c = park[j * 32 + lane];
        if (lane_valid) { su += (double)c.x; sv += (double)c.y; }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        su += __shfl_xor_sync(0xffffffffu, su, o);
        sv += __shfl_xor_sync(0xffffffffu, sv, o);
    }
    const double inv_n = 1.0 / (double)(16 * ds);
    const double mu = su * inv_n, mv = sv * inv_n;
    int worst_tau = 0;
    double uk, vk;                                     // the keypoint's own image under the same polynomial
    tier2_point(L, cam, make_double2(0.0, 0.0), ca, sa, ukx, uky, uk, vk, worst_tau);
    constexpr double kMagic = 6755399441055744.0;
    bool bad = false;
    unsigned out = 0;
#pragma unroll 1
    for (int j = 0; j < PPL; j += 2) {
        int smp[2];
#pragma unroll 1
        for (int e2 = 0; e2 < 2; ++e2) {
            const float2 c = park[(j + e2) * 32 + lane];
            double tu = (double)c.x - mu, tv = (double)c.y - mv;
            double ru = (tu + kMagic) - kMagic, rv = (tv + kMagic) - kMagic;
            if (!(fabs(tu - ru) < 0.5 - (double)kT1Guard) || !(fabs(tv - rv) < 0.5 - (double)kT1Guard)) {
                double u, v;
                const float2 pf = s_patf[(j + e2) * 32 + lane];
                tier2_point(L, cam, make_double2((double)pf.x, (double)pf.y), ca, sa, ukx, uky, u, v, worst_tau);
                tu = (u - uk) - mu; tv = (v - vk) - mv;
                ru = (tu + kMagic) - kMagic; rv = (tv + kMagic) - kMagic;
                bad |= !(fabs(tu - ru) < 0.5 - kT1RepairGuard) || !(fabs(tv - rv) < 0.5 - kT1RepairGuard);
            }
            bad |= !(fabs(tu) < (double)kPatchR + 0.4) || !(fabs(tv) < (double)kPatchR + 0.4);
            int ix = (int)ru, iy = (int)rv;
            ix = min(max(ix, -kPatchR), kPatchR); iy = min(max(iy, -kPatchR), kPatchR);
            smp[e2] = patch[pofs + iy * kPatchS + ix];
        }
        out |= (unsigned)(smp[0] < smp[1]) << (j >> 1);
    }
    if (lane_valid && (bad || worst_tau >= __double2hiint(1.0))) *fail = 1;
    return out;
}

// warp-uniform values of the keypoint a warp works on, kept in shared memory across the pattern loops (see the kernel)
struct __align__(16) WarpCtx {
    float t1[16];                   // tier-1 constants of the keypoint: q[0..7], K0f, gkf, s0f, rk2f, rkf, auk, avk
    double ukx, uky, a_base, ca[3], sa[3];
    const double* row;
    int kx, ky, oidx, b, level;
    uint32_t c;
    float angle;
};
template <int PPL /* pattern points per lane: 16 for descSize <= 32, 32 for descSize 64 */, int MINB = MCS_K3_MINB>
__global__ void __launch_bounds__(kDescWarps * 32, MINB)
describe_kernel(const PyramidGeom* __restrict__ geom, const DescribeArgs args, const mcs_ocam* __restrict__ cams,
                const DistortLut* __restrict__ luts, const int* __restrict__ cam_of_image,
                const uint32_t* __restrict__ sel_xys, const int* __restrict__ sel_count,
                mcs_keypoint* __restrict__ kps_out, uint8_t* __restrict__ desc_out, uint8_t* __restrict__ dmask_out,
                int* __restrict__ counts_out, const int capacity, const int n_images) {
    __shared__ mcs_ocam s_cam[kDescWarps];
    __shared__ WarpCtx s_ctx[kDescWarps];
    __shared__ __align__(8) float2 s_patf[PPL * 32];      // [j][lane] : point 16*byte + k with byte = lane + 32*(j/16), k = j%16, as floats
    // tier 1 parks the projected coordinates of the current pattern here between its two passes ([point][lane], this lane's own
    // slots only): with rolled loops the kernel body stays inside the instruction cache -- the fully unrolled form spent most of
    // its stalled cycles waiting on instruction fetch
    extern __shared__ __align__(8) float2 s_park_dyn[];          // [kDescWarps][PPL * 32], dynamic: 16 KB (descSize <= 32) / 32 KB
    __shared__ __align__(16) uint8_t s_patch[kDescWarps][(2 * kPatchR + 1) * kPatchS];
    const int ds = geom->desc_size;
    // (lanes that own no descriptor byte -- descSize 16 -- carry real pattern points too; every use is guarded by lane_valid)
#pragma unroll
    for (int i = threadIdx.x; i < PPL * 32; i += kDescWarps * 32) s_patf[i] = g_patf[i];
    __syncthreads();

    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    // one warp per slot (a persistent grid-stride variant was slower: static imbalance and more spills)
    const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int sel_total = geom->sel_total;
    const int b = warp_global / sel_total;
    if (b >= n_images) return;
    const int slot = warp_global - b * sel_total;
    const int L = geom->nlevels;
    int level = 0, off = 0;
    for (int l = 0; l < L; ++l)
        if (slot >= geom->lv[l].sel_off) level = l;
    for (int l = 0; l < level; ++l) off += sel_count[b * L + l];
    const LevelGeom& g = geom->lv[level];
    const int p = slot - g.sel_off;
    const int cnt = sel_count[b * L + level];
    if (slot == 0 && lane == 0) {
        int tot = 0;
        for (int l = 0; l < L; ++l) tot += sel_count[b * L + l];
        counts_out[b] = min(tot, capacity);
    }
    if (p >= cnt) return;
    const int oidx = off + p;
    if (oidx >= capacity) return;
    const uint32_t c = sel_xys[(size_t)b * sel_total + slot];
    const int kx = corner_x(c), ky = corner_y(c);
    const uint8_t* uimg = args.lvl[level] + (size_t)b * g.img_bytes;
    const uint8_t* bimg = args.blur[level] + (size_t)b * g.img_bytes;
    const int pitch = g.pitch;

    // ---- stage the blurred 51x51 patch: 2 rows per warp instruction, 15 aligned words per row ----
    uint8_t* patch = s_patch[wib];
    const int x0 = (kx - kPatchR) & ~3;                    // >= 0: keypoints lie >= 25 px inside the level
    {
        const int half = lane >> 4, w = lane & 15;
        const uint32_t* gp = (const uint32_t*)(bimg + (size_t)(ky - kPatchR + half) * pitch + x0) + w;
        uint32_t* sp = (uint32_t*)(patch + half * kPatchS) + w;
        // all loads of a batch are issued before the first store (memory-level parallelism)
#pragma unroll
        for (int k0 = 0; k0 < 26; k0 += 13) {
            uint32_t t[13];
#pragma unroll
            for (int k = 0; k < 13; ++k) {
                const int r = half + 2 * (k0 + k);
                t[k] = (w < 15 && r < 2 * kPatchR + 1) ? __ldg(gp + (size_t)(k0 + k) * (pitch / 2)) : 0u;
            }
#pragma unroll
            for (int k = 0; k < 13; ++k) {
                const int r = half + 2 * (k0 + k);
                if (w < 15 && r < 2 * kPatchR + 1) sp[(k0 + k) * (2 * kPatchS / 4)] = t[k];
            }
        }
    }
    const int pofs = kPatchR * kPatchS + (kx - x0);        // patch byte offset of the keypoint itself

    // ---- IC_Angle (ref :221-248): integer moments over the 845-pixel disc, lane = column u = lane-16 (+ u = 16) ----
    int m10 = 0, m01 = 0;
#if MCS_K3_V3
    {
        // The 33 x 33 neighbourhood of the UNBLURRED level is copied with aligned word loads (3 rows x 10 words per warp
        // instruction) into this warp's slice of the parking buffer, which tier 1 only uses later; the moments are then summed from
        // shared memory with compile-time offsets: row pairs +-k share one disc test, m01 += k (val(+k) - val(-k)).
        constexpr int kIcS = 40;                            // bytes per staged row: 4-byte aligned start + 33 columns
        uint8_t* ic = reinterpret_cast<uint8_t*>(s_park_dyn + wib * (PPL * 32));
        const int xs = (kx - kHalfPatch) & ~3;              // >= 0: keypoints lie >= 25 px inside the level
        {
            const int rr = lane / 10, w = lane - rr * 10;
            const uint32_t* gp = (const uint32_t*)(uimg + (size_t)(ky - kHalfPatch + rr) * pitch + xs) + w;
            uint32_t* sp = (uint32_t*)(ic + rr * kIcS) + w;
            uint32_t t[11];
#pragma unroll
            for (int k = 0; k < 11; ++k) t[k] = (lane < 30) ? __ldg(gp + (size_t)k * 3 * (pitch / 4)) : 0u;
#pragma unroll
            for (int k = 0; k < 11; ++k) if (lane < 30) sp[k * 3 * (kIcS / 4)] = t[k];
        }
        __syncwarp();
        const int u = lane - kHalfPatch;                    // -16 .. 15
        const int au = u < 0 ? -u : u;
        const int vm = c_disc_u[au];                        // |v| <= vmax(|u|) = umax[|u|]: the disc is symmetric (ref :187-202)
        const uint8_t* col = ic + kHalfPatch * kIcS + (kx - kHalfPatch - xs) + lane;
        int sum = col[0];
#pragma unroll
        for (int k = 1; k <= kHalfPatch; ++k) {
            const int a = col[k * kIcS], bb = col[-k * kIcS];
            if (vm >= k) { sum += a + bb; m01 += k * (a - bb); }
        }
        m10 = u * sum;
        const int um = c_disc_u[kHalfPatch];
        if (lane < 2 * um + 1) {                            // column u = +16: rows |v| <= umax[16]
            const int v = lane - um;
            const int val = ic[(kHalfPatch + v) * kIcS + (kx - kHalfPatch - xs) + 2 * kHalfPatch];
            m10 += kHalfPatch * val;
            m01 += v * val;
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            m10 += __shfl_xor_sync(0xffffffffu, m10, o);
            m01 += __shfl_xor_sync(0xffffffffu, m01, o);
        }
        __syncwarp();                                       // the parking buffer is free again
    }
#else
    {
        const uint8_t* ctr = uimg + (size_t)ky * pitch + kx;
        const int u = lane - kHalfPatch;                    // -16 .. 15
        const int au = u < 0 ? -u : u;
        // |v| <= vmax(u): the disc is symmetric (umax table, ref :187-202); vmax(|u|) = umax[|u|]
        const int vm = c_disc_u[au];                        // c_disc_u[0..16] doubles as umax[] (see upload_constants)
#pragma unroll 11
        for (int v = -kHalfPatch; v <= kHalfPatch; ++v) {
            const int val = (v >= -vm && v <= vm) ? (int)ctr[v * pitch + u] : 0;
            m10 += u * val;
            m01 += v * val;
        }
        if (lane < 2 * c_disc_u[kHalfPatch] + 1) {          // column u = +16: rows |v| <= umax[16]
            const int v = lane - c_disc_u[kHalfPatch];
            const int val = ctr[v * pitch + kHalfPatch];
            m10 += kHalfPatch * val;
            m01 += v * val;
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            m10 += __shfl_xor_sync(0xffffffffu, m10, o);
            m01 += __shfl_xor_sync(0xffffffffu, m01, o);
        }
    }
#endif
    const float angle = fast_atan2_deg((float)m01, (float)m10);

    // Everything that is warp-uniform and only needed again in the rare paths or at the very end is parked in this warp's context in
    // shared memory instead of living in registers across the pattern loops: at 80 registers (6 CTAs per SM) the compiler otherwise
    // spills the INVARIANTS OF THE HOT LOOPS, and with 212 KB of the SM's 256 KB configured as shared memory those reloads miss the
    // small L1, and the kernel then waits on local-memory loads.
    WarpCtx& cx = s_ctx[wib];
    const int ci = cam_of_image[b];
    const bool masks = geom->learn_masks != 0, dbrief = geom->do_dbrief != 0 || masks;
    const int npat = masks ? 3 : 1;
    {
        double a0, s0, c0;
        if (masks) a0 = (double)__fdiv_rn(angle, 57.2957763671875f);              // angle / RHOf      (ref :425)
        else a0 = (double)__fmul_rn(angle, 0.01745329238474369f);                   // angle * DEG2RADf  (ref :313,367)
        sincos(a0, &s0, &c0);
        if (lane == 0) {
            cx.kx = kx; cx.ky = ky; cx.oidx = oidx; cx.b = b; cx.level = level; cx.c = c; cx.angle = angle; cx.a_base = a0;
            // angle +- 20 deg (20 / RHOd, ref :424) by the addition theorems (1e-16 away from cos/sin(a0 +- rot); the exact path uses
            // the reference's own cos(angle +- rot) / sin(angle +- rot))
            const double c20 = 0.93969262078590838405, s20 = 0.34202014332566873304;
            cx.ca[0] = c0; cx.sa[0] = s0;
            cx.ca[1] = fma(c0, c20, -s0 * s20); cx.sa[1] = fma(s0, c20, c0 * s20);
            cx.ca[2] = fma(c0, c20, s0 * s20);  cx.sa[2] = fma(s0, c20, -c0 * s20);
        }
    }
    constexpr int BPL = PPL / 16;                 // descriptor bytes per lane
    unsigned v0[BPL], vdiff[BPL];                 // bits of the pattern at the keypoint's angle; bits that differ in a +-20 degree re-test
#pragma unroll
    for (int bb = 0; bb < BPL; ++bb) { v0[bb] = 0u; vdiff[bb] = 0u; }
    auto put = [&](int qi, unsigned e /* byte bb in bits [8bb, 8bb+8) */) {
#pragma unroll
        for (int bb = 0; bb < BPL; ++bb) {
            const unsigned v = (e >> (8 * bb)) & 0xFFu;
            if (qi == 0) v0[bb] = v; else vdiff[bb] |= v ^ v0[bb];
        }
    };
    __syncwarp();                                 // patch staged, context written
    if (!dbrief) {
        // ---- ORB: rotatePattern (ref :285-301) ----
        const double ca0 = cx.ca[0], sa0 = cx.sa[0];
        int ix[PPL], iy[PPL];
        bool far = false;
#pragma unroll
        for (int j = 0; j < PPL; ++j) {
            const float2 pp = s_patf[j * 32 + lane];
            const double px = (double)pp.x, py = (double)pp.y;
            ix[j] = __double2int_rn(px * ca0 - py * sa0);
            iy[j] = __double2int_rn(px * sa0 + py * ca0);
            far |= (unsigned)(ix[j] + kPatchR) > 2u * kPatchR || (unsigned)(iy[j] + kPatchR) > 2u * kPatchR;
        }
        if (__any_sync(0xffffffffu, far)) {
            put(0, orb_pattern_global<PPL>(s_patf, ca0, sa0, lane, bimg, uimg, &g, kx, ky));
        } else {
            unsigned e = 0;
#pragma unroll
            for (int bb = 0; bb < BPL; ++bb) {
#pragma unroll
                for (int bit = 0; bit < 8; ++bit) {
                    const int j0 = 16 * bb + 2 * bit;
                    const int s0 = patch[pofs + iy[j0] * kPatchS + ix[j0]], s1 = patch[pofs + iy[j0 + 1] * kPatchS + ix[j0 + 1]];
                    e |= (unsigned)(s0 < s1) << (8 * bb + bit);
                }
            }
            put(0, e);
        }
    } else {
        // ---- dBRIEF / mdBRIEF: rotateAndDistortPattern (ref :250-283) ----
        if (lane < (int)(sizeof(mcs_ocam) / 8)) ((double*)&s_cam[wib])[lane] = ((const double*)&cams[ci])[lane];
        __syncwarp();
        const mcs_ocam& cam = s_cam[wib];
        const bool lane_valid = (PPL == 32) || (lane < ds);      // descSize 16: lanes 16..31 own no byte
        bool have_lut, t1, mform;
        {
            float q[kT1MCoef], K0f = 0.f, gkf = 0.f, s0f = 0.f, rk2f = 0.f, rkf = 0.f, auk = 0.f, avk = 0.f;
#pragma unroll
            for (int k = 0; k < kT1MCoef; ++k) q[k] = 0.f;
            const DistortLut lut = luts[ci];
            const float scale = g.scale;
            double ukx, uky;   // undistortPointsOcam(pt.x*scale, pt.y*scale, a0)  (ref :1306-1317)
            cam_undistort(cam, (double)__fmul_rn((float)kx, scale), (double)__fmul_rn((float)ky, scale), cam.pol[0], ukx, uky);
            // the table row of this keypoint: centre i = rn(r_k); its polynomials are valid for every pattern point (|r - r_k| <= 21.3)
            const double rk = sqrt(ukx * ukx + uky * uky);
            have_lut = rk < (double)(lut.n - 1);                  // false for NaN as well -> exact path
            const int ci_lut = have_lut ? __double2int_rn(rk) : 0;
            const double* row = lut.coef + (size_t)ci_lut * kLutStride;
            if (lane == 0) { cx.ukx = ukx; cx.uky = uky; cx.row = row; }
            // ---- tier-1 set-up (per keypoint, all lanes redundantly; ~25 FP64 instructions against 48 points x 3 patterns) ----
            t1 = MCS_K3_T1 && have_lut && rk >= kT1MinRadius && __ldg(row + 17) == 1.0;
            mform = MCS_K3_MFORM && t1 && __ldg(row + 23) == 1.0;
            if (mform) {
                // m-form: t_k, K0 = t_k P(t_k), g_k = G(c_i) + K0 in double from the float coefficients the points will use
                const float2 c01 = __ldg((const float2*)(row + 19)), c23 = __ldg((const float2*)(row + 20));
                const float2 c45 = __ldg((const float2*)(row + 21)), c67 = __ldg((const float2*)(row + 22));
                q[0] = c01.x; q[1] = c01.y; q[2] = c23.x; q[3] = c23.y; q[4] = c45.x; q[5] = c45.y; q[6] = c67.x; q[7] = c67.y;
                const double inv_hw = 1.0 / t1m_halfwidth(ci_lut);
                const double tk = (rk * rk - t1m_centre(ci_lut)) * inv_hw;
                double pk = (double)q[7];
#pragma unroll
                for (int k = 6; k >= 0; --k) pk = fma(pk, tk, (double)q[k]);
                const double K0 = tk * pk;
                gkf = (float)(__ldg(row + 18) + K0);
                K0f = (float)K0; s0f = (float)tk; rk2f = (float)inv_hw;              // s0f / rk2f double as t_k / (1 / hw) in the m-form
                auk = (float)(cam.c * ukx + cam.d * uky); avk = (float)(cam.e * ukx + uky);      // A X_k
            } else if (t1) {
                const double Ri = __ldg(row + 12), q0d = __ldg(row + 13);
                const float2 c12 = __ldg((const float2*)(row + 14)), c34 = __ldg((const float2*)(row + 15)), c5x = __ldg((const float2*)(row + 16));
                q[1] = c12.x; q[2] = c12.y; q[3] = c34.x; q[4] = c34.y; q[5] = c5x.x; q[6] = 0.f; q[7] = 0.f;
                const double s0 = (rk - (double)ci_lut) * (1.0 / (double)kT1Scale);          // in units of s'
                double pk = (double)q[5];
                pk = fma(pk, s0, (double)q[4]); pk = fma(pk, s0, (double)q[3]); pk = fma(pk, s0, (double)q[2]);
                pk = fma(pk, s0, (double)q[1]); pk = fma(pk, s0, q0d);
                const double dRk = s0 * pk;                            // R(r_k) - R(i)
                const double gk = (Ri + dRk) / rk;                     // g(r_k)
                // h(s') = s' q'(s') - K0' = R(r) - R(r_k) - g_k (r - r_k):  q'_0 = q_0 - g_k*scale,  K0' = dRk - g_k (r_k - i)
                q[0] = (float)(q0d - gk * (double)kT1Scale);
                K0f = (float)(dRk - gk * (rk - (double)ci_lut));
                gkf = (float)gk; s0f = (float)s0;
                rk2f = (float)(rk * rk); rkf = (float)rk;
                auk = (float)(cam.c * ukx + cam.d * uky); avk = (float)(cam.e * ukx + uky);      // A X_k
            }
            // the tier-1 constants go to the context as well: they are needed in pass 1 of every pattern only, and re-reading them
            // there (four broadcast LDS.128) keeps 15 registers free across pass 2 and the rare-path calls
            if (lane == 0) {
                float4* tp = reinterpret_cast<float4*>(cx.t1);
                tp[0] = make_float4(q[0], q[1], q[2], q[3]); tp[1] = make_float4(q[4], q[5], q[6], q[7]);
                tp[2] = make_float4(K0f, gkf, s0f, rk2f);    tp[3] = make_float4(rkf, auk, avk, 0.f);
            }
        }
        __syncwarp();                             // context complete
#pragma unroll 1                         // one copy of the pattern body: the kernel has to fit the instruction cache
        for (int qi = 0; qi < npat; ++qi) {
            bool done = false;
            float2* park = s_park_dyn + wib * (PPL * 32);
            if (t1) {
                // ---- tier 1: fp32, relative to the keypoint (see the header) ----
                // rotation folded into per-pattern constants (double -> float once): with p the pattern point and d = Rot p,
                //   n = r^2 - r_k^2 = |p|^2 + 2 (Rot^T X_k).p            (|d| = |p|: no rotated point needed for n)
                //   u - u_k = g (A Rot p).x + dg (A X_k).x               (A = affine part [c d; e 1])
                float nx, ny, axx, axy, ayx, ayy;
                {
                    const double caq = cx.ca[qi], saq = cx.sa[qi], ukx = cx.ukx, uky = cx.uky;
                    nx = (float)(2.0 * (ukx * caq + uky * saq)); ny = (float)(2.0 * (uky * caq - ukx * saq));
                    axx = (float)(cam.c * caq + cam.d * saq); axy = (float)(cam.d * caq - cam.c * saq);
                    ayx = (float)(cam.e * caq + saq); ayy = (float)(caq - cam.e * saq);
                }
                float su = 0.f, sv = 0.f;
                {
                const float4* tp = reinterpret_cast<const float4*>(cx.t1);
                const float4 tA = tp[0], tB = tp[1], tC = tp[2], tD = tp[3];
                const float q[kT1MCoef] = {tA.x, tA.y, tA.z, tA.w, tB.x, tB.y, tB.z, tB.w};
                const float K0f = tC.x, gkf = tC.y, s0f = tC.z, rk2f = tC.w, rkf = tD.x, auk = tD.y, avk = tD.z;
                if (mform) {
#pragma unroll kT1Unroll1
                    for (int j = 0; j < PPL; ++j) {
                        const float2 pp = s_patf[j * 32 + lane];
                        const float n = fmaf(pp.x, nx, fmaf(pp.y, ny, fmaf(pp.x, pp.x, pp.y * pp.y)));   // m - m_k
                        const float t = fmaf(n, rk2f, s0f);                       // (m - c_i) / hw_i
                        float pl = q[kT1MCoef - 1];
#pragma unroll
                        for (int k = kT1MCoef - 2; k >= 0; --k) pl = fmaf(pl, t, q[k]);
                        const float dg = fmaf(t, pl, -K0f);                        // g(r) - g(r_k)
                        const float g = gkf + dg;
                        const float du = fmaf(g, fmaf(pp.x, axx, pp.y * axy), dg * auk);   // u - u_k
                        const float dv = fmaf(g, fmaf(pp.x, ayx, pp.y * ayy), dg * avk);   // v - v_k
                        park[j * 32 + lane] = make_float2(du, dv);
                        if (lane_valid) { su += du; sv += dv; }
                    }
                } else
#pragma unroll 4
                for (int j = 0; j < PPL; ++j) {
                    const float2 pp = s_patf[j * 32 + lane];
                    const float n = fmaf(pp.x, nx, fmaf(pp.y, ny, fmaf(pp.x, pp.x, pp.y * pp.y)));
                    const float r2 = rk2f + n;
                    float y, z;
                    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(r2));   // MUFU + one Newton step each: ~1 ulp
                    y = fmaf(0.5f * y, fmaf(-r2 * y, y, 1.f), y);              // 1 / r
                    const float w = fmaf(r2, y, rkf);                          // r + r_k
                    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(z) : "f"(w));
                    z = fmaf(z, fmaf(-w, z, 1.f), z);
                    const float delta = n * z;                                 // r - r_k without cancellation
                    const float sp = fmaf(delta, 1.f / kT1Scale, s0f);
                    float pl = q[5];
                    pl = fmaf(pl, sp, q[4]); pl = fmaf(pl, sp, q[3]); pl = fmaf(pl, sp, q[2]);
                    pl = fmaf(pl, sp, q[1]); pl = fmaf(pl, sp, q[0]);
                    const float dg = fmaf(sp, pl, -K0f) * y;                   // g(r) - g(r_k)
                    const float g = gkf + dg;
                    const float du = fmaf(g, fmaf(pp.x, axx, pp.y * axy), dg * auk);   // u - u_k
                    const float dv = fmaf(g, fmaf(pp.x, ayx, pp.y * ayy), dg * avk);   // v - v_k
                    park[j * 32 + lane] = make_float2(du, dv);
                    if (lane_valid) { su += du; sv += dv; }
                }
                }
                // mean over the 16*ds points: lane partial sums in fp32 (16..32 terms)
                const double inv_n = 1.0 / (double)(16 * ds);
                bool flag = false;
#if MCS_K3_V3
                // ... and the warp sum as ONE integer REDUX per coordinate in 2^-17 px fixed point: a lane's rounding is <= 3.8e-6 px,
                // the mean is off by <= 32 * 3.8e-6 / 512 = 2.4e-7 px (inside the tier-1 error budget, kT1Guard).  A lane sum of 500 px
                // or more (or a NaN) cannot come from a sane pattern (|du| <= ~22 px) and sends the pattern on, so the 32-bit sum
                // (< 32 * 500 * 2^17 = 2^31) never wraps.
                flag = !(fabsf(su) < 500.f) | !(fabsf(sv) < 500.f);
                const int iu = __reduce_add_sync(0xffffffffu, flag ? 0 : __float2int_rn(su * 131072.f));
                const int iv = __reduce_add_sync(0xffffffffu, flag ? 0 : __float2int_rn(sv * 131072.f));
                const float mu = (float)((double)iu * (inv_n * (1.0 / 131072.0))), mv = (float)((double)iv * (inv_n * (1.0 / 131072.0)));
                float wf = 0.f, wt = 0.f;                                      // running maxima of |fraction - tie| and |offset|
#else
                double sud = (double)su, svd = (double)sv;
#pragma unroll
                for (int o = 16; o; o >>= 1) {
                    sud += __shfl_xor_sync(0xffffffffu, sud, o);
                    svd += __shfl_xor_sync(0xffffffffu, svd, o);
                }
                const float mu = (float)(sud * inv_n), mv = (float)(svd * inv_n);
#endif
                constexpr float kMagicF = 12582912.f;                          // 1.5 * 2^23: t + magic rounds t to the nearest even integer
                unsigned bits = 0;                                             // descriptor byte(s) of this lane: points 0..15 | 16..31 << 8
#pragma unroll kT1Unroll2
                for (int j = 0; j < PPL; j += 2) {
                    int smp[2];
#pragma unroll
                    for (int e2 = 0; e2 < 2; ++e2) {
                        const float2 c = park[(j + e2) * 32 + lane];           // this lane's own slot: no synchronisation needed
                        const float tu = c.x - mu, tv = c.y - mv;
                        const float mu_r = tu + kMagicF, mv_r = tv + kMagicF;
                        const float fu = tu - (mu_r - kMagicF), fv = tv - (mv_r - kMagicF);
                        // near a rounding tie, or outside the staged patch
#if MCS_K3_V3
                        // (running maxima, tested once after the loop; a NaN coordinate has already flagged the pattern through its lane sum)
                        wf = fmaxf(wf, fmaxf(fabsf(fu), fabsf(fv)));
                        wt = fmaxf(wt, fmaxf(fabsf(tu), fabsf(tv)));
#else
                        // (the comparisons are written so that a NaN flags too)
                        flag |= !(fabsf(fu) < 0.5f - kT1Guard) | !(fabsf(fv) < 0.5f - kT1Guard) | !(fabsf(tu) < (float)kPatchR + 0.4f) |
                                !(fabsf(tv) < (float)kPatchR + 0.4f);
#endif
                        const int ix = __float_as_int(mu_r) - 0x4B400000, iy = __float_as_int(mv_r) - 0x4B400000;
                        // one clamp of the byte offset keeps the read inside the patch array; an offset that needed it belongs to a
                        // flagged coordinate (|t| >= 25.4) and the pattern is redone
                        const int ofs = min(max(iy * kPatchS + ix, -(kPatchR * kPatchS + kPatchR)), kPatchR * kPatchS + kPatchR);
                        smp[e2] = patch[pofs + ofs];
                    }
                    bits |= (unsigned)(smp[0] < smp[1]) << (j >> 1);          // point pair j/2: bits 0..7 = byte 0, 8..15 = byte 1
                }
#if MCS_K3_V3
                flag |= !(wf < 0.5f - kT1Guard) | !(wt < (float)kPatchR + 0.4f);
#endif
                if (!__any_sync(0xffffffffu, flag && lane_valid)) {
                    put(qi, bits);
                    done = true;
                    if (args.tier_stats && lane == 0) atomicAdd(args.tier_stats, 1ull);
                } else if (MCS_K3_REPAIR) {
                    int fail = 0;
                    const unsigned e = tier1_repair<PPL>(&cam, s_patf, park, cx.row, cx.ca[qi], cx.sa[qi], cx.ukx, cx.uky, lane, ds, patch, pofs, &fail);
                    if (!__any_sync(0xffffffffu, fail != 0)) {
                        put(qi, e);
                        done = true;
                        if (args.tier_stats && lane == 0) atomicAdd(args.tier_stats + 1, 1ull);
                    }
                }
            }
            if (!done) {
                // ---- tier 2 (FP64 polynomial), then tier 3 (exact) where tier 2 cannot decide ----
                unsigned e = 0;
                int need_exact = have_lut ? 0 : 1;
                if (have_lut) e = tier2_pattern<PPL>(&cam, s_patf, cx.row, cx.ca[qi], cx.sa[qi], cx.ukx, cx.uky, lane, ds, patch, pofs, &need_exact);
                const bool exact = __any_sync(0xffffffffu, need_exact != 0);
                if (exact) {
                    const double rot = 20.0 / (180.0 / 3.1415926535897932384626433832795);      // 20 / RHOd         (ref :424)
                    const double aq = qi == 0 ? cx.a_base : (qi == 1 ? cx.a_base + rot : cx.a_base - rot);
                    const int lv = cx.level, bq = cx.b;
                    const LevelGeom& gq = geom->lv[lv];
                    e = exact_pattern<PPL>(&cam, s_patf, aq, cx.ukx, cx.uky, lane, ds, args.blur[lv] + (size_t)bq * gq.img_bytes,
                                           args.lvl[lv] + (size_t)bq * gq.img_bytes, &gq, cx.kx, cx.ky);
                }
                if (args.tier_stats && lane == 0) atomicAdd(args.tier_stats + (exact ? 3 : 2), 1ull);
                put(qi, e);
            }
        }
    }
    {
        const int bo = cx.b, oo = cx.oidx;
#pragma unroll
        for (int bb = 0; bb < BPL; ++bb) {
            const int byte = lane + 32 * bb;
            if (byte < ds) {
                desc_out[((size_t)bo * capacity + oo) * ds + byte] = (uint8_t)v0[bb];
                // stable bit <=> both +-20 degree re-tests agree with the bit (ref :449-451 ...)
                if (dmask_out) dmask_out[((size_t)bo * capacity + oo) * ds + byte] = (uint8_t)(masks ? (~vdiff[bb] & 0xFFu) : 0u);
            }
        }
        if (lane == 0) {
            const int lv = cx.level, kxo = cx.kx, kyo = cx.ky;
            const LevelGeom& go = geom->lv[lv];
            const float scale = go.scale;
            mcs_keypoint k;
            k.x = lv ? __fmul_rn((float)kxo, scale) : (float)kxo;      // pt *= scale for l > 0 (ref :1327-1332)
            k.y = lv ? __fmul_rn((float)kyo, scale) : (float)kyo;
            k.size = go.patch_size; k.angle = cx.angle; k.response = (float)corner_s(cx.c);
            k.octave = lv; k.class_id = -1;
            kps_out[(size_t)bo * capacity + oo] = k;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
cudaError_t upload_constants(const signed char* pairs, const signed char* du, const signed char* dv) {
    cudaError_t e = cudaMemcpyToSymbol(c_pairs, pairs, 2048);
    if (e != cudaSuccess) return e;
    {
        std::vector<float2> pf(1024);
        for (int i = 0; i < 1024; ++i) {
            const int j = i >> 5, ln = i & 31, byte = ln + 32 * (j >> 4), pt = 16 * byte + (j & 15);
            pf[i] = make_float2((float)pairs[2 * pt], (float)pairs[2 * pt + 1]);
        }
        e = cudaMemcpyToSymbol(g_patf, pf.data(), sizeof(float2) * 1024);
        if (e != cudaSuccess) return e;
    }
    e = cudaMemcpyToSymbol(c_disc_u, du, 848);
    if (e != cudaSuccess) return e;
    return cudaMemcpyToSymbol(c_disc_v, dv, 848);
}

// Tabulate R(r) = rho(atan(-z/r)) on [0, n) px in unit intervals: 6 monomial coefficients in
// tau = 2 (r - idx) - 1, interpolating R at the 6 Chebyshev nodes of the interval, all in long double.
void build_distort_lut(const mcs_ocam& cam, std::vector<double>& coef, int& n_out) {
    // table extent: largest undistorted radius of any pixel the mirror mask keeps, plus the pattern reach
    const double scaleF = cam.pol[0];
    double rmax = 64.0;
    const double mcx = cam.u0, mcy = cam.v0, mrad = cam.v0 + 22.0;
    for (int y = 0; y < cam.height; y += 4)
        for (int x = 0; x < cam.width; x += 4) {
            if (cam.mirror_mask == 1 && std::hypot(x - mcx, y - mcy) > mrad + 4.0) continue;
            double wx, wy, wz;
            cam_img_to_world(cam, (double)x, (double)y, wx, wy, wz);
            if (!(wz * scaleF < 0.0)) continue;            // behind / on the undistortion plane: no finite image
            const double ux = -wx / wz * scaleF, uy = -wy / wz * scaleF;
            const double r = std::hypot(ux, uy);
            if (std::isfinite(r) && r > rmax) rmax = r;
        }
    int n = (int)std::min(8192.0, std::ceil(rmax + 64.0));
    n_out = n;
    coef.assign((size_t)n * kLutStride, 0.0);
    const long double z = -(long double)cam.pol[0];
    auto R_exact = [&](long double r) {
        const long double theta = atanl(-z / r);
        long double rho = 0.0L;
        for (int t = 11; t >= 0; --t) rho = rho * theta + (long double)cam.inv_pol[t];
        return rho;
    };
    constexpr int NC = kLutDeg + 1;
    long double nodes[NC];
    for (int k = 0; k < NC; ++k) nodes[k] = cosl((2 * k + 1) * 3.14159265358979323846264338327950288L / (2.0L * NC));
    for (int i = 0; i < n; ++i) {
        // centre i serves keypoints with rn(rk) == i: their pattern points lie in [i - 21.8, i + 21.8] and r >= 0
        const long double lo = std::max(0.0L, (long double)i - (long double)kLutReach), hi = (long double)i + (long double)kLutReach;
        const long double m = 0.5L * (lo + hi), hw = 0.5L * (hi - lo);
        long double A[NC][NC + 1];
        for (int k = 0; k < NC; ++k) {
            long double pw = 1.0L;
            for (int t = 0; t < NC; ++t) { A[k][t] = pw; pw *= nodes[k]; }
            A[k][NC] = R_exact(m + hw * nodes[k]);
        }
        for (int col = 0; col < NC; ++col) {          // Gauss-Jordan with partial pivoting
            int piv = col;
            for (int r2 = col + 1; r2 < NC; ++r2) if (fabsl(A[r2][col]) > fabsl(A[piv][col])) piv = r2;
            for (int t = 0; t <= NC; ++t) std::swap(A[col][t], A[piv][t]);
            for (int r2 = 0; r2 < NC; ++r2) {
                if (r2 == col) continue;
                const long double f = A[r2][col] / A[col][col];
                for (int t = col; t <= NC; ++t) A[r2][t] -= f * A[col][t];
            }
        }
        double* e = coef.data() + (size_t)i * kLutStride;
        const double scale = (double)(1.0L / hw);
        e[0] = (double)(-m / hw); e[1] = scale;
        for (int t = 0; t < NC; ++t) e[2 + t] = (double)(A[t][NC] / A[t][t]);
        // check the fit as the kernel evaluates it (double Horner); a centre whose error could move a rounding
        // decision past the kernel's 5e-7 px tie guard is disabled (NaN coefficients -> exact path)
        double worst = 0.0;
        for (int sidx = 0; sidx <= 96; ++sidx) {
            const double r = (double)(lo + (hi - lo) * ((long double)sidx + 0.37L) / 97.0L);
            const double tau = std::fma(r, e[1], e[0]);
            double gv = e[2 + kLutDeg];
            for (int t = kLutDeg - 1; t >= 0; --t) gv = std::fma(gv, tau, e[2 + t]);
            worst = std::max(worst, (double)fabsl((long double)gv - R_exact((long double)r)));
        }
        if (!(worst < 2e-8))
            for (int t = 0; t < 12; ++t) e[t] = std::nan("");
        // ---- tier-1 entry: R(i + s) - R(i) = s' q(s'), s' = s / kT1Scale, q of degree kT1Coef - 1 interpolating at an even
        // number of Chebyshev nodes of [-reach, reach] (no node at s = 0); enabled where the whole window keeps clear of r = 0
        e[17] = 0.0;
        if ((double)i >= kT1MinRadius - 1.0 && worst < 2e-8) {
            constexpr int NQ = kT1Coef;
            const long double Ri = R_exact((long double)i);
            long double B[NQ][NQ + 1];
            for (int k = 0; k < NQ; ++k) {
                const long double sn = (long double)kLutReach * cosl((2 * k + 1) * 3.14159265358979323846264338327950288L / (2.0L * NQ));
                const long double sp = sn / (long double)kT1Scale;
                long double pw = 1.0L;
                for (int t = 0; t < NQ; ++t) { B[k][t] = pw; pw *= sp; }
                B[k][NQ] = (R_exact((long double)i + sn) - Ri) / sp;
            }
            for (int col = 0; col < NQ; ++col) {
                int piv = col;
                for (int r2 = col + 1; r2 < NQ; ++r2) if (fabsl(B[r2][col]) > fabsl(B[piv][col])) piv = r2;
                for (int t = 0; t <= NQ; ++t) std::swap(B[col][t], B[piv][t]);
                for (int r2 = 0; r2 < NQ; ++r2) {
                    if (r2 == col) continue;
                    const long double f = B[r2][col] / B[col][col];
                    for (int t = col; t <= NQ; ++t) B[r2][t] -= f * B[col][t];
                }
            }
            float qf[NQ + 1] = {0};
            for (int t = 1; t < NQ; ++t) qf[t] = (float)(B[t][NQ] / B[t][t]);
            const double q0 = (double)(B[0][NQ] / B[0][0]);
            // fit error with the coefficients as the kernel holds them (q0 double, q1.. float), evaluated in long double
            long double werr = 0.0L;
            for (int sidx = 0; sidx <= 64; ++sidx) {
                const long double sv = -(long double)kLutReach + 2.0L * (long double)kLutReach * ((long double)sidx + 0.37L) / 65.0L;
                const long double sp = sv / (long double)kT1Scale;
                long double pv = (long double)qf[NQ - 1];
                for (int t = NQ - 2; t >= 1; --t) pv = pv * sp + (long double)qf[t];
                pv = pv * sp + (long double)q0;
                werr = std::max(werr, fabsl(sp * pv - (R_exact((long double)i + sv) - Ri)));
            }
            // Accepted up to 1e-6 px: with the 5e-6 px of fp32 evaluation noise that is still 4x inside kT1Guard, and the repair path
            // (whose mean inherits this systematic part) keeps kT1RepairGuard = 4e-6 > 1e-6 + 1.5e-7.  Centres 40..69 of the Lafida
            // cameras land between 2e-7 and 1e-6; everything farther out is below 1e-7.
            if (werr < 1e-6L) {
                e[12] = (double)Ri; e[13] = q0;
                std::memcpy(&e[14], &qf[1], sizeof(float) * 6);      // q1..q5 + one zero pad float
                e[17] = 1.0;
            }
        }
        // ---- m-form entry of tier 1: G(m) = R(sqrt(m)) / sqrt(m) on the centre's window in m = r^2, G(c + hw t) - G(c) = t P(t) with P
        // of degree kT1MCoef - 1 interpolating at an even number of Chebyshev nodes of [-1, 1] (no node at t = 0).  What the fit error
        // multiplies is the keypoint's own image offset |A X_k| ~ r_k, so it is accepted below 1e-6 px in those terms -- the same bound
        // the s-form entry is held to.
        e[23] = 0.0;
        if (e[17] == 1.0 && (double)i > kLutReach + 1.0) {
            constexpr int NM = kT1MCoef;
            const long double cm = (long double)t1m_centre(i), hm = (long double)t1m_halfwidth(i);
            auto G_exact = [&](long double m) { const long double r = sqrtl(m); return R_exact(r) / r; };
            const long double Gc = G_exact(cm);
            long double B[NM][NM + 1];
            for (int k = 0; k < NM; ++k) {
                const long double tn = cosl((2 * k + 1) * 3.14159265358979323846264338327950288L / (2.0L * NM));
                long double pw = 1.0L;
                for (int t = 0; t < NM; ++t) { B[k][t] = pw; pw *= tn; }
                B[k][NM] = (G_exact(cm + hm * tn) - Gc) / tn;
            }
            for (int col = 0; col < NM; ++col) {
                int piv = col;
                for (int r2 = col + 1; r2 < NM; ++r2) if (fabsl(B[r2][col]) > fabsl(B[piv][col])) piv = r2;
                for (int t = 0; t <= NM; ++t) std::swap(B[col][t], B[piv][t]);
                for (int r2 = 0; r2 < NM; ++r2) {
                    if (r2 == col) continue;
                    const long double f = B[r2][col] / B[col][col];
                    for (int t = col; t <= NM; ++t) B[r2][t] -= f * B[col][t];
                }
            }
            float af[NM];
            for (int t = 0; t < NM; ++t) af[t] = (float)(B[t][NM] / B[t][t]);
            long double werr = 0.0L;
            for (int sidx = 0; sidx <= 96; ++sidx) {
                const long double tv = -1.0L + 2.0L * ((long double)sidx + 0.37L) / 97.0L;
                long double pv = (long double)af[NM - 1];
                for (int t = NM - 2; t >= 0; --t) pv = pv * tv + (long double)af[t];
                werr = std::max(werr, fabsl(tv * pv - (G_exact(cm + hm * tv) - Gc)));
            }
            if (werr * ((long double)i + 1.0L) < 1e-6L) {
                e[18] = (double)Gc;
                std::memcpy(&e[19], af, sizeof(float) * NM);
                e[23] = 1.0;
            }
        }
    }
}

cudaError_t launch_describe(const PyramidGeom& G, const PyramidGeom* G_dev, int n_images, const DescribeArgs& args,
                            const mcs_ocam* cams, const DistortLut* luts, const int* cam_of_image, const uint32_t* sel_xys,
                            const int* sel_count, mcs_keypoint* kps, uint8_t* desc, uint8_t* dmask, int* counts, int capacity,
                            cudaStream_t st) {
    const long long warps = (long long)n_images * G.sel_total;
    const int blocks = (int)std::max<long long>(1, (warps + kDescWarps - 1) / kDescWarps);
    // 96 registers, 5 CTAs of 4 warps per SM (MCS_K3_MINB, measured against 4 and 6 there); the warp context in shared memory keeps
    // the hot-loop invariants out of the spilled set
    const size_t park16 = (size_t)kDescWarps * 16 * 32 * sizeof(float2), park32 = 2 * park16;
    if (G.desc_size > 32) {        // static 23 KB + 32 KB parked coordinates: above the 48 KB default
        cudaError_t e = cudaFuncSetAttribute(describe_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)park32);
        if (e != cudaSuccess) return e;
    }
    if (G.desc_size <= 32)
        describe_kernel<16><<<blocks, kDescWarps * 32, park16, st>>>(G_dev, args, cams, luts, cam_of_image, sel_xys, sel_count, kps, desc,
                                                               dmask, counts, capacity, n_images);
    else
        describe_kernel<32><<<blocks, kDescWarps * 32, park32, st>>>(G_dev, args, cams, luts, cam_of_image, sel_xys, sel_count, kps, desc,
                                                               dmask, counts, capacity, n_images);
    return cudaGetLastError();
}

}  // namespace mcs
