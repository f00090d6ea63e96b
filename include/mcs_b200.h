/*
 * mcs_b200.h -- C ABI of the H100-native (sm_90a) MultiCol-SLAM feature hot path.
 *
 * One shared library (libmcs_b200.so) replaces the arithmetic behind
 *   mdBRIEFextractorOct::operator()            (ref include/mdBRIEFextractorOct.h:355-361,
 *                                               src/mdBRIEFextractorOct.cpp:1244-1337)
 *   cORBmatcher::SearchByProjection(F, MPs)    (ref src/cORBmatcher.cpp:67-166)
 *   cORBmatcher::SearchForInitialization       (ref src/cORBmatcher.cpp:579-726)
 *   cORBmatcher::SearchByBoW(KF, KF)           (ref src/cORBmatcher.cpp:885-966, all-pairs)
 *   DescriptorDistance64[Masked]               (ref src/cORBmatcher.cpp:2438-2474)
 *   cCamModelGeneral_::WorldToImg / ImgToWorld (ref src/cam_model_omni.cpp:49-67,146-161)
 *   CreateMirrorMask level 0                   (ref src/cam_model_omni.cpp:181-220)
 *
 * Plain pointers and sizes only; no C++/torch/OpenCV types cross this boundary.
 * Every function returns an int status (MCS_OK == 0) and never throws.
 * The C++ classes in include/mcs_shim.hpp adapt these entry points to the
 * reference's own class signatures (see INTEGRATION.md).
 *
 * Pointers named *_dev are CUDA device pointers on the extractor's device;
 * everything else is host memory owned by the caller.
 */
#ifndef MCS_B200_H
#define MCS_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MCS_OK                0
#define MCS_ERR_INVALID      -1   /* bad argument (null pointer, size, ...)            */
#define MCS_ERR_UNSUPPORTED  -2   /* option of the reference that is not built (AGAST) */
#define MCS_ERR_CUDA         -3   /* CUDA runtime error; see mcs_last_error()          */
#define MCS_ERR_CAPACITY     -4   /* caller buffer too small                           */
#define MCS_ERR_NO_DEVICE    -5   /* no usable sm_90 (H100) device: there is NO CPU fallback */

#define MCS_MAX_LEVELS       16
#define MCS_FRAME_GRID_COLS  64   /* ref include/cMultiFrame.h:48 */
#define MCS_FRAME_GRID_ROWS  48   /* ref include/cMultiFrame.h:47 */

/* Scaramuzza/OCam interior orientation, the 17 doubles of cCamModelGeneral_
 * (ref include/cam_model_omni.h:47-110; YAML keys Camera.{c,d,e,u0,v0,a0..a4,pol0..pol11,Iw,Ih},
 * loaded zero-padded to 5 / 12 coefficients by src/cSystem.cpp:144-156). */
typedef struct mcs_ocam {
    double c, d, e, u0, v0;
    double pol[5];        /* forward polynomial  f(rho),   p_deg    == 5  */
    double inv_pol[12];   /* backward polynomial rho(theta), invP_deg == 12 */
    int32_t width, height;
    int32_t mirror_mask;  /* Camera.mirrorMask: 1 -> disc mask, 0 -> all ones */
    int32_t _pad;
} mcs_ocam;

/* Constructor arguments of mdBRIEFextractorOct, same order and defaults
 * (ref include/mdBRIEFextractorOct.h:340-352). */
typedef struct mcs_extractor_params {
    int32_t nfeatures;        /* 1000 */
    float   scale_factor;     /* 1.2f (kept as float: the reference widens the float) */
    int32_t nlevels;          /* 8 */
    int32_t edge_threshold;   /* 25 (the reference hard-codes EDGE_THRESHOLD = 25) */
    int32_t first_level;      /* 0, unused by the reference */
    int32_t score_type;       /* parsed, ignored by the reference (FAST score always) */
    int32_t patch_size;       /* 32, unused (PATCH_SIZE constant) */
    int32_t fast_threshold;   /* 20 */
    int32_t use_agast;        /* 0; 1 -> MCS_ERR_UNSUPPORTED */
    int32_t fast_agast_type;  /* 2 == FastFeatureDetector::TYPE_9_16 (only type built) */
    int32_t do_dbrief;        /* 0: ORB, 1: distorted BRIEF */
    int32_t learn_masks;      /* 1: mdBRIEF (descriptor + stability mask) */
    int32_t desc_size;        /* bytes: 16 / 32 / 64 */
} mcs_extractor_params;

/* Binary-compatible with cv::KeyPoint (28 bytes). */
typedef struct mcs_keypoint {
    float   x, y;
    float   size;
    float   angle;
    float   response;
    int32_t octave;
    int32_t class_id;
} mcs_keypoint;

typedef struct mcs_extractor_info {
    int32_t nlevels;
    int32_t capacity;                       /* sum over the levels of max(features_per_level + 2, 16): max keypoints per image */
    int32_t desc_size;
    int32_t features_per_level[MCS_MAX_LEVELS];
    double  scale_factor[MCS_MAX_LEVELS];
    double  inv_scale_factor[MCS_MAX_LEVELS];
} mcs_extractor_info;

typedef struct mcs_extractor mcs_extractor;   /* opaque; one per (camera, thread), not re-entrant */

const char* mcs_last_error(void);             /* thread-local message of the last failure */
int  mcs_device_count(void);                  /* number of visible sm_90 (H100) devices (0 -> none) */
void mcs_params_default(mcs_extractor_params* p);

/* ---- camera model (C1) ------------------------------------------------------------------- */
/* Host-side scalar helpers with the reference's exact double arithmetic; callers (cMultiFrame
 * bearing rays, projection front-ends) use them per point.  The device copies live inside the
 * descriptor kernel. */
void mcs_cam_world_to_img(const mcs_ocam* cam, double x, double y, double z, double* u, double* v);
void mcs_cam_img_to_world(const mcs_ocam* cam, double u, double v, double* x, double* y, double* z);
/* level-0 mirror mask, h*w bytes, 255 inside the disc / 0 outside (or all 1 when mirror_mask==0) */
int  mcs_cam_mirror_mask(const mcs_ocam* cam, uint8_t* mask_out);

/* ---- extractor (E0..E9) ------------------------------------------------------------------ */
int  mcs_extractor_create(const mcs_extractor_params* p, mcs_extractor** out);
void mcs_extractor_destroy(mcs_extractor* ex);
int  mcs_extractor_get_info(const mcs_extractor* ex, mcs_extractor_info* info);

/* The octree sizes of width x height images, as the host plans them (no GPU needed).  DistributeOctTree's first pass divides
 * each of its nIni = cvRound(level width / level height) roots whatever the level's quota, so a level returns up to
 * max(4 nIni, quota + 2) keypoints.  Out: *node_table (K2's nodes per image and level), nodes_ini[l] and sel_cap[l] (selected
 * keypoint slots) per level, *capacity (mcs_extractor_info.capacity).  Returns MCS_OK, or the refusal every extract call makes
 * for that geometry before any launch: MCS_ERR_UNSUPPORTED where the levels' max(4 nIni, quota + 2) sum above the capacity. */
int  mcs_extractor_octree_plan(const mcs_extractor_params* p, int32_t width, int32_t height, int32_t* node_table,
                               int32_t* nodes_ini, int32_t* sel_cap, int32_t* capacity);

/* operator() for one image.  Host buffers, synchronous.
 *   mask: h x w bytes, mandatory (the reference throws on an empty mask);
 *   kps_out[capacity], desc_out[capacity*desc_size], dmask_out[capacity*desc_size] (may be NULL
 *   only when learn_masks==0; when given and learn_masks==0 it is zero-filled like the reference);
 *   *n_out = number of keypoints.  capacity must be >= info.capacity. */
int  mcs_extract(mcs_extractor* ex,
                 const uint8_t* image, int32_t width, int32_t height, int32_t stride,
                 const uint8_t* mask, int32_t mask_stride,
                 const mcs_ocam* cam,
                 mcs_keypoint* kps_out, uint8_t* desc_out, uint8_t* dmask_out,
                 int32_t capacity, int32_t* n_out);

/* Batched form: n_images images of identical size, image i seen by camera cam_of_image[i]
 * (index into cams[]/masks[]).  images: n_images*height*stride bytes; masks: n_cams*height*width.
 * Outputs are fixed-size slots of `capacity` entries per image.  Host buffers (pinned memory
 * recommended), H2D + kernels + D2H inside the call. */
int  mcs_extract_batch(mcs_extractor* ex, int32_t n_images,
                       const uint8_t* images, int32_t width, int32_t height, int32_t stride,
                       const uint8_t* masks, const mcs_ocam* cams, int32_t n_cams,
                       const int32_t* cam_of_image,
                       mcs_keypoint* kps_out, uint8_t* desc_out, uint8_t* dmask_out,
                       int32_t* counts_out, int32_t capacity);

/* Same, all image/output buffers resident in device memory; asynchronous on `stream`
 * (a cudaStream_t passed as void*; NULL = the extractor's own stream, then the call
 * synchronises before returning).  masks/cams/cam_of_image stay host pointers (tiny, cached
 * on the device by the extractor).  With a caller stream the capacity checks of the call (raw corner list, octree node table,
 * keypoint slots: MCS_ERR_CAPACITY) cannot be reported by the call itself: mcs_extractor_check_status does that afterwards. */
int  mcs_extract_batch_device(mcs_extractor* ex, int32_t n_images,
                              const uint8_t* images_dev, int32_t width, int32_t height, int32_t stride,
                              const uint8_t* masks, const mcs_ocam* cams, int32_t n_cams,
                              const int32_t* cam_of_image,
                              mcs_keypoint* kps_dev, uint8_t* desc_dev, uint8_t* dmask_dev,
                              int32_t* counts_dev, int32_t capacity, void* stream);

/* Stream form of the whole path: n_frames multi-camera frames (frame-major: image i = frame i/n_cams,
 * camera i%n_cams) are extracted, and every image is brute-force matched (bit-level Hamming, masked form when
 * learn_masks is set) against the same camera of the previous frame: K best (index, distance) per keypoint
 * slot, (-1, INT_MAX) where none / for frame 0.  match_idx/match_dist: [n_frames*n_cams*capacity*K].
 * Host buffers; H2D, all kernels and D2H happen inside the call. */
int  mcs_extract_match_stream(mcs_extractor* ex, int32_t n_frames, int32_t n_cams,
                              const uint8_t* images, int32_t width, int32_t height, int32_t stride,
                              const uint8_t* masks, const mcs_ocam* cams,
                              mcs_keypoint* kps_out, uint8_t* desc_out, uint8_t* dmask_out,
                              int32_t* counts_out, int32_t capacity,
                              int32_t K, int32_t* match_idx_out, int32_t* match_dist_out);

/* The stream call with two optional extras:
 *  - packed_dev (may be NULL): the features of the batch are also left in the caller's packed exchange buffer (device memory,
 *    mcs_packed_layout(n_frames*n_cams, capacity, descSize) bytes): K3 writes them there, the host copies are taken from there,
 *    and mcs_allgather_features can ship the buffer to the other GPUs of the rig right after the call;
 *  - matches12_out / nmatches_out / redo_out (all three or none): the greedy acceptance of SearchByBoW(KF1, KF2)
 *    (threshold th_low, ratio nnratio, every database keypoint used once; see mcs_match_stream_replay_device) evaluated on the
 *    device over each chunk's K-best lists; host arrays [n_images*capacity], [n_images], [n_images].  In this mode the lists
 *    returned in match_idx_out / match_dist_out hold only the entries that can influence the acceptance (distance below the
 *    relevance bound of mcs_match_stream_greedy_device); shorter lists are padded with (-1, INT_MAX). */
int  mcs_extract_match_stream_packed(mcs_extractor* ex, int32_t n_frames, int32_t n_cams,
                                     const uint8_t* images, int32_t width, int32_t height, int32_t stride,
                                     const uint8_t* masks, const mcs_ocam* cams,
                                     mcs_keypoint* kps_out, uint8_t* desc_out, uint8_t* dmask_out,
                                     int32_t* counts_out, int32_t capacity,
                                     int32_t K, int32_t* match_idx_out, int32_t* match_dist_out, void* packed_dev,
                                     int32_t th_low, double nnratio, int32_t* matches12_out, int32_t* nmatches_out, int32_t* redo_out);

/* Device-resident matching half of the stream form (descriptor slots as written by
 * mcs_extract_batch_device); asynchronous on `stream`. dmask_dev may be NULL (unmasked distance). */
int  mcs_match_stream_device(const uint8_t* desc_dev, const uint8_t* dmask_dev, const int32_t* counts_dev,
                             int32_t n_frames, int32_t n_cams, int32_t capacity, int32_t dim, int32_t K,
                             int32_t* match_idx_dev, int32_t* match_dist_dev, void* stream);

/* The greedy acceptance of SearchByBoW(KF1, KF2) (ref src/cORBmatcher.cpp:899-961: threshold, ratio test, every database
 * keypoint used once, queries in index order) over the K-best lists of mcs_match_stream_device, on the device and on the same
 * stream.  A query is decided from its list whenever the list provably contains the answer (two unmatched entries, or bounds
 * from the last list distance); otherwise the kernel rescans the previous image for that query, so the result equals the
 * reference's sequential loop for every K >= 1.  matches12_dev [n_images*capacity] = matched slot of the previous frame's image
 * or -1, nmatches_dev [n_images]; redo_dev [n_images] is always 0 (kept for callers that check it).  desc_dev / dmask_dev: the
 * descriptor slots the lists were computed from (dmask_dev NULL = unmasked). */
int  mcs_match_stream_replay_device(const int32_t* match_idx_dev, const int32_t* match_dist_dev, const int32_t* counts_dev,
                                    const uint8_t* desc_dev, const uint8_t* dmask_dev,
                                    int32_t n_frames, int32_t n_cams, int32_t capacity, int32_t dim, int32_t K, int32_t th_low, double nnratio,
                                    int32_t* matches12_dev, int32_t* nmatches_dev, int32_t* redo_dev, void* stream);

/* Both steps as one call -- the operation cLoopClosing / cTracking actually want from a brute-force match (SearchByBoW(KF1, KF2)'s
 * acceptance rule, ref src/cORBmatcher.cpp:885-966, of every image against the same camera's image one frame earlier): K-best
 * lists in scratch memory of the stream's pool, then the greedy replay.  Because th_low and nnratio are known to the list kernel
 * here, entries that cannot influence any decision (distance >= the smallest b with (th_low - 1) < nnratio * b) are left out of
 * the lists, so a list shorter than K proves that every relevant entry is in it and the replay rescans less often; the matches
 * are the same as mcs_match_stream_device + mcs_match_stream_replay_device give for any K. */
int  mcs_match_stream_greedy_device(const uint8_t* desc_dev, const uint8_t* dmask_dev, const int32_t* counts_dev,
                                    int32_t n_frames, int32_t n_cams, int32_t capacity, int32_t dim, int32_t th_low, double nnratio,
                                    int32_t* matches12_dev, int32_t* nmatches_dev, void* stream);

/* Per-stage device timings of the LAST extract call, measured with CUDA events on the launching stream when
 * profiling is enabled: ms[0] = K1 (pyramid+blur+FAST, all levels), ms[1] = K2 octree, ms[2] = K3 describe.
 * mcs_extractor_set_profiling(ex, 1) turns the event recording on (off by default). */
int  mcs_extractor_set_profiling(mcs_extractor* ex, int32_t enable);
int  mcs_extractor_get_timings(mcs_extractor* ex, float* ms3);

/* Diagnostics of the descriptor kernel (K3): the distorted patterns are evaluated by the cheapest of three tiers whose error
 * bound still decides every rounding of the reference (fp32 relative to the keypoint / FP64 polynomial / exact operation
 * sequence, multicol_slam_b200/csrc/describe_kernel.cu).  enable != 0 switches counting on for the following extract calls
 * (one atomic per pattern: not for timed runs); counts4 (may be NULL) receives the patterns decided since then by
 * [0] tier 1, [1] tier 1 after the FP64 repair of its near-tie points, [2] tier 2, [3] tier 3. */
int  mcs_extractor_tier_stats(mcs_extractor* ex, int32_t enable, int64_t* counts4);

/* Overflow report of the LAST asynchronous extract call (mcs_extract_batch_device / ..._packed_device on a caller stream):
 * synchronises `stream` (the stream that call ran on; NULL = the extractor's own) and returns MCS_ERR_CAPACITY if a raw corner
 * list, the octree node table or the keypoint slots were too small for some image (results are truncated then), MCS_OK otherwise. */
int  mcs_extractor_check_status(mcs_extractor* ex, void* stream);

/* The per-camera table behind tiers 1 and 2 of the descriptor kernel, as the host builds it (no GPU needed): one row of
 * *row_doubles doubles per integer radius i of the undistorted plane, R(r) = rho(atan(-z / r)) the radial distortion function of
 * cam (ref src/cam_model_omni.cpp:49-67):
 *   [0..1]  tau offset / scale and [2..11] the degree-9 polynomial of R on [i - 22.5, i + 22.5]            (tier 2; NaN = disabled)
 *   [12] R(i), [13] q0, [14..16] q1..q5 as floats: R(i + s) - R(i) = s' q(s'), s' = s / 32, [17] 1.0 = usable (tier 1, s-form)
 *   [18] G(c_i), [19..22] a0..a7 as floats: G(c_i + hw_i t) - G(c_i) = t P(t), G(m) = R(sqrt m) / sqrt m, c_i = i^2 + 22.5^2,
 *           hw_i = 45 i, [23] 1.0 = usable                                                                  (tier 1, m-form)
 * rows_out (may be NULL to query the sizes) receives min(*n_rows, max_rows) rows.  Exists so that the tables can be checked
 * against the camera model independently of the kernel (tests/test_distort_table_cpu.py). */
int  mcs_cam_distort_table(const mcs_ocam* cam, double* rows_out, int32_t max_rows, int32_t* n_rows, int32_t* row_doubles);

/* mcs_extract_batch / mcs_extract with at most 16 images (the per-frame call of cMultiFrame's constructor, ref
 * src/cMultiFrame.cpp:128-139) stage through pinned buffers owned by the extractor, and once a call repeats the previous one's
 * geometry, camera table, camera models and masks the whole copy-in / K1..K3 / copy-out sequence is ONE cudaGraphLaunch.
 * *n receives how many calls were served that way (diagnostics; tests assert the shortcut is taken and changes nothing). */
int  mcs_extractor_graph_replays(mcs_extractor* ex, int64_t* n);

/* Introspection for the parity tests: copy intermediate device buffers of the LAST extract call
 * (image 0 of the batch unless image_index is given) back to the host.
 *   what: 0 = unblurred level (w*h bytes), 1 = blurred level, 2 = mask level,
 *         3 = raw corners of the level as int32 triples (x, y, score) in reference order.
 *   *w_out,*h_out = level size (for what==3: *w_out = number of corners, *h_out = 3). */
int  mcs_extractor_debug_read(mcs_extractor* ex, int32_t image_index, int32_t level, int32_t what,
                              void* out, size_t out_bytes, int32_t* w_out, int32_t* h_out);

/* ---- Hamming distance (M0) --------------------------------------------------------------- */
int  mcs_descriptor_distance64(const uint64_t* a, const uint64_t* b, int32_t dim);
int  mcs_descriptor_distance64_masked(const uint64_t* a, const uint64_t* b,
                                      const uint64_t* mask_a, const uint64_t* mask_b, int32_t dim);

/* ---- brute force (M2 kernel) ------------------------------------------------------------- */
/* For every query q: the K smallest (distance, index) pairs over the nd database descriptors that
 * are not flagged in db_skip (nd bytes, may be NULL), ordered by (distance, index) ascending.
 * Distances are the reference's bit-level popcounts (masked form when qmask/dmask != NULL).
 * Output: topk_idx[nq*K] (-1 = none), topk_dist[nq*K] (0x7FFFFFFF = none).  Host buffers.  nd < 2^21 per call (MCS_ERR_UNSUPPORTED
 * beyond: split the database).  nd may be 0 (d must still be a valid address): every query then gets K "none" entries. */
int  mcs_hamming_topk(const uint8_t* q, const uint8_t* qmask, int32_t nq,
                      const uint8_t* d, const uint8_t* dmask, int32_t nd,
                      const uint8_t* db_skip, int32_t dim, int32_t K,
                      int32_t* topk_idx, int32_t* topk_dist);
int  mcs_hamming_topk_device(const uint8_t* q_dev, const uint8_t* qmask_dev, int32_t nq,
                             const uint8_t* d_dev, const uint8_t* dmask_dev, int32_t nd,
                             const uint8_t* db_skip_dev, int32_t dim, int32_t K,
                             int32_t* topk_idx_dev, int32_t* topk_dist_dev, void* stream);

/* cORBmatcher::SearchByBoW(KF1, KF2, matches12) semantics (ref :885-966): all-pairs scan,
 * best/second best, `best < th_low`, `best < nnratio*second`, every KF2 entry used at most once,
 * queries visited in index order.  valid1/valid2: 1 where the keypoint carries a good map point
 * (NULL = all valid).  matches12[nq] = matched database index or -1.  Returns via *nmatches.
 * nd <= 1 622 016 per call for this entry point and the two below (the acceptance kernel keeps one "used" bit per database
 * entry in shared memory); a larger database returns MCS_ERR_UNSUPPORTED without launching a kernel. */
int  mcs_match_bruteforce(const uint8_t* q, const uint8_t* qmask, const uint8_t* valid1, int32_t nq,
                          const uint8_t* d, const uint8_t* dmask, const uint8_t* valid2, int32_t nd,
                          int32_t dim, int32_t th_low, double nnratio,
                          int32_t* matches12, int32_t* nmatches);
/* Same with query and database descriptors (and masks) resident in device memory -- e.g. the descriptor section of a packed
 * feature buffer against a key-frame database that stays on the GPU; valid1 / valid2 / matches12 / nmatches are host memory.
 * Runs on `stream` and returns when the result is complete. */
int  mcs_match_bruteforce_device(const uint8_t* q_dev, const uint8_t* qmask_dev, const uint8_t* valid1, int32_t nq,
                                 const uint8_t* d_dev, const uint8_t* dmask_dev, const uint8_t* valid2, int32_t nd,
                                 int32_t dim, int32_t th_low, double nnratio, int32_t* matches12, int32_t* nmatches, void* stream);
/* Several query sets against ONE database in one call -- the batched key frames of the loop-closure path (BASELINE config 4:
 * every key frame of a batch against the key-frame database).  seg_start[0..n_seg] delimits the sets inside q_dev; each set is
 * matched exactly as a separate mcs_match_bruteforce_device call would match it (its own "database entry already used" state,
 * as between separate SearchByBoW(KF1, KF2) calls, ref src/cORBmatcher.cpp:885-966), but the K-best lists of all sets come from
 * one kernel launch.  matches12 [seg_start[n_seg]], nmatches [n_seg]. */
int  mcs_match_bruteforce_batch_device(const uint8_t* q_dev, const uint8_t* qmask_dev, const uint8_t* valid1,
                                       const int32_t* seg_start, int32_t n_seg,
                                       const uint8_t* d_dev, const uint8_t* dmask_dev, const uint8_t* valid2, int32_t nd,
                                       int32_t dim, int32_t th_low, double nnratio, int32_t* matches12, int32_t* nmatches, void* stream);

/* Diagnostics: K-best launches the last mcs_match_bruteforce[_batch][_device] call of this thread needed.  Always 1 since the
 * ordered acceptance runs on the device (queries whose list is used up are rescanned inside the replay kernel). */
int  mcs_last_bruteforce_rounds(void);


/* cORBmatcher::SearchForTriangulationRaw(KF1, KF2, ...) (ref src/cORBmatcher.cpp:968-1156): all-pairs scan, same camera only,
 * over the keypoints that carry NO map point (free1/free2 != 0); per query the candidates with distance <= th_low are
 * ordered by (distance, index), and the first one within cvRound(2*best) whose bearing rays satisfy the epipolar constraint
 * CheckDistEpipolarLine(ray1, ray2, E[cam][cam], epi_thresh) (ref src/misc.cpp:53-69) is matched; every KF2 keypoint is used
 * at most once, queries are visited in index order.  rays: [n*3] doubles; E: [n_cams*n_cams*9] row-major 3x3 (ComputeE).
 * matches12[n1] = KF2 index or -1. */
int  mcs_search_for_triangulation(const uint8_t* desc1, const uint8_t* mask1, const int32_t* cam1, const uint8_t* free1,
                                  const double* rays1, int32_t n1,
                                  const uint8_t* desc2, const uint8_t* mask2, const int32_t* cam2, const uint8_t* free2,
                                  const double* rays2, int32_t n2,
                                  int32_t dim, int32_t th_low, const double* E, int32_t n_cams, double epi_thresh,
                                  int32_t* matches12, int32_t* nmatches);

/* ---- multi-camera frame view + grid window search (G1, M1, M3) ---------------------------- */
/* Flat view of the fields of cMultiFrame the matchers read (ref include/cMultiFrame.h:90-175).
 * Keypoints are in the contiguous (camera-major) order of src/cMultiFrame.cpp:168-184. */
typedef struct mcs_frame_view {
    int32_t n_cams;
    int32_t n_keys;                 /* totalN */
    const mcs_keypoint* keys;       /* [n_keys] contiguous index order (mvKeys) */
    const int32_t* key_cam;         /* [n_keys] keypoint_to_cam */
    const uint8_t* desc;            /* [n_keys*dim] descriptor rows in contiguous index order */
    const uint8_t* dmask;           /* [n_keys*dim] or NULL */
    const int32_t* cam_width;       /* [n_cams] mnMaxX - mnMinX */
    const int32_t* cam_height;      /* [n_cams] */
    int32_t dim;                    /* descriptor bytes */
    int32_t n_levels;
    const double* scale_factors;    /* [n_levels] mvScaleFactors */
} mcs_frame_view;

/* Per-frame epilogue of the cMultiFrame constructor on the GPU (SURVEY 8f "next" row 3; ref src/cMultiFrame.cpp:143-184):
 * bearing rays camModel.ImgToWorld(pt) of every keypoint ([n_keys*3] doubles, bit-identical to the host evaluation: only
 * + - * / sqrt) and the 64x48 grid of PosInGrid (:342-353) as CSR over (cam, ix, iy): cell_start [n_cams*64*48 + 1],
 * cell_items [n_keys] (first *n_in_grid valid), ascending keypoint index inside a cell.  keys/key_cam as in mcs_frame_view
 * (cam_width/height are taken from cams[]).  Host buffers.  The window searches build their grid with the same kernel. */
int  mcs_frame_prepare(const mcs_keypoint* keys, const int32_t* key_cam, int32_t n_keys, const mcs_ocam* cams, int32_t n_cams,
                       double* rays_out, int32_t* cell_start_out, int32_t* cell_items_out, int32_t* n_in_grid);

/* One window query: GetFeaturesInArea(cam, x, y, r, min_level, max_level)
 * (ref src/cMultiFrame.cpp:272-340) followed by Hamming distance to every candidate. */
typedef struct mcs_window_query {
    int32_t cam;
    int32_t min_level, max_level;   /* -1,-1 = no level filter */
    int32_t desc_index;             /* row of the query descriptor in the query descriptor array */
    double  x, y, r;
} mcs_window_query;

/* Candidate lists in the reference's visiting order (cell-x outer, cell-y inner, insertion
 * order inside a cell).  cand_idx/cand_dist: [nq*max_cand]; cand_count[nq] holds the TRUE number
 * of candidates (may exceed max_cand: then only the first max_cand are stored and the call
 * returns MCS_ERR_CAPACITY so the caller can retry with a larger max_cand). */
int  mcs_window_search(const mcs_frame_view* frame,
                       const mcs_window_query* queries, int32_t nq,
                       const uint8_t* qdesc, const uint8_t* qmask,
                       int32_t max_cand,
                       int32_t* cand_idx, int32_t* cand_dist, int32_t* cand_count);

/* cORBmatcher::SearchByProjection(F, vpMapPoints, th) (ref :67-166).
 * Map points as parallel arrays: for map point i and camera c, entry i*n_cams+c.
 *   mp_bad[nmp]; in_view[nmp*n_cams]; level[..]; proj_x[..], proj_y[..]; view_cos[..];
 *   mp_desc[nmp*dim] (+ mp_dmask).
 * frame_mp[n_keys]: in/out, index of the map point assigned to each keypoint (-1 = none) --
 * the flat image of F.mvpMapPoints.  having_masks selects the masked distance. */
typedef struct mcs_mappoint_view {
    int32_t n_points;
    const uint8_t* bad;
    const uint8_t* in_view;
    const int32_t* level;
    const double*  proj_x;
    const double*  proj_y;
    const double*  view_cos;
    const uint8_t* desc;
    const uint8_t* dmask;
} mcs_mappoint_view;

int  mcs_search_by_projection(const mcs_frame_view* frame, const mcs_mappoint_view* mps,
                              double th, double nnratio, int32_t th_high, int32_t having_masks,
                              int32_t* frame_mp, int32_t* nmatches);

/* ---- projection front-end of SearchByProjection (SURVEY 8f "next" row 2) ------------------------ */
/* cMultiFrame::isInFrustum(cam, pMP, .) for every (map point, camera) (ref src/cMultiFrame.cpp:218-270) with
 * cMultiCamSys_::WorldToCamHom_fast (ref src/cam_system_omni.cpp:92-112) and isPointInMirrorMask
 * (ref src/cam_model_omni.cpp:163-178): fills exactly the arrays mcs_mappoint_view / mcs_search_by_projection consume.
 *   mtmc_inv, mtmc: [n_cams*16] row-major 4x4 (MtMc_inv[c] and Get_MtMc(c)); masks: n_cams level-0 mirror masks (h*w each);
 *   world_pos, normal: [n_points*3]; min_dist, max_dist: [n_points] (Get{Min,Max}DistanceInvariance);
 *   outputs indexed [point*n_cams + cam].  Host buffers.  Integer outputs (in_view, level) are exact; the projections go
 *   through atan(), so they agree with a CPU evaluation to ~1e-13 px. */
int  mcs_project_mappoints(int32_t n_cams, const double* mtmc_inv, const double* mtmc, const mcs_ocam* cams,
                           const uint8_t* masks, int32_t n_points, const double* world_pos, const double* normal,
                           const double* min_dist, const double* max_dist, const double* scale_factors, int32_t n_levels,
                           uint8_t* in_view, int32_t* level, double* proj_x, double* proj_y, double* view_cos);

/* ---- SearchReferencePointsInFrustum on the device (G1 / M1 without host round trips) ------------------------------------- */
/* Both calls are asynchronous on `stream` (a cudaStream_t as void*; NULL = the default stream, and the call synchronises before
 * returning).  With a stream given neither call waits for it.  Scratch comes from the stream-ordered memory pool.
 *
 * mcs_project_mappoints_device: mcs_project_mappoints with the map-point arrays and the outputs in device memory (the map points
 * stay resident across frames like the cMapPoint members).  mtmc_inv, mtmc, cams and scale_factors are host memory; masks_dev holds
 * the n_cams level-0 mirror masks.  skip_dev ([n_points] bytes, may be NULL): the outputs of a flagged point are left untouched --
 * the reference skips points already matched or bad (ref src/cTracking.cpp:985-988), and SearchByProjection then reads their
 * previous mbTrackInView.  Same kernel and arithmetic as mcs_project_mappoints; cameras of different sizes: MCS_ERR_UNSUPPORTED. */
int  mcs_project_mappoints_device(int32_t n_cams, const double* mtmc_inv, const double* mtmc, const mcs_ocam* cams,
                                  const uint8_t* masks_dev, int32_t n_points, const double* world_pos_dev, const double* normal_dev,
                                  const double* min_dist_dev, const double* max_dist_dev, const double* scale_factors, int32_t n_levels,
                                  const uint8_t* skip_dev, uint8_t* in_view_dev, int32_t* level_dev, double* proj_x_dev,
                                  double* proj_y_dev, double* view_cos_dev, void* stream);

/* mcs_mappoint_view with every pointer in device memory (the arrays mcs_project_mappoints_device fills, plus bad / desc / dmask). */
typedef struct mcs_mappoint_dev_view {
    int32_t n_points;
    const uint8_t* bad;             /* may be NULL: no point is bad */
    const uint8_t* in_view;
    const int32_t* level;
    const double*  proj_x;
    const double*  proj_y;
    const double*  view_cos;
    const uint8_t* desc;
    const uint8_t* dmask;
} mcs_mappoint_dev_view;

/* cORBmatcher::SearchByProjection(F, vpMapPoints, th) (ref :67-166) with the frame in packed feature buffers and every output on
 * the device; the result equals mcs_search_by_projection's.
 *   Frame: camera c is global image first_image + c of packed_dev, which holds n_parts consecutive packed layouts of
 *   part_images images each (mcs_packed_layout(part_images, capacity, dim) bytes apiece): n_parts = 1 is one extraction call's
 *   buffer, n_parts = world with part_images = 1 what mcs_allgather_features leaves for a one-camera-per-GPU rig.  The masks
 *   section is read when having_masks is set.  cam_width / cam_height [n_cams] (mnMaxX - mnMinX, ...) and scale_factors
 *   [n_levels] are host memory.
 *   frame_mp_dev [n_cams * capacity] in/out, indexed by slot c * capacity + j (keypoint j of camera c): -1 = free, accepted
 *   slots receive the map-point index; slots at or beyond a camera's count are ignored.
 *   nmatches_dev: number of acceptances.  status_dev: MCS_ERR_INVALID when an in-view entry of a non-bad point has a level
 *   outside [0, n_levels) -- that query is skipped, the others are unaffected -- MCS_OK otherwise.
 *   diag_dev (may be NULL): int32[4] = fixpoint rounds run, first query the sequential walk took over (-1 = none), queries,
 *   decisions that rescanned their window (DESIGN.md section 4).
 * capacity <= 65535, n_points * n_cams < 2^24. */
int  mcs_search_by_projection_device(const void* packed_dev, int32_t n_parts, int32_t part_images, int32_t first_image,
                                     int32_t n_cams, int32_t capacity, int32_t dim, const int32_t* cam_width, const int32_t* cam_height,
                                     int32_t n_levels, const double* scale_factors, const mcs_mappoint_dev_view* mps,
                                     double th, double nnratio, int32_t th_high, int32_t having_masks,
                                     int32_t* frame_mp_dev, int32_t* nmatches_dev, int32_t* status_dev, int32_t* diag_dev, void* stream);
/* The number of fixpoint rounds mcs_search_by_projection_device runs before the sequential walk finishes the rest. */
int  mcs_search_by_projection_max_rounds(void);

/* A frame in packed feature buffers: camera c is global image first_image + c of packed_dev, which holds n_parts consecutive
 * mcs_packed_layout(part_images, capacity, dim) layouts (see mcs_search_by_projection_device). */
typedef struct mcs_packed_frame {
    const void* packed_dev;
    int32_t n_parts, part_images, first_image;
} mcs_packed_frame;

/* cORBmatcher::SearchByProjection(CurrentFrame, LastFrame, th) (ref :1990-2118, TrackWithMotionModel) with both frames in packed
 * feature buffers and every output on the device.  Asynchronous like mcs_search_by_projection_device (same stream, scratch and
 * staging rules; nothing is read back).
 *   cur / last: the two frames, each in either packed layout; they may share one buffer.  cams [n_cams] host camera models (one
 *   image size for all); masks_dev [n_cams][height][width] their level-0 mirror masks; scale_factors [n_levels] host
 *   (CurrentFrame.mvScaleFactors); mtmc_inv [n_cams * 16] host, the CURRENT rig pose's MtMc_inv (row-major 4x4 per camera).
 *   last_mp_dev [n_cams * capacity]: the last frame's map-point ids by slot (-1 = none), in the frame_mp format of
 *   mcs_search_by_projection_device, so that call's output can be passed on unchanged.  last_outlier_dev (slot-indexed, may be
 *   NULL: no outliers).  world_pos_dev [n_points * 3] and bad_dev [n_points] (may be NULL) are the map points.
 *   For every last-frame keypoint in contiguous order (camera-major): skipped when it has no map point, the point is bad or the
 *   keypoint is an outlier; else the point is projected with WorldToCamHom_fast into the keypoint's own camera and, inside the
 *   mirror mask, searched in GetFeaturesInArea(cam, u, v, th * scale_factors[octave], octave - 1, octave + 1) of the current
 *   frame.  The best candidate not yet assigned (strict < over the visiting order, distance from the last frame's descriptor and
 *   mask) is accepted when its distance is <= th_high; cur_mp_dev receives the map-point id.  No ratio test, no rotation check.
 *   cur_mp_dev [n_cams * capacity] in/out, slot-indexed like frame_mp_dev; slots at or beyond a camera's count are neither read
 *   nor written, in either frame.  nmatches_dev: the acceptances of this call.  status_dev: MCS_ERR_INVALID when a map-point id
 *   is >= n_points or an octave of a query lies outside [0, n_levels) -- that query is dropped, the others are unaffected --
 *   MCS_OK otherwise.  diag_dev (may be NULL): int32[4] as for mcs_search_by_projection_device.
 * capacity <= 65535, n_cams * capacity < 2^24 (MCS_ERR_UNSUPPORTED beyond); cameras of different sizes: MCS_ERR_UNSUPPORTED. */
int  mcs_search_by_projection_last_device(const mcs_packed_frame* cur, const mcs_packed_frame* last, int32_t n_cams, int32_t capacity,
                                          int32_t dim, const mcs_ocam* cams, const uint8_t* masks_dev, int32_t n_levels,
                                          const double* scale_factors, const double* mtmc_inv, const int32_t* last_mp_dev,
                                          const uint8_t* last_outlier_dev, int32_t n_points, const double* world_pos_dev,
                                          const uint8_t* bad_dev, double th, int32_t th_high, int32_t having_masks, int32_t* cur_mp_dev,
                                          int32_t* nmatches_dev, int32_t* status_dev, int32_t* diag_dev, void* stream);

/* TrackPreviousFrame's two searches (ref src/cTracking.cpp:724-788) with both frames in packed feature buffers and every output on
 * the device, F1 = last, F2 = cur.  Same conventions as mcs_search_by_projection_last_device: asynchronous, host validation before
 * any launch, both frames may share one buffer, last_mp_dev / cur_mp_dev [n_cams * capacity] slot-indexed map-point ids (-1 =
 * none), slots at or beyond a camera's count neither read nor written in either frame, nmatches_dev / status_dev / diag_dev as
 * there.  Acceptance is MCS_RULE_RATIO: the best candidate not yet assigned (strict < over the visiting order) is accepted when
 * best <= second * nnratio (second = INT_MAX without one) and best <= th_high; cur_mp_dev receives the map-point id.  Neither call
 * reads scale factors: -1 as an octave is "no level filter" and an octave >= the frame's levels finds no candidate, so octaves
 * raise no status.
 *
 * mcs_window_search_device: WindowSearch(last, cur, window, ., min_level, max_level) (ref src/cORBmatcher.cpp:326-473).
 *   cur_mp_dev is an output: every slot below a camera's count is first set to -1 (the reference starts from an all-NULL vector).
 *   Each last-frame keypoint in contiguous order whose map point exists and is not bad, with min_level <= 0 or octave >=
 *   min_level, and max_level == INT_MAX or octave <= max_level, searches GetFeaturesInArea(cam, x, y, window) of the same camera of
 *   cur, all levels.  cam_width / cam_height [n_cams] host.  status_dev: MCS_ERR_INVALID when a map-point id is >= n_points (that
 *   query is dropped).  n_cams * capacity < 2^24.
 * mcs_search_by_projection_frames_device: SearchByProjection(last, cur, window, .) (ref :476-577).
 *   cur_mp_dev is in/out and holds cur's map points on entry; the points it holds are "already found" and their keypoints are
 *   taken.  A last-frame keypoint searches when its map point exists, is not bad, is not already found and the keypoint is the
 *   first to carry it; the point is projected with WorldToCamHom_fast into EVERY camera c of the current pose (mtmc_inv [n_cams *
 *   16] host, row-major MtMc_inv) and, inside c's mirror mask (masks_dev [n_cams][height][width]), searched in
 *   GetFeaturesInArea(c, u, v, window, octave, octave).  Each camera's search may be accepted.  cams [n_cams] host, one image
 *   size for all (MCS_ERR_UNSUPPORTED otherwise); world_pos_dev [n_points * 3], bad_dev [n_points] (may be NULL).
 *   status_dev: MCS_ERR_INVALID when a last-frame map-point id is >= n_points (that keypoint is dropped); ids >= n_points in
 *   cur_mp_dev mark their keypoint taken and find no point.  n_cams * n_cams * capacity < 2^24.
 * capacity <= 65535; beyond the query bounds MCS_ERR_UNSUPPORTED. */
int  mcs_window_search_device(const mcs_packed_frame* cur, const mcs_packed_frame* last, int32_t n_cams, int32_t capacity, int32_t dim,
                              const int32_t* cam_width, const int32_t* cam_height, const int32_t* last_mp_dev, int32_t n_points,
                              const uint8_t* bad_dev, int32_t window, int32_t min_level, int32_t max_level, double nnratio,
                              int32_t th_high, int32_t having_masks, int32_t* cur_mp_dev, int32_t* nmatches_dev, int32_t* status_dev,
                              int32_t* diag_dev, void* stream);
int  mcs_search_by_projection_frames_device(const mcs_packed_frame* cur, const mcs_packed_frame* last, int32_t n_cams, int32_t capacity,
                                            int32_t dim, const mcs_ocam* cams, const uint8_t* masks_dev, const double* mtmc_inv,
                                            const int32_t* last_mp_dev, int32_t n_points, const double* world_pos_dev,
                                            const uint8_t* bad_dev, int32_t window, double nnratio, int32_t th_high, int32_t having_masks,
                                            int32_t* cur_mp_dev, int32_t* nmatches_dev, int32_t* status_dev, int32_t* diag_dev,
                                            void* stream);

/* Generic projection-window search: the shape shared by the remaining cORBmatcher searches (SURVEY 8a row M4).
 * Queries are visited in order; for each one the candidates of GetFeaturesInArea(cam, x, y, r, min_level, max_level)
 * that are not yet taken (assigned[idx] >= 0) are scanned in the reference's order, best / second best are tracked
 * with strict `<`, and the best candidate is accepted by `rule`:
 *   MCS_RULE_RATIO        best <= second*nnratio && best <= threshold   WindowSearch (ref src/cORBmatcher.cpp:420),
 *                                                                       SearchByProjection(F1,F2,win,..) (:556-558)
 *   MCS_RULE_BEST         best <= threshold                             SearchByProjection(Current, Last, th) (:2070)
 *   MCS_RULE_LEVEL_RATIO  best <= threshold && !(bestLevel == secondLevel && best > nnratio*second)
 *                                                                       SearchByProjection(F, MapPoints, th) (:151-158)
 *   MCS_RULE_BEST_FREE    best <= threshold, candidates are NOT skipped when taken and nothing is marked: the per-query
 *                         answer is written to assigned[q] (best index or -1; `assigned` is then an output of nq entries).
 *                         This is the matching core of Fuse(pKF, curKF, ..) (:1326-1366), Fuse(pKF, Scw, ..) (:1620-1660) and
 *                         SearchBySim3 (:1793-1830, :1869-1906): their level filter {l-1, l} goes into the query.
 *   MCS_RULE_FIRST_FREE   Fuse(pKF, vpMapPoints, th) (:1420-1568, the overload cLocalMapping calls at src/cLocalMapping.cpp:450)
 *                         as the reference really behaves: it computes the descriptor distance and DISCARDS it (:1506-1514, `dist`
 *                         stays 0), so the first candidate of the window that passes the level filter wins with distance
 *                         0 <= threshold.  Stateless like MCS_RULE_BEST_FREE: assigned[q] = that candidate or -1.
 *   MCS_RULE_SCW          SearchByProjection(pKF, Scw, vpPoints, vpMatched, th) (:2265-2392) as written: taken candidates
 *                         (vpMatched[idx], i.e. assigned[idx] >= 0) are skipped; the descriptor compared for candidate idx of a
 *                         query of camera c is ROW idx OF CAMERA c's MATRIX -- the contiguous keypoint id used as a per-camera row
 *                         (:2367, :2372) -- i.e. contiguous keypoint first(c) + idx; candidates whose row lies beyond camera c's own
 *                         rows (where the reference reads past the matrix: undefined) are dropped; accepted when
 *                         best <= threshold && bestIdx > 0 (:2385, keypoint 0 can never be matched).  Needs camera-major keypoints.
 * On acceptance assigned[bestIdx] = query_tag[q] (tags must be >= 0).  The caller builds the queries (projection
 * front-end, "bad"/duplicate filters of the reference loops) and owns `assigned` (in/out, [n_keys], -1 = free). */
#define MCS_RULE_RATIO        0
#define MCS_RULE_BEST         1
#define MCS_RULE_LEVEL_RATIO  2
#define MCS_RULE_BEST_FREE    3
#define MCS_RULE_FIRST_FREE   4
#define MCS_RULE_SCW          5
int  mcs_search_windows(const mcs_frame_view* frame, const mcs_window_query* queries, int32_t nq,
                        const uint8_t* qdesc, const uint8_t* qmask, const int32_t* query_tag,
                        int32_t rule, double nnratio, int32_t threshold, int32_t* assigned, int32_t* nmatches);

/* cORBmatcher::SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize)
 * (ref :579-726, checkOrientation is compile-time false: include/cORBmatcher.h:40).
 * prev_matched[2*n1] in/out (x,y doubles); matches12[n1] out. */
int  mcs_search_for_initialization(const mcs_frame_view* f1, const mcs_frame_view* f2,
                                   double* prev_matched, int32_t window_size,
                                   double nnratio, int32_t th_low, int32_t having_masks,
                                   int32_t* matches12, int32_t* nmatches);

/* Map initialisation's search, cTracking::Initialize's SearchForInitialization(mInitialFrame, mCurrentFrame, mvbPrevMatched,
 * mvIniMatches, windowSize) (ref src/cTracking.cpp:405-409, src/cORBmatcher.cpp:579-726), with both frames in packed feature
 * buffers and its state on the device.  Conventions of mcs_window_search_device: asynchronous on `stream` (NULL synchronises),
 * host validation before any launch, nothing read back, f1 / f2 in either packed layout and possibly one buffer.
 *   Every F1 keypoint below its camera's count is a query, in contiguous order: GetFeaturesInArea(cam, prev.x, prev.y,
 *   window_size, octave, octave) in the same camera of F2; candidates whose vMatchedDistance is <= their distance are skipped;
 *   the best is accepted when best <= th_low and best < second * nnratio (second = INT_MAX without one), and takes its F2
 *   keypoint from an earlier query.  checkOrientation is compile-time false (include/cORBmatcher.h:40).
 *   cam_width / cam_height [n_cams] host.  prev_matched_dev [n_cams * capacity * 2] doubles, in/out, F1 slot-indexed (c * capacity +
 *   j): the window centres, read before any is written; afterwards a surviving match's centre is its F2 keypoint's position.
 *   matches12_dev [n_cams * capacity] out, F1 slot-indexed: the F2 SLOT matched, or -1; every F1 slot below a camera's count is
 *   written.  Slots at or beyond a camera's count are neither read nor written, in any array or frame.  nmatches_dev [1]: the
 *   reference's return value (F2 keypoints with an owner).  diag_dev (may be NULL): int32[2], the queries and the decisions that
 *   rescanned their window.  No input is invalid in a data-dependent way (an octave outside the frame's levels finds no
 *   candidate), so there is no status.
 * capacity <= 65535 (visiting positions and walk state are 16-bit); n_cams * capacity < 2^24 (MCS_ERR_UNSUPPORTED beyond).
 * mcs_search_for_initialization_seed_device: FirstInitialization's fill of mvbPrevMatched (ref src/cTracking.cpp:383-386):
 *   prev_matched_dev[2 * slot .. +1] = (double) the keypoint's position, for every F1 slot below its camera's count. */
int  mcs_search_for_initialization_device(const mcs_packed_frame* f1, const mcs_packed_frame* f2, int32_t n_cams, int32_t capacity,
                                          int32_t dim, const int32_t* cam_width, const int32_t* cam_height, double* prev_matched_dev,
                                          int32_t window_size, double nnratio, int32_t th_low, int32_t having_masks,
                                          int32_t* matches12_dev, int32_t* nmatches_dev, int32_t* diag_dev, void* stream);
int  mcs_search_for_initialization_seed_device(const mcs_packed_frame* f1, int32_t n_cams, int32_t capacity, int32_t dim,
                                               double* prev_matched_dev, void* stream);

/* The matching part of the three Fuse overloads (ref src/cORBmatcher.cpp:1265-1418, :1420-1567, :1570-1719) for n_kf target key
 * frames in one call, with every target in packed feature buffers: cLocalMapping::SearchInNeighbors' Fuse(pKFi, curKF, .) per
 * neighbour and its Fuse(curKF, candidates), cLoopClosing::SearchAndFuse's Fuse(pKF, Scw, ., 4) per corrected key frame.
 * Conventions of mcs_search_by_projection_last_device: asynchronous on `stream` (NULL synchronises), host validation before any
 * launch, nothing read back, stream-ordered scratch; the targets' frames in either packed layout, possibly sharing one buffer.
 * The call decides which keypoint each (key frame, query, camera) hits; the map bookkeeping (Replace, AddObservation,
 * AddMapPoint) stays with the caller, which replays the hits in row order over the live map.
 *   kfs [n_kf] host: per target its frame, its slot-indexed map-point ids mp_dev [n_cams * capacity] (the frame_mp_dev format; NULL
 *   = no "already in the key frame" pre-filter for it), mtmc_inv [n_cams * 16] host (row-major MtMc_inv of the pose to project
 *   with) and ow, the centre the depth test measures from (GetCameraCenter, or the Sim3's rigid part for MCS_FUSE_SIM3).
 *   cams [n_cams] host camera models (one image size for all), masks_dev [n_cams][height][width] their mirror masks,
 *   scale_factors [n_levels] host.  query_mp_dev [n_q]: map-point ids, -1 = NULL (the array may be NULL when n_q is 0).  The map points: world_pos_dev [n_points * 3],
 *   min_dist_dev / max_dist_dev [n_points] (GetMin/MaxDistanceInvariance), desc_dev / dmask_dev [n_points * dim] (dmask_dev only
 *   read when having_masks), bad_dev [n_points] (may be NULL).
 *   For every key frame k, query q, camera c, in that order: q is skipped when its id is -1, the point is bad, or a slot of
 *   kfs[k].mp_dev below its camera's count holds it.  Otherwise the point is projected (WorldToCamHom_fast, mirror mask), its
 *   distance to ow tested against [min, max] -- a float for MCS_FUSE_NEIGHBOUR / MCS_FUSE_FIRST, a double for MCS_FUSE_SIM3 --,
 *   its level l predicted by lower_bound over the scale factors, and GetFeaturesInArea(c, u, v, th * scale_factors[l]) searched on
 *   levels {l - 1, l}.  MCS_FUSE_NEIGHBOUR / MCS_FUSE_SIM3: the best candidate (strict < over the visiting order) hits when its
 *   distance is <= th_low.  MCS_FUSE_FIRST: the first candidate in visiting order hits (the reference discards the distance).
 *   The pre-filter relies on the caller's map: a point a key frame's slot holds is IsInKeyFrame of that key frame (the reference
 *   always pairs AddMapPoint with AddObservation), and bad never reverts.  Skipping such a query changes no decision.
 *   hits_dev [max_hits][3] out (may be NULL when max_hits is 0): (k, q, slot) rows in the order above, slot = c * capacity + j in key frame k.  n_hits_dev [1]: the
 *   true number of hits.  status_dev [1]: MCS_ERR_CAPACITY when n_hits exceeds max_hits (only the first max_hits rows are written,
 *   nothing past them), MCS_ERR_INVALID when a query id is >= n_points (that query is dropped, the others are unaffected; this
 *   error is kept over MCS_ERR_CAPACITY), MCS_OK otherwise.
 *   Scratch: 4 * n_points + n_kf * n_q bytes for the pre-filter, about 170 bytes per (k, q, c) entry, and the front end's
 *   per-slot arrays for n_kf * n_cams images.
 * capacity <= 65535; n_kf * n_cams * capacity < 2^24 and n_kf * n_q * n_cams < 2^24 (MCS_ERR_UNSUPPORTED beyond: split the
 * batch); cameras of different sizes: MCS_ERR_UNSUPPORTED. */
typedef struct mcs_fuse_target {
    mcs_packed_frame frame;      /* the key frame's features */
    const int32_t*   mp_dev;     /* [n_cams * capacity] slot-indexed map-point ids, or NULL */
    const double*    mtmc_inv;   /* host [n_cams * 16] */
    double           ow[3];
} mcs_fuse_target;

#define MCS_FUSE_NEIGHBOUR 0     /* Fuse(pKF, curKF, vpMapPoints, th)  :1265  float dist3D, best <= th_low          */
#define MCS_FUSE_FIRST     1     /* Fuse(pKF, vpMapPoints, th)         :1420  float dist3D, first in-level candidate */
#define MCS_FUSE_SIM3      2     /* Fuse(pKF, Scw, vpPoints, th)       :1570  double dist3D, best <= th_low         */

int  mcs_fuse_device(const mcs_fuse_target* kfs, int32_t n_kf, int32_t n_cams, int32_t capacity, int32_t dim, const mcs_ocam* cams,
                     const uint8_t* masks_dev, int32_t n_levels, const double* scale_factors, int32_t variant, const int32_t* query_mp_dev,
                     int32_t n_q, int32_t n_points, const double* world_pos_dev, const double* min_dist_dev, const double* max_dist_dev,
                     const uint8_t* desc_dev, const uint8_t* dmask_dev, const uint8_t* bad_dev, double th, int32_t th_low,
                     int32_t having_masks, int32_t* hits_dev, int32_t max_hits, int32_t* n_hits_dev, int32_t* status_dev, void* stream);

/* Loop closing's two Sim3 searches (cLoopClosing::ComputeSim3, ref src/cLoopClosing.cpp:343 and :401) with the key frames in packed
 * feature buffers.  Conventions of mcs_search_by_projection_last_device: asynchronous on `stream` (NULL synchronises), host
 * validation before any launch, nothing read back, stream-ordered scratch; frames in either packed layout, possibly one buffer;
 * map-point rows slot-indexed (c * capacity + j), slots at or beyond a camera's count neither read nor written.  cams [n_cams] host
 * camera models (one image size for all, MCS_ERR_UNSUPPORTED otherwise), masks_dev [n_cams][height][width] their mirror masks,
 * scale_factors [n_levels] host.  The map points: world_pos_dev [n_points * 3], min_dist_dev / max_dist_dev [n_points]
 * (GetMin/MaxDistanceInvariance), desc_dev / dmask_dev [n_points * dim] (dmask_dev read only when having_masks), bad_dev
 * [n_points] (may be NULL).  capacity <= 65535; n_cams * capacity < 2^24 (MCS_ERR_UNSUPPORTED beyond).
 *
 * mcs_search_by_sim3_device: SearchBySim3(pKF1, pKF2, vpMatches12, s12, R12, t12, th) (ref src/cORBmatcher.cpp:1721-1988).
 *   kf1 / kf2 may be the same frame.  t1w / t2w host row-major 4x4, each key frame's GetPoseInverse(); mc_inv [n_cams * 16] host,
 *   invMat(Get_M_c(c)) of the rig both key frames share; r12 [9] row-major, t12 [3], s12 != 0 (MCS_ERR_INVALID otherwise).  The
 *   launcher forms sR12 = s12 * R12, sR21 = (1 / s12) * R12^T and t21 = -sR21 * t12 in cv::Matx order.
 *   Direction 1: every KF1 slot in slot order whose id in mp1_dev exists, whose matches12_dev entry is -1 on entry (vbAlreadyMatched1)
 *   and whose point is not bad: p3Dc1 = R1w * X + t1w, p3Dc2 = sR21 * p3Dc1 + t21, p4 = mc_inv[c] * (p3Dc2, 1) with c the keypoint's
 *   camera; dropped when p3Dc2.z < 0 (the rig frame's z, not the camera's), when WorldToImg(p4) lies outside camera c's mirror mask,
 *   or when |p4.xyz| (a double) lies outside [min, max]; else level l = lower_bound over the scale factors, clamped, and the best
 *   candidate (strict < over the visiting order, nothing skipped) of GetFeaturesInArea(c, u, v, th * scale_factors[l]) of KF2 on
 *   levels {l - 1, l} counts when its distance is <= th_high.  Direction 2 is the mirror image, KF2 into KF1 with sR12 and t12,
 *   already2_dev (KF2 slot-indexed bytes, may be NULL: vbAlreadyMatched2, which the caller builds from GetIndexInKeyFrame(pKF2)[0])
 *   as its skip list.  matches12_dev (KF1 slot-indexed map-point ids, in/out): matches12[s1] = mp2[s2] where direction 1 found s2
 *   for s1 and direction 2 found s1 for s2.  nfound_dev [1]: those agreements.  status_dev: MCS_ERR_INVALID when an id in mp1_dev,
 *   mp2_dev or matches12_dev is >= n_points (that slot is dropped, the others are unaffected), MCS_OK otherwise.
 *
 * mcs_search_by_projection_scw_device: SearchByProjection(pKF, Scw, vpPoints, vpMatched, th) (ref :2265-2392) as written there.
 *   mtmc_inv [n_cams * 16] host and ow [3] host: the rigid part of Scw (MtMc_inv and centre of the rig posed by
 *   invMat(Rt2Hom(Rcw, tcw)), as mcs_fuse_target for MCS_FUSE_SIM3).  points_dev [n_q] map-point ids, -1 = NULL (may be NULL when
 *   n_q is 0).  matched_dev: vpMatched, slot-indexed map-point ids, in/out; the points it holds on entry are spAlreadyFound for the
 *   whole call, its slots holding an id are taken.  Entry i of points_dev in order, unless NULL, bad or already found: projected
 *   (WorldToCamHom_fast, mirror mask) into the camera of CONTIGUOUS KEYPOINT i of the key frame (keypoint_to_cam.find(iMP), :2307),
 *   its double distance to ow tested against [min, max], its level l predicted, and GetFeaturesInArea(cam, u, v, th *
 *   scale_factors[l]) searched on levels {l - 1, l} without the taken keypoints.  Candidate j of camera c is compared through row
 *   first(c) + j of camera c's descriptors (the reference indexes the camera's matrix with the contiguous id, :2367, :2372), and
 *   dropped when that row is at or beyond camera c's count (the reference reads past the matrix there).  The best is accepted when
 *   best <= th_low and it is not contiguous keypoint 0 (`bestIdx > 0`, :2385: the first slot of the first camera with keypoints),
 *   greedily in entry order: matched_dev receives the point.  nmatches_dev [1]: the acceptances of this call (the reference's
 *   return value; ComputeSim3's nTotalMatches counts every slot of matched_dev that holds a point).  status_dev: MCS_ERR_INVALID
 *   when an id is >= n_points, or when an entry that reaches the camera look-up lies at or beyond the key frame's keypoint count
 *   (the reference dereferences unordered_map::end() there: undefined); such an entry is dropped, the others are unaffected.
 *   diag_dev (may be NULL): int32[4] as for mcs_search_by_projection_device.  n_q < 2^24 (MCS_ERR_UNSUPPORTED beyond). */
/* Loop closing's first matcher call, SearchByBoW(mpCurrentKF, pKF, vvpMapPointMatches[i]) (cLoopClosing::ComputeSim3, ref
 * src/cLoopClosing.cpp:281; src/cORBmatcher.cpp:885-966), for n_kf candidate key frames in one call.  Per candidate k,
 * independently of the others (n_kf candidates in one call give what n_kf calls with one candidate give):
 *   Queries: the KF1 slots below each camera's count, in slot order (the reference's contiguous order), whose mp1_dev id is >= 0
 *   and whose point is not bad.  Database: the slots of kfs[k] below each camera's count whose mp_dev[k] id is >= 0 and not bad.
 *   Each query takes the best and second-best distance (strict <, in slot order) over the database slots this candidate has not
 *   yet taken; accepted when best < th_low and (double)best < nnratio * (double)second (second = INT_MAX without one), and the
 *   slot is then taken for the rest of the candidate's walk.  Distances are DescriptorDistance64 / DescriptorDistance64Masked
 *   (having_masks) between the packed descriptor rows, dim 16 / 32 / 64.
 *   matches12_dev [n_kf][n_cams * capacity]: per KF1 slot the map-point id of the candidate slot it matched (vpMapPoints2[bestIdx2]),
 *   or -1: the matches12_dev row mcs_search_by_sim3_device takes, once the caller's RANSAC has cleared the outliers.
 *   match_slot_dev (same shape, may be NULL): the candidate slot matched, or -1.  Both are set below each camera's count of KF1;
 *   slots at or beyond a count are neither read nor written, in any frame.  nmatches_dev [n_kf]: the reference's return value.
 *   status_dev [1]: MCS_ERR_INVALID when a map-point id is >= n_points -- that slot is dropped, the others are unaffected --,
 *   MCS_OK otherwise.  bad_dev [n_points] may be NULL.
 * Conventions of mcs_search_by_bow_device: asynchronous on `stream` (NULL synchronises), every argument checked on the host before
 * any launch, stream-ordered scratch, nothing read back.  Each frame in either packed layout; KF1 and the candidates may share
 * buffers, and KF1 may be one of its own candidates.  n_kf = 0 is a successful no-op.
 * Limits (MCS_ERR_UNSUPPORTED beyond, before any launch): n_cams * capacity <= 1 622 016, the "taken" bits of one candidate's
 * database held in the shared memory of one acceptance CTA (and below the lists' 21-bit index); n_cams * capacity < 2^24 (the
 * query bound of the device searches); n_kf * n_cams * capacity < 2^31.  capacity <= 65535.
 * Scratch, one stream-ordered block: per slot of each of the 1 + n_kf frames, dim bytes of compact descriptors (2 * dim with
 * having_masks) and 4 of slot map; per (candidate, slot), 32 * splits bytes of partial K-best lists, 64 of merged lists and 4 of
 * compact matches, with NS = n_cams * capacity and splits <= min(ceil(NS / 256), max(1, ceil(32 * SMs / (ceil(NS / 128) * n_kf))))
 * database chunks: on a 132-SM device and a config-3 frame (NS = 8 000), 32 chunks (about 1.1 KB per row) for one candidate, 5
 * for 16.  The limits above bound indices, not memory: near n_kf * NS = 2^31 the scratch would be about 200 GB, and the call
 * then fails with MCS_ERR_CUDA from the scratch allocation, before any kernel is launched. */
int  mcs_search_by_bow_keyframes_device(const mcs_packed_frame* kf1, const int32_t* mp1_dev, const mcs_packed_frame* kfs,
                                        const int32_t* const* mp_dev, int32_t n_kf, int32_t n_cams, int32_t capacity, int32_t dim,
                                        int32_t n_points, const uint8_t* bad_dev, int32_t th_low, double nnratio, int32_t having_masks,
                                        int32_t* matches12_dev, int32_t* match_slot_dev, int32_t* nmatches_dev, int32_t* status_dev,
                                        void* stream);
/* Local mapping's search, SearchForTriangulationRaw(mpCurrentMultiKeyFrame, pKF2, ...) (cLocalMapping::CreateNewMapPoints, ref
 * src/cLocalMapping.cpp:226-380; src/cORBmatcher.cpp:968-1107, no rotation check), for ONE neighbour key frame per call:
 *   Queries: the KF1 slots below each camera's count whose mp1_dev id is -1 (free; any other id is taken, bad or not), in slot order
 *   (the reference's contiguous order).  Candidates of a query: the free KF2 slots of the SAME camera, below its count, not taken
 *   by an earlier query of this call, at distance <= th_low (DescriptorDistance64 / DescriptorDistance64Masked with having_masks,
 *   dim 16 / 32 / 64).  With best the smallest candidate distance, the candidates are walked in (distance, slot) order while
 *   distance <= 2 * best and the first with CheckDistEpipolarLine(ray1, ray2, E[c][c], epi_thresh) (ref src/misc.cpp:53-69) is
 *   matched and taken.  Rays are mvKeysRays: cam_img_to_world of the keypoint's float position under cams[c].
 *   cams [n_cams] and E [n_cams * n_cams * 9] (row-major 3x3 blocks E[c1][c2], the layout of mcs_search_for_triangulation and of
 *   the settings' essential matrices; only the blocks E[c][c] are read) are host memory.  Cameras may differ in size.
 *   mp1_dev / mp2_dev: slot-indexed map-point ids [n_cams * capacity].  matches12_dev [n_cams * capacity]: per KF1 slot the KF2
 *   slot matched, or -1, for every slot below its camera's count; no slot at or beyond a count is read or written, in either frame.
 *   nmatches_dev [1]: the reference's return value.  diag_dev (may be NULL): int32[2], the queries and the decisions that rescanned
 *   a camera's database because the K-best lists could not decide them.
 * The reference's CreateNewMapPoints adds the points it triangulates to KF1 before it searches the next neighbour, which removes
 * their keypoints from the next call's queries: call once per neighbour and write the new ids into mp1_dev / mp2_dev in between.
 * Conventions of mcs_search_for_initialization_device: asynchronous on `stream` (NULL synchronises), every argument checked on the
 * host before any launch, stream-ordered scratch, nothing read back.  Each frame in either packed layout; KF1 and KF2 may share
 * buffers or be the same frame.
 * Limits (MCS_ERR_UNSUPPORTED beyond, before any launch): capacity <= 65535 (a camera's rows and "taken" bits in one CTA);
 * n_cams * capacity < 2^24.  Scratch, one stream-ordered block: per slot of each frame dim bytes of compact descriptors (2 * dim
 * with having_masks), 24 of ray and 4 of slot map; per KF1 slot 32 * splits + 72 bytes of K-best lists and flags, splits <=
 * ceil(capacity / 256) database chunks. */
int  mcs_search_for_triangulation_device(const mcs_packed_frame* kf1, const int32_t* mp1_dev, const mcs_packed_frame* kf2,
                                         const int32_t* mp2_dev, int32_t n_cams, int32_t capacity, int32_t dim, const mcs_ocam* cams,
                                         const double* E, double epi_thresh, int32_t th_low, int32_t having_masks,
                                         int32_t* matches12_dev, int32_t* nmatches_dev, int32_t* diag_dev, void* stream);
int  mcs_search_by_sim3_device(const mcs_packed_frame* kf1, const mcs_packed_frame* kf2, int32_t n_cams, int32_t capacity, int32_t dim,
                               const mcs_ocam* cams, const uint8_t* masks_dev, int32_t n_levels, const double* scale_factors, const double* t1w,
                               const double* t2w, const double* mc_inv, double s12, const double* r12, const double* t12, double th,
                               const int32_t* mp1_dev, const int32_t* mp2_dev, int32_t n_points, const double* world_pos_dev,
                               const double* min_dist_dev, const double* max_dist_dev, const uint8_t* desc_dev, const uint8_t* dmask_dev,
                               const uint8_t* bad_dev, const uint8_t* already2_dev, int32_t th_high, int32_t having_masks,
                               int32_t* matches12_dev, int32_t* nfound_dev, int32_t* status_dev, void* stream);
int  mcs_search_by_projection_scw_device(const mcs_packed_frame* kf, int32_t n_cams, int32_t capacity, int32_t dim, const mcs_ocam* cams,
                                         const uint8_t* masks_dev, int32_t n_levels, const double* scale_factors, const double* mtmc_inv,
                                         const double* ow, const int32_t* points_dev, int32_t n_q, int32_t n_points,
                                         const double* world_pos_dev, const double* min_dist_dev, const double* max_dist_dev,
                                         const uint8_t* desc_dev, const uint8_t* dmask_dev, const uint8_t* bad_dev, int32_t th, int32_t th_low,
                                         int32_t having_masks, int32_t* matched_dev, int32_t* nmatches_dev, int32_t* status_dev,
                                         int32_t* diag_dev, void* stream);

/* ---- map-point tables on the device: cMapPoint::ComputeDistinctiveDescriptors and UpdateNormalAndDepth ------------------------ */
/* The producer of the map-point tables the device searches read (desc_dev / dmask_dev, normal_dev, min_dist_dev / max_dist_dev):
 * for every listed point, the reference's methods over its observations, with the key frames in packed feature buffers.
 * Conventions of the device searches: asynchronous on `stream` (NULL synchronises), every argument checked on the host before any
 * launch, small host tables staged in stream order, stream-ordered scratch, status on the device, nothing read back.
 *   kfs [n_kf] host: the key frames the observations name.  frame: either packed layout, several key frames may share a buffer;
 *   ow: GetCameraCenter(); bad: isBad() (its rows are no descriptor candidates, it still adds its term to the normal).
 *   scale_factors [n_levels] host (mvScaleFactors).  point_ids_dev [n_upd]: the points to update, repeats allowed (every point
 *   depends only on its own inputs, so a repeated id writes the same bytes).
 *   Observations, a CSR indexed by map-point id: obs_offsets_dev [n_points + 1], and per entry obs_kf_dev (index into kfs) and
 *   obs_slot_dev (c * capacity + j in that key frame).  Entries come in mObservations order -- a std::map keyed by key-frame
 *   address, so the caller lists the order it wants -- with each key frame's slots adjacent, in AddObservation order.
 *   ref_kf_dev [n_points] (index into kfs: mpRefKF), bad_dev [n_points] (may be NULL: no point is bad; a bad point is left
 *   untouched), world_pos_dev [n_points * 3].
 *   what = MCS_MP_DESCRIPTOR: ComputeDistinctiveDescriptors(having_masks) (ref src/cMapPoint.cpp:294-388).  The rows of the
 *   non-bad key frames' observations in list order; none: nothing changes; N <= 2: row 0; else the row i < N - 1 whose median
 *   of its upper part {D(i, j) : j > i} (the element of rank floor((N - 1 - i) / 2)) is strictly smallest, the first on ties.
 *   D is DescriptorDistance64, or DescriptorDistance64Masked when having_masks.  desc_dev [n_points * dim] receives the row,
 *   dmask_dev [n_points * dim] its mask only when having_masks (otherwise dmask_dev is neither read nor written).
 *   what = MCS_MP_NORMAL_DEPTH: UpdateNormalAndDepth() (:449-492).  normal_dev [n_points * 3] = the mean over the listed KEY
 *   FRAMES (bad ones included) of (X - Ow) / |X - Ow|, with OpenCV's Vec / scalar = multiplication by the rounded reciprocal;
 *   NaN for a point without observations (0 * (1. / 0)).  level = octave of the ref key frame's first observation, 1 when it
 *   has none; s = scale_factors[level], dist = |X - Ow_ref|; min_dist_dev = 0.8 * (((1 / s) * dist) / s) and max_dist_dev =
 *   1.2 * ((s * dist) * scale_factors[n_levels - 1 - level]): GetMin/MaxDistanceInvariance, the values the searches take.
 *   Only the listed rows of the arrays `what` selects are written; the arrays it does not select may be NULL.
 *   status_dev [1]: MCS_ERR_INVALID when a listed id is outside [0, n_points), an obs_kf or (MCS_MP_NORMAL_DEPTH) ref_kf index
 *   is outside [0, n_kf), a slot lies at or beyond its camera's count, a key frame's observations are not adjacent, or the level
 *   read lies outside [0, n_levels) -- that point is left untouched, the others are unaffected --, MCS_OK otherwise.
 * capacity <= 65535, dim 16 / 32 / 64. */
typedef struct mcs_mp_keyframe {
    mcs_packed_frame frame;   /* the key frame's features, either packed layout */
    double ow[3];             /* GetCameraCenter() */
    int32_t bad;              /* isBad(): no descriptor rows, still counted in the normal */
} mcs_mp_keyframe;
#define MCS_MP_DESCRIPTOR   1 /* ComputeDistinctiveDescriptors */
#define MCS_MP_NORMAL_DEPTH 2 /* UpdateNormalAndDepth */
int  mcs_update_mappoints_device(const mcs_mp_keyframe* kfs, int32_t n_kf, int32_t n_cams, int32_t capacity, int32_t dim,
                                 int32_t n_levels, const double* scale_factors, int32_t what, int32_t having_masks,
                                 const int32_t* point_ids_dev, int32_t n_upd, int32_t n_points,
                                 const int32_t* obs_offsets_dev, const int32_t* obs_kf_dev, const int32_t* obs_slot_dev,
                                 const int32_t* ref_kf_dev, const uint8_t* bad_dev, const double* world_pos_dev,
                                 uint8_t* desc_dev, uint8_t* dmask_dev, double* normal_dev, double* min_dist_dev, double* max_dist_dev,
                                 int32_t* status_dev, void* stream);

/* ---- bag of words: ORBVocabulary::transform and the feature-vector guided search (SURVEY 8f, rank 4) ------- */
/* The vocabulary tree of DBoW2::TemplatedVocabulary<FORB::TDescriptor, FORB> (ref include/cORBVocabulary.h:34,
 * ThirdParty/DBoW2/DBoW2/TemplatedVocabulary.h) as flat arrays.  Node 0 is the root; parent[0] is ignored.
 * descriptors: n_nodes x 32 bytes (FORB::L = 32; row 0 unused).  weight[i]: node weight (word weight for leaves).
 * node_order: the n_nodes-1 non-root node ids in the order the reference's load() appends them to their parent's
 * children (ref :1596-1608 / :1382-1421); NULL = ascending id.  word_node[w] = node id of word w.
 * scoring: 0 L1_NORM, 1 L2_NORM, 2 CHI_SQUARE, 3 KL, 4 BHATTACHARYYA, 5 DOT_PRODUCT; weighting: 0 TF_IDF, 1 TF, 2 IDF,
 * 3 BINARY (ref ThirdParty/DBoW2/DBoW2/BowVector.h:36-59). */
typedef struct mcs_vocabulary mcs_vocabulary;
int  mcs_vocabulary_create(int32_t k, int32_t L, int32_t scoring, int32_t weighting, int32_t n_nodes,
                           const int32_t* parent, const double* weight, const uint8_t* descriptors,
                           const int32_t* node_order, int32_t n_words, const int32_t* word_node,
                           mcs_vocabulary** out);
void mcs_vocabulary_destroy(mcs_vocabulary* voc);

/* transform(feature, word_id, weight, &nid, levelsup) for n descriptors of 32 bytes (ref :1218-1261): the tree
 * descent on the GPU, one 16-lane group per descriptor, FORB::distance (ref FORB.cpp:84-104), first minimum wins.
 * node_id[i] = ancestor at level L - levelsup (0 when that level is <= 0).  The reference leaves nid indeterminate
 * when the leaf is shallower than that level; this library returns the leaf's node id there.  Any output may be NULL. */
int  mcs_bow_transform(const mcs_vocabulary* voc, const uint8_t* desc, int32_t n, int32_t levelsup,
                       int32_t* word_id, double* weight, int32_t* node_id);

/* transform(features, BowVector&, FeatureVector&, levelsup) (ref :1126-1194; call sites src/cMultiFrame.cpp:356-363,
 * src/cMultiKeyFrame.cpp:105-114).  desc = the frame's descriptors of all cameras concatenated in camera order
 * (cConverter::toDescriptorVector, ref src/cConverter.cpp:58-66).
 * BowVector: bow_words/bow_values[<= n] ascending word id (std::map order), *n_bow entries, weights accumulated in
 * feature order and normalised as the scoring type asks.
 * FeatureVector: CSR -- fv_nodes[<= n] ascending node id, fv_offsets[*n_fv + 1], fv_features[<= n] (ascending feature
 * index inside a node). */
int  mcs_bow_vectors(const mcs_vocabulary* voc, const uint8_t* desc, int32_t n, int32_t levelsup,
                     int32_t* bow_words, double* bow_values, int32_t* n_bow,
                     int32_t* fv_nodes, int32_t* fv_offsets, int32_t* n_fv, int32_t* fv_features);

/* ORBVocabulary::score(v1, v2) with the vocabulary's scoring type (ref ScoringObject.cpp:23-313); host arithmetic. */
int  mcs_bow_score(const mcs_vocabulary* voc, const int32_t* words1, const double* values1, int32_t n1,
                   const int32_t* words2, const double* values2, int32_t n2, double* score);

/* cORBmatcher::SearchByBoW(cMultiKeyFrame*, cMultiFrame&, vpMapPointMatches) (ref src/cORBmatcher.cpp:179-324; call site
 * src/cTracking.cpp:1177): for every vocabulary node both feature vectors hold, each key-frame keypoint that carries a
 * good map point (valid1) looks for its best / second best among the frame keypoints of that node that are still
 * unmatched; accepted if best <= th_low and best < nnratio * second.  Distances for all (node, keypoint) groups are
 * computed on the GPU, the order-dependent bookkeeping is replayed on the host.  desc1/desc2: n x dim rows in the
 * concatenated keypoint order the feature vectors index; masks NULL = unmasked.  match_of_2[n2] = key-frame keypoint
 * index or -1.  checkOrientation is compile-time false in the reference (include/cORBmatcher.h:40). */
int  mcs_search_by_bow(const uint8_t* desc1, const uint8_t* mask1, const uint8_t* valid1, int32_t n1,
                       const int32_t* fv1_nodes, const int32_t* fv1_offsets, int32_t n_fv1, const int32_t* fv1_features,
                       const uint8_t* desc2, const uint8_t* mask2, int32_t n2,
                       const int32_t* fv2_nodes, const int32_t* fv2_offsets, int32_t n_fv2, const int32_t* fv2_features,
                       int32_t dim, int32_t th_low, double nnratio, int32_t* match_of_2, int32_t* nmatches);

/* ---- Relocalisation's bag-of-words step on the device (ref src/cTracking.cpp:1125-1312): ComputeBoW and SearchByBoW(KF, F) on
 * frames that stay in their packed feature buffers.  Conventions of mcs_search_by_projection_last_device: frames as
 * mcs_packed_frame, everything per keypoint indexed by slot c * capacity + j, asynchronous on `stream` (NULL = the default
 * stream, synchronised before returning), scratch from the stream-ordered pool, every argument checked on the host before any
 * launch, results and status in device memory, nothing read back.  Slot order is the reference's contiguous keypoint order
 * (camera-major, ref src/cMultiFrame.cpp:168-184), so "ascending feature index" in DBoW2's containers is "ascending slot". */

/* The largest number of distinct node ids a FeatureVector built with `levelsup` can hold: the nodes at depth
 * max(L - levelsup, 0) plus the leaves shallower than that (see mcs_bow_transform).  Sizes fv_nodes / fv_offsets and max_nodes
 * below.  Host arithmetic. */
int  mcs_vocabulary_level_nodes(const mcs_vocabulary* voc, int32_t levelsup, int32_t* n_nodes);

/* transform(features, BowVector&, FeatureVector&, levelsup) (ref TemplatedVocabulary.h:1126-1194; ComputeBoW, ref
 * src/cMultiFrame.cpp:356-363, src/cMultiKeyFrame.cpp:105-114) over the descriptors of the n_cams cameras of `frame`, each
 * camera's slots below its device-side count, in camera order.  The values equal mcs_bow_vectors on the concatenated descriptors
 * bit for bit, feature indices being slots.  All outputs are device memory:
 *   word_dev / weight_dev / node_dev [n_cams * capacity] (each may be NULL): what mcs_bow_transform returns, per slot; untouched
 *     at or beyond a camera's count.
 *   FeatureVector as CSR: fv_nodes_dev [max_nodes] ascending node ids, fv_offsets_dev [max_nodes + 1], n_fv_dev [1],
 *     fv_features_dev [n_cams * capacity] slots, ascending inside a node; fv_offsets_dev[*n_fv_dev] entries are written.
 *   BowVector: bow_words_dev / bow_values_dev [n_cams * capacity] ascending word ids and their values, n_bow_dev [1].
 *   status_dev [1]: MCS_OK, or MCS_ERR_CAPACITY when the frame holds more than max_nodes nodes: the FeatureVector then holds the
 *     max_nodes smallest node ids, complete and consistent, and nothing is written beyond the arrays.  The BowVector is unaffected.
 * dim must be 32 (FORB::L; MCS_ERR_UNSUPPORTED otherwise); the vocabulary's device must be current (MCS_ERR_INVALID otherwise);
 * capacity <= 65535, n_cams * capacity < 2^24.  Scratch: 4 bytes per vocabulary node and 8 per word, cleared per call. */
int  mcs_bow_vectors_device(const mcs_vocabulary* voc, const mcs_packed_frame* frame, int32_t n_cams, int32_t capacity, int32_t dim,
                            int32_t levelsup, int32_t max_nodes, int32_t* word_dev, double* weight_dev, int32_t* node_dev,
                            int32_t* fv_nodes_dev, int32_t* fv_offsets_dev, int32_t* n_fv_dev, int32_t* fv_features_dev,
                            int32_t* bow_words_dev, double* bow_values_dev, int32_t* n_bow_dev, int32_t* status_dev, void* stream);

/* A frame or key frame whose FeatureVector is on the device (mcs_bow_vectors_device's CSR outputs, or arrays of the same form). */
typedef struct mcs_bow_frame {
    mcs_packed_frame frame;
    const int32_t* fv_nodes_dev;        /* [<= max_nodes] strictly ascending node ids          */
    const int32_t* fv_offsets_dev;      /* [*n_fv_dev + 1] non-decreasing                      */
    const int32_t* n_fv_dev;            /* [1]; entries beyond max_nodes are not visited       */
    const int32_t* fv_features_dev;     /* slots                                               */
    const int32_t* mp_dev;              /* [n_cams * capacity] slot-indexed map-point ids, -1 = none; NULL for the current frame */
} mcs_bow_frame;

/* cORBmatcher::SearchByBoW(pKF, F, vpMapPointMatches) (ref src/cORBmatcher.cpp:179-324, mbCheckOrientation compile-time false)
 * for n_kf key frames against one current frame, as Relocalisation calls it for every candidate (ref src/cTracking.cpp:1170-1177).
 * Per key frame k, independently of the others (n_kf key frames in one call give what n_kf calls with one key frame give):
 *   match_mp_dev [n_kf][n_cams * capacity]: the map-point id matched to each current-frame slot, -1 = none; match_slot_dev (same
 *   shape, may be NULL): the key-frame slot it came from.  Both are first set to -1 below each camera's count of `cur`; slots at
 *   or beyond a count are neither read nor written, in any frame.
 *   For every node id both feature vectors hold, ascending, and every key-frame slot of that node in list order whose mp_dev is
 *   >= 0 and not bad: best and second-best distance (strict <, in list order) over the current frame's slots of that node that no
 *   earlier keypoint of this key frame has taken; accepted when best <= th_low and (double)best < nnratio * (double)second
 *   (second = INT_MAX without one).  Distances are DescriptorDistance64 / DescriptorDistance64Masked (having_masks) between the
 *   packed descriptor rows, dim 16 / 32 / 64.
 *   nmatches_dev [n_kf].  status_dev [1]: MCS_ERR_INVALID when a map-point id is >= n_points or a feature-vector entry is no
 *   keypoint of its frame -- that keypoint is dropped, the others are unaffected -- MCS_OK otherwise.  bad_dev [n_points] may be NULL.
 * The key frames may live in different packed buffers from each other and from `cur`, or share one.  max_nodes bounds the node
 * lists visited (mcs_vocabulary_level_nodes); the grid is sized from n_kf * max_nodes.  n_kf = 0 is a successful no-op.
 * capacity <= 65535, n_cams * capacity < 2^24 (MCS_ERR_UNSUPPORTED beyond). */
int  mcs_search_by_bow_device(const mcs_bow_frame* kfs, int32_t n_kf, const mcs_bow_frame* cur, int32_t n_cams, int32_t capacity,
                              int32_t dim, int32_t max_nodes, int32_t n_points, const uint8_t* bad_dev, int32_t th_low, double nnratio,
                              int32_t having_masks, int32_t* match_mp_dev, int32_t* match_slot_dev, int32_t* nmatches_dev,
                              int32_t* status_dev, void* stream);

/* ---- multi-GPU: one camera (or stream chunk) per GPU, ONE allgather of the packed feature buffer (SURVEY 8e) -------------- */
/* Packed feature buffer of a batch of n_images images: the four output arrays of the batched extractor in one allocation,
 *   [ counts int32[n_images] | mcs_keypoint[n_images][capacity] | desc u8[n_images][capacity][dim] | dmask u8[n_images][capacity][dim] ]
 * every section on a 256-byte boundary.  offsets4 (may be NULL) receives the four byte offsets; returns the total size.  It is
 * the only layout that travels between GPUs: K3 writes it in place, the allgather moves it, the matchers read it in place. */
size_t mcs_packed_layout(int32_t n_images, int32_t capacity, int32_t dim, size_t* offsets4);
size_t mcs_slot_bytes(int32_t capacity, int32_t dim);     /* == mcs_packed_layout(1, capacity, dim, NULL): one camera of a rig */

/* mcs_extract_batch_device with the four outputs laid out as above inside packed_dev (device memory, mcs_packed_layout bytes). */
int  mcs_extract_batch_packed_device(mcs_extractor* ex, int32_t n_images,
                                     const uint8_t* images_dev, int32_t width, int32_t height, int32_t stride,
                                     const uint8_t* masks, const mcs_ocam* cams, int32_t n_cams, const int32_t* cam_of_image,
                                     void* packed_dev, int32_t capacity, void* stream);

/* Communicator of the rig's GPUs: one process per GPU.  Rank 0 draws the 128-byte rendezvous token (ncclGetUniqueId) and the host
 * program hands it to the other ranks by whatever it already has (MPI, torch.distributed, a socket); every rank then calls
 * mcs_comm_create on its current CUDA device (collective; ncclCommInitRank).  NCCL is loaded at run time: the copy the process
 * already carries (e.g. PyTorch's) or the system libnccl.so.2; MCS_ERR_UNSUPPORTED when there is none. */
typedef struct mcs_comm mcs_comm;
int  mcs_comm_unique_id(uint8_t* id128);
int  mcs_comm_create(const uint8_t* id128, int32_t rank, int32_t world, mcs_comm** out);
void mcs_comm_destroy(mcs_comm* comm);
int  mcs_comm_info(const mcs_comm* comm, int32_t* rank, int32_t* world, int32_t* nccl_version);

/* The single exchange of the path, the device-side counterpart of cMultiFrame's camera-order concatenation (ref
 * src/cMultiFrame.cpp:168-184): every rank contributes its packed buffer (`bytes` identical on all ranks) and receives
 * world * bytes in rank order in gathered_dev.  One ncclAllGather on `stream` (a cudaStream_t as void*), asynchronous: issue it
 * right behind the extraction on the same stream, or on a second stream behind an event to overlap it with the next batch. */
int  mcs_allgather_features(mcs_comm* comm, const void* packed_dev, size_t bytes, void* gathered_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MCS_B200_H */
