/*
 * derp_b200.h — C ABI of the H100-native depth-estimation hot path.
 *
 * The reference (facebook360_dep, source/depth_estimation) has no FFI for this path: its
 * stages are free functions over PyramidLevel<cv::Vec3w>& (Derp.h:57-161) linked statically
 * into DerpCLI / TemporalBilateralFilter / UpsampleDisparity.  This header is the boundary a
 * maintainer would bind instead: one opaque context per (GPU, stream) that owns all device
 * buffers of one pyramid level of one frame, and one entry point per reference stage.
 * Every entry point cites the reference function it replaces.
 *
 * Conventions
 *   - all functions return 0 on success, a negative DERP_E* code on failure;
 *     derp_last_error() returns a thread-local human readable message.
 *   - in the CUDA library, every image, plane, mask and output argument (and every entry of an array of them) may be
 *     pageable or pinned host memory, memory of any CUDA device, or managed memory; the checker libraries take host
 *     memory.  Descriptors, options, arrays of pointers and scalar results are host memory.  The caller owns its
 *     buffers; the library owns device memory inside DerpCtx.
 *   - images are row-major, top row first, tightly packed:
 *       colour  : uint16_t[H][W][3]  (B,G,R — cv::Vec3w, DerpUtil.h:19)
 *       float   : float[H][W]
 *       mask    : uint8_t[H][W]      (0 / non-zero — cv::Mat_<bool>)
 *       warp    : float[H][W][2]     (x,y — cv::Vec2f)
 *   - `dst` is an index into the destination list given to derp_create (rigDst),
 *     `src` an index into the camera list (rigSrc).
 *   - a context is not thread-safe; different contexts are independent.
 *
 * Two shared libraries export exactly this ABI:
 *   facebook360_dep_b200/libderp_b200.so  — the product: hand-written sm_90a CUDA
 *   oracle/libderp_oracle.so              — TEST INFRASTRUCTURE ONLY: CPU restatement
 */
#ifndef DERP_B200_H_
#define DERP_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DERP_OK 0
#define DERP_EINVAL (-1)   /* bad argument / precondition (reference: glog CHECK failure) */
#define DERP_ECUDA (-2)    /* CUDA runtime error */
#define DERP_ENOMEM (-3)
#define DERP_ESTATE (-4)   /* call sequence error (e.g. stage before derp_reproject) */
#define DERP_ECOVERAGE (-5)/* Derp.cpp:339 CHECK(partialCoverage || useForegroundMasks) */

/* Camera::Type, source/util/Camera.h:43 */
#define DERP_CAM_FTHETA 0
#define DERP_CAM_RECTILINEAR 1
#define DERP_CAM_EQUISOLID 2
#define DERP_CAM_ORTHOGRAPHIC 3

/* One camera exactly as the rig JSON states it (Camera.cpp:30-75, docs/rig.md).
 * Derived state (re-unitarised rotation Camera.cpp:77-87, distortionMax Camera.cpp:119-154,
 * cosFov Camera.cpp:204-207) is computed inside the library. */
typedef struct DerpCameraDesc {
  int32_t type;           /* DERP_CAM_* */
  int32_t has_principal;  /* 0 => principal = resolution / 2 (Camera.cpp:47-51) */
  int32_t has_fov;        /* 0 => default fov (Camera.cpp:183-195) */
  int32_t reserved;
  double origin[3];
  double forward[3];
  double up[3];
  double right[3];
  double resolution[2];
  double principal[2];
  double focal[2];
  double distortion[3];   /* missing trailing entries = 0 (Camera.cpp:53-63) */
  double fov;             /* radians from the optical axis */
} DerpCameraDesc;

/* What PyramidLevel's constructor receives (PyramidLevel.h:93-167, DerpCLI.cpp:250-271). */
typedef struct DerpLevelParams {
  int32_t width, height;            /* sizeLevel */
  int32_t level, num_levels;        /* brute force runs iff level == num_levels-1 */
  int32_t full_width, full_height;  /* rigDst[0].resolution before normalisation (DerpCLI.cpp:212-214) */
  float var_noise_floor;            /* --var_noise_floor (full-size); level value derived per PyramidLevel.h:232-236 */
  float var_high_thresh;            /* --var_high_thresh */
  int32_t use_foreground_masks;     /* --use_foreground_masks */
  int32_t reserved;
} DerpLevelParams;

/* Arguments of processLevel (Derp.cpp:1005-1034) + the constants the north-star makes tunable. */
typedef struct DerpProcessOpts {
  int32_t num_depths;             /* kNumDepths, Derp.h:33 (reference: 150) */
  float min_depth_m;              /* --min_depth_m */
  float max_depth_m;              /* --max_depth_m */
  int32_t partial_coverage;       /* --partial_coverage */
  int32_t random_proposals;       /* --random_proposals */
  int32_t ping_pong_iterations;   /* --ping_pong_iterations */
  int32_t mismatches_start_level; /* --mismatches_start_level */
  int32_t do_bilateral_filter;    /* --do_bilateral_filter */
  int32_t do_median_filter;       /* --do_median_filter */
  int32_t reserved;
} DerpProcessOpts;

typedef struct DerpCtx DerpCtx;

/* Identification: "cuda-sm_90a" for the product, "oracle-cpu" for the test oracle. */
const char* derp_backend(void);
const char* derp_last_error(void);

/* Number of host worker threads for CPU-side loops (oracle only; the CUDA library ignores it).
 * Mirrors --threads (ThreadPool.h:30-45): -1 = hardware_concurrency, 0 = inline. */
int derp_set_threads(int threads);

/* rigSrc = cams[0..num_cams), rigDst[i] = cams[dst_to_src[i]] (DerpUtil.cpp:75-88 mapSrcToDstIndexes,
 * ImageUtil.cpp:110-125 filterDestinations).  Cameras are given at full resolution; the library
 * normalises them (Camera::normalizeRig, Camera.cpp:236-242) like DerpCLI.cpp:216-218.
 * The CUDA library takes rigs of up to 64 cameras (DERP_EINVAL above; the count is checked before the
 * device is looked up); the oracle has no limit. */
int derp_create(const DerpCameraDesc* cams, int num_cams, const int32_t* dst_to_src, int num_dsts,
                int device, DerpCtx** out);
void derp_destroy(DerpCtx* ctx);

/* Stream control (CUDA library; no-ops in the oracle).  derp_set_stream makes the context enqueue
 * all its work on the caller's cudaStream_t (e.g. the stream a benchmark times with CUDA events);
 * stage functions that return no host data are then asynchronous.  derp_sync waits for the stream.
 * derp_get_launch_count reports how many kernels this context has launched so far. */
int derp_set_stream(DerpCtx* ctx, void* cuda_stream);
int derp_sync(DerpCtx* ctx);
int derp_get_launch_count(DerpCtx* ctx, uint64_t* out);
/* Optional timing of the dominant kernel (the fused sweep of derp_brute_force): while enabled, every
 * sweep launch is bracketed by CUDA events on the context's stream; derp_get_profile synchronises and
 * returns the summed device time and the number of launches since derp_profile(ctx, 1). */
int derp_profile(DerpCtx* ctx, int enable);
int derp_get_profile(DerpCtx* ctx, double* sweep_ms, uint64_t* sweep_launches);
/* The same for the dominant kernel of a fine level (pingPongKernel): summed device time, launches, and the cost
 * evaluations / contributing sources those launches performed, since derp_profile(ctx, 1). */
int derp_get_profile_ping_pong(DerpCtx* ctx, double* ms, uint64_t* launches, uint64_t* evals, uint64_t* hits);

/* How derp_brute_force sweeps (CUDA library; accepted and ignored by the CPU libraries).  Every mode produces the same
 * bytes; they differ in how much exact arithmetic runs:
 *   0  automatic: filtered when the sweep has >= 32 M (pixel, candidate) pairs (e.g. 512^2 x 128) and the bound buffer
 *      (num_depths x W x H floats) fits in memory; plain otherwise (small sweeps: the filter's extra launches cost more)
 *   1  plain sweep: the exact cost of every (pixel, candidate) (sweepKernel)
 *   2  filtered sweep: a proven lower bound of every (pixel, candidate), the exact cost only where the bound does not
 *      exclude the candidate (derp_refine.cuh)
 * derp_get_sweep_stats: exact evaluations the last filtered derp_brute_force performed (list entries, seed pixels);
 * both 0 after a plain sweep.  The work counters of derp_get_counters always count the algorithmic work
 * (every (pixel, candidate) and its contributing sources), whichever mode ran. */
int derp_set_sweep_mode(DerpCtx* ctx, int mode);
int derp_get_sweep_stats(DerpCtx* ctx, uint64_t* refined, uint64_t* seeds);

/* Starts one (frame, level): allocates level buffers, zero-fills disparity/cost/confidence/
 * mismatch mask (PyramidLevel.h:206-230) and builds the dst FOV masks
 * (generateFovMasks, DerpUtil.cpp:259-276).  Invalidates everything from the previous level. */
int derp_level_begin(DerpCtx* ctx, const DerpLevelParams* p);

/* Source colours of all cameras, colors[s] = uint16_t[H][W][3] (e.g. a level that derp_downscale_area produced on
 * the device); also computes the per-source
 * variance (PyramidLevel::computeVariances PyramidLevel.h:232-247, computeImageVariance
 * DerpUtil.cpp:214-237). */
int derp_set_colors(DerpCtx* ctx, const uint16_t* const* colors);
/* Optional (use_foreground_masks): masks[s] per source camera, background[d] per destination. */
int derp_set_foreground_masks(DerpCtx* ctx, const uint8_t* const* masks);
int derp_set_background_disparity(DerpCtx* ctx, const float* const* background);

/* reprojectColors + precomputeProjections for ONE destination (Derp.cpp:955-1003): builds, for
 * every source s, projWarp(dst,s) (src px -> dst px at infinity), projColor(dst,s)
 * (cv::remap INTER_CUBIC of the source through projWarpInv) and projColorBias (3x3 box mean).
 * The tables of one destination are resident at a time; cost-evaluating stages below require
 * them to be current for their `dst`. */
int derp_reproject(DerpCtx* ctx, int dst);

/* computeBruteForceDisparity (Derp.cpp:264-382): fused sweep + winner-takes-all.
 * best_index (optional, int32_t[H][W]) receives the winning candidate index, -1 where no
 * candidate had a finite cost, -2 outside FOV, -3 outside the foreground mask; border pixels get
 * the index of the clamped interior pixel. */
int derp_brute_force(DerpCtx* ctx, int dst, int num_depths, float min_depth_m, float max_depth_m,
                     int partial_coverage, int32_t* best_index);
/* randomProposal(s) (Derp.cpp:750-873) — no level test here; the caller decides (processLevel). */
int derp_random_proposals(DerpCtx* ctx, int dst, int num_proposals, float min_depth_m,
                          float max_depth_m);
/* pingPong (Derp.cpp:480-538) */
int derp_ping_pong(DerpCtx* ctx, int dst, int iterations);
/* handleDisparityMismatches body for all destinations (Derp.cpp:685-748); needs num_dsts == num_cams. */
int derp_mismatches(DerpCtx* ctx);
/* The same stage when the destination cameras of one frame are dealt to several contexts (one per GPU,
 * SURVEY.md 8(e)(i)): the Jacobi update of handleDisparityMismatches (Derp.cpp:734-747) reads the
 * pre-update disparity of EVERY camera, so one all-gather per level is the only exchange.
 *   derp_disparity_device_ptr  address of this context's disparity plane of `dst` (device memory on the
 *                              CUDA library, host memory on the oracle) for a zero-copy exchange;
 *   derp_gather_disparities    planes[s] = disparity of camera s (num_cams entries): host memory, memory
 *                              of this device or of a peer device (NVLink copy), or NULL for a camera
 *                              this context owns as a destination.  Copies into a context-owned
 *                              all-camera buffer and returns when the copies are complete;
 *   derp_mismatches_gathered   the stage for this context's destinations against the gathered planes.
 * Callers put a barrier between the last two calls so that no peer still reads a plane being updated. */
const float* derp_disparity_device_ptr(DerpCtx* ctx, int dst);
int derp_gather_disparities(DerpCtx* ctx, const float* const* planes);
int derp_mismatches_gathered(DerpCtx* ctx);
/* bilateralFilter (Derp.cpp:875-902) / medianFilter (Derp.cpp:904-920) / maskFov (Derp.cpp:940-951) */
int derp_bilateral(DerpCtx* ctx, int dst);
int derp_median(DerpCtx* ctx, int dst);
int derp_mask_fov(DerpCtx* ctx, int dst);

/* upsampleDisparities for one destination (UpsampleDisparityLib.cpp:98-182): writes the level's
 * disparity from a coarser map.  coarse_mask / fine_mask are the destination's foreground masks at
 * both sizes (ignored unless use_foreground_masks). */
int derp_upsample_from(DerpCtx* ctx, int dst, const float* coarse, int coarse_w, int coarse_h,
                       const uint8_t* coarse_mask, const uint8_t* fine_mask);

/* In-memory level hand-off.  The reference writes every level's disparities as PFM files and reads the coarser level
 * back from disk before it upsamples it (DerpCLI.cpp:276-303, loadImages of getLevelDisparityDir(level + 1)).
 * derp_level_keep snapshots the finished level's disparity planes inside the context (device memory on the CUDA library,
 * stream-ordered, no host copy); after derp_level_begin + derp_set_colors of the next finer level,
 * derp_upsample_from_kept does what derp_upsample_from does, from that snapshot.  Same bytes as the file round trip. */
int derp_level_keep(DerpCtx* ctx);
int derp_upsample_from_kept(DerpCtx* ctx, int dst, const uint8_t* coarse_mask, const uint8_t* fine_mask);

/* processLevel minus file output (Derp.cpp:1005-1034) for all destinations. */
int derp_process_level(DerpCtx* ctx, const DerpProcessOpts* opts);
/* The two halves of derp_process_level around the mismatch stage, for callers that exchange
 * disparities between contexts there: estimate = reprojection + brute force | proposals + ping-pong
 * (Derp.cpp:1024-1027), filter = bilateral + median + maskFov (Derp.cpp:1029-1035).
 * derp_process_level == estimate; derp_mismatches when the level asks for it; filter. */
int derp_level_estimate(DerpCtx* ctx, const DerpProcessOpts* opts);
int derp_level_filter(DerpCtx* ctx, const DerpProcessOpts* opts);

/* Cost of one hypothesis per pixel: out_cost/out_conf[y][x] = computeCost(dst, disparity[y][x], x, y)
 * (Derp.cpp:104-226) on interior pixels, NaN on the 1-px border.  Test/diagnostic entry. */
int derp_eval_cost(DerpCtx* ctx, int dst, const float* disparity, float* out_cost, float* out_conf);

/* Caller <-> context state. NULL pointers are skipped. */
int derp_set_disparity(DerpCtx* ctx, int dst, const float* disparity, const float* cost,
                       const float* confidence);
int derp_get_disparity(DerpCtx* ctx, int dst, float* disparity, float* cost, float* confidence);
int derp_get_fov_mask(DerpCtx* ctx, int dst, uint8_t* mask);
int derp_get_mismatch_mask(DerpCtx* ctx, int dst, uint8_t* mask);
int derp_get_variance(DerpCtx* ctx, int src, float* variance);
int derp_get_var_noise_floor(DerpCtx* ctx, float* out);
/* Tables of the destination last passed to derp_reproject. */
int derp_get_proj_warp(DerpCtx* ctx, int src, float* warp_xy);
int derp_get_proj_color(DerpCtx* ctx, int src, uint16_t* bgr);
int derp_get_proj_bias(DerpCtx* ctx, int src, uint16_t* bgr);
/* Work counters of the last cost-evaluating stage: number of computeCost calls and the number
 * of (call, source) pairs whose source camera saw the point (sum of ssdCount). */
int derp_get_counters(DerpCtx* ctx, uint64_t* cost_evals, uint64_t* src_hits);

/* temporalJointBilateralFilter (TemporalBilateralFilter.h:126-215) for one camera.
 * guides[t] colour, disps[t] float, masks[t] uint8 (fg & fov of frame t), t in [0, num_frames). */
int derp_temporal_filter(int device, int width, int height, int num_frames,
                         const uint16_t* const* guides, const float* const* disps,
                         const uint8_t* const* masks, int frame_offset, float sigma,
                         int spatial_radius, float weight0, float weight1, float weight2,
                         float* out);

/* generalizedJointBilateralFilter<float, Vec3f> exactly as UpsampleDisparity.cpp:118-128 calls it
 * (that file re-defines PixelType = cv::Vec3f, UpsampleDisparity.cpp:57; TemporalBilateralFilter.h:39-124):
 * guide = float BGR in [0,1] as cv_util::loadImage<Vec3f> produces it (u16 * (1/65535.f), u8 * (1/255.f)),
 * mask as given (not AND-ed with the FOV mask), weights passed as (weight_b, weight_g, weight_r). */
int derp_joint_bilateral_f32(int device, int width, int height, const float* image,
                             const float* guide_bgr, const uint8_t* mask, int radius, float sigma,
                             float weight0, float weight1, float weight2, float* out);

/* Stand-alone upsampling as the UpsampleDisparity app needs it (UpsampleDisparityLib.cpp:98-182)
 * for one camera; fov masks are derived from `cam`. */
int derp_upsample_disparity(int device, const DerpCameraDesc* cam, const float* coarse, int coarse_w,
                            int coarse_h, const float* background_up, const uint8_t* coarse_mask,
                            const uint8_t* fine_mask, int out_w, int out_h,
                            int use_foreground_masks, float* out);

/* Device memory for callers that keep frames resident between calls (e.g. the temporal filter's sliding window):
 * derp_device_alloc / derp_device_free on `device`; derp_device_copy copies `bytes` between any two addresses — host,
 * this device or a PEER device (NVLink copy; peer access is enabled on first use).  The CPU libraries implement the
 * three with malloc / free / memcpy so that callers need no second code path in tests. */
int derp_device_alloc(int device, size_t bytes, void** out);
int derp_device_free(int device, void* p);
int derp_device_copy(int device, void* dst, const void* src, size_t bytes);

/* cv::resize(..., INTER_AREA) of a 3-channel 16-bit image, shrinking only: the resize scripts/render/resize.py:51-85
 * builds every pyramid level with (each level from the FULL-SIZE image, widths scripts/render/config.py:46), and the resize of
 * GenerateForegroundMasks' 16-bit inputs.  Bit-identical to OpenCV for integer
 * ratios (resizeAreaFast_) and general ratios (computeResizeAreaTab / ResizeArea_Invoker<ushort, float>). */
int derp_downscale_area(int device, const uint16_t* src, int src_w, int src_h, uint16_t* dst, int dst_w, int dst_h);

/* generateForegroundMask<cv::Vec3w, cv::Vec3f> (source/render/BackgroundSubtractionUtil.h:20-59), the per-camera body of
 * the GenerateForegroundMasks app that produces the masks --use_foreground_masks consumes: Gaussian blur of template
 * (background) and frame (blur_radius 0 or 1 = the app's default 3 x 3 kernel), conversion to [0, 1] floats,
 * mask = ||template - frame||_2 > threshold, morphological closing with a morph_closing_size^2 rectangle.
 * Images u16 HxWx3, mask uint8 HxW with values 0 / 1. */
int derp_foreground_mask(int device, const uint16_t* templ, const uint16_t* frame, int width, int height, int blur_radius,
                         float threshold, int morph_closing_size, uint8_t* mask);

/* Camera mesh of one disparity map, the geometry half of ConvertToBinary's convertDepth BEFORE mesh simplification
 * (source/mesh_stream/ConvertToBinary.cpp:150-183; SURVEY §8(f) rank 4, first slice): depth = 1 / disparity, optional
 * INTER_NEAREST shrink by depth_scale (< 1; 1 = none), mesh_util::getVertexesEquiError (source/render/MeshUtil.h:313-338),
 * mesh_util::getFaces(wrapHorizontally = false, isRigCoordinates = false, tear_ratio) (MeshUtil.h:162-298), vertex mask =
 * !isnan(depth) [& bit 0 of the foreground mask, resized INTER_NEAREST to the depth grid],
 * mesh_util::applyMaskToVertexesAndFaces (MeshUtil.h:342-403).  Outputs in the layout mesh_util::writeDepth stores as
 * .vtx / .idx (MeshUtil.h:74-93): float32 x, y, z per vertex, uint32 x 3 per face, in the reference's order.
 * resolution_* / scalar_focal: the camera's (possibly rescaled, ConvertToBinary.cpp:322-343) resolution and
 * Camera::getScalarFocal().  `vertexes` needs room for 3 floats per grid cell, `faces` for 6 uint32 per grid cell
 * (derp_camera_mesh_size gives the grid).
 * derp_camera_mesh_simplified adds the simplification step (ConvertToBinary.cpp:186-203): render::MeshSimplifier
 * (source/render/MeshSimplifier.cpp: quadric-error edge contraction, equi-error costs, strictness 0.2, boundary edges kept)
 * down to `triangles` faces when the mesh has more, then z < 0 -> FLT_MIN.  That stage is a chain of dependent
 * contractions (one thread in the reference's call): the GPU builds the mesh in double precision, the contraction sweeps
 * run on the host inside the library. */
int derp_camera_mesh_size(int width, int height, double depth_scale, int* mesh_width, int* mesh_height);
int derp_camera_mesh(int device, const float* disparity, int width, int height, double depth_scale, double resolution_x,
                     double resolution_y, double scalar_focal, float tear_ratio, const uint8_t* foreground_mask,
                     int mask_width, int mask_height, float* vertexes, uint32_t* faces, uint64_t* num_vertexes,
                     uint64_t* num_faces);
int derp_camera_mesh_simplified(int device, const float* disparity, int width, int height, double depth_scale,
                                double resolution_x, double resolution_y, double scalar_focal, float tear_ratio,
                                const uint8_t* foreground_mask, int mask_width, int mask_height, int triangles,
                                float* vertexes, uint32_t* faces, uint64_t* num_vertexes, uint64_t* num_faces);

/* BC7 colour of ConvertToBinary's convertColor (ConvertToBinary.cpp:122-138; the default --output_formats holds bc7).
 * derp_bc7_compress replaces CompressBlocksBC7(&surface, out, &settings) with GetProfile_veryfast(&settings)
 * (source/conversion/BC7Util.h:69-76; the ISPC texture compressor vendored under source/thirdparty/bc7_compressor,
 * ispc_texcomp.cpp:61-93, kernel.ispc:615-2036): an RGBA8 surface (width * 4 bytes per row, alpha ignored = opaque) to
 * 16-byte blocks, block row r starting at byte r * width * 4; `blocks` holds width * height bytes and is zeroed first,
 * partial edge blocks (width or height not a multiple of 4) are not encoded — all as the reference does.
 * derp_bc7_compress_image replaces bc7_util::compressBC7(image, ...) up to the file write (BC7Util.h:45-76): `pixels` is the
 * image as cv::imread(IMREAD_UNCHANGED) returns it (B, G, R[, A] interleaved, 8 or 16 bits per channel); conversion to
 * [0, 1] floats (CvUtil.h:196-207), bc7_util::gammaCorrect (BC7Util.h:41-43) and the RGBA packing are fused into the
 * block loads through a lookup table over the stored channel values, built on the host with the host's powf.
 * Modes tried: 1 and 3 (best 3 / 1 of the 64 partitions by the residual bound), 6; same operation order, x86 conversion
 * semantics and end-point quantisation as the reference BUILD, IEEE division / square root where that build uses the
 * RCPPS / RSQRTPS estimates (so individual blocks can differ where an estimate's last bit decides; see derp_bc7.cuh). */
int derp_bc7_compress(int device, const uint8_t* rgba, int width, int height, uint8_t* blocks);
int derp_bc7_compress_image(int device, const void* pixels, int bits_per_channel, int channels, int width, int height,
                            float gamma, uint8_t* blocks);

#ifdef __cplusplus
}
#endif
#endif /* DERP_B200_H_ */
