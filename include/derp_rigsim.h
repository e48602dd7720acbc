/*
 * derp_rigsim.h — C ABI of RigSimulator (source/rig/RigSimulator.cpp): the synthetic scene, its sphere-tree BVH and the
 * ray tracer that renders rig cameras and equirects with ground-truth depth, on the H100.
 *
 * Exported by facebook360_dep_b200/libderp_b200.so next to the depth ABI of derp_b200.h, whose conventions it follows:
 * 0 on success, a negative DERP_E* code on failure with the message in derp_last_error(); images row-major, top row
 * first, tightly packed; every output pointer may be host or device memory (device memory of the current device is
 * written in place).
 *
 * Scene and BVH (host code, because they consume the process's rand() stream in the reference's order; the caller seeds
 * it with srand, the reference app never does):
 *   derp_rigsim_scene_create: makeIcosahedronScene / makeCubesScene / makeGroundPlaneScene (RigSimulator.cpp:264-358),
 *     selfIdx binding and BoundingVolumeHierarchy::makeBVH(triangles, 20, 5, 0, 50) (RigSimulator.cpp:680-696,
 *     BoundingVolumeHierarchy.h:32-112).  The BVH is flattened in preorder: node k holds its sphere, the range
 *     [first, first + count) of leaf triangles (count = 0 for an inner node) and `escape`, the preorder index of the
 *     first node after its subtree.  leaf_tris lists, in preorder, the scene index of every leaf's triangles.
 *   derp_rigsim_scene_info / derp_rigsim_scene_get: the counts, then copies of the triangles (Triangle's constructor,
 *     RaytracingPrimitives.h:45-49: e1, e2 and the normalised normal), the nodes and the leaf triangle list.
 *
 * Rendering (the trace kernel: one thread per supersample ray; the area kernel: INTER_AREA by the integer factor aas):
 *   derp_rigsim_render_cameras: renderCamera (RigSimulator.cpp:591-625) for every camera, without the noise
 *     (corruptImageWithNoise stays on the host): bgr[i] receives [res.y][res.x][3] floats (255 * B, G, R) and depth[i]
 *     [res.y][res.x] floats (FLT_MAX where nothing is hit or the supersample is outside the image circle; INTER_AREA
 *     sums of FLT_MAX overflow to inf as in OpenCV).  Cameras are used as given (not normalised); the resolution must
 *     be integral.
 *   derp_rigsim_render_equirect: renderMonoEquirect (stereo = 0: out0 = BGR, out1 = clamp(1 / depth, 0, 1)) or
 *     renderStereoEquirect (stereo = 1: out0 = left BGR, out1 = right BGR) (RigSimulator.cpp:519-589), width x height.
 *   The sky texel (traceRayToGetColor's acosf / atan2f, RigSimulator.cpp:222-237) is decided on the device only where
 *   an interval evaluation proves the C library's result; the other rays are recomputed on the host with the same code
 *   (derp_rigsim.cuh documents the bound).  derp_rigsim_last_host_rays: the number of rays the calling thread's last
 *   render resolved on the host (its share of derp_rigsim_last_rays, the supersample rays traced).
 *   derp_test_rigsim_area: the area kernel alone on src ([dh k][dw k][cn] floats) into dst ([dh][dw][cn]), for tests.
 *   derp_test_sky_texel: a probe of the device's proof of the sky texel, for tests: skyTexelDevice of the directions
 *     dirs[3 i .. 3 i + 2] of a rows x cols skybox into texel[2 i] (row) and texel[2 i + 1] (column), or (-1, -1) where
 *     the device leaves the ray to the host; on `device` with host pointers.
 *   derp_test_sky_texel_host: its host twin (the C library's acosf and atan2f), which always decides.
 *   derp_rigsim_trace_host: traceRayToGetColor (RigSimulator.cpp:196-262) on the host for n fp32 rays {origin, dir}:
 *     out[4 i .. 4 i + 3] = B, G, R (0..1), depth.  For tests without a GPU.
 */
#ifndef DERP_RIGSIM_H_
#define DERP_RIGSIM_H_

#include "derp_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

enum { DERP_RIGSIM_ICOSAHEDRON = 0, DERP_RIGSIM_CUBE = 1, DERP_RIGSIM_GROUND_PLANE = 2 };

/* The scene flags of RigSimulator.cpp:46-121 */
typedef struct DerpRigsimSceneParams {
  int32_t scene;                   /* --scene: DERP_RIGSIM_* */
  int32_t num_random_icosahedrons; /* --num_random_icosahedrons */
  int32_t red_triangle;            /* --red_triangle */
  int32_t reserved;
  double min_icosahedron_dist;     /* --min_icosahedron_dist */
  double max_icosahedron_dist;     /* --max_icosahedron_dist */
  double min_icosahedron_radius;   /* --min_icosahedron_radius */
  double max_icosahedron_radius;   /* --max_icosahedron_radius */
  double ground_plane_dist_m;      /* --ground_plane_dist_m */
} DerpRigsimSceneParams;

/* Triangle (RaytracingPrimitives.h:36-50) without selfIdx, which is the triangle's index in the scene */
typedef struct DerpRigsimTriangle {
  float v0[3], v1[3], v2[3], e1[3], e2[3], normal[3], color[3];
} DerpRigsimTriangle;

typedef struct DerpRigsimNode {
  float center[3];
  float radius;
  int32_t first, count, escape, reserved;
} DerpRigsimNode;

/* The rendering flags of RigSimulator.cpp:46-121 and the images they name */
typedef struct DerpRigsimRender {
  int32_t anti_alias_supersample; /* --anti_alias_supersample, >= 1 */
  int32_t marble;                 /* --marble */
  double marble_scale;            /* --marble_scale */
  double interpupillary_radius;   /* --interpupillary_radius (stereo equirect) */
  const uint8_t* skybox_bgr;      /* the skybox, 8-bit B, G, R, host memory */
  int32_t skybox_width, skybox_height;
  const uint8_t* ceiling_bgr;     /* the --ceiling_path image, 8-bit B, G, R, host memory; NULL: no ceiling */
  int32_t ceiling_cols, ceiling_rows;
  double ceiling_position;        /* --ceiling_position */
  double ceiling_width;           /* --ceiling_width */
  double ceiling_depth;           /* --ceiling_depth */
} DerpRigsimRender;

typedef struct DerpRigsimScene DerpRigsimScene;

int derp_rigsim_scene_create(const DerpRigsimSceneParams* params, DerpRigsimScene** out);
void derp_rigsim_scene_destroy(DerpRigsimScene* scene);
int derp_rigsim_scene_info(const DerpRigsimScene* scene, int32_t* num_triangles, int32_t* num_nodes,
                           int32_t* num_leaf_tris);
int derp_rigsim_scene_get(const DerpRigsimScene* scene, DerpRigsimTriangle* triangles, DerpRigsimNode* nodes,
                          int32_t* leaf_tris);

int derp_rigsim_render_cameras(int device, const DerpRigsimScene* scene, const DerpRigsimRender* opts,
                               const DerpCameraDesc* cams, int num_cams, float* const* bgr, float* const* depth);
int derp_rigsim_render_equirect(int device, const DerpRigsimScene* scene, const DerpRigsimRender* opts, int stereo,
                                int width, int height, float* out0, float* out1);
uint64_t derp_rigsim_last_host_rays(void);
uint64_t derp_rigsim_last_rays(void);

int derp_test_rigsim_area(int device, const float* src, int dw, int dh, int cn, int k, float* dst);
int derp_test_sky_texel(int device, const float* dirs, int n, int rows, int cols, int32_t* texel);
int derp_test_sky_texel_host(const float* dirs, int n, int rows, int cols, int32_t* texel);
int derp_rigsim_trace_host(const DerpRigsimScene* scene, const DerpRigsimRender* opts, const float* rays, int n,
                           float* out);

#ifdef __cplusplus
}
#endif
#endif /* DERP_RIGSIM_H_ */
