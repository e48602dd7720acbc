// include/derp_rigsim.h: RigSimulator's trace and INTER_AREA kernels on sm_90a (per-ray code in derp_rigsim.cuh), the
// host scene and BVH, and the host instantiation of the per-ray code for the CPU tests.
#include "derp_host.cuh"
#include "derp_rigsim.cuh"

using namespace derp;
using namespace derp::rigsim;

struct DerpRigsimScene {
  std::vector<DerpRigsimTriangle> tris;
  std::vector<DerpRigsimNode> nodes;
  std::vector<int> leafTris;
};

namespace {

// A supersample whose sky texel the device left undecided: its index in the supersampled plane and its direction
struct SkyRay {
  unsigned pixel;
  float d[3];
};
// What the second plane of a render holds: the depth (cameras), clamp(1 / depth, 0, 1) (mono equirect) or nothing
enum Plane2 { kDepth = 0, kInvDepth = 1, kNone = 2 };

struct RigsimScratch {
  DevBuf<DerpRigsimNode> nodes;
  DevBuf<int> leafTris;
  DevBuf<DerpRigsimTriangle> tris;
  DevBuf<uint8_t> sky, ceil;
  DevBuf<float> bgrSS, p2SS, out0, out1, tables;
  UndecidedList<SkyRay> undecided;
  DevBuf<int2> texels;
  DevBuf<DevCamera> cam;
};
thread_local RigsimScratch g_rig;
thread_local unsigned long long g_rigHostRays = 0, g_rigRays = 0;

// One supersample's result into the supersampled planes: 255 * BGR and the second plane
__device__ __forceinline__ void store(const float* c, size_t at, float* bgr, float* p2, int plane2) {
  bgr[3 * at] = 255.0f * c[0];
  bgr[3 * at + 1] = 255.0f * c[1];
  bgr[3 * at + 2] = 255.0f * c[2];
  if (plane2 == kDepth) {
    p2[at] = c[3];
  } else if (plane2 == kInvDepth) {
    const float v = 1.0f / c[3];
    p2[at] = v < 0.0f ? 0.0f : v > 1.0f ? 1.0f : v;  // math_util::clamp
  }
}

// The rest of traceRayToGetColor on the device: the sky texel when the interval proves it, else the ray is listed
__device__ __forceinline__ void shadeRay(const SceneView& s, V3 o, V3 d, size_t at, float* bgr, float* p2, int plane2,
                                         UndecidedView<SkyRay> undecided) {
  float c[4];
  if (!traceRay(s, o, d, c)) {
    int row, col;
    if (!skyTexelDevice(d, s.skyH, s.skyW, &row, &col)) {
      undecided.append(SkyRay{(unsigned)at, {d.x, d.y, d.z}});
      return;
    }
    skyColor(s, row, col, c);
  }
  store(c, at, bgr, p2, plane2);
}

// renderCamera's supersamples (RigSimulator.cpp:598-621): pixel = ((x + 0.5f) / aas, (y + 0.5f) / aas) in fp32;
// outside the image circle (0, 0, 0, FLT_MAX), else cam.rig(pixel) narrowed to fp32 and traced
__global__ void __launch_bounds__(kTraceThreadsX* kTraceThreadsY)
    traceCameraKernel(SceneView s, const DevCamera* __restrict__ cam, int W, int H, int aas, float* bgr, float* depth,
                      UndecidedView<SkyRay> undecided) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  const DevCamera& c = *cam;
  const size_t at = (size_t)y * W + x;
  const double px = (x + 0.5f) / aas, py = (y + 0.5f) / aas;
  if (outsideImageCircle(c, px, py)) {
    const float zero[4] = {0, 0, 0, FLT_MAX};
    store(zero, at, bgr, depth, kDepth);
    return;
  }
  double dir[3];
  pixelRay(c, px, py, dir);
  shadeRay(s, v3((float)c.pos[0], (float)c.pos[1], (float)c.pos[2]), v3((float)dir[0], (float)dir[1], (float)dir[2]),
           at, bgr, depth, kDepth, undecided);
}

// renderMonoEquirect / renderStereoEquirect's supersamples (RigSimulator.cpp:529-545, 558-585): the direction
// (sinf(phi) cosf(theta), sinf(phi) sinf(theta), cosf(phi)) from the host's per-row and per-column tables, in fp32; the
// origin 0 (mono) or the column's eye (stereo)
__global__ void __launch_bounds__(kTraceThreadsX* kTraceThreadsY)
    traceEquirectKernel(SceneView s, int W, int H, const float* __restrict__ tab, const float* __restrict__ eyes,
                        float* bgr, float* p2, int plane2, UndecidedView<SkyRay> undecided) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  const float sinP = tab[y], cosP = tab[H + y], cosT = tab[2 * H + x], sinT = tab[2 * H + W + x];
  const V3 o = eyes ? v3(eyes + 3 * x) : v3(0.0f, 0.0f, 0.0f);
  shadeRay(s, o, v3(sinP * cosT, sinP * sinT, cosP), (size_t)y * W + x, bgr, p2, plane2, undecided);
}

// The listed supersamples, with the texels the host found
__global__ void resolveSkyKernel(SceneView s, const SkyRay* __restrict__ list, const int2* __restrict__ texels, int n,
                                 float* bgr, float* p2, int plane2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float c[4];
  skyColor(s, texels[i].x, texels[i].y, c);
  store(c, list[i].pixel, bgr, p2, plane2);
}

// INTER_AREA by the integer factor k of an image of cn channels (resizeAreaFast_, as csrc/host/area_resize.h states
// and tests/golden/rigsim_vectors.npz pins to cv2): factor 2 with 1 channel takes ((a + b) + (c + d)) * 0.25f; any
// other case sums the k * k samples in row order into a float, four at a time (sum += ((s0 + s1) + s2) + s3), then
// multiplies by 1.f / (k * k).  k = 1 copies.
__global__ void areaKernel(const float* __restrict__ src, int dw, int dh, int cn, int k, float* __restrict__ dst) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t n = (size_t)dw * dh * cn;
  if (i >= n) return;
  const int c = (int)(i % cn);
  const size_t p = i / cn;
  const int x = (int)(p % dw), y = (int)(p / dw);
  const size_t row = (size_t)dw * k * cn;
  const float* S = src + (size_t)y * k * row + (size_t)x * k * cn + c;
  if (k == 1) {
    dst[i] = S[0];
    return;
  }
  if (k == 2 && cn == 1) {
    dst[i] = ((S[0] + S[cn]) + (S[row] + S[row + cn])) * 0.25f;
    return;
  }
  const int area = k * k;
  float sum = 0;
  int j = 0;
  for (; j <= area - 4; j += 4)
    sum += S[(size_t)(j / k) * row + (size_t)(j % k) * cn] + S[(size_t)((j + 1) / k) * row + (size_t)((j + 1) % k) * cn] +
           S[(size_t)((j + 2) / k) * row + (size_t)((j + 2) % k) * cn] +
           S[(size_t)((j + 3) / k) * row + (size_t)((j + 3) % k) * cn];
  for (; j < area; ++j) sum += S[(size_t)(j / k) * row + (size_t)(j % k) * cn];
  dst[i] = sum * (1.f / area);
}

int checkRender(const char* who, const DerpRigsimScene* scene, const DerpRigsimRender* o) {
  const std::string w(who);
  if (!scene || !o) return fail(DERP_EINVAL, w + ": scene and options are required");
  if (o->anti_alias_supersample < 1) return fail(DERP_EINVAL, w + ": anti_alias_supersample must be at least 1");
  if (!o->skybox_bgr || o->skybox_width < 1 || o->skybox_height < 1 ||
      (long long)o->skybox_width * o->skybox_height >= (1ll << 30))
    return fail(DERP_EINVAL, w + ": a skybox image is required");
  if (o->ceiling_bgr && (o->ceiling_cols < 1 || o->ceiling_rows < 1 ||
                         (long long)o->ceiling_cols * o->ceiling_rows >= (1ll << 30)))
    return fail(DERP_EINVAL, w + ": bad ceiling image");
  return DERP_OK;
}

SceneView hostView(const DerpRigsimScene* sc, const DerpRigsimRender* o) {
  return SceneView{sc->nodes.data(),  sc->leafTris.data(), sc->tris.data(),     o->skybox_bgr,     o->skybox_width,
                   o->skybox_height,  o->ceiling_bgr,      o->ceiling_cols,     o->ceiling_rows,   o->ceiling_position,
                   o->ceiling_width,  o->ceiling_depth,    o->marble,           o->marble_scale};
}

// Device copies of the scene and the images
int uploadScene(const DerpRigsimScene* sc, const DerpRigsimRender* o, SceneView& v) {
  RigsimScratch& g = g_rig;
  if (int rc = upload(g.nodes, sc->nodes.data(), sc->nodes.size())) return rc;
  if (sc->tris.empty()) {  // a scene without triangles: the root is an empty leaf, nothing is read
    CU(g.leafTris.ensure(1));
    CU(g.tris.ensure(1));
  } else {
    if (int rc = upload(g.leafTris, sc->leafTris.data(), sc->leafTris.size())) return rc;
    if (int rc = upload(g.tris, sc->tris.data(), sc->tris.size())) return rc;
  }
  if (int rc = upload(g.sky, o->skybox_bgr, (size_t)o->skybox_width * o->skybox_height * 3)) return rc;
  v = hostView(sc, o);
  v.nodes = g.nodes.p;
  v.leafTris = g.leafTris.p;
  v.tris = g.tris.p;
  v.sky = g.sky.p;
  if (o->ceiling_bgr) {
    if (int rc = upload(g.ceil, o->ceiling_bgr, (size_t)o->ceiling_cols * o->ceiling_rows * 3)) return rc;
    v.ceil = g.ceil.p;
  }
  return DERP_OK;
}

// Launches `trace` (which lists undecided sky rays), resolves the listed rays on the host and writes them; returns the
// number of host rays in *hostRays
template <class Launch>
int traceAndResolve(const SceneView& v, Launch trace, float* bgr, float* p2, int plane2, unsigned long long* hostRays) {
  RigsimScratch& g = g_rig;
  std::vector<SkyRay> list;
  if (int rc = g.undecided.collect(trace, list)) return rc;
  const size_t count = list.size();
  *hostRays += count;
  if (!count) return DERP_OK;
  std::vector<int2> tex(count);
  for (size_t k = 0; k < count; ++k) {
    int row, col;
    skyTexelHost(v3(list[k].d), v.skyH, v.skyW, &row, &col);
    tex[k] = make_int2(row, col);
  }
  if (int rc = upload(g.texels, tex.data(), count)) return rc;
  resolveSkyKernel<<<grid1(count), 256>>>(v, g.undecided.items.p, g.texels.p, (int)count, bgr, p2, plane2);
  CU(cudaGetLastError());
  return DERP_OK;
}

// INTER_AREA of the supersampled plane src (dw * k x dh * k, cn channels) into the caller's dst (in place or staged)
int downscaleInto(const float* src, int dw, int dh, int cn, int k, float* dst, DevBuf<float>& stage) {
  const size_t n = (size_t)dw * dh * cn;
  float* d = dst;
  if (int rc = outBuffer(d, n, stage)) return rc;
  areaKernel<<<grid1(n), 256>>>(src, dw, dh, cn, k, d);
  CU(cudaGetLastError());
  return stageOut(dst, d, n);
}

// Test probe: skyTexelDevice of the directions dirs[3 i .. 3 i + 2] into texel[2 i .. 2 i + 1], (-1, -1) when undecided
__global__ void skyTexelKernel(const float* dirs, int n, int rows, int cols, int32_t* texel) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int row = -1, col = -1;
  if (!skyTexelDevice(v3(dirs + 3 * i), rows, cols, &row, &col)) row = col = -1;
  texel[2 * i] = row;
  texel[2 * i + 1] = col;
}

}  // namespace

extern "C" {

int derp_rigsim_scene_create(const DerpRigsimSceneParams* p, DerpRigsimScene** out) {
  if (!p || !out) return fail(DERP_EINVAL, "derp_rigsim_scene_create: params and out are required");
  *out = nullptr;
  if (p->num_random_icosahedrons < 0 || p->num_random_icosahedrons > (1 << 20))
    return fail(DERP_EINVAL, "derp_rigsim_scene_create: num_random_icosahedrons must be 0..2^20");
  DerpRigsimScene* s = new DerpRigsimScene;
  if (p->scene == DERP_RIGSIM_ICOSAHEDRON) {
    rigsim::host::makeIcosahedronScene(*p, s->tris);
  } else if (p->scene == DERP_RIGSIM_CUBE) {
    rigsim::host::makeCubesScene(s->tris);
  } else if (p->scene == DERP_RIGSIM_GROUND_PLANE) {
    rigsim::host::makeGroundPlaneScene(*p, s->tris);
  } else {
    delete s;
    return fail(DERP_EINVAL, "derp_rigsim_scene_create: unknown scene " + std::to_string(p->scene));
  }
  std::vector<int> all(s->tris.size());
  for (size_t i = 0; i < all.size(); ++i) all[i] = (int)i;
  rigsim::host::makeBVH(s->tris, all, 20, 5, 0, 50, s->nodes, s->leafTris);  // RigSimulator.cpp:688-696
  *out = s;
  return DERP_OK;
}

void derp_rigsim_scene_destroy(DerpRigsimScene* scene) { delete scene; }

int derp_rigsim_scene_info(const DerpRigsimScene* s, int32_t* nt, int32_t* nn, int32_t* nl) {
  if (!s || !nt || !nn || !nl) return fail(DERP_EINVAL, "derp_rigsim_scene_info: bad arguments");
  *nt = (int32_t)s->tris.size();
  *nn = (int32_t)s->nodes.size();
  *nl = (int32_t)s->leafTris.size();
  return DERP_OK;
}

int derp_rigsim_scene_get(const DerpRigsimScene* s, DerpRigsimTriangle* tris, DerpRigsimNode* nodes, int32_t* leaf) {
  if (!s || !tris || !nodes || !leaf) return fail(DERP_EINVAL, "derp_rigsim_scene_get: bad arguments");
  std::copy(s->tris.begin(), s->tris.end(), tris);
  std::copy(s->nodes.begin(), s->nodes.end(), nodes);
  std::copy(s->leafTris.begin(), s->leafTris.end(), leaf);
  return DERP_OK;
}

int derp_rigsim_render_cameras(int device, const DerpRigsimScene* scene, const DerpRigsimRender* opts,
                               const DerpCameraDesc* cams, int num_cams, float* const* bgr, float* const* depth) {
  static const char* who = "derp_rigsim_render_cameras";
  if (int rc = checkRender(who, scene, opts)) return rc;
  if (!cams || num_cams < 1 || !bgr || !depth) return fail(DERP_EINVAL, std::string(who) + ": bad arguments");
  const int aas = opts->anti_alias_supersample;
  std::vector<DevCamera> c(num_cams);
  for (int i = 0; i < num_cams; ++i) {
    if (!derp::host::makeCamera(cams[i], &c[i])) return fail(DERP_EINVAL, std::string(who) + ": invalid camera " + std::to_string(i));
    const double w = c[i].res[0], h = c[i].res[1];
    if (!bgr[i] || !depth[i] || w != (double)(int)w || h != (double)(int)h || w < 1 || h < 1 ||
        w * h * aas * aas >= (double)(1ll << 30))
      return fail(DERP_EINVAL, std::string(who) + ": camera " + std::to_string(i) +
                                   " needs an integral resolution, at most 2^30 supersamples and outputs");
  }
  CU(cudaSetDevice(device));
  SceneView v;
  if (int rc = uploadScene(scene, opts, v)) return rc;
  RigsimScratch& g = g_rig;
  unsigned long long hostRays = 0, rays = 0;
  for (int i = 0; i < num_cams; ++i) {
    const int w = (int)c[i].res[0], h = (int)c[i].res[1], W = w * aas, H = h * aas;
    const size_t n = (size_t)W * H;
    CU(g.bgrSS.ensure(3 * n));
    CU(g.p2SS.ensure(n));
    if (int rc = upload(g.cam, &c[i], 1)) return rc;
    const dim3 block(kTraceThreadsX, kTraceThreadsY), grid((W + block.x - 1) / block.x, (H + block.y - 1) / block.y);
    const DevCamera* cam = g.cam.p;
    float *b = g.bgrSS.p, *d = g.p2SS.p;
    auto trace = [&](UndecidedView<SkyRay> undecided) {
      traceCameraKernel<<<grid, block>>>(v, cam, W, H, aas, b, d, undecided);
      return DERP_OK;
    };
    if (int rc = traceAndResolve(v, trace, b, d, kDepth, &hostRays)) return rc;
    rays += n;
    if (int rc = downscaleInto(b, w, h, 3, aas, bgr[i], g.out0)) return rc;
    if (int rc = downscaleInto(d, w, h, 1, aas, depth[i], g.out1)) return rc;
  }
  g_rigHostRays = hostRays;
  g_rigRays = rays;
  return DERP_OK;
}

int derp_rigsim_render_equirect(int device, const DerpRigsimScene* scene, const DerpRigsimRender* opts, int stereo,
                                int width, int height, float* out0, float* out1) {
  static const char* who = "derp_rigsim_render_equirect";
  if (int rc = checkRender(who, scene, opts)) return rc;
  const int aas = opts->anti_alias_supersample;
  if (width < 1 || height < 1 || (double)width * height * aas * aas >= (double)(1ll << 30) || !out0 || !out1)
    return fail(DERP_EINVAL, std::string(who) + ": bad size or outputs");
  const int W = width * aas, H = height * aas;
  // Host tables in the overloads the reference resolves (float sinf / cosf of float angles for the direction, double
  // sin / cos of double angles for the stereo eyes; RigSimulator.cpp:536-576)
  std::vector<float> tab(2 * (size_t)H + 2 * (size_t)W), eyes[2];
  for (int y = 0; y < H; ++y) {
    const float phi = (float)(kPi * (y + 0.5f) / float(H));
    tab[y] = sinf(phi);
    tab[H + y] = cosf(phi);
  }
  std::vector<float> theta(W);
  for (int x = 0; x < W; ++x) {
    theta[x] = (float)(2.0f * kPi * (1.0f - (x + 0.5f) / float(W)));
    tab[2 * H + x] = cosf(theta[x]);
    tab[2 * H + W + x] = sinf(theta[x]);
  }
  if (stereo) {
    for (int e = 0; e < 2; ++e) {
      eyes[e].resize(3 * (size_t)W);
      const double turn = e == 0 ? kPi / 2.0f : -kPi / 2.0f;  // theta + M_PI / 2.0f (left), theta - M_PI / 2.0f (right)
      for (int x = 0; x < W; ++x) {
        const float ex = (float)cos(theta[x] + turn), ey = (float)sin(theta[x] + turn);
        eyes[e][3 * x] = (float)(ex * opts->interpupillary_radius);
        eyes[e][3 * x + 1] = (float)(ey * opts->interpupillary_radius);
        eyes[e][3 * x + 2] = (float)(0.0f * opts->interpupillary_radius);
      }
    }
  }
  CU(cudaSetDevice(device));
  SceneView v;
  if (int rc = uploadScene(scene, opts, v)) return rc;
  RigsimScratch& g = g_rig;
  const size_t n = (size_t)W * H, nt = tab.size();
  CU(g.tables.ensure(nt + (stereo ? 6 * (size_t)W : 0)));
  CU(cudaMemcpy(g.tables.p, tab.data(), nt * sizeof(float), cudaMemcpyHostToDevice));
  if (stereo)
    for (int e = 0; e < 2; ++e)
      CU(cudaMemcpy(g.tables.p + nt + 3 * (size_t)W * e, eyes[e].data(), 3 * (size_t)W * sizeof(float),
                    cudaMemcpyHostToDevice));
  CU(g.bgrSS.ensure(3 * n));
  CU(g.p2SS.ensure(stereo ? 3 * n : n));
  const dim3 block(kTraceThreadsX, kTraceThreadsY), grid((W + block.x - 1) / block.x, (H + block.y - 1) / block.y);
  unsigned long long hostRays = 0;
  for (int e = 0; e < (stereo ? 2 : 1); ++e) {
    // mono: BGR and 1 / depth; stereo: the left eye's BGR, then the right eye's (in the second buffer)
    float* b = e == 0 ? g.bgrSS.p : g.p2SS.p;
    float* p2 = stereo ? nullptr : g.p2SS.p;
    const int plane2 = stereo ? kNone : kInvDepth;
    const float* tabs = g.tables.p;
    const float* eye = stereo ? g.tables.p + nt + 3 * (size_t)W * e : nullptr;
    auto trace = [&](UndecidedView<SkyRay> undecided) {
      traceEquirectKernel<<<grid, block>>>(v, W, H, tabs, eye, b, p2, plane2, undecided);
      return DERP_OK;
    };
    if (int rc = traceAndResolve(v, trace, b, p2, plane2, &hostRays)) return rc;
  }
  if (int rc = downscaleInto(g.bgrSS.p, width, height, 3, aas, out0, g.out0)) return rc;
  if (int rc = downscaleInto(g.p2SS.p, width, height, stereo ? 3 : 1, aas, out1, g.out1)) return rc;
  g_rigHostRays = hostRays;
  g_rigRays = n * (stereo ? 2 : 1);
  return DERP_OK;
}

int derp_test_rigsim_area(int device, const float* src, int dw, int dh, int cn, int k, float* dst) {
  if (!src || !dst || dw < 1 || dh < 1 || cn < 1 || k < 1 || (double)dw * dh * cn * k * k >= (double)(1ll << 30))
    return fail(DERP_EINVAL, "derp_test_rigsim_area: bad arguments");
  CU(cudaSetDevice(device));
  RigsimScratch& g = g_rig;
  const size_t n = (size_t)dw * dh * cn * k * k;
  if (int rc = stageIn(src, n, g.bgrSS)) return rc;
  return downscaleInto(src, dw, dh, cn, k, dst, g.out0);
}

uint64_t derp_rigsim_last_host_rays(void) { return g_rigHostRays; }
uint64_t derp_rigsim_last_rays(void) { return g_rigRays; }

int derp_rigsim_trace_host(const DerpRigsimScene* scene, const DerpRigsimRender* opts, const float* rays, int n,
                           float* out) {
  if (int rc = checkRender("derp_rigsim_trace_host", scene, opts)) return rc;
  if (!rays || !out || n < 0) return fail(DERP_EINVAL, "derp_rigsim_trace_host: bad arguments");
  const SceneView v = hostView(scene, opts);
  for (int i = 0; i < n; ++i) {
    const V3 o = v3(rays + 6 * i), d = v3(rays + 6 * i + 3);
    if (!traceRay(v, o, d, out + 4 * i)) {
      int row, col;
      skyTexelHost(d, v.skyH, v.skyW, &row, &col);
      skyColor(v, row, col, out + 4 * i);
    }
  }
  return DERP_OK;
}

int derp_test_sky_texel(int device, const float* dirs, int n, int rows, int cols, int32_t* texel) {
  if (!dirs || n < 1 || rows < 1 || cols < 1 || !texel) return fail(DERP_EINVAL, "derp_test_sky_texel: bad arguments");
  CU(cudaSetDevice(device));
  DevBuf<float> dd;
  DevBuf<int32_t> dt;
  if (int rc = upload(dd, dirs, 3 * (size_t)n)) return rc;
  CU(dt.ensure(2 * (size_t)n));
  skyTexelKernel<<<grid1(n), 256>>>(dd.p, n, rows, cols, dt.p);
  CU(cudaGetLastError());
  CU(cudaMemcpy(texel, dt.p, 2 * (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost));
  return DERP_OK;
}

int derp_test_sky_texel_host(const float* dirs, int n, int rows, int cols, int32_t* texel) {
  if (!dirs || n < 1 || rows < 1 || cols < 1 || !texel) return fail(DERP_EINVAL, "derp_test_sky_texel_host: bad arguments");
  for (int i = 0; i < n; ++i) skyTexelHost(v3(dirs + 3 * i), rows, cols, &texel[2 * i], &texel[2 * i + 1]);
  return DERP_OK;
}

}  // extern "C"
