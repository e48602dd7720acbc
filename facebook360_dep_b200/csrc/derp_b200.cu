// libderp_b200.so — the product: C ABI of include/derp_b200.h implemented with hand-written
// sm_90a CUDA kernels (derp_kernels.cuh).  No CPU fallback: every entry point that computes
// needs a CUDA device and fails with DERP_ECUDA otherwise.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -fmad=false (see Makefile).
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/derp_b200.h"
#include "derp_kernels.cuh"
#include "derp_refine.cuh"
#include "derp_mesh.cuh"
#include "derp_simplify.h"
#include "derp_bc7.cuh"
#include "derp_rephoto.cuh"
#include "derp_sweepview.cuh"
#include "../../include/derp_rephoto.h"
#include "../../include/derp_canopy.h"
#include "../../include/derp_sweepview.h"

using namespace derp;

namespace {

thread_local std::string g_err;

int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

#define CU(call)                                                                                     \
  do {                                                                                               \
    cudaError_t e_ = (call);                                                                         \
    if (e_ != cudaSuccess)                                                                           \
      return fail(DERP_ECUDA, std::string(#call) + ": " + cudaGetErrorString(e_) + " (" + __FILE__ + ":" + \
                                  std::to_string(__LINE__) + ")");                                   \
  } while (0)

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  ~DevBuf() { release(); }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
  }
  cudaError_t ensure(size_t count) {
    if (count <= n && p) return cudaSuccess;
    release();
    cudaError_t e = cudaMalloc(&p, std::max<size_t>(count, 1) * sizeof(T));
    if (e == cudaSuccess) n = count;
    return e;
  }
};

inline dim3 grid2(int W, int H, int z = 1) { return dim3((W + kBlockX - 1) / kBlockX, (H + kBlockY - 1) / kBlockY, z); }
inline dim3 block2() { return dim3(kBlockX, kBlockY, 1); }
// Grid of the kernels that walk the active-pixel list: one CTA per kPatchThreads list slots of the largest
// possible list (its length is only known on the device); CTAs past the end exit before staging anything.  A
// capped grid with more loop trips per CTA is not faster.
inline unsigned listGrid(int W, int H, int threads = kPatchThreads) {
  const size_t all = ((size_t)(W - 2) * (H - 2) + threads - 1) / threads;
  return (unsigned)std::max<size_t>(1, all);
}
inline size_t bilateralSmem(int radius) {  // float4 tile + mask bytes of bilateralKernel
  const size_t cells = (size_t)(kBlockX + 2 * radius) * (kBlockY + 2 * radius);
  return cells * sizeof(float4) + ((cells + 15) / 16) * 16;
}
inline unsigned grid1(size_t n, int t = 256) { return (unsigned)((n + t - 1) / t); }

// OpenCV's float bicubic table (imgwarp.cpp: interpolateCubic A=-0.75, initInterTab2D, INTER_TAB_SIZE 32)
void buildBicubicTable(std::vector<float>& tab) {
  float t1[32][4];
  const float scale = 1.f / 32;
  for (int i = 0; i < 32; ++i) {
    const float x = i * scale, A = -0.75f;
    t1[i][0] = ((A * (x + 1) - 5 * A) * (x + 1) + 8 * A) * (x + 1) - 4 * A;
    t1[i][1] = ((A + 2) * x - (A + 3)) * x * x + 1;
    t1[i][2] = ((A + 2) * (1 - x) - (A + 3)) * (1 - x) * (1 - x) + 1;
    t1[i][3] = 1.f - t1[i][0] - t1[i][1] - t1[i][2];
  }
  // the 2-D table entry (fy, fx)[k1][k2] = t1[fy][k1] * t1[fx][k2] (initInterTab2D) is formed in reprojectKernel
  tab.resize(32 * 4);
  for (int i = 0; i < 32; ++i)
    for (int k = 0; k < 4; ++k) tab[i * 4 + k] = t1[i][k];
}

// resize.cpp interpolateLanczos4
void lanczosTaps(float x, float* c) {
  static const double s45 = 0.70710678118654752440084436210485;
  static const double cs[][2] = {{1, 0}, {-s45, -s45}, {0, 1}, {s45, -s45}, {-1, 0}, {s45, s45}, {0, -1}, {-s45, s45}};
  if (x < 1.1920928955078125e-07f) {
    for (int i = 0; i < 8; ++i) c[i] = 0;
    c[3] = 1;
    return;
  }
  float sum = 0;
  const double y0 = -(x + 3) * M_PI * 0.25, s0 = std::sin(y0), c0 = std::cos(y0);
  for (int i = 0; i < 8; ++i) {
    const double y = -(x + 3 - i) * M_PI * 0.25;
    c[i] = (float)((cs[i][0] * s0 + cs[i][1] * c0) / (y * y));
    sum += c[i];
  }
  sum = 1.f / sum;
  for (int i = 0; i < 8; ++i) c[i] *= sum;
}
int floorD(double v) {
  int i = (int)v;
  return i - (i > v);
}
void lanczosAxis(int sn, int dn, std::vector<int>& ofs, std::vector<float>& taps) {
  const double inv = (double)dn / sn, scale = 1. / inv;
  ofs.resize(dn);
  taps.resize((size_t)dn * 8);
  for (int d = 0; d < dn; ++d) {
    float f = (float)((d + 0.5) * scale - 0.5);
    const int s = floorD(f);
    f -= s;
    ofs[d] = s;
    lanczosTaps(f, &taps[(size_t)d * 8]);
  }
}
void nearestAxis(int sn, int dn, std::vector<int>& ofs) {
  const double inv = (double)dn / sn, ifx = 1. / inv;
  ofs.resize(dn);
  for (int d = 0; d < dn; ++d) ofs[d] = std::min(floorD(d * ifx), sn - 1);
}
// UpsampleDisparityLib.cpp:27-52: clock-wise outward spiral of diameter w
void spiralOffsets(int w, std::vector<short2>& locs) {
  int x = 0, y = 0, dx = 0, dy = -1, t = w;
  const int samples = t * t;
  locs.clear();
  for (int i = 0; i < samples; ++i) {
    if ((-w / 2 <= x) && (x <= w / 2) && (-w / 2 <= y) && (y <= w / 2)) locs.push_back(make_short2((short)x, (short)y));
    if (x == y || ((x < 0) && (x == -y)) || ((x > 0) && (x == 1 - y))) {
      t = dx;
      dx = -dy;
      dy = t;
    }
    x += dx;
    y += dy;
  }
}

// The kernels that evaluate costs, instantiated for one visibility-mask width (evalCost in derp_cost.cuh).
struct CostKernels {
  void (*sweep)(SweepArgs);
  void (*evalCost)(CostView, const float*, float*, float*, unsigned long long*);
  void (*proposal)(ProposalArgs);
  void (*pingPong)(PingPongArgs);
  void (*sweepLower)(LowerArgs);
  void (*sweepSeed)(SeedArgs);
  void (*refine)(RefineArgs);
  void (*lowerBoundCheck)(CheckArgs);
};
template <class Mask>
CostKernels costKernelsOf() {
  return CostKernels{sweepKernel<Mask>,      evalCostKernel<Mask>,  proposalKernel<Mask>, pingPongKernel<Mask>,
                     sweepLowerKernel<Mask>, sweepSeedKernel<Mask>, refineKernel<Mask>,   lowerBoundCheckKernel<Mask>};
}
// The one place the rig size selects code: a 32-bit mask for rigs of up to 32 cameras, a 64-bit one up to 64.
const CostKernels& costKernels(int numCams) {
  static const CostKernels narrow = costKernelsOf<uint32_t>(), wide = costKernelsOf<uint64_t>();
  return numCams <= kNarrowMaxCams ? narrow : wide;
}

// The most dynamic shared memory an H100 grants one CTA.
constexpr size_t kMaxDynSmem = 227 * 1024;

}  // namespace

struct DerpCtx {
  int device = 0;
  int numSMs = 0;
  cudaStream_t stream = nullptr;
  bool ownStream = false;
  int S = 0, Sd = 0;
  CostKernels k{};  // costKernels(S)
  std::vector<int> dst2src;
  std::vector<DevCamera> camsNorm;  // normalised (Camera::normalizeRig)
  DevBuf<DevCamera> dCams, dCamsPx;
  DevBuf<float> dWtab;
  // level
  bool levelOpen = false, haveColors = false, haveFg = false, haveBg = false, haveGathered = false;
  bool accumulateCounters = false;
  DerpLevelParams lp{};
  int W = 0, H = 0;
  size_t plane = 0;
  float varNoiseFloor = 0;
  DevBuf<uint2> dColor;
  DevBuf<float4> dProjColor, dProjBias;  // integer-valued float texels (see derp_cost.cuh)
  DevBuf<unsigned> dSelTab;
  DevBuf<uint2> dProjColor16, dProjBias16;  // the same tables as 4 x u16 for the compacted kernels (built on demand)
  bool tabF32 = false, tabU16 = false;     // which bias/final tables of projDst are built
  DevBuf<float2> dProjWarp, dWarpInv;  // per-destination scratch when the geometry cache is off
  // geometry cache: projWarp / projWarpInv of every (dst, src) pair depend on the rig and the level size only
  // one cache per level size (all levels of cfg-2 together: 21 GB, created only while it fits in half of the free
  // memory), so both level-major (DerpCLI) and
  // frame-major pipelines hit it from the second frame on
  struct GeomCache {
    DevBuf<float2> buf;  // [Sd][2][S][H][W]
    std::vector<uint8_t> valid;
  };
  std::map<std::pair<int, int>, std::unique_ptr<GeomCache>> geomCaches;
  GeomCache* geom = nullptr;  // cache of the current level size, or null (maps go to the scratch buffers)
  bool geomCached = false;
  DevBuf<float> dVariance, dBg, dDisp, dCost, dConf, dScratchA, dScratchB, dScratchC, dDisparities, dGathered;
  DevBuf<uint8_t> dFg, dFov, dMismatch, dChangedA, dChangedB, dStage;
  DevBuf<unsigned long long> dBest, dCounters;
  // filtered sweep (derp_refine.cuh): lower bounds of every (candidate, pixel), seeds, refine list
  DevBuf<float> dLb;
  DevBuf<unsigned long long> dSeed, dRefList, dRefCount;
  unsigned long long lastRefined = 0, lastSeeds = 0;  // exact evaluations of the last filtered sweep
  int sweepMode = 0;                                  // derp_set_sweep_mode
  // in-memory level hand-off (derp_level_keep / derp_upsample_from_kept): the finished level's disparity planes
  DevBuf<float> dKept, dUpA, dUpB, dUpCoarse;
  DevBuf<uint8_t> dUpMc, dUpMu, dUpFovC;
  int keptW = 0, keptH = 0, keptSd = 0;
  DevBuf<unsigned> dUncovered;
  DevBuf<int> dPrefix, dIdx, dOfs, dRowCount, dTileCount, dTileOffset, dList;
  DevBuf<float> dTaps;
  DevBuf<short2> dSpiral;
  int projDst = -1;
  uint64_t launches = 0;
  uint64_t lastEvals = 0, lastHits = 0;
  bool countersOnDevice = false;
  int tableD = -1;
  float tableMin = 0, tableMax = 0;  // candidate table currently in dDisparities
  // optional per-kernel timing of the dominant kernel (sweepKernel) with CUDA events on c->stream
  bool profiling = false;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> sweepEvents;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pingEvents;  // pingPongKernel launches while profiling
  DevBuf<unsigned long long> dCountersPP;                         // their own (evaluations, source hits)

  float2* warpOf(int dst) const { return geomCached ? geom->buf.p + (size_t)dst * 2 * S * plane : dProjWarp.p; }
  float2* warpInvOf(int dst) const { return geomCached ? geom->buf.p + ((size_t)dst * 2 + 1) * S * plane : dWarpInv.p; }
  const uint8_t* fgOf(int src) const { return haveFg ? dFg.p + (size_t)src * plane : nullptr; }
  const float* bgOf(int dst) const { return haveBg ? dBg.p + (size_t)dst * plane : nullptr; }
  CostView view(int dst) const {
    CostView v;
    v.W = W;
    v.H = H;
    v.S = S;
    v.self = dst2src[dst];
    v.projColor = dProjColor.p;
    v.projBias = dProjBias.p;
    v.projColor16 = dProjColor16.p;
    v.projBias16 = dProjBias16.p;
    v.selTab = dSelTab.p;
    v.projWarp = warpOf(dst);
    v.variance = dVariance.p + (size_t)v.self * plane;
    v.cams = dCams.p;
    v.one = 1.0f;
    v.b23 = 8388608.0f;
    return v;
  }
  // dynamic smem of the cost kernels: S cameras + the destination patch tile
  // + S - 1 (ssdB, ssdU) pairs per thread for the robust camera mean (one slot per possible source)
  int selSlots() const { return S > 1 ? S - 1 : 1; }
  size_t camSmem(int threads = kBlockX * kBlockY) const {
    return (size_t)S * sizeof(DevCamera) + kTileFloats * sizeof(float) + (size_t)selSlots() * threads * sizeof(float2);
  }
  // compacted kernels: S cameras + one 3x3 patch per thread + the selection slots
  size_t patchSmem(int threads = kPatchThreads) const {
    return (size_t)S * sizeof(DevCamera) + (size_t)2 * 9 * threads * 2 * sizeof(float) + (size_t)selSlots() * threads * sizeof(float2);
  }
  // CTA height of the dense sweep: the tallest up to `rows` whose shared memory fits (`rows` itself up to 42 cameras;
  // the 63 slots per thread of a 64-camera rig leave room for 12 rows)
  int sweepRows(int rows) const {
    while (rows > 1 && camSmem(kBlockX * rows) > kMaxDynSmem) --rows;
    return rows;
  }
};

namespace {

int useDevice(DerpCtx* c) {
  CU(cudaSetDevice(c->device));
  return DERP_OK;
}

int checkDst(DerpCtx* c, int dst, const char* who, bool needProj) {
  if (!c) return fail(DERP_EINVAL, std::string(who) + ": null ctx");
  if (!c->levelOpen) return fail(DERP_ESTATE, std::string(who) + ": no level");
  if (dst < 0 || dst >= c->Sd) return fail(DERP_EINVAL, std::string(who) + ": dst out of range");
  if (needProj && c->projDst != dst)
    return fail(DERP_ESTATE, std::string(who) + ": derp_reproject(dst) must precede this stage");
  return useDevice(c);
}

int launchCheck(DerpCtx* c, const char* what) {
  c->launches++;
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) return fail(DERP_ECUDA, std::string(what) + ": " + cudaGetErrorString(e));
  return DERP_OK;
}
#define LAUNCHED(what)                      \
  do {                                      \
    int rc_ = launchCheck(c, what);         \
    if (rc_) return rc_;                    \
  } while (0)

// A cost kernel's dynamic shared memory (cameras, tile or patches, selection slots) grows with the rig: refuse a
// launch that would not fit instead of letting it fail.
int checkSmem(size_t bytes, const char* what) {
  if (bytes <= kMaxDynSmem) return DERP_OK;
  return fail(DERP_EINVAL, std::string(what) + ": needs " + std::to_string(bytes) + " B of shared memory per CTA, more than the " +
                               std::to_string(kMaxDynSmem) + " B an H100 grants");
}
#define SMEM_FITS(bytes, what)                \
  do {                                        \
    int rc_ = checkSmem(bytes, what);         \
    if (rc_) return rc_;                      \
  } while (0)

int resetCounters(DerpCtx* c) {
  if (c->accumulateCounters) return DERP_OK;  // derp_level_estimate: one reset / one read-back for all stages
  CU(cudaMemsetAsync(c->dCounters.p, 0, 2 * sizeof(unsigned long long), c->stream));
  c->countersOnDevice = true;
  return DERP_OK;
}

int readCounters(DerpCtx* c) {
  unsigned long long h[2];
  CU(cudaMemcpyAsync(h, c->dCounters.p, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  c->lastEvals = h[0];
  c->lastHits = h[1];
  return DERP_OK;
}

// list of active pixels of one destination, tile-major (activeScan -> tile counts -> offsets -> scatter);
// left in dList, the total in dTileOffset[numTiles] (see listCountPtr)
int buildActiveList(DerpCtx* c, const uint8_t* fov, const uint8_t* fg, const float* variance, float varThresh) {
  const int W = c->W, H = c->H;
  const dim3 tg = grid2(W, H);
  const int numTiles = (int)(tg.x * tg.y);
  activeScanKernel<<<(H + 7) / 8, 256, 0, c->stream>>>(W, H, fov, fg, variance, varThresh, c->dPrefix.p, c->dRowCount.p);
  LAUNCHED("activeScanKernel");
  tileCountKernel<<<tg, block2(), 0, c->stream>>>(W, H, c->dPrefix.p, c->dTileCount.p);
  LAUNCHED("tileCountKernel");
  rowOffsetKernel<<<1, 1024, 0, c->stream>>>(numTiles, c->dTileCount.p, c->dTileOffset.p);
  LAUNCHED("rowOffsetKernel");
  activeScatterKernel<<<tg, block2(), 0, c->stream>>>(W, H, c->dPrefix.p, c->dTileOffset.p, c->dList.p);
  LAUNCHED("activeScatterKernel");
  return DERP_OK;
}
const int* listCountPtr(DerpCtx* c) {
  const dim3 tg = grid2(c->W, c->H);
  return c->dTileOffset.p + (size_t)tg.x * tg.y;
}

// candidate table of the brute-force sweep (Derp.cpp:279-285, probeDisparity ImageUtil.cpp:100-107)
std::vector<float> probeDisparities(int num_depths, float min_depth_m, float max_depth_m) {
  std::vector<float> disparities(num_depths);
  const float minDisparity = 1.0f / max_depth_m, maxDisparity = 1.0f / min_depth_m;
  for (int i = 0; i < num_depths; ++i) {
    const double fraction = double(i) / double(num_depths - 1);
    disparities[i] = (float)(fraction * (double)minDisparity + (1 - fraction) * (double)maxDisparity);
  }
  return disparities;
}

// arguments of sweepLowerKernel for one destination: bounds go to dLb, per-pixel seeds to dSeed
LowerArgs lowerArgs(DerpCtx* c, int dst, const float* disparities, int num_depths, int chunk) {
  const bool useFg = c->lp.use_foreground_masks != 0;
  const int self = c->dst2src[dst];
  LowerArgs la;
  la.v = c->view(dst);
  la.fov = c->dFov.p + (size_t)dst * c->plane;
  la.fg = useFg ? c->fgOf(self) : nullptr;
  la.bg = useFg ? c->bgOf(dst) : nullptr;
  la.disparities = disparities;
  la.D = num_depths;
  la.chunk = chunk;
  la.lb = c->dLb.p;
  la.seed = c->dSeed.p;
  la.counters = c->dCounters.p;
  return la;
}

}  // namespace

extern "C" {

const char* derp_backend(void) { return "cuda-sm_90a"; }
const char* derp_last_error(void) { return g_err.c_str(); }
int derp_set_threads(int) { return DERP_OK; }

int derp_create(const DerpCameraDesc* cams, int num_cams, const int32_t* dst_to_src, int num_dsts, int device,
                DerpCtx** out) {
  if (!cams || !dst_to_src || !out || num_cams <= 0 || num_dsts <= 0)
    return fail(DERP_EINVAL, "derp_create: bad arguments");
  if (num_cams > kMaxCams) return fail(DERP_EINVAL, "derp_create: at most 64 cameras are supported");
  std::unique_ptr<DerpCtx> c(new DerpCtx);
  c->device = device;
  c->S = num_cams;
  c->k = costKernels(num_cams);
  c->Sd = num_dsts;
  c->camsNorm.resize(num_cams);
  for (int i = 0; i < num_cams; ++i) {
    if (!host::makeCamera(cams[i], &c->camsNorm[i]))
      return fail(DERP_EINVAL, "derp_create: invalid camera " + std::to_string(i));
  }
  for (int i = 1; i < num_cams; ++i)  // PyramidLevel::checkParams (PyramidLevel.h:169-184)
    if (c->camsNorm[i].res[0] != c->camsNorm[0].res[0] || c->camsNorm[i].res[1] != c->camsNorm[0].res[1])
      return fail(DERP_EINVAL, "derp_create: cameras must share one resolution");
  for (auto& cam : c->camsNorm)
    if (!(cam.res[0] == 1 && cam.res[1] == 1)) host::normalise(cam);
  c->dst2src.assign(dst_to_src, dst_to_src + num_dsts);
  for (int d : c->dst2src)
    if (d < 0 || d >= num_cams) return fail(DERP_EINVAL, "derp_create: dst_to_src out of range");
  int ndev = 0;
  CU(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) return fail(DERP_ECUDA, "derp_create: no such CUDA device " + std::to_string(device));
  CU(cudaSetDevice(device));
  CU(cudaDeviceGetAttribute(&c->numSMs, cudaDevAttrMultiProcessorCount, device));
  CU(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  c->ownStream = true;
  CU(c->dCams.ensure(num_cams));
  CU(c->dCamsPx.ensure(num_cams));
  CU(cudaMemcpy(c->dCams.p, c->camsNorm.data(), num_cams * sizeof(DevCamera), cudaMemcpyHostToDevice));
  std::vector<float> tab;
  buildBicubicTable(tab);
  CU(c->dWtab.ensure(tab.size()));
  CU(cudaMemcpy(c->dWtab.p, tab.data(), tab.size() * sizeof(float), cudaMemcpyHostToDevice));
  CU(c->dCounters.ensure(2));
  CU(c->dUncovered.ensure(1));
  std::vector<unsigned> selTab(kSelTabSize);
  buildSelectTable(selTab.data());
  CU(c->dSelTab.ensure(selTab.size()));
  CU(cudaMemcpy(c->dSelTab.p, selTab.data(), selTab.size() * sizeof(unsigned), cudaMemcpyHostToDevice));
  // the cost kernels keep cameras, the destination patch tile / per-thread patches and the selection slots in
  // dynamic shared memory: 92 KB for a 640-thread sweep CTA of a 16-camera rig, 177 KB with 32 cameras, 216 KB for a
  // 384-thread one with 64 cameras (DerpCtx::sweepRows); kMaxDynSmem is the most an H100 grants one CTA
  const int maxSmem = (int)kMaxDynSmem;
  CU(cudaFuncSetAttribute(c->k.sweep, cudaFuncAttributeMaxDynamicSharedMemorySize, maxSmem));
  CU(cudaFuncSetAttribute(c->k.evalCost, cudaFuncAttributeMaxDynamicSharedMemorySize, maxSmem));
  CU(cudaFuncSetAttribute(c->k.proposal, cudaFuncAttributeMaxDynamicSharedMemorySize, maxSmem));
  CU(cudaFuncSetAttribute(c->k.pingPong, cudaFuncAttributeMaxDynamicSharedMemorySize, maxSmem));
  CU(cudaFuncSetAttribute(c->k.sweepLower, cudaFuncAttributeMaxDynamicSharedMemorySize, maxSmem));
  CU(cudaFuncSetAttribute(c->k.sweepSeed, cudaFuncAttributeMaxDynamicSharedMemorySize, maxSmem));
  CU(cudaFuncSetAttribute(c->k.refine, cudaFuncAttributeMaxDynamicSharedMemorySize, maxSmem));
  CU(cudaFuncSetAttribute(c->k.lowerBoundCheck, cudaFuncAttributeMaxDynamicSharedMemorySize, maxSmem));
  *out = c.release();
  return DERP_OK;
}

void derp_destroy(DerpCtx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  if (c->ownStream && c->stream) cudaStreamDestroy(c->stream);
  delete c;
}

int derp_set_stream(DerpCtx* c, void* cuda_stream) {
  if (!c) return fail(DERP_EINVAL, "null ctx");
  int rc = useDevice(c);
  if (rc) return rc;
  CU(cudaStreamSynchronize(c->stream));
  if (c->ownStream && c->stream) cudaStreamDestroy(c->stream);
  c->ownStream = false;
  c->stream = (cudaStream_t)cuda_stream;
  return DERP_OK;
}

int derp_sync(DerpCtx* c) {
  if (!c) return fail(DERP_EINVAL, "null ctx");
  int rc = useDevice(c);
  if (rc) return rc;
  CU(cudaStreamSynchronize(c->stream));
  return DERP_OK;
}

int derp_profile(DerpCtx* c, int enable) {
  if (!c) return fail(DERP_EINVAL, "null ctx");
  for (auto& e : c->sweepEvents) {
    cudaEventDestroy(e.first);
    cudaEventDestroy(e.second);
  }
  c->sweepEvents.clear();
  for (auto& e : c->pingEvents) {
    cudaEventDestroy(e.first);
    cudaEventDestroy(e.second);
  }
  c->pingEvents.clear();
  c->profiling = enable != 0;
  if (c->profiling) {
    CU(c->dCountersPP.ensure(2));
    CU(cudaMemsetAsync(c->dCountersPP.p, 0, 2 * sizeof(unsigned long long), c->stream));
  }
  return DERP_OK;
}

int derp_get_profile_ping_pong(DerpCtx* c, double* ms, uint64_t* launches, uint64_t* evals, uint64_t* hits) {
  if (!c) return fail(DERP_EINVAL, "null ctx");
  int rc = useDevice(c);
  if (rc) return rc;
  CU(cudaStreamSynchronize(c->stream));
  double total = 0;
  for (auto& e : c->pingEvents) {
    float t = 0;
    CU(cudaEventElapsedTime(&t, e.first, e.second));
    total += t;
  }
  unsigned long long h[2] = {0, 0};
  if (c->dCountersPP.p) CU(cudaMemcpy(h, c->dCountersPP.p, sizeof(h), cudaMemcpyDeviceToHost));
  if (ms) *ms = total;
  if (launches) *launches = c->pingEvents.size();
  if (evals) *evals = h[0];
  if (hits) *hits = h[1];
  return DERP_OK;
}

int derp_get_profile(DerpCtx* c, double* sweep_ms, uint64_t* sweep_launches) {
  if (!c) return fail(DERP_EINVAL, "null ctx");
  int rc = useDevice(c);
  if (rc) return rc;
  CU(cudaStreamSynchronize(c->stream));
  double total = 0;
  for (auto& e : c->sweepEvents) {
    float ms = 0;
    CU(cudaEventElapsedTime(&ms, e.first, e.second));
    total += ms;
  }
  if (sweep_ms) *sweep_ms = total;
  if (sweep_launches) *sweep_launches = c->sweepEvents.size();
  return DERP_OK;
}

int derp_get_launch_count(DerpCtx* c, uint64_t* out) {
  if (!c || !out) return fail(DERP_EINVAL, "bad arguments");
  *out = c->launches;
  return DERP_OK;
}

int derp_level_begin(DerpCtx* c, const DerpLevelParams* p) {
  if (!c || !p || p->width < 3 || p->height < 3 || p->num_levels <= 0 || p->full_height <= 0)
    return fail(DERP_EINVAL, "derp_level_begin: bad arguments");
  int rc = useDevice(c);
  if (rc) return rc;
  c->lp = *p;
  c->W = p->width;
  c->H = p->height;
  c->plane = (size_t)c->W * c->H;
  const size_t n = c->plane;
  // PyramidLevel::computeVariances (PyramidLevel.h:232-236): width / heightFullSize, as written
  const float scale = float(c->W) / p->full_height;
  const float scaleVar = scale * scale;
  c->varNoiseFloor = std::max(p->var_noise_floor * scaleVar, kMinVarF);
  CU(c->dColor.ensure(n * c->S));
  CU(c->dVariance.ensure(n * c->S));
  CU(c->dProjColor16.ensure(n * c->S));  // the float4 / u16 bias tables are allocated by the first stage that reads them
  {  // geometry cache of this level size: create it if all pairs' maps fit in (half of the free) HBM
    const auto key = std::make_pair(c->W, c->H);
    auto it = c->geomCaches.find(key);
    if (it == c->geomCaches.end()) {
      size_t freeB = 0, totalB = 0;
      CU(cudaMemGetInfo(&freeB, &totalB));
      const size_t need = (size_t)c->Sd * 2 * c->S * n * sizeof(float2);
      const size_t levelBuffers = n * (size_t)c->S * 64;  // what the rest of this function is about to allocate
      std::unique_ptr<DerpCtx::GeomCache> g(new DerpCtx::GeomCache);
      if (need + levelBuffers < freeB / 2 && g->buf.ensure(need / sizeof(float2)) == cudaSuccess) {
        g->valid.assign(c->Sd, 0);
        it = c->geomCaches.emplace(key, std::move(g)).first;
      }
      cudaGetLastError();
    }
    c->geom = it == c->geomCaches.end() ? nullptr : it->second.get();
    c->geomCached = c->geom != nullptr;
  }
  if (!c->geomCached) {
    CU(c->dProjWarp.ensure(n * c->S));
    CU(c->dWarpInv.ensure(n * c->S));
  }
  CU(c->dFov.ensure(n * c->Sd));
  CU(c->dDisp.ensure(n * c->Sd));
  CU(c->dCost.ensure(n * c->Sd));
  CU(c->dConf.ensure(n * c->Sd));
  CU(c->dMismatch.ensure(n * c->Sd));
  CU(c->dScratchA.ensure(n));
  CU(c->dScratchB.ensure(n));
  CU(c->dChangedA.ensure(n));
  CU(c->dChangedB.ensure(n));
  CU(c->dBest.ensure(n));
  CU(c->dPrefix.ensure(n));
  CU(c->dList.ensure(n));
  CU(c->dRowCount.ensure(c->H));
  {
    const dim3 tg = grid2(c->W, c->H);
    CU(c->dTileCount.ensure((size_t)tg.x * tg.y));
    CU(c->dTileOffset.ensure((size_t)tg.x * tg.y + 1));
  }
  CU(c->dIdx.ensure(n));
  CU(c->dStage.ensure(n * 6 * (size_t)c->S));
  CU(cudaMemsetAsync(c->dDisp.p, 0, n * c->Sd * sizeof(float), c->stream));
  CU(cudaMemsetAsync(c->dCost.p, 0, n * c->Sd * sizeof(float), c->stream));
  CU(cudaMemsetAsync(c->dConf.p, 0, n * c->Sd * sizeof(float), c->stream));
  CU(cudaMemsetAsync(c->dMismatch.p, 0, n * c->Sd, c->stream));
  // cameras rescaled to the level's pixel size (Derp.cpp:961,968)
  std::vector<DevCamera> px(c->S);
  for (int s = 0; s < c->S; ++s) px[s] = host::rescaled(c->camsNorm[s], c->W, c->H);
  CU(cudaMemcpyAsync(c->dCamsPx.p, px.data(), c->S * sizeof(DevCamera), cudaMemcpyHostToDevice, c->stream));
  CU(cudaStreamSynchronize(c->stream));  // px goes out of scope
  for (int d = 0; d < c->Sd; ++d) {
    fovMaskKernel<<<grid2(c->W, c->H), block2(), 0, c->stream>>>(c->dCams.p + c->dst2src[d], c->W, c->H,
                                                                 c->dFov.p + (size_t)d * n);
    LAUNCHED("fovMaskKernel");
  }
  c->projDst = -1;
  c->haveColors = c->haveFg = c->haveBg = c->haveGathered = false;
  c->levelOpen = true;
  return DERP_OK;
}

int derp_set_colors(DerpCtx* c, const uint16_t* const* colors) {
  if (!c || !colors) return fail(DERP_EINVAL, "derp_set_colors: bad arguments");
  if (!c->levelOpen) return fail(DERP_ESTATE, "derp_set_colors: no level");
  int rc = useDevice(c);
  if (rc) return rc;
  const size_t n = c->plane;
  for (int s = 0; s < c->S; ++s) {
    if (!colors[s]) return fail(DERP_EINVAL, "derp_set_colors: null image");
    uint8_t* st = c->dStage.p + (size_t)s * n * 6;
    CU(cudaMemcpyAsync(st, colors[s], n * 6, cudaMemcpyDefault, c->stream));  // host or device image
    packColorKernel<<<grid1(n), 256, 0, c->stream>>>(n, reinterpret_cast<const uint16_t*>(st), c->dColor.p + (size_t)s * n);
    LAUNCHED("packColorKernel");
  }
  varianceKernel<<<grid2(c->W, c->H, c->S), block2(), 0, c->stream>>>(c->W, c->H, c->dColor.p, c->dVariance.p);
  LAUNCHED("varianceKernel");
  c->haveColors = true;
  c->projDst = -1;
  return DERP_OK;
}

int derp_set_foreground_masks(DerpCtx* c, const uint8_t* const* masks) {
  if (!c || !masks) return fail(DERP_EINVAL, "derp_set_foreground_masks: bad arguments");
  if (!c->levelOpen) return fail(DERP_ESTATE, "no level");
  int rc = useDevice(c);
  if (rc) return rc;
  const size_t n = c->plane;
  CU(c->dFg.ensure(n * c->S));
  for (int s = 0; s < c->S; ++s)
    CU(cudaMemcpyAsync(c->dFg.p + (size_t)s * n, masks[s], n, cudaMemcpyHostToDevice, c->stream));
  c->haveFg = true;
  return DERP_OK;
}

int derp_set_background_disparity(DerpCtx* c, const float* const* background) {
  if (!c || !background) return fail(DERP_EINVAL, "derp_set_background_disparity: bad arguments");
  if (!c->levelOpen) return fail(DERP_ESTATE, "no level");
  int rc = useDevice(c);
  if (rc) return rc;
  const size_t n = c->plane;
  CU(c->dBg.ensure(n * c->Sd));
  for (int d = 0; d < c->Sd; ++d)
    CU(cudaMemcpyAsync(c->dBg.p + (size_t)d * n, background[d], n * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  c->haveBg = true;
  return DERP_OK;
}

int derp_reproject(DerpCtx* c, int dst) {
  int rc = checkDst(c, dst, "derp_reproject", false);
  if (rc) return rc;
  if (!c->haveColors) return fail(DERP_ESTATE, "derp_reproject: colours not set");
  const int self = c->dst2src[dst];
  if (!c->geomCached || !c->geom->valid[dst]) {  // rig + level size only: computed once per destination when cached
    projWarpKernel<<<grid2(c->W, c->H, c->S), block2(), 0, c->stream>>>(c->dCamsPx.p, c->S, self, c->W, c->H, c->warpOf(dst));
    LAUNCHED("projWarpKernel");
    warpInvKernel<<<grid2(c->W, c->H, c->S), block2(), 0, c->stream>>>(c->dCamsPx.p, c->S, self, c->W, c->H, c->warpInvOf(dst));
    LAUNCHED("warpInvKernel");
    if (c->geomCached) c->geom->valid[dst] = 1;
  }
  reprojectKernel<<<grid2(c->W, c->H, c->S), block2(), 0, c->stream>>>(c->warpInvOf(dst), c->S, self, c->W, c->H, c->dColor.p,
                                                                       c->dWtab.p, c->dProjColor16.p);
  LAUNCHED("reprojectKernel");
  c->projDst = dst;
  c->tabF32 = c->tabU16 = false;  // colour bias + final table layout: built by the first stage that needs them
  return DERP_OK;
}

// K4 in the table format the calling stage reads: float4 for the dense sweep / evalCost / the getters, 4 x u16 for
// the compacted fine-level kernels.  A level normally needs exactly one of them per destination.
static int ensureTablesF32(DerpCtx* c) {
  if (c->tabF32) return DERP_OK;
  CU(c->dProjColor.ensure(c->plane * c->S));
  CU(c->dProjBias.ensure(c->plane * c->S));
  biasKernel<<<grid2(c->W, c->H, c->S), block2(), 0, c->stream>>>(c->W, c->H, c->dProjColor16.p, c->dProjColor.p,
                                                                  c->dProjBias.p);
  LAUNCHED("biasKernel");
  c->tabF32 = true;
  return DERP_OK;
}
static int ensureTablesU16(DerpCtx* c) {
  if (c->tabU16) return DERP_OK;
  CU(c->dProjBias16.ensure(c->plane * c->S));
  bias16Kernel<<<grid2(c->W, c->H, c->S), block2(), 0, c->stream>>>(c->W, c->H, c->dProjColor16.p, c->dProjBias16.p);
  LAUNCHED("bias16Kernel");
  c->tabU16 = true;
  return DERP_OK;
}

int derp_eval_cost(DerpCtx* c, int dst, const float* disparity, float* out_cost, float* out_conf) {
  if (!disparity) return fail(DERP_EINVAL, "derp_eval_cost: bad arguments");
  int rc = checkDst(c, dst, "derp_eval_cost", true);
  if (rc) return rc;
  const size_t n = c->plane;
  CU(c->dScratchC.ensure(n));
  CU(cudaMemcpyAsync(c->dScratchA.p, disparity, n * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  if ((rc = resetCounters(c))) return rc;
  if ((rc = ensureTablesF32(c))) return rc;
  SMEM_FITS(c->camSmem(), "evalCostKernel");
  c->k.evalCost<<<grid2(c->W, c->H), block2(), c->camSmem(), c->stream>>>(c->view(dst), c->dScratchA.p, c->dScratchB.p,
                                                                         c->dScratchC.p, c->dCounters.p);
  LAUNCHED("evalCostKernel");
  if (out_cost) CU(cudaMemcpyAsync(out_cost, c->dScratchB.p, n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  if (out_conf) CU(cudaMemcpyAsync(out_conf, c->dScratchC.p, n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  rc = readCounters(c);
  c->countersOnDevice = false;
  return rc;
}

int derp_brute_force(DerpCtx* c, int dst, int num_depths, float min_depth_m, float max_depth_m, int partial_coverage,
                     int32_t* best_index) {
  if (num_depths < 2) return fail(DERP_EINVAL, "derp_brute_force: bad arguments");
  int rc = checkDst(c, dst, "derp_brute_force", true);
  if (rc) return rc;
  const bool useFg = c->lp.use_foreground_masks != 0;
  if (useFg && (!c->haveBg || !c->haveFg))
    return fail(DERP_ESTATE, "derp_brute_force: foreground masks / background disparity not set");
  const int W = c->W, H = c->H;
  const size_t n = c->plane;
  const int self = c->dst2src[dst];
  const float minDisparity = 1.0f / max_depth_m;
  if (c->tableD != num_depths || c->tableMin != min_depth_m || c->tableMax != max_depth_m) {
    const std::vector<float> disparities = probeDisparities(num_depths, min_depth_m, max_depth_m);
    CU(c->dDisparities.ensure(num_depths));
    CU(cudaMemcpyAsync(c->dDisparities.p, disparities.data(), num_depths * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    CU(cudaStreamSynchronize(c->stream));  // host vector lifetime (tiny copy, only when the table changes)
    c->tableD = num_depths;
    c->tableMin = min_depth_m;
    c->tableMax = max_depth_m;
  }
  if ((rc = ensureTablesF32(c))) return rc;
  fillKernel<unsigned long long><<<grid1(n), 256, 0, c->stream>>>(n, c->dBest.p, 0x7f7fffffffffffffull);
  LAUNCHED("fillKernel");
  if ((rc = resetCounters(c))) return rc;
  CU(cudaMemsetAsync(c->dUncovered.p, 0, sizeof(unsigned), c->stream));
  // candidate chunks: enough CTAs to fill every SM with 8 resident CTAs even on the coarse levels
  // CTA height of the sweep: kSweepMaxRows rows (one 640-thread CTA per SM, 96 registers) on large levels —
  // its warps share more texel rows — and half of that (two CTAs per SM, same 20 warps) on small ones, where CTA count matters
  // more.  Rigs of more than 42 cameras get shorter CTAs (sweepRows).
  const int sweepBY = c->sweepRows(H >= 1024 ? kSweepMaxRows : kSweepMaxRows / 2);
  const size_t sweepSmem = c->camSmem(kBlockX * sweepBY);
  SMEM_FITS(sweepSmem, "sweepKernel");
  SMEM_FITS(c->camSmem(), "sweepSeedKernel");
  SMEM_FITS(c->patchSmem(), "refineKernel");
  const dim3 g = grid2(W, H);
  const dim3 gs((W + kBlockX - 1) / kBlockX, (H + sweepBY - 1) / sweepBY, 1);
  const long ctas = (long)gs.x * gs.y * std::max(1, sweepBY / 8);
  int chunks = (int)std::min<long>(num_depths, std::max<long>(1, ((long)c->numSMs * 8 * 4 + ctas - 1) / ctas));
  const int chunk = (num_depths + chunks - 1) / chunks;
  chunks = (num_depths + chunk - 1) / chunk;
  SweepArgs a;
  a.v = c->view(dst);
  a.fov = c->dFov.p + (size_t)dst * n;
  a.fg = useFg ? c->fgOf(self) : nullptr;
  a.bg = useFg ? c->bgOf(dst) : nullptr;
  a.disparities = c->dDisparities.p;
  a.D = num_depths;
  a.chunk = chunk;
  a.best = c->dBest.p;
  a.counters = c->dCounters.p;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  if (c->profiling) {
    CU(cudaEventCreate(&ev0));
    CU(cudaEventCreate(&ev1));
    CU(cudaEventRecord(ev0, c->stream));
  }
  // Filtered sweep (derp_refine.cuh) unless derp_set_sweep_mode chose the plain one, the candidate count is tiny or the
  // bound buffer does not fit: lower bound of every (pixel, candidate), exact cost only where the bound does not exclude
  // the candidate.
  const int mode = c->sweepMode;
  // automatic: the filter pays off when the bound pass amortises its extra launches and the read-back of the list
  // length: >= 32 M (pixel, candidate) pairs (512^2 x 128); BASELINE.json configs[0] (512^2 x 32) and the coarsest
  // pyramid levels stay on the plain sweep
  bool filtered = mode == 2 || (mode == 0 && num_depths >= 8 && (unsigned long long)n * (unsigned long long)num_depths >= (32ull << 20));
  const unsigned long long capacity = (unsigned long long)n * (unsigned long long)std::max(2, num_depths / 8);
  if (filtered) {
    size_t freeB = 0, totalB = 0;
    cudaMemGetInfo(&freeB, &totalB);
    const size_t need = (size_t)num_depths * n * sizeof(float) + capacity * sizeof(unsigned long long) + n * 8;
    if (c->dLb.n < (size_t)num_depths * n && need > freeB / 2) filtered = false;
  }
  c->lastRefined = c->lastSeeds = 0;
  if (filtered) {
    CU(c->dLb.ensure((size_t)num_depths * n));
    CU(c->dSeed.ensure(n));
    CU(c->dRefList.ensure(capacity));
    CU(c->dRefCount.ensure(1));
    fillKernel<unsigned long long><<<grid1(n), 256, 0, c->stream>>>(n, c->dSeed.p, 0x7f7fffffffffffffull);
    LAUNCHED("fillKernel");
    CU(cudaMemsetAsync(c->dRefCount.p, 0, sizeof(unsigned long long), c->stream));
    const LowerArgs la = lowerArgs(c, dst, a.disparities, num_depths, chunk);
    c->k.sweepLower<<<dim3(gs.x, gs.y, chunks), dim3(kBlockX, sweepBY, 1), sweepSmem, c->stream>>>(la);
    LAUNCHED("sweepLowerKernel");
    SeedArgs sa;
    sa.v = a.v;
    sa.fov = a.fov;
    sa.fg = a.fg;
    sa.disparities = a.disparities;
    sa.seed = c->dSeed.p;
    sa.best = c->dBest.p;
    c->k.sweepSeed<<<g, block2(), c->camSmem(), c->stream>>>(sa);
    LAUNCHED("sweepSeedKernel");
    ListArgs li;
    li.W = W;
    li.H = H;
    li.D = num_depths;
    li.fov = a.fov;
    li.fg = a.fg;
    li.lb = c->dLb.p;
    li.seed = c->dSeed.p;
    li.best = c->dBest.p;
    li.list = c->dRefList.p;
    li.capacity = capacity;
    li.count = c->dRefCount.p;
    refineListKernel<<<g, block2(), 0, c->stream>>>(li);
    LAUNCHED("refineListKernel");
    unsigned long long count = 0;
    CU(cudaMemcpyAsync(&count, c->dRefCount.p, sizeof(count), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    if (count > capacity) {
      // more survivors than the list holds (bounds useless on this input): redo the destination with the plain sweep
      filtered = false;
      fillKernel<unsigned long long><<<grid1(n), 256, 0, c->stream>>>(n, c->dBest.p, 0x7f7fffffffffffffull);
      LAUNCHED("fillKernel");
      CU(cudaMemsetAsync(c->dCounters.p, 0, 2 * sizeof(unsigned long long), c->stream));
    } else {
      c->lastRefined = count;
      c->lastSeeds = n;
      if (count > 0) {
        RefineArgs ra;
        ra.v = a.v;
        ra.disparities = a.disparities;
        ra.list = c->dRefList.p;
        ra.count = count;
        ra.best = c->dBest.p;
        c->k.refine<<<(unsigned)((count + kPatchThreads - 1) / kPatchThreads), kPatchThreads, c->patchSmem(), c->stream>>>(ra);
        LAUNCHED("refineKernel");
      }
    }
  }
  if (!filtered) {
    c->k.sweep<<<dim3(gs.x, gs.y, chunks), dim3(kBlockX, sweepBY, 1), sweepSmem, c->stream>>>(a);
    LAUNCHED("sweepKernel");
  }
  if (c->profiling) {
    CU(cudaEventRecord(ev1, c->stream));
    c->sweepEvents.emplace_back(ev0, ev1);
  }
  float* disp = c->dDisp.p + (size_t)dst * n;
  float* cost = c->dCost.p + (size_t)dst * n;
  float* conf = c->dConf.p + (size_t)dst * n;
  int* idx = best_index ? c->dIdx.p : nullptr;
  sweepFinalizeKernel<<<g, block2(), 0, c->stream>>>(W, H, a.fov, a.fg, a.bg, a.v.variance, c->dDisparities.p, minDisparity,
                                                     c->dBest.p, disp, cost, conf, idx, c->dUncovered.p);
  LAUNCHED("sweepFinalizeKernel");
  extendBorderKernel<<<grid1(2 * W + 2 * (H - 2)), 256, 0, c->stream>>>(W, H, a.fg, a.bg, disp, cost, conf, idx);
  LAUNCHED("extendBorderKernel");
  if (best_index) CU(cudaMemcpyAsync(best_index, c->dIdx.p, n * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  if (!(partial_coverage || useFg)) {
    unsigned unc = 0;
    CU(cudaMemcpyAsync(&unc, c->dUncovered.p, sizeof(unsigned), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    if (unc > 0)  // Derp.cpp:339 CHECK(partialCoverage || useForegroundMasks)
      return fail(DERP_ECOVERAGE, "Insufficient coverage at " + std::to_string(unc) + " pixels");
  } else if (best_index) {
    CU(cudaStreamSynchronize(c->stream));
  }
  return DERP_OK;
}

int derp_random_proposals(DerpCtx* c, int dst, int num_proposals, float min_depth_m, float max_depth_m) {
  int rc = checkDst(c, dst, "derp_random_proposals", true);
  if (rc) return rc;
  if (num_proposals < 0) return fail(DERP_EINVAL, "derp_random_proposals: negative count");
  const bool useFg = c->lp.use_foreground_masks != 0;
  if (useFg && (!c->haveBg || !c->haveFg)) return fail(DERP_ESTATE, "derp_random_proposals: masks not set");
  const int W = c->W, H = c->H;
  const size_t n = c->plane;
  const int self = c->dst2src[dst];
  const float kRandomPropHighVarDeviation = 0.1f;  // Derp.h:37
  const float varHighDev = kRandomPropHighVarDeviation * c->lp.var_high_thresh;
  const float varThresh = std::max(varHighDev, c->varNoiseFloor);
  ProposalArgs a;
  a.v = c->view(dst);
  a.fov = c->dFov.p + (size_t)dst * n;
  a.fg = useFg ? c->fgOf(self) : nullptr;
  a.bg = useFg ? c->bgOf(dst) : nullptr;
  a.prefix = c->dPrefix.p;
  a.disp = c->dDisp.p + (size_t)dst * n;
  a.cost = c->dCost.p + (size_t)dst * n;
  a.conf = c->dConf.p + (size_t)dst * n;
  a.numProposals = num_proposals;
  a.level = c->lp.level;
  a.minDispGlobal = 1.0f / max_depth_m;
  a.maxDisp = 1.0f / min_depth_m;
  a.counters = c->dCounters.p;
  a.list = c->dList.p;
  a.listCount = listCountPtr(c);
  if ((rc = resetCounters(c))) return rc;
  if ((rc = ensureTablesU16(c))) return rc;
  a.v = c->view(dst);  // the u16 tables may just have been allocated
  if ((rc = buildActiveList(c, a.fov, a.fg, a.v.variance, varThresh))) return rc;
  if (useFg) {
    backgroundFillKernel<<<grid2(W, H), block2(), 0, c->stream>>>(W, H, a.fov, a.fg, a.bg, a.disp);
    LAUNCHED("backgroundFillKernel");
  }
  SMEM_FITS(c->patchSmem(), "proposalKernel");
  c->k.proposal<<<listGrid(W, H), kPatchThreads, c->patchSmem(), c->stream>>>(a);
  LAUNCHED("proposalKernel");
  return DERP_OK;
}

int derp_ping_pong(DerpCtx* c, int dst, int iterations) {
  int rc = checkDst(c, dst, "derp_ping_pong", true);
  if (rc) return rc;
  const bool useFg = c->lp.use_foreground_masks != 0;
  if (useFg && (!c->haveBg || !c->haveFg)) return fail(DERP_ESTATE, "derp_ping_pong: masks not set");
  const int W = c->W, H = c->H;
  const size_t n = c->plane;
  const int self = c->dst2src[dst];
  float* disp = c->dDisp.p + (size_t)dst * n;
  float* cost = c->dCost.p + (size_t)dst * n;
  const uint8_t* fov = c->dFov.p + (size_t)dst * n;
  const uint8_t* fg = useFg ? c->fgOf(self) : nullptr;
  const float* bg = useFg ? c->bgOf(dst) : nullptr;
  if ((rc = resetCounters(c))) return rc;
  if ((rc = ensureTablesU16(c))) return rc;
  // active pixels: interior, in FOV, foreground, variance >= noise floor (Derp.cpp:420-437)
  if ((rc = buildActiveList(c, fov, fg, c->view(dst).variance, c->varNoiseFloor))) return rc;
  fillKernel<uint8_t><<<grid1(n), 256, 0, c->stream>>>(n, c->dChangedA.p, (uint8_t)1);
  LAUNCHED("fillKernel");
  uint8_t* chIn = c->dChangedA.p;
  uint8_t* chOut = c->dChangedB.p;
  SMEM_FITS(c->patchSmem(kPingThreads), "pingPongKernel");
  for (int it = 1; it <= iterations; ++it) {
    pingPongInitKernel<<<grid2(W, H), block2(), 0, c->stream>>>(W, H, fov, fg, bg, disp, c->dScratchA.p, c->dScratchB.p, chOut);
    LAUNCHED("pingPongInitKernel");
    PingPongArgs a;
    a.v = c->view(dst);
    a.fov = fov;
    a.fg = fg;
    a.bg = bg;
    a.disp = disp;
    a.changed = chIn;
    a.dispRes = c->dScratchA.p;
    a.costRes = c->dScratchB.p;
    a.changedNext = chOut;
    a.list = c->dList.p;
    a.listCount = listCountPtr(c);
    a.counters = c->dCounters.p;
    a.counters2 = c->profiling ? c->dCountersPP.p : nullptr;
    cudaEvent_t p0 = nullptr, p1 = nullptr;
    if (c->profiling) {
      CU(cudaEventCreate(&p0));
      CU(cudaEventCreate(&p1));
      CU(cudaEventRecord(p0, c->stream));
    }
    c->k.pingPong<<<listGrid(W, H, kPingThreads), kPingThreads, c->patchSmem(kPingThreads), c->stream>>>(a);
    LAUNCHED("pingPongKernel");
    if (c->profiling) {
      CU(cudaEventRecord(p1, c->stream));
      c->pingEvents.emplace_back(p0, p1);
    }
    // disp <- dispRes, cost <- costsRes (Derp.cpp:527-529); confidence is not written back
    CU(cudaMemcpyAsync(disp, c->dScratchA.p, n * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));
    CU(cudaMemcpyAsync(cost, c->dScratchB.p, n * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));
    std::swap(chIn, chOut);
  }
  return DERP_OK;
}

// K9 for this context's destinations; dispAll = [S] planes indexed by rig camera (pre-update values of every camera).
static int launchMismatches(DerpCtx* c, const float* dispAll) {
  const size_t n = c->plane;
  DevBuf<float> dNew;
  CU(dNew.ensure(n * c->Sd));
  for (int d = 0; d < c->Sd; ++d) {
    const int self = c->dst2src[d];
    MismatchArgs a;
    a.W = c->W;
    a.H = c->H;
    a.S = c->S;
    a.self = self;
    a.cams = c->dCams.p;
    a.dispAll = dispAll;
    a.variance = c->dVariance.p + (size_t)self * n;
    a.fov = c->dFov.p + (size_t)d * n;
    a.fg = (c->lp.use_foreground_masks && c->haveFg) ? c->fgOf(self) : nullptr;
    a.varNoiseFloor = c->varNoiseFloor;
    a.varHighThresh = c->lp.var_high_thresh;
    a.dispNew = dNew.p + (size_t)d * n;
    a.mask = c->dMismatch.p + (size_t)d * n;
    mismatchKernel<<<grid2(c->W, c->H), block2(), (size_t)c->S * sizeof(DevCamera), c->stream>>>(a);  // cameras only
    LAUNCHED("mismatchKernel");
  }
  CU(cudaMemcpyAsync(c->dDisp.p, dNew.p, n * c->Sd * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));
  CU(cudaStreamSynchronize(c->stream));  // dNew is freed on return
  return DERP_OK;
}

int derp_mismatches(DerpCtx* c) {
  if (!c) return fail(DERP_EINVAL, "null ctx");
  if (!c->levelOpen) return fail(DERP_ESTATE, "derp_mismatches: no level");
  if (c->Sd != c->S) return fail(DERP_EINVAL, "Mismatches only valid when considering all cameras");
  for (int d = 0; d < c->Sd; ++d)
    if (c->dst2src[d] != d) return fail(DERP_EINVAL, "derp_mismatches: dst list must equal camera list");
  int rc = useDevice(c);
  if (rc) return rc;
  return launchMismatches(c, c->dDisp.p);
}

// ---- destination cameras dealt to several contexts: all-gather of disparities, then K9 per shard ---------
const float* derp_disparity_device_ptr(DerpCtx* c, int dst) {
  if (checkDst(c, dst, "derp_disparity_device_ptr", false)) return nullptr;
  return c->dDisp.p + (size_t)dst * c->plane;
}

int derp_gather_disparities(DerpCtx* c, const float* const* planes) {
  if (!c || !planes) return fail(DERP_EINVAL, "derp_gather_disparities: bad arguments");
  if (!c->levelOpen) return fail(DERP_ESTATE, "derp_gather_disparities: no level");
  int rc = useDevice(c);
  if (rc) return rc;
  const size_t n = c->plane, b = n * sizeof(float);
  CU(c->dGathered.ensure(n * c->S));
  std::vector<int> ownDst(c->S, -1);
  for (int d = 0; d < c->Sd; ++d) ownDst[c->dst2src[d]] = d;
  for (int s = 0; s < c->S; ++s) {
    float* to = c->dGathered.p + (size_t)s * n;
    const float* from = planes[s];
    if (!from) {
      if (ownDst[s] < 0) return fail(DERP_EINVAL, "derp_gather_disparities: no plane for a camera this context does not own");
      CU(cudaMemcpyAsync(to, c->dDisp.p + (size_t)ownDst[s] * n, b, cudaMemcpyDeviceToDevice, c->stream));
      continue;
    }
    cudaPointerAttributes at{};
    CU(cudaPointerGetAttributes(&at, from));
    if (at.type == cudaMemoryTypeDevice && at.device != c->device) {
      // a peer context's plane: device-to-device over NVLink (the runtime stages through the host if the two
      // devices have no peer path)
      int can = 0;
      CU(cudaDeviceCanAccessPeer(&can, c->device, at.device));
      if (can) {
        const cudaError_t e = cudaDeviceEnablePeerAccess(at.device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CU(e);
        (void)cudaGetLastError();
      }
      CU(cudaMemcpyPeerAsync(to, c->device, from, at.device, b, c->stream));
    } else {
      CU(cudaMemcpyAsync(to, from, b, cudaMemcpyDefault, c->stream));
    }
  }
  CU(cudaStreamSynchronize(c->stream));
  c->haveGathered = true;
  return DERP_OK;
}

int derp_mismatches_gathered(DerpCtx* c) {
  if (!c) return fail(DERP_EINVAL, "null ctx");
  if (!c->levelOpen) return fail(DERP_ESTATE, "derp_mismatches_gathered: no level");
  if (!c->haveGathered) return fail(DERP_ESTATE, "derp_mismatches_gathered: derp_gather_disparities not called for this level");
  int rc = useDevice(c);
  if (rc) return rc;
  c->haveGathered = false;  // one exchange per stage
  return launchMismatches(c, c->dGathered.p);
}

int derp_bilateral(DerpCtx* c, int dst) {
  int rc = checkDst(c, dst, "derp_bilateral", false);
  if (rc) return rc;
  if (!c->haveColors) return fail(DERP_ESTATE, "derp_bilateral: colours not set");
  const size_t n = c->plane;
  const int self = c->dst2src[dst];
  // Derp.cpp:876-878: pow(float, int) promotes to double, result narrowed to float
  const float scale = (float)std::pow((double)0.9f, (double)c->lp.level);
  const int spaceRadius = (int)std::max(std::ceil(5 * scale), float(1));
  const uint8_t* fg = (c->lp.use_foreground_masks && c->haveFg) ? c->fgOf(self) : nullptr;
  float* disp = c->dDisp.p + (size_t)dst * n;
  const float sigma = 0.005f;
  DivConst three, denom;
  CU(makeDivConst(3.0f, c->stream, &three));
  CU(makeDivConst(2.0f * (sigma * sigma), c->stream, &denom));
  bilateralKernel<GuideU16><<<grid2(c->W, c->H), block2(), bilateralSmem(spaceRadius), c->stream>>>(
      c->W, c->H, disp, GuideU16{c->dColor.p + (size_t)self * n}, c->dFov.p + (size_t)dst * n, fg, spaceRadius, three, denom,
      0.5f, 1.0f, 1.0f, c->dScratchA.p);
  LAUNCHED("bilateralKernel");
  CU(cudaMemcpyAsync(disp, c->dScratchA.p, n * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));
  return DERP_OK;
}

int derp_median(DerpCtx* c, int dst) {
  int rc = checkDst(c, dst, "derp_median", false);
  if (rc) return rc;
  const size_t n = c->plane;
  const int self = c->dst2src[dst];
  const uint8_t* fg = (c->lp.use_foreground_masks && c->haveFg) ? c->fgOf(self) : nullptr;
  float* disp = c->dDisp.p + (size_t)dst * n;
  medianKernel<<<grid2(c->W, c->H), block2(), 0, c->stream>>>(c->W, c->H, disp, c->bgOf(dst), c->dFov.p + (size_t)dst * n, fg,
                                                             c->dScratchA.p);
  LAUNCHED("medianKernel");
  CU(cudaMemcpyAsync(disp, c->dScratchA.p, n * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));
  return DERP_OK;
}

int derp_mask_fov(DerpCtx* c, int dst) {
  int rc = checkDst(c, dst, "derp_mask_fov", false);
  if (rc) return rc;
  const size_t n = c->plane;
  maskFovKernel<<<grid1(n), 256, 0, c->stream>>>(n, c->dFov.p + (size_t)dst * n, c->dDisp.p + (size_t)dst * n);
  LAUNCHED("maskFovKernel");
  return DERP_OK;
}

}  // extern "C"

namespace {

// upsampleDisparityInPlace (UpsampleDisparityLib.cpp:98-147) on device buffers.
// dCoarse: cw*ch floats; maskC / maskUp: already AND-ed with the FOV masks (nullable when !useFg).
int upsampleDevice(DerpCtx* c, cudaStream_t st, const float* dCoarse, int cw, int ch, const float* dBgUp,
                   const uint8_t* dMaskC, const uint8_t* dMaskUp, int W, int H, bool useFg, float* dOut,
                   DevBuf<float>& tmpA, DevBuf<float>& tmpB, DevBuf<int>& dOfs, DevBuf<float>& dTaps,
                   DevBuf<short2>& dSpiral) {
  if (useFg) {
    if (!dBgUp || !dMaskC || !dMaskUp) return fail(DERP_EINVAL, "upsample: masks and background required");
    const float scale = float(W) / float(cw);  // getRadius (UpsampleDisparityLib.cpp:93-96)
    const int radius = (int)(scale * scale + 1);
    std::vector<int> xo, yo;
    nearestAxis(cw, W, xo);
    nearestAxis(ch, H, yo);
    std::vector<int> ofs(xo);
    ofs.insert(ofs.end(), yo.begin(), yo.end());
    CU(dOfs.ensure(ofs.size()));
    CU(cudaMemcpyAsync(dOfs.p, ofs.data(), ofs.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    std::vector<short2> sp;
    spiralOffsets(radius * 2 + 1, sp);
    CU(dSpiral.ensure(sp.size()));
    CU(cudaMemcpyAsync(dSpiral.p, sp.data(), sp.size() * sizeof(short2), cudaMemcpyHostToDevice, st));
    CU(cudaStreamSynchronize(st));
    CU(tmpA.ensure((size_t)W * H));
    nearestMaskedKernel<<<grid2(W, H), block2(), 0, st>>>(cw, ch, W, H, dCoarse, dMaskC, dMaskUp, dOfs.p, dOfs.p + W, tmpA.p);
    if (c) c->launches++;
    replaceNansKernel<<<grid2(W, H), block2(), 0, st>>>(W, H, tmpA.p, dBgUp, dMaskUp, dSpiral.p, (int)sp.size(), dOut);
    if (c) c->launches++;
  } else {
    std::vector<int> xo, yo;
    std::vector<float> al, be;
    lanczosAxis(cw, W, xo, al);
    lanczosAxis(ch, H, yo, be);
    std::vector<int> ofs(xo);
    ofs.insert(ofs.end(), yo.begin(), yo.end());
    std::vector<float> taps(al);
    taps.insert(taps.end(), be.begin(), be.end());
    CU(dOfs.ensure(ofs.size()));
    CU(dTaps.ensure(taps.size()));
    CU(cudaMemcpyAsync(dOfs.p, ofs.data(), ofs.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(dTaps.p, taps.data(), taps.size() * sizeof(float), cudaMemcpyHostToDevice, st));
    CU(cudaStreamSynchronize(st));
    CU(tmpA.ensure((size_t)cw * ch));
    CU(tmpB.ensure((size_t)W * ch));
    nanToKernel<<<grid1((size_t)cw * ch), 256, 0, st>>>((size_t)cw * ch, dCoarse, 1e-4f, tmpA.p);
    lanczosHKernel<<<grid2(W, ch), block2(), 0, st>>>(cw, ch, W, tmpA.p, dOfs.p, dTaps.p, tmpB.p);
    lanczosVKernel<<<grid2(W, H), block2(), 0, st>>>(ch, W, H, tmpB.p, dOfs.p + W, dTaps.p + (size_t)W * 8, dOut);
    if (c) c->launches += 3;
  }
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) return fail(DERP_ECUDA, std::string("upsample kernels: ") + cudaGetErrorString(e));
  return DERP_OK;
}

__global__ void andMaskKernel(size_t n, const uint8_t* a, const uint8_t* b, uint8_t* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (a[i] && b[i]) ? 1 : 0;
}

}  // namespace

extern "C" {

// shared body of derp_upsample_from / derp_upsample_from_kept: dCoarse is a device plane; every temporary belongs to the
// context (no allocation, no host synchronisation per call)
static int upsampleIntoLevel(DerpCtx* c, int dst, const float* dCoarse, int cw, int ch, const uint8_t* coarse_mask,
                             const uint8_t* fine_mask, const char* who) {
  const bool useFg = c->lp.use_foreground_masks != 0;
  const int W = c->W, H = c->H;
  const size_t nc = (size_t)cw * ch, n = c->plane;
  if (useFg) {
    if (!coarse_mask || !fine_mask) return fail(DERP_EINVAL, std::string(who) + ": masks required");
    if (!c->haveBg) return fail(DERP_ESTATE, std::string(who) + ": background disparity not set");
    CU(c->dUpMc.ensure(nc));
    CU(c->dUpMu.ensure(n));
    CU(c->dUpFovC.ensure(nc));
    CU(cudaMemcpyAsync(c->dUpMc.p, coarse_mask, nc, cudaMemcpyDefault, c->stream));
    CU(cudaMemcpyAsync(c->dUpMu.p, fine_mask, n, cudaMemcpyDefault, c->stream));
    // FOV masks at both sizes (UpsampleDisparityLib.cpp:163-176)
    fovMaskKernel<<<grid2(cw, ch), block2(), 0, c->stream>>>(c->dCams.p + c->dst2src[dst], cw, ch, c->dUpFovC.p);
    andMaskKernel<<<grid1(nc), 256, 0, c->stream>>>(nc, c->dUpFovC.p, c->dUpMc.p, c->dUpMc.p);
    andMaskKernel<<<grid1(n), 256, 0, c->stream>>>(n, c->dFov.p + (size_t)dst * n, c->dUpMu.p, c->dUpMu.p);
    c->launches += 3;
  }
  return upsampleDevice(c, c->stream, dCoarse, cw, ch, useFg ? c->bgOf(dst) : nullptr, useFg ? c->dUpMc.p : nullptr,
                        useFg ? c->dUpMu.p : nullptr, W, H, useFg, c->dDisp.p + (size_t)dst * n, c->dUpA, c->dUpB, c->dOfs,
                        c->dTaps, c->dSpiral);
}

int derp_upsample_from(DerpCtx* c, int dst, const float* coarse, int coarse_w, int coarse_h, const uint8_t* coarse_mask,
                       const uint8_t* fine_mask) {
  if (!coarse || coarse_w < 1 || coarse_h < 1) return fail(DERP_EINVAL, "derp_upsample_from: bad arguments");
  int rc = checkDst(c, dst, "derp_upsample_from", false);
  if (rc) return rc;
  const size_t nc = (size_t)coarse_w * coarse_h;
  cudaPointerAttributes a;
  const bool onDevice = cudaPointerGetAttributes(&a, coarse) == cudaSuccess &&
      (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged);
  cudaGetLastError();
  const float* dCoarse = coarse;
  if (!onDevice) {  // host plane (the PFM a caller read back): staged once into a context buffer
    CU(c->dUpCoarse.ensure(nc));
    CU(cudaMemcpyAsync(c->dUpCoarse.p, coarse, nc * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    dCoarse = c->dUpCoarse.p;
  }
  rc = upsampleIntoLevel(c, dst, dCoarse, coarse_w, coarse_h, coarse_mask, fine_mask, "derp_upsample_from");
  if (rc == DERP_OK && !onDevice) CU(cudaStreamSynchronize(c->stream));  // the caller's host plane may be reused on return
  return rc;
}

int derp_level_keep(DerpCtx* c) {
  if (!c || !c->levelOpen) return fail(DERP_ESTATE, "derp_level_keep: no level is open");
  const size_t n = c->plane * (size_t)c->Sd;
  CU(cudaSetDevice(c->device));
  CU(c->dKept.ensure(n));
  CU(cudaMemcpyAsync(c->dKept.p, c->dDisp.p, n * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));
  c->keptW = c->W;
  c->keptH = c->H;
  c->keptSd = c->Sd;
  return DERP_OK;
}

int derp_upsample_from_kept(DerpCtx* c, int dst, const uint8_t* coarse_mask, const uint8_t* fine_mask) {
  int rc = checkDst(c, dst, "derp_upsample_from_kept", false);
  if (rc) return rc;
  if (c->keptW < 1 || c->keptSd != c->Sd) return fail(DERP_ESTATE, "derp_upsample_from_kept: derp_level_keep has not been called");
  const size_t nc = (size_t)c->keptW * c->keptH;
  return upsampleIntoLevel(c, dst, c->dKept.p + (size_t)dst * nc, c->keptW, c->keptH, coarse_mask, fine_mask,
                           "derp_upsample_from_kept");
}

// computeResizeAreaTab (resize.cpp) as per-destination tap ranges
static void areaTaps(int ssize, int dsize, std::vector<int>& ofs, std::vector<int>& si, std::vector<float>& alpha) {
  const double scale = (double)ssize / dsize;
  ofs.assign(1, 0);
  si.clear();
  alpha.clear();
  for (int dx = 0; dx < dsize; ++dx) {
    const double fsx1 = dx * scale, fsx2 = fsx1 + scale;
    const double cellWidth = std::min(scale, ssize - fsx1);
    int sx1 = (int)std::ceil(fsx1), sx2 = (int)std::floor(fsx2);
    sx2 = std::min(sx2, ssize - 1);
    sx1 = std::min(sx1, sx2);
    if (sx1 - fsx1 > 1e-3) {
      si.push_back(sx1 - 1);
      alpha.push_back((float)((sx1 - fsx1) / cellWidth));
    }
    for (int sx = sx1; sx < sx2; ++sx) {
      si.push_back(sx);
      alpha.push_back(float(1.0 / cellWidth));
    }
    if (fsx2 - sx2 > 1e-3) {
      si.push_back(sx2);
      alpha.push_back((float)(std::min(std::min(fsx2 - sx2, 1.), cellWidth) / cellWidth));
    }
    ofs.push_back((int)si.size());
  }
}

int derp_downscale_area(int device, const uint16_t* src, int src_w, int src_h, uint16_t* dst, int dst_w, int dst_h) {
  if (!src || !dst || src_w < 1 || src_h < 1 || dst_w < 1 || dst_h < 1 || dst_w > src_w || dst_h > src_h)
    return fail(DERP_EINVAL, "derp_downscale_area: bad arguments (INTER_AREA is only used to shrink on this path)");
  CU(cudaSetDevice(device));
  const size_t ns = (size_t)src_w * src_h * 3, nd = (size_t)dst_w * dst_h * 3;
  // device-resident images are used in place; host images are staged
  auto onDevice = [](const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
      cudaGetLastError();
      return false;
    }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
  };
  const bool srcDev = onDevice(src), dstDev = onDevice(dst);
  DevBuf<uint16_t> dS, dD;
  const uint16_t* sp = src;
  uint16_t* dp = dst;
  if (!srcDev) {
    CU(dS.ensure(ns));
    CU(cudaMemcpy(dS.p, src, ns * sizeof(uint16_t), cudaMemcpyHostToDevice));
    sp = dS.p;
  }
  if (!dstDev) {
    CU(dD.ensure(nd));
    dp = dD.p;
  }
  const double sx = (double)src_w / dst_w, sy = (double)src_h / dst_h;
  const int kx = (int)std::floor(sx + 0.5), ky = (int)std::floor(sy + 0.5);
  const dim3 grid((dst_w * 3 + 255) / 256, dst_h);
  if (std::fabs(sx - kx) < 2.220446049250313e-16 && std::fabs(sy - ky) < 2.220446049250313e-16) {
    areaResizeFastKernel<<<grid, 256>>>(sp, src_w, dp, dst_w, dst_h, kx, ky);
  } else {
    std::vector<int> xo, xs, yo, ys;
    std::vector<float> xa, ya;
    areaTaps(src_w, dst_w, xo, xs, xa);
    areaTaps(src_h, dst_h, yo, ys, ya);
    DevBuf<int> dXo, dXs, dYo, dYs;
    DevBuf<float> dXa, dYa;
    CU(dXo.ensure(xo.size()));
    CU(dXs.ensure(xs.size()));
    CU(dXa.ensure(xa.size()));
    CU(dYo.ensure(yo.size()));
    CU(dYs.ensure(ys.size()));
    CU(dYa.ensure(ya.size()));
    CU(cudaMemcpy(dXo.p, xo.data(), xo.size() * sizeof(int), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(dXs.p, xs.data(), xs.size() * sizeof(int), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(dXa.p, xa.data(), xa.size() * sizeof(float), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(dYo.p, yo.data(), yo.size() * sizeof(int), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(dYs.p, ys.data(), ys.size() * sizeof(int), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(dYa.p, ya.data(), ya.size() * sizeof(float), cudaMemcpyHostToDevice));
    areaResizeKernel<<<grid, 256>>>(sp, src_w, src_h, dp, dst_w, dst_h, dXo.p, dXs.p, dXa.p, dYo.p, dYs.p, dYa.p);
    CU(cudaDeviceSynchronize());  // tables are freed on return
  }
  CU(cudaGetLastError());
  if (!dstDev) CU(cudaMemcpy(dst, dD.p, nd * sizeof(uint16_t), cudaMemcpyDeviceToHost));
  else if (!srcDev) CU(cudaDeviceSynchronize());  // the staged source is freed on return
  return DERP_OK;
}

int derp_device_alloc(int device, size_t bytes, void** out) {
  if (!out) return fail(DERP_EINVAL, "derp_device_alloc: null out");
  CU(cudaSetDevice(device));
  CU(cudaMalloc(out, bytes ? bytes : 1));
  return DERP_OK;
}
int derp_device_free(int device, void* p) {
  if (!p) return DERP_OK;
  CU(cudaSetDevice(device));
  CU(cudaFree(p));
  return DERP_OK;
}
int derp_device_copy(int device, void* dst, const void* src, size_t bytes) {
  if (!dst || !src) return fail(DERP_EINVAL, "derp_device_copy: null pointer");
  CU(cudaSetDevice(device));
  // a source (or destination) on another GPU: make sure the direct NVLink path is enabled
  for (const void* p : {src, (const void*)dst}) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) == cudaSuccess && a.type == cudaMemoryTypeDevice && a.device != device) {
      int can = 0;
      if (cudaDeviceCanAccessPeer(&can, device, a.device) == cudaSuccess && can) {
        const cudaError_t e = cudaDeviceEnablePeerAccess(a.device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return fail(DERP_ECUDA, cudaGetErrorString(e));
      }
    }
    cudaGetLastError();
  }
  CU(cudaMemcpy(dst, src, bytes, cudaMemcpyDefault));
  return DERP_OK;
}

int derp_foreground_mask(int device, const uint16_t* templ, const uint16_t* frame, int width, int height, int blur_radius,
                         float threshold, int morph_closing_size, uint8_t* mask) {
  if (!templ || !frame || !mask || width < 1 || height < 1 || morph_closing_size < 0)
    return fail(DERP_EINVAL, "derp_foreground_mask: bad arguments");
  if (blur_radius < 0 || blur_radius > 1)
    return fail(DERP_EINVAL, "derp_foreground_mask: blur_radius 0 or 1 (the app's default 3 x 3 Gaussian)");
  CU(cudaSetDevice(device));
  const size_t n = (size_t)width * height;
  DevBuf<uint16_t> dT, dF, dTb, dFb;
  DevBuf<uint8_t> dM, dM2;
  CU(dT.ensure(n * 3));
  CU(dF.ensure(n * 3));
  CU(dM.ensure(n));
  CU(cudaMemcpy(dT.p, templ, n * 6, cudaMemcpyDefault));
  CU(cudaMemcpy(dF.p, frame, n * 6, cudaMemcpyDefault));
  const uint16_t *pt = dT.p, *pf = dF.p;
  if (blur_radius == 1) {
    CU(dTb.ensure(n * 3));
    CU(dFb.ensure(n * 3));
    const dim3 g((width * 3 + 255) / 256, height);
    gaussian3Kernel<<<g, 256>>>(dT.p, width, height, dTb.p);
    gaussian3Kernel<<<g, 256>>>(dF.p, width, height, dFb.p);
    pt = dTb.p;
    pf = dFb.p;
  }
  foregroundDiffKernel<<<grid1(n), 256>>>(n, pt, pf, threshold, dM.p);
  if (morph_closing_size > 0) {  // MORPH_CLOSE = dilate, then erode
    CU(dM2.ensure(n));
    morphRectKernel<<<grid2(width, height), block2()>>>(dM.p, width, height, morph_closing_size, 1, dM2.p);
    morphRectKernel<<<grid2(width, height), block2()>>>(dM2.p, width, height, morph_closing_size, 0, dM.p);
  }
  CU(cudaGetLastError());
  CU(cudaMemcpy(mask, dM.p, n, cudaMemcpyDefault));
  return DERP_OK;
}

// cv::resize(depth, depth, Size(), s, s, INTER_NEAREST) (ConvertToBinary.cpp:153-156): dsize = cvRound(size * s),
// source index = min(floor(d * (1 / s)), size - 1) (resize.cpp resizeNN with the caller's scale factors)
static void meshAxis(int sn, double scale, std::vector<int>& ofs) {
  if (!(scale < 1)) {
    ofs.resize(sn);
    for (int d = 0; d < sn; ++d) ofs[d] = d;
    return;
  }
  const int dn = (int)std::nearbyint(sn * scale);
  const double ifx = 1. / scale;
  ofs.resize(std::max(dn, 0));
  for (int d = 0; d < dn; ++d) ofs[d] = std::min(floorD(d * ifx), sn - 1);
}

int derp_camera_mesh_size(int width, int height, double depth_scale, int* mesh_width, int* mesh_height) {
  if (width < 1 || height < 1 || !(depth_scale > 0) || depth_scale > 1 || !mesh_width || !mesh_height)
    return fail(DERP_EINVAL, "derp_camera_mesh_size: bad arguments (depth_scale in (0, 1], ConvertToBinary.cpp:348)");
  *mesh_width = depth_scale < 1 ? (int)std::nearbyint(width * depth_scale) : width;
  *mesh_height = depth_scale < 1 ? (int)std::nearbyint(height * depth_scale) : height;
  return DERP_OK;
}

static int cameraMesh(int device, const float* disparity, int width, int height, double depth_scale, double resolution_x,
                      double resolution_y, double scalar_focal, float tear_ratio, const uint8_t* foreground_mask,
                      int mask_width, int mask_height, int triangles, float* vertexes, uint32_t* faces,
                      uint64_t* num_vertexes, uint64_t* num_faces) {
  int W = 0, H = 0;
  int rc = derp_camera_mesh_size(width, height, depth_scale, &W, &H);
  if (rc) return rc;
  if (!disparity || !vertexes || !faces || !num_vertexes || !num_faces || W < 1 || H < 1 ||
      (foreground_mask && (mask_width < 1 || mask_height < 1)))
    return fail(DERP_EINVAL, "derp_camera_mesh: bad arguments");
  CU(cudaSetDevice(device));
  const size_t n = (size_t)W * H, nsrc = (size_t)width * height;
  if (n >= (1ull << 31)) return fail(DERP_EINVAL, "derp_camera_mesh: grid too large for 32-bit indexes");
  std::vector<int> ofs, tmp;
  meshAxis(width, depth_scale, ofs);
  meshAxis(height, depth_scale, tmp);
  ofs.insert(ofs.end(), tmp.begin(), tmp.end());
  if (foreground_mask) {  // cv::resize(mask, mask, depth.size(), 0, 0, INTER_NEAREST), ConvertToBinary.cpp:171-174
    nearestAxis(mask_width, W, tmp);
    ofs.insert(ofs.end(), tmp.begin(), tmp.end());
    nearestAxis(mask_height, H, tmp);
    ofs.insert(ofs.end(), tmp.begin(), tmp.end());
  }
  // grow-only scratch per host thread (the app converts one (frame, camera) after the other on each GPU worker thread)
  struct MeshScratch {
    DevBuf<float> dDisp, dVtx;
    DevBuf<double> dVtx64;
    DevBuf<int> dOfs;
    DevBuf<uint8_t> dFg, dQuad, dUsed;
    DevBuf<unsigned> dTiles, dIndex, dFaces;
    DevBuf<unsigned long long> dTotals;
    int device = -1;
  };
  static thread_local MeshScratch sc;
  if (sc.device != device) {  // the thread moved to another GPU: the old buffers belong to the old device
    if (sc.device >= 0) {
      cudaSetDevice(sc.device);
      sc.dDisp.release();
      sc.dVtx.release();
      sc.dVtx64.release();
      sc.dOfs.release();
      sc.dFg.release();
      sc.dQuad.release();
      sc.dUsed.release();
      sc.dTiles.release();
      sc.dIndex.release();
      sc.dFaces.release();
      sc.dTotals.release();
      CU(cudaSetDevice(device));
    }
    sc.device = device;
  }
  DevBuf<float>&dDisp = sc.dDisp, &dVtx = sc.dVtx;
  DevBuf<int>& dOfs = sc.dOfs;
  DevBuf<uint8_t>&dFg = sc.dFg, &dQuad = sc.dQuad, &dUsed = sc.dUsed;
  DevBuf<unsigned>&dTiles = sc.dTiles, &dIndex = sc.dIndex, &dFaces = sc.dFaces;
  DevBuf<unsigned long long>& dTotals = sc.dTotals;
  const float* disp = disparity;
  const uint8_t* fg = foreground_mask;
  cudaPointerAttributes at{};
  if (cudaPointerGetAttributes(&at, disparity) != cudaSuccess || at.type != cudaMemoryTypeDevice) {
    (void)cudaGetLastError();
    CU(dDisp.ensure(nsrc));
    CU(cudaMemcpy(dDisp.p, disparity, nsrc * sizeof(float), cudaMemcpyDefault));
    disp = dDisp.p;
  }
  if (fg && (cudaPointerGetAttributes(&at, fg) != cudaSuccess || at.type != cudaMemoryTypeDevice)) {
    (void)cudaGetLastError();
    CU(dFg.ensure((size_t)mask_width * mask_height));
    CU(cudaMemcpy(dFg.p, fg, (size_t)mask_width * mask_height, cudaMemcpyDefault));
    fg = dFg.p;
  }
  const int tiles = (int)((n + kScanTile - 1) / kScanTile);
  CU(dOfs.ensure(ofs.size()));
  CU(cudaMemcpy(dOfs.p, ofs.data(), ofs.size() * sizeof(int), cudaMemcpyHostToDevice));
  CU(dQuad.ensure(n));
  CU(dUsed.ensure(n));
  CU(dTiles.ensure(2 * (size_t)tiles));
  CU(dIndex.ensure(n));
  CU(dTotals.ensure(2));
  CU(cudaMemset(dUsed.p, 0, n));
  MeshGrid g;
  g.W = W;
  g.H = H;
  g.srcW = width;
  g.disp = disp;
  g.xofs = dOfs.p;
  g.yofs = dOfs.p + W;
  g.fg = fg;
  g.fgW = mask_width;
  g.fgx = dOfs.p + W + H;
  g.fgy = dOfs.p + 2 * (size_t)W + H;
  g.stepX = resolution_x / W;
  g.stepY = resolution_y / H;
  g.scale = scalar_focal * 1.0;  // kRadius = 1 (MeshUtil.h:316)
  g.tearRatio = tear_ratio;
  g.floorZ = 0;
  meshQuadKernel<<<grid2(W, H), block2()>>>(g, dQuad.p, dUsed.p);
  meshTileCountKernel<<<tiles, kScanThreads>>>(n, dQuad.p, dUsed.p, dTiles.p, dTiles.p + tiles);
  meshTileScanKernel<<<1, kScanThreads>>>(tiles, dTiles.p, dTiles.p + tiles, dTotals.p);
  CU(cudaGetLastError());
  unsigned long long totals[2] = {0, 0};
  CU(cudaMemcpy(totals, dTotals.p, sizeof(totals), cudaMemcpyDeviceToHost));
  if (triangles > 0 && totals[0] > (unsigned long long)triangles) {
    // Simplification (ConvertToBinary.cpp:186-203): the mesh in double precision goes to the host, where the strictly
    // sequential edge-contraction sweeps run (derp_simplify.h), like MeshSimplifier with kThreads = 1 in the reference.
    DevBuf<double>& dVtx64 = sc.dVtx64;
    CU(dVtx64.ensure(std::max<size_t>(1, totals[1] * 3)));
    CU(dFaces.ensure(std::max<size_t>(1, totals[0] * 3)));
    g.floorZ = 0;  // the simplifier works on the raw values; the floor is applied to its output below
    meshEmitVertexesKernel<double><<<tiles, kScanThreads>>>(g, dUsed.p, dTiles.p + tiles, dIndex.p, dVtx64.p);
    meshEmitFacesKernel<<<tiles, kScanThreads>>>(W, n, dQuad.p, dTiles.p, dIndex.p, dFaces.p);
    CU(cudaGetLastError());
    std::vector<double> hv(totals[1] * 3);
    std::vector<uint32_t> hf(totals[0] * 3);
    CU(cudaMemcpy(hv.data(), dVtx64.p, hv.size() * sizeof(double), cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(hf.data(), dFaces.p, hf.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    simplify::Mesh mesh(hv.data(), totals[1], hf.data(), totals[0]);
    mesh.run(triangles, 0.2f, false);  // kStrictness, kRemoveBoundaryEdges (ConvertToBinary.cpp:193-195)
    std::vector<float> ov(mesh.verts.size() * 3);
    std::vector<uint32_t> of(mesh.faces.size() * 3);
    for (size_t i = 0; i < mesh.verts.size(); ++i) {
      const simplify::V3& p = mesh.verts[i].p;
      ov[3 * i] = (float)p.x;
      ov[3 * i + 1] = (float)p.y;
      ov[3 * i + 2] = (float)(p.z < 0 ? (double)FLT_MIN : p.z);  // ConvertToBinary.cpp:199-203
    }
    for (size_t i = 0; i < mesh.faces.size(); ++i)
      for (int j = 0; j < 3; ++j) of[3 * i + j] = (uint32_t)mesh.faces[i].v[j];
    CU(cudaMemcpy(vertexes, ov.data(), ov.size() * sizeof(float), cudaMemcpyDefault));
    CU(cudaMemcpy(faces, of.data(), of.size() * sizeof(uint32_t), cudaMemcpyDefault));
    *num_vertexes = mesh.verts.size();
    *num_faces = mesh.faces.size();
    return DERP_OK;
  }
  g.floorZ = triangles > 0;  // the reference applies it after the (here: no-op) simplification
  // outputs: written in place when the caller's buffers are device memory, else staged
  float* vtx = vertexes;
  uint32_t* fac = faces;
  if (cudaPointerGetAttributes(&at, vertexes) != cudaSuccess || at.type != cudaMemoryTypeDevice) {
    (void)cudaGetLastError();
    CU(dVtx.ensure(std::max<size_t>(1, totals[1] * 3)));
    vtx = dVtx.p;
  }
  if (cudaPointerGetAttributes(&at, faces) != cudaSuccess || at.type != cudaMemoryTypeDevice) {
    (void)cudaGetLastError();
    CU(dFaces.ensure(std::max<size_t>(1, totals[0] * 3)));
    fac = dFaces.p;
  }
  meshEmitVertexesKernel<float><<<tiles, kScanThreads>>>(g, dUsed.p, dTiles.p + tiles, dIndex.p, vtx);
  meshEmitFacesKernel<<<tiles, kScanThreads>>>(W, n, dQuad.p, dTiles.p, dIndex.p, fac);
  CU(cudaGetLastError());
  if (vtx != vertexes) CU(cudaMemcpy(vertexes, vtx, totals[1] * 3 * sizeof(float), cudaMemcpyDefault));
  if (fac != faces) CU(cudaMemcpy(faces, fac, totals[0] * 3 * sizeof(uint32_t), cudaMemcpyDefault));
  CU(cudaDeviceSynchronize());
  *num_faces = totals[0];
  *num_vertexes = totals[1];
  return DERP_OK;
}

int derp_camera_mesh(int device, const float* disparity, int width, int height, double depth_scale, double resolution_x,
                     double resolution_y, double scalar_focal, float tear_ratio, const uint8_t* foreground_mask,
                     int mask_width, int mask_height, float* vertexes, uint32_t* faces, uint64_t* num_vertexes,
                     uint64_t* num_faces) {
  return cameraMesh(device, disparity, width, height, depth_scale, resolution_x, resolution_y, scalar_focal, tear_ratio,
                    foreground_mask, mask_width, mask_height, 0, vertexes, faces, num_vertexes, num_faces);
}

int derp_camera_mesh_simplified(int device, const float* disparity, int width, int height, double depth_scale,
                                double resolution_x, double resolution_y, double scalar_focal, float tear_ratio,
                                const uint8_t* foreground_mask, int mask_width, int mask_height, int triangles,
                                float* vertexes, uint32_t* faces, uint64_t* num_vertexes, uint64_t* num_faces) {
  return cameraMesh(device, disparity, width, height, depth_scale, resolution_x, resolution_y, scalar_focal, tear_ratio,
                    foreground_mask, mask_width, mask_height, triangles, vertexes, faces, num_vertexes, num_faces);
}

int derp_upsample_disparity(int device, const DerpCameraDesc* cam, const float* coarse, int coarse_w, int coarse_h,
                            const float* background_up, const uint8_t* coarse_mask, const uint8_t* fine_mask, int out_w,
                            int out_h, int use_foreground_masks, float* out) {
  if (!cam || !coarse || !out || coarse_w < 1 || coarse_h < 1 || out_w < 1 || out_h < 1)
    return fail(DERP_EINVAL, "derp_upsample_disparity: bad arguments");
  CU(cudaSetDevice(device));
  const size_t nc = (size_t)coarse_w * coarse_h, n = (size_t)out_w * out_h;
  DevBuf<float> dCoarse, dBg, dOut, tA, tB, dTaps;
  DevBuf<uint8_t> dMc, dMu, dFovC, dFovU;
  DevBuf<int> dOfs;
  DevBuf<short2> dSpiral;
  DevBuf<DevCamera> dCam;
  cudaStream_t st = nullptr;  // legacy default stream: this entry point is synchronous
  CU(dCoarse.ensure(nc));
  CU(dOut.ensure(n));
  CU(cudaMemcpy(dCoarse.p, coarse, nc * sizeof(float), cudaMemcpyHostToDevice));
  if (use_foreground_masks) {
    if (!coarse_mask || !fine_mask || !background_up) return fail(DERP_EINVAL, "derp_upsample_disparity: masks/background required");
    DevCamera hc;
    if (!host::makeCamera(*cam, &hc)) return fail(DERP_EINVAL, "derp_upsample_disparity: invalid camera");
    host::normalise(hc);
    CU(dCam.ensure(1));
    CU(cudaMemcpy(dCam.p, &hc, sizeof(hc), cudaMemcpyHostToDevice));
    CU(dBg.ensure(n));
    CU(dMc.ensure(nc));
    CU(dMu.ensure(n));
    CU(dFovC.ensure(nc));
    CU(dFovU.ensure(n));
    CU(cudaMemcpy(dBg.p, background_up, n * sizeof(float), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(dMc.p, coarse_mask, nc, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(dMu.p, fine_mask, n, cudaMemcpyHostToDevice));
    fovMaskKernel<<<grid2(coarse_w, coarse_h), block2(), 0, st>>>(dCam.p, coarse_w, coarse_h, dFovC.p);
    fovMaskKernel<<<grid2(out_w, out_h), block2(), 0, st>>>(dCam.p, out_w, out_h, dFovU.p);
    andMaskKernel<<<grid1(nc), 256, 0, st>>>(nc, dFovC.p, dMc.p, dMc.p);
    andMaskKernel<<<grid1(n), 256, 0, st>>>(n, dFovU.p, dMu.p, dMu.p);
  }
  int rc = upsampleDevice(nullptr, st, dCoarse.p, coarse_w, coarse_h, use_foreground_masks ? dBg.p : nullptr,
                          use_foreground_masks ? dMc.p : nullptr, use_foreground_masks ? dMu.p : nullptr, out_w, out_h,
                          use_foreground_masks != 0, dOut.p, tA, tB, dOfs, dTaps, dSpiral);
  if (rc) return rc;
  CU(cudaMemcpy(out, dOut.p, n * sizeof(float), cudaMemcpyDeviceToHost));
  return DERP_OK;
}

int derp_level_estimate(DerpCtx* c, const DerpProcessOpts* o) {
  if (!c || !o) return fail(DERP_EINVAL, "derp_level_estimate: bad arguments");
  if (!c->levelOpen || !c->haveColors) return fail(DERP_ESTATE, "derp_level_estimate: level/colours not set");
  const bool coarsest = c->lp.level == c->lp.num_levels - 1;
  // The work counters accumulate on the device across all stages and destinations and are read back once: a
  // read-back per stage would drain the stream ~3 times per destination, which dominates the small levels.
  int rc = useDevice(c);
  if (rc) return rc;
  if ((rc = resetCounters(c))) return rc;
  c->accumulateCounters = true;
  for (int d = 0; d < c->Sd && !rc; ++d) {
    if ((rc = derp_reproject(c, d))) break;
    if (coarsest)  // preprocessLevel (Derp.cpp:826-842)
      rc = derp_brute_force(c, d, o->num_depths, o->min_depth_m, o->max_depth_m, o->partial_coverage, nullptr);
    if (!rc && o->random_proposals > 0 && !coarsest)  // Derp.cpp:851-853
      rc = derp_random_proposals(c, d, o->random_proposals, o->min_depth_m, o->max_depth_m);
    if (!rc && !coarsest)  // Derp.cpp:545-547
      rc = derp_ping_pong(c, d, o->ping_pong_iterations);
  }
  c->accumulateCounters = false;
  if (rc) return rc;
  if ((rc = readCounters(c))) return rc;  // synchronises the stream
  c->countersOnDevice = false;
  return DERP_OK;
}

int derp_level_filter(DerpCtx* c, const DerpProcessOpts* o) {
  if (!c || !o) return fail(DERP_EINVAL, "derp_level_filter: bad arguments");
  if (!c->levelOpen || !c->haveColors) return fail(DERP_ESTATE, "derp_level_filter: level/colours not set");
  int rc;
  for (int d = 0; d < c->Sd; ++d) {
    if (o->do_bilateral_filter && (rc = derp_bilateral(c, d))) return rc;
    if (o->do_median_filter && (rc = derp_median(c, d))) return rc;
    if ((rc = derp_mask_fov(c, d))) return rc;
  }
  CU(cudaStreamSynchronize(c->stream));
  return DERP_OK;
}

int derp_process_level(DerpCtx* c, const DerpProcessOpts* o) {
  int rc = derp_level_estimate(c, o);
  if (rc) return rc;
  const bool coarsest = c->lp.level == c->lp.num_levels - 1;
  if (!(c->lp.level > o->mismatches_start_level || coarsest)) {  // Derp.cpp:726-728
    if ((rc = derp_mismatches(c))) return rc;
  }
  const uint64_t evals = c->lastEvals, hits = c->lastHits;
  if ((rc = derp_level_filter(c, o))) return rc;
  c->lastEvals = evals;
  c->lastHits = hits;
  c->countersOnDevice = false;
  return DERP_OK;
}

// ---- state access ------------------------------------------------------------------------------------
int derp_set_disparity(DerpCtx* c, int dst, const float* disparity, const float* cost, const float* confidence) {
  int rc = checkDst(c, dst, "derp_set_disparity", false);
  if (rc) return rc;
  const size_t n = c->plane, b = n * sizeof(float);
  if (disparity) CU(cudaMemcpyAsync(c->dDisp.p + (size_t)dst * n, disparity, b, cudaMemcpyDefault, c->stream));
  if (cost) CU(cudaMemcpyAsync(c->dCost.p + (size_t)dst * n, cost, b, cudaMemcpyDefault, c->stream));
  if (confidence) CU(cudaMemcpyAsync(c->dConf.p + (size_t)dst * n, confidence, b, cudaMemcpyDefault, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return DERP_OK;
}

int derp_get_disparity(DerpCtx* c, int dst, float* disparity, float* cost, float* confidence) {
  int rc = checkDst(c, dst, "derp_get_disparity", false);
  if (rc) return rc;
  const size_t n = c->plane, b = n * sizeof(float);
  if (disparity) CU(cudaMemcpyAsync(disparity, c->dDisp.p + (size_t)dst * n, b, cudaMemcpyDefault, c->stream));
  if (cost) CU(cudaMemcpyAsync(cost, c->dCost.p + (size_t)dst * n, b, cudaMemcpyDefault, c->stream));
  if (confidence) CU(cudaMemcpyAsync(confidence, c->dConf.p + (size_t)dst * n, b, cudaMemcpyDefault, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return DERP_OK;
}

int derp_get_fov_mask(DerpCtx* c, int dst, uint8_t* mask) {
  if (!mask) return fail(DERP_EINVAL, "bad arguments");
  int rc = checkDst(c, dst, "derp_get_fov_mask", false);
  if (rc) return rc;
  CU(cudaMemcpyAsync(mask, c->dFov.p + (size_t)dst * c->plane, c->plane, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return DERP_OK;
}

int derp_get_mismatch_mask(DerpCtx* c, int dst, uint8_t* mask) {
  if (!mask) return fail(DERP_EINVAL, "bad arguments");
  int rc = checkDst(c, dst, "derp_get_mismatch_mask", false);
  if (rc) return rc;
  CU(cudaMemcpyAsync(mask, c->dMismatch.p + (size_t)dst * c->plane, c->plane, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return DERP_OK;
}

int derp_get_variance(DerpCtx* c, int src, float* variance) {
  if (!c || !variance) return fail(DERP_EINVAL, "bad arguments");
  if (!c->levelOpen || !c->haveColors) return fail(DERP_ESTATE, "derp_get_variance: colours not set");
  if (src < 0 || src >= c->S) return fail(DERP_EINVAL, "src out of range");
  int rc = useDevice(c);
  if (rc) return rc;
  CU(cudaMemcpyAsync(variance, c->dVariance.p + (size_t)src * c->plane, c->plane * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return DERP_OK;
}

int derp_get_var_noise_floor(DerpCtx* c, float* out) {
  if (!c || !out || !c->levelOpen) return fail(DERP_EINVAL, "bad arguments");
  *out = c->varNoiseFloor;
  return DERP_OK;
}

static int checkProj(DerpCtx* c, int src, const char* who) {
  if (!c) return fail(DERP_EINVAL, "null ctx");
  if (!c->levelOpen || c->projDst < 0) return fail(DERP_ESTATE, std::string(who) + ": no projection tables");
  if (src < 0 || src >= c->S) return fail(DERP_EINVAL, std::string(who) + ": src out of range");
  return useDevice(c);
}

int derp_get_proj_warp(DerpCtx* c, int src, float* warp_xy) {
  if (!warp_xy) return fail(DERP_EINVAL, "bad arguments");
  int rc = checkProj(c, src, "derp_get_proj_warp");
  if (rc) return rc;
  CU(cudaMemcpyAsync(warp_xy, c->warpOf(c->projDst) + (size_t)src * c->plane, c->plane * sizeof(float2), cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return DERP_OK;
}

static int getTexels(DerpCtx* c, const float4* plane, uint16_t* bgr) {
  const size_t n = c->plane;
  uint16_t* st = reinterpret_cast<uint16_t*>(c->dStage.p);
  unpackTexelF32Kernel<<<grid1(n), 256, 0, c->stream>>>(n, plane, st);
  LAUNCHED("unpackTexelF32Kernel");
  CU(cudaMemcpyAsync(bgr, st, n * 6, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return DERP_OK;
}

int derp_get_proj_color(DerpCtx* c, int src, uint16_t* bgr) {
  if (!bgr) return fail(DERP_EINVAL, "bad arguments");
  int rc = checkProj(c, src, "derp_get_proj_color");
  if (rc) return rc;
  if ((rc = ensureTablesF32(c))) return rc;
  return getTexels(c, c->dProjColor.p + (size_t)src * c->plane, bgr);
}

int derp_get_proj_bias(DerpCtx* c, int src, uint16_t* bgr) {
  if (!bgr) return fail(DERP_EINVAL, "bad arguments");
  int rc = checkProj(c, src, "derp_get_proj_bias");
  if (rc) return rc;
  if ((rc = ensureTablesF32(c))) return rc;
  return getTexels(c, c->dProjBias.p + (size_t)src * c->plane, bgr);
}

int derp_get_counters(DerpCtx* c, uint64_t* cost_evals, uint64_t* src_hits) {
  if (!c) return fail(DERP_EINVAL, "null ctx");
  int rc = useDevice(c);
  if (rc) return rc;
  if (c->countersOnDevice) {  // stage-level calls leave their counters on the device
    if ((rc = readCounters(c))) return rc;
    c->countersOnDevice = false;
  }
  if (cost_evals) *cost_evals = c->lastEvals;
  if (src_hits) *src_hits = c->lastHits;
  return DERP_OK;
}

int derp_set_sweep_mode(DerpCtx* c, int mode) {
  if (!c || mode < 0 || mode > 2) return fail(DERP_EINVAL, "derp_set_sweep_mode: bad arguments");
  c->sweepMode = mode;
  return DERP_OK;
}

/* Exact evaluations of the last derp_brute_force when it ran as the filtered sweep (derp_refine.cuh): refined list
 * entries and seeds (one per pixel plane entry launched); both 0 after a plain sweep. */
int derp_get_sweep_stats(DerpCtx* c, uint64_t* refined, uint64_t* seeds) {
  if (!c) return fail(DERP_EINVAL, "derp_get_sweep_stats: null context");
  if (refined) *refined = c->lastRefined;
  if (seeds) *seeds = c->lastSeeds;
  return DERP_OK;
}

/* Test hook: validates the lower bounds of the filtered sweep against the exact cost of EVERY (pixel, candidate) of one
 * destination.  stats[5]: evaluations compared, violations (bound > exact cost; must be 0), bounds not formed,
 * bounds within 5 % of the exact cost, candidates a threshold at the true per-pixel minimum keeps. */
int derp_debug_lower_bound(DerpCtx* c, int dst, int num_depths, float min_depth_m, float max_depth_m, uint64_t* stats) {
  int rc = checkDst(c, dst, "derp_debug_lower_bound", true);
  if (rc) return rc;
  if (num_depths < 2 || !stats) return fail(DERP_EINVAL, "derp_debug_lower_bound: bad arguments");
  const int W = c->W, H = c->H;
  const size_t n = c->plane;
  const std::vector<float> disparities = probeDisparities(num_depths, min_depth_m, max_depth_m);
  DevBuf<float> dTab;
  DevBuf<unsigned long long> dStats;
  CU(dTab.ensure(num_depths));
  CU(dStats.ensure(5));
  CU(cudaMemcpyAsync(dTab.p, disparities.data(), num_depths * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  CU(cudaMemsetAsync(dStats.p, 0, 5 * sizeof(unsigned long long), c->stream));
  if ((rc = ensureTablesF32(c))) return rc;
  CU(c->dLb.ensure((size_t)num_depths * n));
  CU(c->dSeed.ensure(n));
  fillKernel<unsigned long long><<<grid1(n), 256, 0, c->stream>>>(n, c->dSeed.p, 0x7f7fffffffffffffull);
  LAUNCHED("fillKernel");
  if ((rc = resetCounters(c))) return rc;
  const LowerArgs la = lowerArgs(c, dst, dTab.p, num_depths, num_depths);
  const int by = kBlockY;
  SMEM_FITS(c->camSmem(kBlockX * by), "sweepLowerKernel");
  SMEM_FITS(c->camSmem(), "lowerBoundCheckKernel");
  c->k.sweepLower<<<dim3((W + kBlockX - 1) / kBlockX, (H + by - 1) / by, 1), dim3(kBlockX, by, 1), c->camSmem(kBlockX * by), c->stream>>>(la);
  LAUNCHED("sweepLowerKernel");
  CheckArgs ca;
  ca.v = la.v;
  ca.fov = la.fov;
  ca.fg = la.fg;
  ca.bg = la.bg;
  ca.disparities = dTab.p;
  ca.D = num_depths;
  ca.lb = c->dLb.p;
  ca.stats = dStats.p;
  c->k.lowerBoundCheck<<<grid2(W, H), block2(), c->camSmem(), c->stream>>>(ca);
  LAUNCHED("lowerBoundCheckKernel");
  unsigned long long h[5];
  CU(cudaMemcpyAsync(h, dStats.p, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  for (int i = 0; i < 5; ++i) stats[i] = h[i];
  return DERP_OK;
}

// temporalJointBilateralFilter (TemporalBilateralFilter.h:126-215) for one camera
int derp_temporal_filter(int device, int width, int height, int num_frames, const uint16_t* const* guides,
                         const float* const* disps, const uint8_t* const* masks, int frame_offset, float sigma,
                         int spatial_radius, float weight0, float weight1, float weight2, float* out) {
  if (!guides || !disps || !masks || !out || num_frames < 1 || frame_offset < 0 || frame_offset >= num_frames || width < 1 ||
      height < 1 || spatial_radius < 0)
    return fail(DERP_EINVAL, "derp_temporal_filter: bad arguments");
  CU(cudaSetDevice(device));
  const size_t n = (size_t)width * height;
  // grow-only scratch per host thread (one thread drives one GPU): a sequence filters thousands of (frame, camera)
  // windows of the same size, cudaMalloc per call would dominate the 0.8 ms kernel
  struct Scratch {
    DevBuf<uint2> dG;
    DevBuf<float> dD, dOut;
    DevBuf<uint8_t> dM, dStage;
    int device = -1;
  };
  static thread_local Scratch sc;
  if (sc.device != device) {  // the thread moved to another GPU: the old buffers belong to the old device
    if (sc.device >= 0) {
      cudaSetDevice(sc.device);
      sc.dG.release();
      sc.dD.release();
      sc.dOut.release();
      sc.dM.release();
      sc.dStage.release();
      CU(cudaSetDevice(device));
    }
    sc.device = device;
  }
  DevBuf<uint2>& dG = sc.dG;
  DevBuf<float>&dD = sc.dD, &dOut = sc.dOut;
  DevBuf<uint8_t>&dM = sc.dM, &dStage = sc.dStage;
  CU(dG.ensure(n * num_frames));
  CU(dD.ensure(n * num_frames));
  CU(dM.ensure(n * num_frames));
  CU(dOut.ensure(n));
  CU(dStage.ensure(n * 6));
  for (int t = 0; t < num_frames; ++t) {  // frames may live in host or device memory (e.g. halo frames received over NVLink)
    CU(cudaMemcpy(dStage.p, guides[t], n * 6, cudaMemcpyDefault));
    packColorKernel<<<grid1(n), 256>>>(n, reinterpret_cast<const uint16_t*>(dStage.p), dG.p + (size_t)t * n);
    CU(cudaMemcpy(dD.p + (size_t)t * n, disps[t], n * sizeof(float), cudaMemcpyDefault));
    CU(cudaMemcpy(dM.p + (size_t)t * n, masks[t], n, cudaMemcpyDefault));
  }
  TemporalArgs a;
  a.W = width;
  a.H = height;
  a.T = num_frames;
  a.frameOffset = frame_offset;
  a.radius = spatial_radius;
  a.guides = dG.p;
  a.disps = dD.p;
  a.masks = dM.p;
  CU(makeDivConst(65535.0f, 0, &a.maxPix));
  CU(makeDivConst(sigma * sigma, 0, &a.sig2));
  a.w0 = weight0;
  a.w1 = weight1;
  a.w2 = weight2;
  a.out = dOut.p;
  temporalKernel<<<grid2(width, height), block2()>>>(a);
  CU(cudaGetLastError());
  CU(cudaMemcpy(out, dOut.p, n * sizeof(float), cudaMemcpyDefault));
  return DERP_OK;
}

int derp_joint_bilateral_f32(int device, int width, int height, const float* image, const float* guide_bgr,
                             const uint8_t* mask, int radius, float sigma, float weight0, float weight1, float weight2,
                             float* out) {
  if (!image || !guide_bgr || !mask || !out || radius < 0 || width < 1 || height < 1)
    return fail(DERP_EINVAL, "derp_joint_bilateral_f32: bad arguments");
  CU(cudaSetDevice(device));
  const size_t n = (size_t)width * height;
  DevBuf<float> dI, dG, dO;
  DevBuf<uint8_t> dM;
  CU(dI.ensure(n));
  CU(dG.ensure(n * 3));
  CU(dO.ensure(n));
  CU(dM.ensure(n));
  CU(cudaMemcpy(dI.p, image, n * sizeof(float), cudaMemcpyHostToDevice));
  CU(cudaMemcpy(dG.p, guide_bgr, n * 3 * sizeof(float), cudaMemcpyHostToDevice));
  CU(cudaMemcpy(dM.p, mask, n, cudaMemcpyHostToDevice));
  DivConst three, denom;
  CU(makeDivConst(3.0f, 0, &three));
  CU(makeDivConst(2.0f * (sigma * sigma), 0, &denom));
  if (bilateralSmem(radius) <= kBilMaxSmem)
    bilateralKernel<GuideF32><<<grid2(width, height), block2(), bilateralSmem(radius)>>>(
        width, height, dI.p, GuideF32{dG.p}, dM.p, nullptr, radius, three, denom, weight0, weight1, weight2, dO.p);
  else
    bilateralWideKernel<GuideF32><<<grid2(width, height), block2()>>>(width, height, dI.p, GuideF32{dG.p}, dM.p, nullptr, radius,
                                                                    three, denom, weight0, weight1, weight2, dO.p);
  CU(cudaGetLastError());
  CU(cudaMemcpy(out, dO.p, n * sizeof(float), cudaMemcpyDeviceToHost));
  return DERP_OK;
}


// ---- BC7 colour (ConvertToBinary's default colour format) ----
static int bc7Launch(int device, const void* src, size_t srcBytes, int mode, int channels, int width, int height,
                     const uint8_t* lutHost, size_t lutBytes, uint8_t* blocks) {
  CU(cudaSetDevice(device));
  const size_t outBytes = (size_t)width * height;
  DevBuf<uint8_t> dSrc, dOut, dLut;
  const void* s = src;
  cudaPointerAttributes at{};
  if (cudaPointerGetAttributes(&at, src) != cudaSuccess || at.type != cudaMemoryTypeDevice) {
    (void)cudaGetLastError();
    CU(dSrc.ensure(srcBytes));
    CU(cudaMemcpy(dSrc.p, src, srcBytes, cudaMemcpyDefault));
    s = dSrc.p;
  }
  uint8_t* o = blocks;
  const bool outOnDevice = cudaPointerGetAttributes(&at, blocks) == cudaSuccess && at.type == cudaMemoryTypeDevice;
  if (!outOnDevice) {
    (void)cudaGetLastError();
    CU(dOut.ensure(outBytes));
    o = dOut.p;
  }
  CU(cudaMemset(o, 0, outBytes));  // the reference's output vector starts zeroed; partial edge blocks are never written
  const int bx = width / 4, by = height / 4;
  if (bx > 0 && by > 0) {
    const unsigned grid = (unsigned)(((size_t)bx * by + derp::bc7::kBc7Threads - 1) / derp::bc7::kBc7Threads);
    if (mode == 0) {
      derp::bc7::bc7Kernel<<<grid, derp::bc7::kBc7Threads>>>(derp::bc7::Rgba8Source{(const uint8_t*)s, width}, width, bx, by, o);
    } else {
      CU(dLut.ensure(lutBytes));
      CU(cudaMemcpy(dLut.p, lutHost, lutBytes, cudaMemcpyHostToDevice));
      if (mode == 8)
        derp::bc7::bc7Kernel<<<grid, derp::bc7::kBc7Threads>>>(
            derp::bc7::BgrSource<uint8_t>{(const uint8_t*)s, width, channels, dLut.p}, width, bx, by, o);
      else
        derp::bc7::bc7Kernel<<<grid, derp::bc7::kBc7Threads>>>(
            derp::bc7::BgrSource<uint16_t>{(const uint16_t*)s, width, channels, dLut.p}, width, bx, by, o);
    }
    CU(cudaGetLastError());
  }
  if (!outOnDevice) CU(cudaMemcpy(blocks, o, outBytes, cudaMemcpyDeviceToHost));
  else CU(cudaDeviceSynchronize());
  return DERP_OK;
}

int derp_bc7_compress(int device, const uint8_t* rgba, int width, int height, uint8_t* blocks) {
  if (!rgba || !blocks || width < 1 || height < 1) return fail(DERP_EINVAL, "derp_bc7_compress: bad arguments");
  return bc7Launch(device, rgba, (size_t)width * height * 4, 0, 4, width, height, nullptr, 0, blocks);
}

int derp_bc7_compress_image(int device, const void* pixels, int bits_per_channel, int channels, int width, int height,
                            float gamma, uint8_t* blocks) {
  if (!pixels || !blocks || width < 1 || height < 1 || (bits_per_channel != 8 && bits_per_channel != 16) ||
      (channels != 3 && channels != 4))
    return fail(DERP_EINVAL, "derp_bc7_compress_image: 8 or 16 bits per channel, 3 (BGR) or 4 (BGRA) channels");
  std::vector<uint8_t> lut((size_t)1 << bits_per_channel);
  derp::bc7::gammaTable(bits_per_channel, gamma, lut.data());
  return bc7Launch(device, pixels, (size_t)width * height * channels * (bits_per_channel / 8), bits_per_channel, channels,
                   width, height, lut.data(), lut.size(), blocks);
}

}  // extern "C"

// ---- rephotography (derp_rephoto.cuh) ----------------------------------------------------------------
// Grow-only scratch per host thread, like the camera mesh: the app renders four cubemaps and one score per camera.
namespace {
struct RephotoScratch {
  DevBuf<float> disp, bgra, vtx, out, f32, mats, trig, eq;
  DevBuf<ushort4> texC, texD;
  DevBuf<unsigned long long> keys;
  DevBuf<float4> accC, accD;
  DevBuf<int> flags;
  DevBuf<int32_t> win;
  DevBuf<uint8_t> mask;
  DevBuf<double> partial;
  int device = -1;
  void release() {
    disp.release(); bgra.release(); vtx.release(); out.release(); f32.release(); mats.release(); trig.release();
    eq.release(); texC.release(); texD.release();
    keys.release(); accC.release(); accD.release(); flags.release(); win.release(); mask.release(); partial.release();
  }
};
thread_local RephotoScratch g_rephoto;

int rephotoScratch(int device) {
  RephotoScratch& s = g_rephoto;
  if (s.device != device) {
    if (s.device >= 0) {
      cudaSetDevice(s.device);
      s.release();
    }
    s.device = device;
  }
  CU(cudaSetDevice(device));
  return DERP_OK;
}

// CanopyScene::cubemap / equirect / render (derp_canopy.h) in every mode; rephotography is the cubemap, ipd 0,
// alpha-blended, on-screen case with NaN set to 0.  When the colour and the disparity colour are both wanted at one
// texture size, one raster serves both; otherwise each scene is a pass of its own (the alpha test and the LOD depend on
// the texture's size).
int canopyRender(const char* who, int device, const DerpCameraDesc* cams, int num_cams, const float* const* disparities,
                 int mw, int mh, const float* const* colors_bgra, int cw, int ch, int projection, const float* position,
                 const float* matrix, int outW, int outH, float ipd, int alphaBlend, int shader, bool zeroNan,
                 float* out_color, float* out_disparity, int32_t* winners) {
  using namespace derp::rephoto;
  const std::string name(who);
  if (!cams || num_cams < 0 || (num_cams > 0 && !disparities) || mw < 2 || mh < 2 || !position ||
      (!out_color && !out_disparity) || (out_color && num_cams > 0 && !colors_bgra) || (out_color && (cw < 1 || ch < 1)))
    return fail(DERP_EINVAL, name + ": bad arguments");
  if (shader != DERP_CANOPY_ON_SCREEN && shader != DERP_CANOPY_SVD)
    return fail(DERP_EINVAL, name + ": shader must be DERP_CANOPY_ON_SCREEN or DERP_CANOPY_SVD");
  int views, W, H;  // the raster: `views` viewports of W x H
  if (projection == DERP_CANOPY_CUBEMAP || projection == DERP_CANOPY_EQUIRECT) {
    const bool ok = projection == DERP_CANOPY_CUBEMAP ? outW == outH : outW == 2 * outH;
    if (!ok || outH < 2) return fail(DERP_EINVAL, name + ": bad output size for the projection");
    views = kFaces;
    W = H = outH;
  } else if (projection == DERP_CANOPY_PERSPECTIVE) {
    if (!matrix || outW < 1 || outH < 1) return fail(DERP_EINVAL, name + ": perspective needs a matrix and a size");
    views = 1;
    W = outW;
    H = outH;
  } else {
    return fail(DERP_EINVAL, name + ": unknown projection");
  }
  if ((long long)mw * mh >= (1ll << 30) || (out_color && (long long)cw * ch >= (1ll << 30)) ||
      (long long)W * H * views >= (1ll << 31))
    return fail(DERP_EINVAL, name + ": image or output too large");
  std::vector<DevCamera> dcMesh(num_cams), dcTex(num_cams);
  for (int i = 0; i < num_cams; ++i) {
    DevCamera c;
    if (!host::makeCamera(cams[i], &c)) return fail(DERP_EINVAL, name + ": invalid camera " + std::to_string(i));
    dcMesh[i] = host::rescaled(c, mw, mh);  // camera.rescale({disparity.cols, disparity.rows})
    if (out_color) dcTex[i] = host::rescaled(c, cw, ch);  // alphaFov: camera.rescale({color.cols, color.rows})
  }
  std::vector<float> mats(16 * views);
  if (views == kFaces) {
    FaceMats fm;
    faceMatrices(position, &fm);
    for (int f = 0; f < kFaces; ++f) std::memcpy(&mats[16 * f], fm.m[f], 16 * sizeof(float));
  } else {
    std::memcpy(mats.data(), matrix, 16 * sizeof(float));
  }
  struct Pass {
    bool color, disp;
  };
  std::vector<Pass> passes;
  if (out_color && out_disparity && cw == mw && ch == mh) {
    passes.push_back({true, true});
  } else {
    if (out_color) passes.push_back({true, false});
    if (out_disparity) passes.push_back({false, true});
  }
  int rc = rephotoScratch(device);
  if (rc) return rc;
  RephotoScratch& s = g_rephoto;
  const size_t n = (size_t)mw * mh, nc = out_color ? (size_t)cw * ch : 0;
  const size_t pixels = (size_t)views * W * H;
  CU(s.disp.ensure(n));
  CU(s.vtx.ensure(n * 3));
  CU(s.keys.ensure(pixels));
  CU(s.flags.ensure(1));
  CU(s.mats.ensure(mats.size()));
  CU(cudaMemcpy(s.mats.p, mats.data(), mats.size() * sizeof(float), cudaMemcpyHostToDevice));
  if (out_color) {
    CU(s.bgra.ensure(nc * 4));
    CU(s.accC.ensure(pixels));
    CU(cudaMemset(s.accC.p, 0, pixels * sizeof(float4)));
  }
  if (out_disparity) {
    CU(s.accD.ensure(pixels));
    CU(cudaMemset(s.accD.p, 0, pixels * sizeof(float4)));
  }
  if (winners) CU(s.win.ensure(pixels * std::max(num_cams, 1)));
  CU(s.out.ensure(pixels * 4));
  const int prims = (mw - 1) * (mh - 1) * 2;
  for (size_t pi = 0; pi < passes.size(); ++pi) {
    const Pass& ps = passes[pi];
    const int tw = ps.color ? cw : mw, th = ps.color ? ch : mh;
    int levels = 1;
    while ((tw >> levels) > 0 || (th >> levels) > 0) ++levels;
    if (levels > kMaxLevels) return fail(DERP_EINVAL, name + ": image too large");
    Canopy cv{};
    cv.mw = mw;
    cv.mh = mh;
    cv.levels = levels;
    cv.svd = shader == DERP_CANOPY_SVD;
    cv.alphaBlend = alphaBlend != 0;
    long long texels = 0;
    for (int l = 0; l < levels; ++l) {
      cv.lw[l] = std::max(1, tw >> l);
      cv.lh[l] = std::max(1, th >> l);
      cv.lofs[l] = texels;
      texels += (long long)cv.lw[l] * cv.lh[l];
    }
    if (ps.color) CU(s.texC.ensure(texels));
    if (ps.disp) CU(s.texD.ensure(texels));
    ushort4* texC = ps.color ? s.texC.p : nullptr;
    ushort4* texD = ps.disp ? s.texD.p : nullptr;
    cv.vtx = s.vtx.p;
    cv.tex[0] = texC;
    cv.tex[1] = texD;
    int32_t* win = winners && pi == 0 ? s.win.p : nullptr;
    const bool ownGrid = ps.color && (cw != mw || ch != mh);  // the colour texture on a grid of its own
    for (int i = 0; i < num_cams; ++i) {  // canopies in camera order: the blend sums are order-dependent
      CU(cudaMemcpy(s.disp.p, disparities[i], n * sizeof(float), cudaMemcpyDefault));
      if (ps.color) CU(cudaMemcpy(s.bgra.p, colors_bgra[i], nc * 4 * sizeof(float), cudaMemcpyDefault));
      CU(cudaMemset(s.flags.p, 0, sizeof(int)));
      if (ownGrid) {
        rephotoPrepKernel<<<dim3((cw + 127) / 128, ch), 128>>>(dcTex[i], nullptr, s.bgra.p, cw, ch, position[0], position[1],
                                                              position[2], 0.0f, nullptr, texC, nullptr, s.flags.p);
        rephotoPrepKernel<<<dim3((mw + 127) / 128, mh), 128>>>(dcMesh[i], s.disp.p, nullptr, mw, mh, position[0],
                                                              position[1], position[2], ipd, s.vtx.p, nullptr, nullptr,
                                                              s.flags.p);
      } else {
        rephotoPrepKernel<<<dim3((mw + 127) / 128, mh), 128>>>(dcMesh[i], s.disp.p, s.bgra.p, mw, mh, position[0],
                                                              position[1], position[2], ipd, s.vtx.p, texC, texD,
                                                              s.flags.p);
      }
      for (int l = 1; l < levels; ++l)
        for (int t = 0; t < 2; ++t) {
          ushort4* tex = t == 0 ? texC : texD;
          if (!tex) continue;
          rephotoMipKernel<<<dim3((cv.lw[l] + 127) / 128, cv.lh[l]), 128>>>(tex + cv.lofs[l - 1], cv.lw[l - 1],
                                                                            cv.lh[l - 1], tex + cv.lofs[l], cv.lw[l],
                                                                            cv.lh[l]);
        }
      CU(cudaMemcpy(&cv.anyZeroAlpha, s.flags.p, sizeof(int), cudaMemcpyDeviceToHost));
      CU(cudaMemset(s.keys.p, 0xff, pixels * sizeof(unsigned long long)));
      rephotoRasterKernel<<<dim3((prims + 255) / 256, views), 256>>>(cv, s.mats.p, W, H, prims, s.keys.p);
      rephotoResolveKernel<<<grid1(pixels), 256>>>(cv, s.mats.p, W, H, views, s.keys.p, ps.color ? s.accC.p : nullptr,
                                                   ps.disp ? s.accD.p : nullptr, win ? win + (size_t)i * pixels : nullptr);
      CU(cudaGetLastError());
    }
  }
  std::vector<float> trig;
  if (projection == DERP_CANOPY_EQUIRECT) {  // equirectFS' texel-centre directions, fp64 rounded to fp32
    const int e = outH;
    trig.resize((size_t)6 * e);
    const double kPi = 3.14159265358979323846;
    for (int y = 0; y < e; ++y) {
      const double lat = -(((y + 0.5) / e) - 0.5) * kPi;
      trig[y] = (float)std::cos(lat);
      trig[e + y] = (float)std::sin(lat);
    }
    for (int x = 0; x < 2 * e; ++x) {
      const double lon = (1 - (x + 0.5) / (2 * e)) * 2.0 * kPi;
      trig[2 * e + x] = (float)std::cos(lon);
      trig[4 * e + x] = (float)std::sin(lon);
    }
    CU(s.trig.ensure(trig.size()));
    CU(cudaMemcpy(s.trig.p, trig.data(), trig.size() * sizeof(float), cudaMemcpyHostToDevice));
    CU(s.eq.ensure((size_t)2 * e * e * 4));
  }
  for (int t = 0; t < 2; ++t) {
    float* dst = t == 0 ? out_color : out_disparity;
    if (!dst) continue;
    rephotoUnpremulKernel<<<grid1(pixels), 256>>>(pixels, t == 0 ? s.accC.p : s.accD.p, zeroNan, s.out.p);
    CU(cudaGetLastError());
    if (projection == DERP_CANOPY_EQUIRECT) {
      const int e = outH;
      canopyEquirectKernel<<<dim3((2 * e + 127) / 128, e), 128>>>(s.out.p, e, s.trig.p, s.eq.p);
      CU(cudaGetLastError());
      CU(cudaMemcpy(dst, s.eq.p, (size_t)2 * e * e * 4 * sizeof(float), cudaMemcpyDefault));
    } else {
      CU(cudaMemcpy(dst, s.out.p, pixels * 4 * sizeof(float), cudaMemcpyDefault));
    }
  }
  if (winners && num_cams > 0)
    CU(cudaMemcpy(winners, s.win.p, pixels * num_cams * sizeof(int32_t), cudaMemcpyDefault));
  CU(cudaDeviceSynchronize());
  return DERP_OK;
}
}  // namespace

extern "C" {

int derp_rephoto_cubemap(int device, const DerpCameraDesc* cams, int num_cams, const float* const* disparities,
                         const float* const* colors_bgra, int width, int height, const float* center, int edge,
                         float* out_color, float* out_disparity, int32_t* winners) {
  return canopyRender("derp_rephoto_cubemap", device, cams, num_cams, disparities, width, height, colors_bgra, width, height,
                      DERP_CANOPY_CUBEMAP, center, nullptr, edge, edge, 0.0f, 1, DERP_CANOPY_ON_SCREEN, true, out_color,
                      out_disparity, winners);
}

int derp_canopy_render(int device, const DerpCameraDesc* cams, int num_cams, const float* const* disparities,
                       int mesh_width, int mesh_height, const float* const* colors_bgra, int color_width,
                       int color_height, int projection, const float* position, const float* matrix, int out_width,
                       int out_height, float ipd, int alpha_blend, int shader, float* out_color, float* out_disparity,
                       int32_t* winners) {
  return canopyRender("derp_canopy_render", device, cams, num_cams, disparities, mesh_width, mesh_height, colors_bgra,
                      color_width, color_height, projection, position, matrix, out_width, out_height, ipd, alpha_blend,
                      shader, false, out_color, out_disparity, winners);
}

int derp_canopy_snapshot_matrix(const float* position, const float* forward, const float* up, double horizontal_fov_deg,
                                int width, int height, float* matrix) {
  if (!position || !forward || !up || !matrix || width < 1 || height < 1)
    return fail(DERP_EINVAL, "derp_canopy_snapshot_matrix: bad arguments");
  if (!derp::rephoto::snapshotMatrix(position, forward, up, horizontal_fov_deg, width, height, matrix))
    return fail(DERP_EINVAL, "derp_canopy_snapshot_matrix: forward and up do not give a unitary basis");
  return DERP_OK;
}

int derp_rephoto_score(int device, const float* ref_bgr, const float* ren_bgr, const uint8_t* mask, int width, int height,
                       int method, int stat_radius, float* score_map, double* avg) {
  using namespace derp::rephoto;
  if (!ref_bgr || !ren_bgr || !mask || width < 1 || height < 1 || !score_map || !avg)
    return fail(DERP_EINVAL, "derp_rephoto_score: bad arguments");
  if (method != DERP_REPHOTO_MSSIM && method != DERP_REPHOTO_NCC)
    return fail(DERP_EINVAL, "derp_rephoto_score: method must be DERP_REPHOTO_MSSIM or DERP_REPHOTO_NCC");
  if (stat_radius < 1 || stat_radius > 31) return fail(DERP_EINVAL, "derp_rephoto_score: stat_radius in [1, 31]");
  int rc = rephotoScratch(device);
  if (rc) return rc;
  RephotoScratch& s = g_rephoto;
  const size_t pixels = (size_t)width * height, n = pixels * 3;
  // f32 layout: [x | y | mu (2n) | moments (3n) | sig (3n) | tmp (3n) | weights (64)]
  CU(s.f32.ensure(13 * n + 64));
  float *x = s.f32.p, *y = x + n, *mu = y + n, *mom = mu + 2 * n, *sig = mom + 3 * n, *tmp = sig + 3 * n,
        *wt = tmp + 3 * n;
  float hw[64];
  gaussianWeights(stat_radius, hw);
  const unsigned blocks = grid1(pixels);
  CU(s.mask.ensure(pixels));
  CU(s.out.ensure(n));
  CU(s.partial.ensure((size_t)blocks * 6));
  CU(cudaMemcpy(x, ref_bgr, n * sizeof(float), cudaMemcpyDefault));
  CU(cudaMemcpy(y, ren_bgr, n * sizeof(float), cudaMemcpyDefault));
  CU(cudaMemcpy(s.mask.p, mask, pixels, cudaMemcpyDefault));
  CU(cudaMemcpy(wt, hw, (2 * stat_radius + 1) * sizeof(float), cudaMemcpyHostToDevice));
  const dim3 g2((width + 127) / 128, height, 2), g3((width + 127) / 128, height, 3);
  rephotoBlurRowsKernel<<<g2, 128>>>(x, width, height, stat_radius, wt, tmp);  // x, y are adjacent: two images
  rephotoBlurColsKernel<<<g2, 128>>>(tmp, width, height, stat_radius, wt, mu);
  rephotoMomentsKernel<<<grid1(n), 256>>>(n, x, y, mu, mom);
  rephotoBlurRowsKernel<<<g3, 128>>>(mom, width, height, stat_radius, wt, tmp);
  rephotoBlurColsKernel<<<g3, 128>>>(tmp, width, height, stat_radius, wt, sig);
  rephotoScoreKernel<<<blocks, 256>>>(pixels, mu, sig, s.mask.p, method == DERP_REPHOTO_NCC, s.out.p, s.partial.p);
  CU(cudaGetLastError());
  std::vector<double> part((size_t)blocks * 6);
  CU(cudaMemcpy(score_map, s.out.p, n * sizeof(float), cudaMemcpyDefault));
  CU(cudaMemcpy(part.data(), s.partial.p, part.size() * sizeof(double), cudaMemcpyDeviceToHost));
  for (int c = 0; c < 3; ++c) {  // cv::mean(channel, mask without NaN): 0 for an empty mask
    double sum = 0, cnt = 0;
    for (unsigned b = 0; b < blocks; ++b) {
      sum += part[b * 6 + c];
      cnt += part[b * 6 + 3 + c];
    }
    avg[c] = cnt > 0 ? sum / cnt : 0.0;
  }
  return DERP_OK;
}

}  // extern "C"

// ---- host-side test hooks ---------------------------------------------------------------------------
// The selection, RNG and camera code is __host__ __device__; these entry points run the HOST
// instantiation so that CPU-only tests (-m "not gpu") can check it against libstdc++ / the oracle.
extern "C" {

// 1 if the three-instruction constant division (derp_divconst.cuh) was validated exact for divisor c on `device`
// (every dividend mantissa against __fdiv_rn), 0 if it failed and the kernels use the plain division, < 0 on error.
int derp_test_div_const(int device, float c) {
  if (cudaSetDevice(device) != cudaSuccess) return DERP_ECUDA;
  DivConst k;
  if (makeDivConst(c, 0, &k) != cudaSuccess) return DERP_ECUDA;
  return k.fast;
}

// Host instantiation of the table-driven selection (derp_select.cuh): returns 1 and the sum when the table path
// applies (4 <= n <= 8, distinct non-NaN first keys), 0 when the caller must run the general algorithm.
int derp_test_select_table(const float* first, const float* second, int n, int keep, float* out) {
  static const std::vector<unsigned> tab = [] {
    std::vector<unsigned> t(derp::kSelTabSize);
    derp::buildSelectTable(t.data());
    return t;
  }();
  if (n < derp::kSelTabMinN || n > derp::kSelTabMaxN) return 0;
  float a[8], b[8];
  for (int i = 0; i < n; ++i) {
    a[i] = first[i];
    b[i] = second[i];
  }
  float out6 = 0;
  const bool ok8 = derp::robustSumTable<8>(derp::ArrayPairs{a, b}, n, keep, tab.data(), out);
  if (n <= 6) {  // the 6-slot instance must agree wherever it applies
    const bool ok6 = derp::robustSumTable<6>(derp::ArrayPairs{a, b}, n, keep, tab.data(), &out6);
    if (ok6 != ok8 || (ok8 && memcmp(&out6, out, 4) != 0)) return -1;
  }
  return ok8 ? 1 : 0;
}

// host-only hook for tests/test_mesh.py: the simplifier on an arbitrary mesh (double xyz, uint32 indices); outputs sized
// like the inputs
int derp_test_simplify(const double* xyz, uint64_t nv, const uint32_t* idx, uint64_t nf, int triangles, float strictness,
                       int remove_boundary_edges, double* out_xyz, uint32_t* out_idx, uint64_t* out_nv, uint64_t* out_nf) {
  derp::simplify::Mesh mesh(xyz, nv, idx, nf);
  mesh.run(triangles, strictness, remove_boundary_edges != 0);
  for (size_t i = 0; i < mesh.verts.size(); ++i) {
    out_xyz[3 * i] = mesh.verts[i].p.x;
    out_xyz[3 * i + 1] = mesh.verts[i].p.y;
    out_xyz[3 * i + 2] = mesh.verts[i].p.z;
  }
  for (size_t i = 0; i < mesh.faces.size(); ++i)
    for (int j = 0; j < 3; ++j) out_idx[3 * i + j] = (uint32_t)mesh.faces[i].v[j];
  *out_nv = mesh.verts.size();
  *out_nf = mesh.faces.size();
  return 0;
}

// HOST instantiation of the BC7 block encoder (derp_bc7.cuh) for tests/test_bc7.py -m "not gpu"; the apps call
// derp_bc7_compress* (CUDA) only.
int derp_test_bc7_blocks_host(const uint8_t* rgba, int width, int height, uint8_t* blocks) {
  if (!rgba || !blocks || width < 1 || height < 1) return DERP_EINVAL;
  std::memset(blocks, 0, (size_t)width * height);
  derp::bc7::encodeSurfaceOnHost(rgba, width, height, blocks);
  return DERP_OK;
}
int derp_test_bc7_gamma_table(int bits_per_channel, float gamma, uint8_t* lut) {
  if ((bits_per_channel != 8 && bits_per_channel != 16) || !lut) return DERP_EINVAL;
  derp::bc7::gammaTable(bits_per_channel, gamma, lut);
  return DERP_OK;
}

float derp_test_robust_sum(const float* first, const float* second, int n, int keep) {
  float a[64], b[64];
  if (n > 64 || n < 0) return NAN;
  for (int i = 0; i < n; ++i) {
    a[i] = first[i];
    b[i] = second[i];
  }
  return derp::robustSum(a, b, n, keep);
}

void derp_test_minstd_uniform(uint32_t seed, uint64_t skip, int n, float lo, float hi, float* out) {
  derp::MinstdRand0 r;
  r.seed(seed);
  r.discard(skip);
  for (int i = 0; i < n; ++i) out[i] = r.uniform(lo, hi);
}

// sees() of the (optionally normalised) camera for n rig-space points; pix = pixel coordinates
int derp_test_camera_sees(const DerpCameraDesc* d, int normalized, const double* pts, int n, double* pix, uint8_t* seen) {
  derp::DevCamera c;
  if (!derp::host::makeCamera(*d, &c)) return fail(DERP_EINVAL, "invalid camera");
  if (normalized) derp::host::normalise(c);
  for (int i = 0; i < n; ++i) {
    double x = NAN, y = NAN;
    seen[i] = derp::sees(c, pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], &x, &y) ? 1 : 0;
    pix[2 * i] = x;
    pix[2 * i + 1] = y;
  }
  return DERP_OK;
}

// rig(pixel, depth) and isOutsideImageCircle(pixel)
int derp_test_camera_rig(const DerpCameraDesc* d, const double* pix, int n, double depth, double* pts, uint8_t* outside) {
  derp::DevCamera c;
  if (!derp::host::makeCamera(*d, &c)) return fail(DERP_EINVAL, "invalid camera");
  for (int i = 0; i < n; ++i) {
    double dir[3];
    derp::pixelRay(c, pix[2 * i], pix[2 * i + 1], dir);
    for (int k = 0; k < 3; ++k) pts[3 * i + k] = c.pos[k] + dir[k] * depth;
    outside[i] = derp::outsideImageCircle(c, pix[2 * i], pix[2 * i + 1]) ? 1 : 0;
  }
  return DERP_OK;
}

int derp_test_camera_info(const DerpCameraDesc* d, double* rotation9, double* distortion_max, double* cos_fov) {
  derp::DevCamera c;
  if (!derp::host::makeCamera(*d, &c)) return fail(DERP_EINVAL, "invalid camera");
  for (int i = 0; i < 9; ++i) rotation9[i] = c.rot[i];
  *distortion_max = c.distMax;
  *cos_fov = c.cosFov;
  return DERP_OK;
}

}  // extern "C"

// ---- sweep-view slices (derp_sweepview.h) ---------------------------------------------------------------------
namespace {
using derp::sweep::SrcImage;

struct SweepScratch {
  DevBuf<DevCamera> cams;
  DevBuf<SrcImage> imgs;
  DevBuf<float4> upload, out;
  DevBuf<double> tabs;
  DevBuf<float> depths;
  DevBuf<int> widths, box;
  DevBuf<float4*> outs;
  DevBuf<unsigned long long> hits;
  int device = -1;
  void release() {
    cams.release(); imgs.release(); upload.release(); out.release(); tabs.release(); depths.release();
    widths.release(); box.release(); outs.release(); hits.release();
  }
};
thread_local SweepScratch g_sweep;
thread_local unsigned long long g_sweepHits = 0;  // contributing (sample, camera) pairs of the last call

int sweepScratch(int device) {
  SweepScratch& s = g_sweep;
  if (s.device != device) {
    if (s.device >= 0) {
      cudaSetDevice(s.device);
      s.release();
    }
    s.device = device;
  }
  CU(cudaSetDevice(device));
  return DERP_OK;
}

// Cameras as the apps hold them (already rescaled), optionally centred on camera `center`
int sweepCameras(const char* who, const DerpCameraDesc* cams, int n, int center, std::vector<DevCamera>& out) {
  const std::string name(who);
  if (!cams || n < 1 || n > derp::sweep::kMaxCams)
    return fail(DERP_EINVAL, name + ": between 1 and " + std::to_string(derp::sweep::kMaxCams) + " cameras");
  std::vector<DerpCameraDesc> d(cams, cams + n);
  if (center >= n) return fail(DERP_EINVAL, name + ": center index out of range");
  if (center >= 0 && !derp::sweep::host::centerRig(d.data(), n, center))
    return fail(DERP_EINVAL, name + ": centerRig produced an invalid rotation");
  out.resize(n);
  for (int i = 0; i < n; ++i)
    if (!host::makeCamera(d[i], &out[i])) return fail(DERP_EINVAL, name + ": invalid camera " + std::to_string(i));
  return DERP_OK;
}

int checkImages(const char* who, const float* const* images, const int32_t* sizes, int n) {
  if (!images || !sizes) return fail(DERP_EINVAL, std::string(who) + ": images and sizes are required");
  for (int i = 0; i < n; ++i)
    if (!images[i] || sizes[2 * i] < 1 || sizes[2 * i + 1] < 1 || (long long)sizes[2 * i] * sizes[2 * i + 1] >= (1ll << 30))
      return fail(DERP_EINVAL, std::string(who) + ": bad image " + std::to_string(i));
  return DERP_OK;
}

// The equirect reads images[c](int(py), int(px)) unclamped: every camera's resolution must fit its image
int checkFit(const char* who, const std::vector<DevCamera>& c, const int32_t* sizes) {
  for (size_t i = 0; i < c.size(); ++i)
    if (c[i].res[0] > sizes[2 * i] || c[i].res[1] > sizes[2 * i + 1])
      return fail(DERP_EINVAL, std::string(who) + ": camera " + std::to_string(i) + "'s resolution " +
                                   std::to_string(c[i].res[0]) + " x " + std::to_string(c[i].res[1]) +
                                   " exceeds its image " + std::to_string(sizes[2 * i]) + " x " +
                                   std::to_string(sizes[2 * i + 1]));
  return DERP_OK;
}

// Device copies of the rig and its images: device-resident images are used in place (16-byte aligned float4)
int stageSweepRig(const std::vector<DevCamera>& cams, const float* const* images, const int32_t* sizes) {
  SweepScratch& s = g_sweep;
  const int n = (int)cams.size();
  CU(s.cams.ensure(n));
  CU(cudaMemcpy(s.cams.p, cams.data(), n * sizeof(DevCamera), cudaMemcpyHostToDevice));
  if (!images) return DERP_OK;
  std::vector<SrcImage> im(n);
  std::vector<size_t> hostAt(n, SIZE_MAX);
  size_t total = 0;
  for (int i = 0; i < n; ++i) {
    cudaPointerAttributes at;
    const bool dev = cudaPointerGetAttributes(&at, images[i]) == cudaSuccess && at.type == cudaMemoryTypeDevice &&
                     ((uintptr_t)images[i] % 16) == 0;
    cudaGetLastError();
    if (!dev) {
      hostAt[i] = total;
      total += (size_t)sizes[2 * i] * sizes[2 * i + 1];
    }
    im[i] = SrcImage{reinterpret_cast<const float4*>(images[i]), sizes[2 * i], sizes[2 * i + 1]};
  }
  if (total) {
    CU(s.upload.ensure(total));
    for (int i = 0; i < n; ++i) {
      if (hostAt[i] == SIZE_MAX) continue;
      const size_t px = (size_t)sizes[2 * i] * sizes[2 * i + 1];
      CU(cudaMemcpy(s.upload.p + hostAt[i], images[i], px * sizeof(float4), cudaMemcpyDefault));
      im[i].p = s.upload.p + hostAt[i];
    }
  }
  CU(s.imgs.ensure(n));
  CU(cudaMemcpy(s.imgs.p, im.data(), n * sizeof(SrcImage), cudaMemcpyHostToDevice));
  return DERP_OK;
}

size_t sweepSmem(int n) { return (size_t)n * (sizeof(DevCamera) + sizeof(SrcImage)); }

// Host tables of one equirect slice set: full (bounds == NULL, one shared table) or cropped (one table per slice)
struct EquirectPlan {
  std::vector<double> cosT, sinT, sinP, cosP;
  std::vector<int> widths;
  int tStride = 0, pStride = 0, maxW = 0;
};
int planEquirect(const char* who, uint64_t height, int num, const double* bounds, EquirectPlan& p) {
  if (height < 1 || height > (1u << 15)) return fail(DERP_EINVAL, std::string(who) + ": height must be 1..32768");
  const double width = (double)(2 * height);
  if (!bounds) {
    std::vector<double> xs(2 * height), ys(height);
    for (uint64_t i = 0; i < 2 * height; ++i) xs[i] = (double)i;
    for (uint64_t i = 0; i < height; ++i) ys[i] = (double)i;
    p.cosT.resize(xs.size()); p.sinT.resize(xs.size()); p.sinP.resize(height); p.cosP.resize(height);
    derp::sweep::host::thetaTable(xs.data(), (int)xs.size(), width, p.cosT.data(), p.sinT.data());
    derp::sweep::host::phiTable(ys.data(), (int)height, (double)height, p.sinP.data(), p.cosP.data());
    p.widths.assign(num, (int)(2 * height));
    p.maxW = (int)(2 * height);
    return DERP_OK;
  }
  std::vector<uint64_t> ws(num);
  for (int k = 0; k < num; ++k) {
    if (!derp::sweep::host::cropWidth(height, bounds + 4 * k, &ws[k]))
      return fail(DERP_EINVAL, std::string(who) + ": slice " + std::to_string(k) +
                                   ": the crop box is empty or has zero width or height (nothing visible)");
    p.maxW = std::max<int>(p.maxW, (int)ws[k]);
  }
  p.tStride = p.maxW;
  p.pStride = (int)height;
  p.cosT.assign((size_t)num * p.maxW, 0); p.sinT.assign((size_t)num * p.maxW, 0);
  p.sinP.assign((size_t)num * height, 0); p.cosP.assign((size_t)num * height, 0);
  for (int k = 0; k < num; ++k) {
    std::vector<double> xs, ys;
    derp::sweep::host::cropSamples(height, ws[k], bounds + 4 * k, xs, ys);
    derp::sweep::host::thetaTable(xs.data(), (int)ws[k], width, &p.cosT[(size_t)k * p.maxW], &p.sinT[(size_t)k * p.maxW]);
    derp::sweep::host::phiTable(ys.data(), (int)height, (double)height, &p.sinP[(size_t)k * height],
                                &p.cosP[(size_t)k * height]);
    p.widths.push_back((int)ws[k]);
  }
  return DERP_OK;
}

// Device copy of an EquirectPlan; `outs` (device pointers) are filled by the caller
int uploadPlan(const EquirectPlan& p, const float* depths, int num, derp::sweep::EquirectSlices& s) {
  SweepScratch& g = g_sweep;
  const size_t nt = p.cosT.size(), np = p.sinP.size();
  CU(g.tabs.ensure(2 * nt + 2 * np));
  CU(cudaMemcpy(g.tabs.p, p.cosT.data(), nt * 8, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(g.tabs.p + nt, p.sinT.data(), nt * 8, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(g.tabs.p + 2 * nt, p.sinP.data(), np * 8, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(g.tabs.p + 2 * nt + np, p.cosP.data(), np * 8, cudaMemcpyHostToDevice));
  CU(g.depths.ensure(num));
  CU(cudaMemcpy(g.depths.p, depths, num * sizeof(float), cudaMemcpyDefault));
  CU(g.widths.ensure(num));
  CU(cudaMemcpy(g.widths.p, p.widths.data(), num * sizeof(int), cudaMemcpyHostToDevice));
  s.cosT = g.tabs.p;
  s.sinT = g.tabs.p + nt;
  s.sinP = g.tabs.p + 2 * nt;
  s.cosP = g.tabs.p + 2 * nt + np;
  s.depths = g.depths.p;
  s.widths = g.widths.p;
  s.tStride = p.tStride;
  s.pStride = p.pStride;
  s.height = (int)(p.sinP.size() / (p.pStride ? (size_t)num : 1));
  s.numSlices = num;
  return DERP_OK;
}

// an output the kernels can write in place: device memory, 16-byte aligned for float4 stores.  Anything else is staged
// in scratch and copied back with cudaMemcpyDefault, which infers the direction from the address
bool onDevice(const void* p) {
  cudaPointerAttributes at;
  const bool d = cudaPointerGetAttributes(&at, p) == cudaSuccess && at.type == cudaMemoryTypeDevice &&
                 ((uintptr_t)p % 16) == 0;
  cudaGetLastError();
  return d;
}

}  // namespace

extern "C" {

int derp_sweep_overlaps(int device, const DerpCameraDesc* cams, int num_cams, const float* const* images_bgra,
                        const int32_t* image_sizes, int dst, const float* disparities, int num_slices, float* out) {
  static const char* who = "derp_sweep_overlaps";
  std::vector<DevCamera> c;
  if (int rc = sweepCameras(who, cams, num_cams, -1, c)) return rc;
  if (int rc = checkImages(who, images_bgra, image_sizes, num_cams)) return rc;
  if (dst < 0 || dst >= num_cams || !disparities || num_slices < 1 || !out)
    return fail(DERP_EINVAL, std::string(who) + ": bad arguments");
  const int W = (int)c[dst].res[0], H = (int)c[dst].res[1];  // Image colorDst(resolution.y(), resolution.x())
  if (W < 1 || H < 1) return fail(DERP_EINVAL, std::string(who) + ": the destination has no pixels");
  if ((long long)W * H * num_slices >= (1ll << 31)) return fail(DERP_EINVAL, std::string(who) + ": output too large");
  if (int rc = sweepScratch(device)) return rc;
  if (int rc = stageSweepRig(c, images_bgra, image_sizes)) return rc;
  SweepScratch& s = g_sweep;
  const size_t plane = (size_t)W * H;
  float4* dOut;
  if (onDevice(out)) {
    dOut = reinterpret_cast<float4*>(out);
  } else {
    CU(s.out.ensure(plane * num_slices));
    dOut = s.out.p;
  }
  CU(s.depths.ensure(num_slices));
  CU(cudaMemcpy(s.depths.p, disparities, num_slices * sizeof(float), cudaMemcpyDefault));
  CU(s.hits.ensure(1));
  CU(cudaMemset(s.hits.p, 0, sizeof(unsigned long long)));
  const int chunk = derp::sweep::kOverlapSlicesPerThread;
  const dim3 block(derp::sweep::kSweepThreadsX, derp::sweep::kSweepThreadsY);
  const dim3 grid((W + block.x - 1) / block.x, (H + block.y - 1) / block.y, (num_slices + chunk - 1) / chunk);
  derp::sweep::overlapsKernel<<<grid, block, sweepSmem(num_cams)>>>(s.cams.p, s.imgs.p, num_cams, dst, W, H, s.depths.p,
                                                                     num_slices, chunk, dOut, s.hits.p);
  CU(cudaGetLastError());
  if (dOut != reinterpret_cast<float4*>(out))
    CU(cudaMemcpy(out, dOut, plane * num_slices * sizeof(float4), cudaMemcpyDefault));
  CU(cudaMemcpy(&g_sweepHits, s.hits.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  return DERP_OK;
}

int derp_sweep_crop_bounds(int device, const DerpCameraDesc* cams, int num_cams, int center, uint64_t height,
                           const float* depths, int num_depths, double* bounds) {
  static const char* who = "derp_sweep_crop_bounds";
  std::vector<DevCamera> c;
  if (int rc = sweepCameras(who, cams, num_cams, center, c)) return rc;
  if (!depths || num_depths < 1 || num_depths > 65535 || !bounds)
    return fail(DERP_EINVAL, std::string(who) + ": bad arguments");
  EquirectPlan p;
  if (int rc = planEquirect(who, height, num_depths, nullptr, p)) return rc;
  if (int rc = sweepScratch(device)) return rc;
  if (int rc = stageSweepRig(c, nullptr, nullptr)) return rc;
  derp::sweep::EquirectSlices sl{};
  if (int rc = uploadPlan(p, depths, num_depths, sl)) return rc;
  SweepScratch& s = g_sweep;
  std::vector<int> box(4 * num_depths);
  for (int k = 0; k < num_depths; ++k) {
    box[4 * k] = (int)(2 * height);  // minX = width, maxX = 0, minY = height, maxY = 0
    box[4 * k + 1] = 0;
    box[4 * k + 2] = (int)height;
    box[4 * k + 3] = 0;
  }
  CU(s.box.ensure(box.size()));
  CU(cudaMemcpy(s.box.p, box.data(), box.size() * sizeof(int), cudaMemcpyHostToDevice));
  const dim3 block(derp::sweep::kSweepThreadsX, derp::sweep::kSweepThreadsY);
  const dim3 grid((p.maxW + block.x - 1) / block.x, ((int)height + block.y - 1) / block.y, num_depths);
  derp::sweep::cropBoundsKernel<<<grid, block, sweepSmem(num_cams)>>>(s.cams.p, num_cams, sl, s.box.p);
  CU(cudaGetLastError());
  CU(cudaMemcpy(box.data(), s.box.p, box.size() * sizeof(int), cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < box.size(); ++i) bounds[i] = (double)box[i];
  return DERP_OK;
}

int derp_sweep_crop_width(uint64_t height, const double* bounds, uint64_t* width) {
  if (!bounds || !width) return fail(DERP_EINVAL, "derp_sweep_crop_width: bad arguments");
  if (!derp::sweep::host::cropWidth(height, bounds, width))
    return fail(DERP_EINVAL, "derp_sweep_crop_width: the crop box is empty or has zero width or height (nothing visible)");
  return DERP_OK;
}

int derp_sweep_equirect(int device, const DerpCameraDesc* cams, int num_cams, int center, const float* const* images_bgra,
                        const int32_t* image_sizes, uint64_t height, const float* depths, int num_depths,
                        const double* bounds, int black_bg, float* const* out) {
  static const char* who = "derp_sweep_equirect";
  std::vector<DevCamera> c;
  if (int rc = sweepCameras(who, cams, num_cams, center, c)) return rc;
  if (int rc = checkImages(who, images_bgra, image_sizes, num_cams)) return rc;
  if (int rc = checkFit(who, c, image_sizes)) return rc;
  if (!depths || num_depths < 1 || num_depths > 65535 || !out) return fail(DERP_EINVAL, std::string(who) + ": bad arguments");
  for (int k = 0; k < num_depths; ++k)
    if (!out[k]) return fail(DERP_EINVAL, std::string(who) + ": NULL output");
  EquirectPlan p;
  if (int rc = planEquirect(who, height, num_depths, bounds, p)) return rc;
  if (int rc = sweepScratch(device)) return rc;
  if (int rc = stageSweepRig(c, images_bgra, image_sizes)) return rc;
  derp::sweep::EquirectSlices sl{};
  if (int rc = uploadPlan(p, depths, num_depths, sl)) return rc;
  SweepScratch& s = g_sweep;
  // device-resident outputs are written in place; the others are staged in one scratch buffer and copied back
  std::vector<float4*> outs(num_depths);
  std::vector<size_t> at(num_depths, SIZE_MAX);
  size_t total = 0;
  for (int k = 0; k < num_depths; ++k) {
    if (onDevice(out[k])) continue;
    at[k] = total;
    total += (size_t)p.widths[k] * height;
  }
  if (total) CU(s.out.ensure(total));
  for (int k = 0; k < num_depths; ++k)
    outs[k] = at[k] == SIZE_MAX ? reinterpret_cast<float4*>(out[k]) : s.out.p + at[k];
  CU(s.outs.ensure(num_depths));
  CU(cudaMemcpy(s.outs.p, outs.data(), num_depths * sizeof(float4*), cudaMemcpyHostToDevice));
  sl.outs = s.outs.p;
  CU(s.hits.ensure(1));
  CU(cudaMemset(s.hits.p, 0, sizeof(unsigned long long)));
  const float4 bg = black_bg ? make_float4(0.f, 0.f, 0.f, 1.f) : make_float4(0.f, 0.f, 1.f, 1.f);
  const dim3 block(derp::sweep::kSweepThreadsX, derp::sweep::kSweepThreadsY);
  const dim3 grid((p.maxW + block.x - 1) / block.x, ((int)height + block.y - 1) / block.y, num_depths);
  derp::sweep::equirectKernel<<<grid, block, sweepSmem(num_cams)>>>(s.cams.p, s.imgs.p, num_cams, sl, bg, s.hits.p);
  CU(cudaGetLastError());
  for (int k = 0; k < num_depths; ++k)
    if (outs[k] != reinterpret_cast<float4*>(out[k]))
      CU(cudaMemcpy(out[k], outs[k], (size_t)p.widths[k] * height * sizeof(float4), cudaMemcpyDefault));
  CU(cudaMemcpy(&g_sweepHits, s.hits.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  return DERP_OK;
}

int derp_sweep_center_rig(const DerpCameraDesc* cams, int num_cams, int center, DerpCameraDesc* out, double* rotation9) {
  if (!cams || num_cams < 1 || center < 0 || center >= num_cams || !out)
    return fail(DERP_EINVAL, "derp_sweep_center_rig: bad arguments");
  std::vector<DerpCameraDesc> d(cams, cams + num_cams);
  if (!derp::sweep::host::centerRig(d.data(), num_cams, center))
    return fail(DERP_EINVAL, "derp_sweep_center_rig: invalid camera rotation");
  for (int i = 0; i < num_cams; ++i) {
    out[i] = d[i];
    if (rotation9) {
      DevCamera c;
      if (!host::makeCamera(d[i], &c)) return fail(DERP_EINVAL, "derp_sweep_center_rig: invalid camera");
      for (int k = 0; k < 9; ++k) rotation9[9 * i + k] = c.rot[k];
    }
  }
  return DERP_OK;
}

uint64_t derp_sweep_last_hits(void) { return g_sweepHits; }

int derp_test_sweep_overlaps_host(const DerpCameraDesc* cams, int num_cams, const float* const* images_bgra,
                                  const int32_t* image_sizes, int dst, const float* disparities, int num_slices,
                                  float* out) {
  static const char* who = "derp_test_sweep_overlaps_host";
  std::vector<DevCamera> c;
  if (int rc = sweepCameras(who, cams, num_cams, -1, c)) return rc;
  if (int rc = checkImages(who, images_bgra, image_sizes, num_cams)) return rc;
  if (dst < 0 || dst >= num_cams || !disparities || num_slices < 1 || !out) return fail(DERP_EINVAL, "bad arguments");
  std::vector<SrcImage> im(num_cams);
  for (int i = 0; i < num_cams; ++i)
    im[i] = SrcImage{reinterpret_cast<const float4*>(images_bgra[i]), image_sizes[2 * i], image_sizes[2 * i + 1]};
  const int W = (int)c[dst].res[0], H = (int)c[dst].res[1];
  float4* o = reinterpret_cast<float4*>(out);
  int hits = 0;
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      const double px = x + 0.5, py = y + 0.5;
      const bool outside = outsideImageCircle(c[dst], px, py);
      double dir[3];
      if (!outside) pixelRay(c[dst], px, py, dir);
      for (int k = 0; k < num_slices; ++k)
        o[(size_t)k * W * H + (size_t)y * W + x] =
            outside ? make_float4(0.f, 0.f, 0.f, 0.f)
                    : derp::sweep::overlapPixel(c.data(), im.data(), num_cams, c[dst].pos, dir, disparities[k], &hits);
    }
  return DERP_OK;
}

int derp_test_sweep_equirect_host(const DerpCameraDesc* cams, int num_cams, int center,
                                  const float* const* images_bgra, const int32_t* image_sizes, uint64_t height,
                                  const float* depths, int num_depths, const double* bounds, int black_bg,
                                  float* const* out) {
  static const char* who = "derp_test_sweep_equirect_host";
  std::vector<DevCamera> c;
  if (int rc = sweepCameras(who, cams, num_cams, center, c)) return rc;
  if (int rc = checkImages(who, images_bgra, image_sizes, num_cams)) return rc;
  if (int rc = checkFit(who, c, image_sizes)) return rc;
  if (!depths || num_depths < 1 || !out) return fail(DERP_EINVAL, "bad arguments");
  EquirectPlan p;
  if (int rc = planEquirect(who, height, num_depths, bounds, p)) return rc;
  std::vector<SrcImage> im(num_cams);
  for (int i = 0; i < num_cams; ++i)
    im[i] = SrcImage{reinterpret_cast<const float4*>(images_bgra[i]), image_sizes[2 * i], image_sizes[2 * i + 1]};
  const float4 bg = black_bg ? make_float4(0.f, 0.f, 0.f, 1.f) : make_float4(0.f, 0.f, 1.f, 1.f);
  int hits = 0;
  for (int k = 0; k < num_depths; ++k) {
    const double depth = (double)depths[k];
    const int W = p.widths[k];
    for (uint64_t y = 0; y < height; ++y)
      for (int x = 0; x < W; ++x) {
        const double r = depth * p.sinP[(size_t)k * p.pStride + y];
        reinterpret_cast<float4*>(out[k])[y * W + x] = derp::sweep::equirectPixel(
            c.data(), im.data(), num_cams, r * p.cosT[(size_t)k * p.tStride + x], r * p.sinT[(size_t)k * p.tStride + x],
            depth * p.cosP[(size_t)k * p.pStride + y], bg, &hits);
      }
  }
  return DERP_OK;
}

}  // extern "C"
