// libderp_b200.so — the product: C ABI of include/derp_b200.h implemented with hand-written
// sm_90a CUDA kernels (derp_kernels.cuh).  No CPU fallback: every entry point that computes
// needs a CUDA device and fails with DERP_ECUDA otherwise.  This file holds the depth context (DerpCtx) and the
// stand-alone depth stages; derp_convert.cu, derp_canopy.cu and derp_sweepview.cu hold the other entry points.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -fmad=false (see Makefile).
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>

#include "derp_host.cuh"
#include "derp_kernels.cuh"
#include "derp_refine.cuh"

using namespace derp;

thread_local std::string g_err;

static_assert(kBlock2X == kBlockX && kBlock2Y == kBlockY, "grid2 / block2 must launch the kernels' CTA");

namespace {

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
    const int peer = deviceOf(from);
    if (peer >= 0 && peer != c->device) {
      // a peer context's plane: device-to-device over NVLink (the runtime stages through the host if the two
      // devices have no peer path)
      if ((rc = enablePeer(c->device, peer))) return rc;
      CU(cudaMemcpyPeerAsync(to, c->device, from, peer, b, c->stream));
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
  const float* dCoarse = coarse;  // a host plane (the PFM a caller read back) is staged into a context buffer
  if ((rc = stageIn(dCoarse, nc, c->dUpCoarse, alignof(float), c->stream))) return rc;
  rc = upsampleIntoLevel(c, dst, dCoarse, coarse_w, coarse_h, coarse_mask, fine_mask, "derp_upsample_from");
  if (rc == DERP_OK && dCoarse != coarse) CU(cudaStreamSynchronize(c->stream));  // the caller's plane may be reused on return
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
  DevBuf<uint16_t> dS, dD;
  const uint16_t* sp = src;
  uint16_t* dp = dst;
  int rc = stageIn(sp, ns, dS);
  if (rc || (rc = outBuffer(dp, nd, dD))) return rc;
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
  if (dp != dst) return stageOut(dst, dp, nd);
  if (sp != src) CU(cudaDeviceSynchronize());  // the staged source is freed on return
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
    const int other = deviceOf(p);
    if (other >= 0 && other != device)
      if (int rc = enablePeer(device, other)) return rc;
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
  };
  static thread_local Scratch sc;
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
