// libderp_b200.so — the product: C ABI of include/derp_b200.h implemented with hand-written
// sm_90a CUDA kernels (derp_kernels.cuh).  No CPU fallback: every entry point that computes
// needs a CUDA device and fails with DERP_ECUDA otherwise.  This file holds the depth context (DerpCtx) and the
// stand-alone depth stages; derp_convert.cu, derp_canopy.cu and derp_sweepview.cu hold the other entry points.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -fmad=false (see Makefile).
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>

#include "../../include/derp_blur.h"
#include "../../include/derp_resize.h"
#include "derp_host.cuh"
#include "derp_kernels.cuh"
#include "derp_refine.cuh"
#include "derp_resize.cuh"

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

// Temporaries of one upsampling: the masks of fovAndMasks, the tables and intermediate planes of upsampleDevice
struct UpsampleScratch {
  DevBuf<uint8_t> maskC, maskUp, fovC, fovUp;
  DevBuf<float> tmpA, tmpB, taps;
  DevBuf<int> ofs;
  DevBuf<short2> spiral;
};

// CUDA events around launches on one stream, destroyed by clear() and the destructor: ev holds (start, stop) of every
// logged launch, then the start of one in progress.  A launch that fails between begin() and end() is not counted: the
// next begin() records over its start.
struct EventLog {
  std::vector<cudaEvent_t> ev;
  EventLog() = default;
  EventLog(const EventLog&) = delete;
  EventLog& operator=(const EventLog&) = delete;
  ~EventLog() { clear(); }
  int begin(cudaStream_t st) { return ev.size() % 2 ? rerecord(st) : record(st); }
  int end(cudaStream_t st) { return record(st); }
  size_t count() const { return ev.size() / 2; }
  // the summed device time of the logged launches; the stream must have been synchronised
  int totalMs(double* ms) const {
    *ms = 0;
    for (size_t i = 0; i < 2 * count(); i += 2) {
      float t = 0;
      CU(cudaEventElapsedTime(&t, ev[i], ev[i + 1]));
      *ms += t;
    }
    return DERP_OK;
  }
  void clear() {
    for (cudaEvent_t e : ev) cudaEventDestroy(e);
    ev.clear();
  }
  int record(cudaStream_t st) {
    cudaEvent_t e;
    CU(cudaEventCreate(&e));
    ev.push_back(e);
    return rerecord(st);
  }
  int rerecord(cudaStream_t st) {
    CU(cudaEventRecord(ev.back(), st));
    return DERP_OK;
  }
};

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
  DevBuf<float> dDispNext;  // the mismatch stage's Jacobi update of every destination
  // in-memory level hand-off (derp_level_keep / derp_upsample_from_kept): the finished level's disparity planes
  DevBuf<float> dKept, dUpCoarse;
  int keptW = 0, keptH = 0, keptSd = 0;
  UpsampleScratch up;  // derp_upsample_from[_kept]
  DevBuf<unsigned> dUncovered;
  DevBuf<int> dPrefix, dIdx, dRowCount, dTileCount, dTileOffset, dList;
  int projDst = -1;
  uint64_t launches = 0;
  uint64_t lastEvals = 0, lastHits = 0;
  bool countersOnDevice = false;
  int tableD = -1;
  float tableMin = 0, tableMax = 0;  // candidate table currently in dDisparities
  // optional timing of the brute-force sweeps and the pingPongKernel launches (derp_profile)
  bool profiling = false;
  EventLog sweepLog, pingLog;
  DevBuf<unsigned long long> dCountersPP;  // the ping-pong launches' own (evaluations, source hits)

  float2* warpOf(int dst) const { return geomCached ? geom->buf.p + (size_t)dst * 2 * S * plane : dProjWarp.p; }
  float2* warpInvOf(int dst) const { return geomCached ? geom->buf.p + ((size_t)dst * 2 + 1) * S * plane : dWarpInv.p; }
  // the stages read the foreground mask (and the cost stages the background) only when the level uses foreground masks
  const uint8_t* fgFor(int dst) const {
    return lp.use_foreground_masks && haveFg ? dFg.p + (size_t)dst2src[dst] * plane : nullptr;
  }
  const float* bgOf(int dst) const { return haveBg ? dBg.p + (size_t)dst * plane : nullptr; }
  CostView view(int dst) const {
    const int self = dst2src[dst];
    return CostView{W, H, S, self, dProjColor.p, dProjBias.p, dProjColor16.p, dProjBias16.p, dSelTab.p,
                    warpOf(dst), dVariance.p + (size_t)self * plane, dCams.p, 1.0f, 8388608.0f};
  }
  // Call it after the stage's ensureTables*, which may reallocate the tables the view points at.
  DstArgs dstArgs(int dst) const {
    return DstArgs{view(dst), dFov.p + (size_t)dst * plane, fgFor(dst), lp.use_foreground_masks ? bgOf(dst) : nullptr};
  }
  // dynamic smem of the cost kernels: S cameras + the destination patch tile
  // + S - 1 (ssdB, ssdU) pairs per thread for the robust camera mean (one slot per possible source)
  int selSlots() const { return S > 1 ? S - 1 : 1; }
  size_t camSmem(int threads = kBlockX * kBlockY) const {
    return (size_t)S * sizeof(DevCamera) + kTileFloats * sizeof(float) + (size_t)selSlots() * threads * sizeof(float2);
  }
  // the bound pass of the filtered sweep keeps no selection slots (KeptBound): S cameras + the destination tile, which
  // leaves the rest of the SM's L1 to its gathers
  size_t lowerSmem() const { return (size_t)S * sizeof(DevCamera) + kTileFloats * sizeof(float); }
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

int checkMasks(DerpCtx* c, const char* msg) {
  if (c->lp.use_foreground_masks && (!c->haveBg || !c->haveFg)) return fail(DERP_ESTATE, msg);
  return DERP_OK;
}

// Copies (to, from) between a caller's buffer and the context, returned with the copies done; a null end skips one
int copyPlanes(DerpCtx* c, size_t bytes, std::initializer_list<std::pair<void*, const void*>> copies) {
  for (const auto& p : copies)
    if (p.first && p.second) CU(cudaMemcpyAsync(p.first, p.second, bytes, cudaMemcpyDefault, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return DERP_OK;
}

// The candidate table in dDisparities, uploaded only when it changes
int candidateTable(DerpCtx* c, int num_depths, float min_depth_m, float max_depth_m) {
  if (c->tableD == num_depths && c->tableMin == min_depth_m && c->tableMax == max_depth_m) return DERP_OK;
  const std::vector<float> disparities = probeDisparities(num_depths, min_depth_m, max_depth_m);
  if (int rc = upload(c->dDisparities, disparities.data(), num_depths, c->stream)) return rc;
  CU(cudaStreamSynchronize(c->stream));  // host vector lifetime (tiny copy, only when the table changes)
  c->tableD = num_depths;
  c->tableMin = min_depth_m;
  c->tableMax = max_depth_m;
  return DERP_OK;
}

// Launch shape of sweepKernel and sweepLowerKernel: CTAs of kBlockX x rows threads, grid.z = chunks of `chunk` candidates
struct SweepShape {
  int rows, chunks, chunk;
  dim3 grid(int W, int H) const { return dim3((W + kBlockX - 1) / kBlockX, (H + rows - 1) / rows, chunks); }
};

// CTA height: kSweepMaxRows rows (one 640-thread CTA per SM, 96 registers) on large levels — its warps share more texel
// rows — and half of that (two CTAs per SM, same 20 warps) on small ones, where CTA count matters more.  Rigs of more
// than 42 cameras get shorter CTAs (sweepRows).  Candidate chunks: enough CTAs to fill every SM with 8 resident CTAs
// even on the coarse levels.
SweepShape sweepShape(const DerpCtx* c, int num_depths) {
  const int rows = c->sweepRows(c->H >= 1024 ? kSweepMaxRows : kSweepMaxRows / 2);
  const long ctas = (long)((c->W + kBlockX - 1) / kBlockX) * ((c->H + rows - 1) / rows) * std::max(1, rows / 8);
  const int chunks = (int)std::min<long>(num_depths, std::max<long>(1, ((long)c->numSMs * 8 * 4 + ctas - 1) / ctas));
  const int chunk = (num_depths + chunks - 1) / chunks;
  return SweepShape{rows, (num_depths + chunk - 1) / chunk, chunk};
}

// Filtered sweep (derp_refine.cuh) unless derp_set_sweep_mode chose the plain one, the candidate count is tiny or the
// bound buffer does not fit: lower bound of every (pixel, candidate), exact cost only where the bound does not exclude
// the candidate.  Automatic: the filter pays off when the bound pass amortises its extra launches and the read-back of
// the list length: >= 32 M (pixel, candidate) pairs (512^2 x 128); BASELINE.json configs[0] (512^2 x 32) and the
// coarsest pyramid levels stay on the plain sweep.
bool useFilteredSweep(const DerpCtx* c, int num_depths, unsigned long long capacity) {
  const int mode = c->sweepMode;
  const size_t n = c->plane;
  if (!(mode == 2 || (mode == 0 && num_depths >= 8 && (unsigned long long)n * (unsigned long long)num_depths >= (32ull << 20))))
    return false;
  size_t freeB = 0, totalB = 0;
  cudaMemGetInfo(&freeB, &totalB);
  const size_t need = (size_t)num_depths * n * sizeof(float) + capacity * sizeof(unsigned long long) + n * 8;
  return !(c->dLb.n < (size_t)num_depths * n && need > freeB / 2);
}

// Pass 1 of the filtered sweep: the lower bound of every (pixel, candidate) into dLb, the per-pixel seeds into dSeed
// (both allocated by the caller)
int boundPass(DerpCtx* c, const DstArgs& da, const float* disparities, int num_depths, const SweepShape& shape) {
  const size_t n = c->plane;
  fillKernel<unsigned long long><<<grid1(n), 256, 0, c->stream>>>(n, c->dSeed.p, 0x7f7fffffffffffffull);
  LAUNCHED("fillKernel");
  const LowerArgs la{da, disparities, num_depths, shape.chunk, c->dLb.p, c->dSeed.p, c->dCounters.p};
  c->k.sweepLower<<<shape.grid(c->W, c->H), dim3(kBlockX, shape.rows), c->lowerSmem(), c->stream>>>(la);
  LAUNCHED("sweepLowerKernel");
  return DERP_OK;
}

// The filtered sweep into dBest: bound pass, seed, refine list, its length read back, refine.  *finished is false when
// more candidates survived than the list holds (the bounds are useless on this input): dBest and the counters are then
// reset for the plain sweep.
int filteredSweep(DerpCtx* c, const DstArgs& da, int num_depths, const SweepShape& shape, unsigned long long capacity,
                  bool* finished) {
  const size_t n = c->plane;
  CU(c->dLb.ensure((size_t)num_depths * n));
  CU(c->dSeed.ensure(n));
  CU(c->dRefList.ensure(capacity));
  CU(c->dRefCount.ensure(1));
  CU(cudaMemsetAsync(c->dRefCount.p, 0, sizeof(unsigned long long), c->stream));
  int rc = boundPass(c, da, c->dDisparities.p, num_depths, shape);
  if (rc) return rc;
  const SeedArgs sa{da.v, da.fov, da.fg, c->dDisparities.p, c->dSeed.p, c->dBest.p};
  c->k.sweepSeed<<<grid2(c->W, c->H), block2(), c->camSmem(), c->stream>>>(sa);
  LAUNCHED("sweepSeedKernel");
  const ListArgs li{c->W, c->H, num_depths, da.fov, da.fg, c->dLb.p, c->dSeed.p, c->dBest.p, c->dRefList.p, capacity,
                    c->dRefCount.p};
  refineListKernel<<<grid2(c->W, c->H), block2(), 0, c->stream>>>(li);
  LAUNCHED("refineListKernel");
  unsigned long long count = 0;
  CU(cudaMemcpyAsync(&count, c->dRefCount.p, sizeof(count), cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  *finished = count <= capacity;
  if (!*finished) {
    fillKernel<unsigned long long><<<grid1(n), 256, 0, c->stream>>>(n, c->dBest.p, 0x7f7fffffffffffffull);
    LAUNCHED("fillKernel");
    CU(cudaMemsetAsync(c->dCounters.p, 0, 2 * sizeof(unsigned long long), c->stream));
    return DERP_OK;
  }
  c->lastRefined = count;
  c->lastSeeds = n;
  if (count > 0) {
    const RefineArgs ra{da.v, c->dDisparities.p, c->dRefList.p, count, c->dBest.p};
    c->k.refine<<<(unsigned)((count + kPatchThreads - 1) / kPatchThreads), kPatchThreads, c->patchSmem(), c->stream>>>(ra);
    LAUNCHED("refineKernel");
  }
  return DERP_OK;
}

int plainSweep(DerpCtx* c, const DstArgs& da, int num_depths, const SweepShape& shape) {
  const SweepArgs a{da, c->dDisparities.p, num_depths, shape.chunk, c->dBest.p, c->dCounters.p};
  c->k.sweep<<<shape.grid(c->W, c->H), dim3(kBlockX, shape.rows), c->camSmem(kBlockX * shape.rows), c->stream>>>(a);
  LAUNCHED("sweepKernel");
  return DERP_OK;
}

// dBest to the destination's disparity, cost and confidence with their borders extended; best_index (nullable) receives
// the winning candidates.  Uncovered pixels fail the call unless partial_coverage or foreground masks allow them.
int finishSweep(DerpCtx* c, int dst, const DstArgs& da, float minDisparity, int partial_coverage, int32_t* best_index) {
  const int W = c->W, H = c->H;
  const size_t n = c->plane;
  float* disp = c->dDisp.p + (size_t)dst * n;
  float* cost = c->dCost.p + (size_t)dst * n;
  float* conf = c->dConf.p + (size_t)dst * n;
  int* idx = best_index ? c->dIdx.p : nullptr;
  sweepFinalizeKernel<<<grid2(W, H), block2(), 0, c->stream>>>(W, H, da.fov, da.fg, da.bg, da.v.variance, c->dDisparities.p,
                                                               minDisparity, c->dBest.p, disp, cost, conf, idx, c->dUncovered.p);
  LAUNCHED("sweepFinalizeKernel");
  extendBorderKernel<<<grid1(2 * W + 2 * (H - 2)), 256, 0, c->stream>>>(W, H, da.fg, da.bg, disp, cost, conf, idx);
  LAUNCHED("extendBorderKernel");
  if (best_index) CU(cudaMemcpyAsync(best_index, c->dIdx.p, n * sizeof(int), cudaMemcpyDefault, c->stream));
  if (!(partial_coverage || c->lp.use_foreground_masks)) {
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
  CU(c->dCamsPx.ensure(num_cams));
  int rc = upload(c->dCams, c->camsNorm.data(), num_cams);
  if (rc) return rc;
  std::vector<float> tab;
  buildBicubicTable(tab);
  if ((rc = upload(c->dWtab, tab.data(), tab.size()))) return rc;
  CU(c->dCounters.ensure(2));
  CU(c->dUncovered.ensure(1));
  std::vector<unsigned> selTab(kSelTabSize);
  buildSelectTable(selTab.data());
  if ((rc = upload(c->dSelTab, selTab.data(), selTab.size()))) return rc;
  // the cost kernels keep cameras, the destination patch tile / per-thread patches and the selection slots in
  // dynamic shared memory: 92 KB for a 640-thread sweep CTA of a 16-camera rig, 177 KB with 32 cameras, 216 KB for a
  // 384-thread one with 64 cameras (DerpCtx::sweepRows); kMaxDynSmem is the most an H100 grants one CTA
  const CostKernels& k = c->k;
  for (const void* f : {(const void*)k.sweep, (const void*)k.evalCost, (const void*)k.proposal, (const void*)k.pingPong,
                        (const void*)k.sweepLower, (const void*)k.sweepSeed, (const void*)k.refine, (const void*)k.lowerBoundCheck})
    CU(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxDynSmem));
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

int derp_sync(DerpCtx* c) {
  if (!c) return fail(DERP_EINVAL, "null ctx");
  int rc = useDevice(c);
  if (rc) return rc;
  CU(cudaStreamSynchronize(c->stream));
  return DERP_OK;
}

int derp_set_stream(DerpCtx* c, void* cuda_stream) {
  if (int rc = derp_sync(c)) return rc;
  if (c->ownStream && c->stream) cudaStreamDestroy(c->stream);
  c->ownStream = false;
  c->stream = (cudaStream_t)cuda_stream;
  return DERP_OK;
}

int derp_profile(DerpCtx* c, int enable) {
  if (!c) return fail(DERP_EINVAL, "null ctx");
  c->sweepLog.clear();
  c->pingLog.clear();
  c->profiling = enable != 0;
  if (c->profiling) {
    CU(c->dCountersPP.ensure(2));
    CU(cudaMemsetAsync(c->dCountersPP.p, 0, 2 * sizeof(unsigned long long), c->stream));
  }
  return DERP_OK;
}

int derp_get_profile_ping_pong(DerpCtx* c, double* ms, uint64_t* launches, uint64_t* evals, uint64_t* hits) {
  int rc = derp_sync(c);
  if (rc) return rc;
  double total = 0;
  if ((rc = c->pingLog.totalMs(&total))) return rc;
  unsigned long long h[2] = {0, 0};
  if (c->dCountersPP.p) CU(cudaMemcpy(h, c->dCountersPP.p, sizeof(h), cudaMemcpyDeviceToHost));
  if (ms) *ms = total;
  if (launches) *launches = c->pingLog.count();
  if (evals) *evals = h[0];
  if (hits) *hits = h[1];
  return DERP_OK;
}

int derp_get_profile(DerpCtx* c, double* sweep_ms, uint64_t* sweep_launches) {
  int rc = derp_sync(c);
  if (rc) return rc;
  double total = 0;
  if ((rc = c->sweepLog.totalMs(&total))) return rc;
  if (sweep_ms) *sweep_ms = total;
  if (sweep_launches) *sweep_launches = c->sweepLog.count();
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
    CU(cudaMemcpyAsync(c->dFg.p + (size_t)s * n, masks[s], n, cudaMemcpyDefault, c->stream));
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
    CU(cudaMemcpyAsync(c->dBg.p + (size_t)d * n, background[d], n * sizeof(float), cudaMemcpyDefault, c->stream));
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
  CU(cudaMemcpyAsync(c->dScratchA.p, disparity, n * sizeof(float), cudaMemcpyDefault, c->stream));
  if ((rc = resetCounters(c))) return rc;
  if ((rc = ensureTablesF32(c))) return rc;
  if ((rc = checkSmem(c->camSmem(), "evalCostKernel"))) return rc;
  c->k.evalCost<<<grid2(c->W, c->H), block2(), c->camSmem(), c->stream>>>(c->view(dst), c->dScratchA.p, c->dScratchB.p,
                                                                         c->dScratchC.p, c->dCounters.p);
  LAUNCHED("evalCostKernel");
  if (out_cost) CU(cudaMemcpyAsync(out_cost, c->dScratchB.p, n * sizeof(float), cudaMemcpyDefault, c->stream));
  if (out_conf) CU(cudaMemcpyAsync(out_conf, c->dScratchC.p, n * sizeof(float), cudaMemcpyDefault, c->stream));
  rc = readCounters(c);
  c->countersOnDevice = false;
  return rc;
}

int derp_brute_force(DerpCtx* c, int dst, int num_depths, float min_depth_m, float max_depth_m, int partial_coverage,
                     int32_t* best_index) {
  if (num_depths < 2) return fail(DERP_EINVAL, "derp_brute_force: bad arguments");
  int rc = checkDst(c, dst, "derp_brute_force", true);
  if (rc) return rc;
  if ((rc = checkMasks(c, "derp_brute_force: foreground masks / background disparity not set"))) return rc;
  if ((rc = candidateTable(c, num_depths, min_depth_m, max_depth_m))) return rc;
  if ((rc = ensureTablesF32(c))) return rc;
  const size_t n = c->plane;
  fillKernel<unsigned long long><<<grid1(n), 256, 0, c->stream>>>(n, c->dBest.p, 0x7f7fffffffffffffull);
  LAUNCHED("fillKernel");
  if ((rc = resetCounters(c))) return rc;
  CU(cudaMemsetAsync(c->dUncovered.p, 0, sizeof(unsigned), c->stream));
  const SweepShape shape = sweepShape(c, num_depths);
  if ((rc = checkSmem(c->camSmem(kBlockX * shape.rows), "sweepKernel"))) return rc;
  if ((rc = checkSmem(c->camSmem(), "sweepSeedKernel"))) return rc;
  if ((rc = checkSmem(c->patchSmem(), "refineKernel"))) return rc;
  const DstArgs da = c->dstArgs(dst);  // after ensureTablesF32 (see dstArgs)
  if (c->profiling && (rc = c->sweepLog.begin(c->stream))) return rc;
  c->lastRefined = c->lastSeeds = 0;
  const unsigned long long capacity = (unsigned long long)n * std::max(2, num_depths / 8);  // refine list entries
  bool finished = false;
  if (useFilteredSweep(c, num_depths, capacity) && (rc = filteredSweep(c, da, num_depths, shape, capacity, &finished)))
    return rc;
  if (!finished && (rc = plainSweep(c, da, num_depths, shape))) return rc;
  if (c->profiling && (rc = c->sweepLog.end(c->stream))) return rc;
  return finishSweep(c, dst, da, 1.0f / max_depth_m, partial_coverage, best_index);
}

int derp_random_proposals(DerpCtx* c, int dst, int num_proposals, float min_depth_m, float max_depth_m) {
  int rc = checkDst(c, dst, "derp_random_proposals", true);
  if (rc) return rc;
  if (num_proposals < 0) return fail(DERP_EINVAL, "derp_random_proposals: negative count");
  if ((rc = checkMasks(c, "derp_random_proposals: masks not set"))) return rc;
  const int W = c->W, H = c->H;
  const size_t n = c->plane;
  const float kRandomPropHighVarDeviation = 0.1f;  // Derp.h:37
  const float varHighDev = kRandomPropHighVarDeviation * c->lp.var_high_thresh;
  const float varThresh = std::max(varHighDev, c->varNoiseFloor);
  if ((rc = resetCounters(c))) return rc;
  if ((rc = ensureTablesU16(c))) return rc;
  const size_t o = (size_t)dst * n;  // dstArgs after ensureTablesU16 (see dstArgs)
  const ProposalArgs a{c->dstArgs(dst), c->dPrefix.p, c->dList.p, listCountPtr(c), c->dDisp.p + o, c->dCost.p + o,
                       c->dConf.p + o, num_proposals, c->lp.level, 1.0f / max_depth_m, 1.0f / min_depth_m, c->dCounters.p};
  if ((rc = buildActiveList(c, a.fov, a.fg, a.v.variance, varThresh))) return rc;
  if (c->lp.use_foreground_masks) {
    backgroundFillKernel<<<grid2(W, H), block2(), 0, c->stream>>>(W, H, a.fov, a.fg, a.bg, a.disp);
    LAUNCHED("backgroundFillKernel");
  }
  if ((rc = checkSmem(c->patchSmem(), "proposalKernel"))) return rc;
  c->k.proposal<<<listGrid(W, H), kPatchThreads, c->patchSmem(), c->stream>>>(a);
  LAUNCHED("proposalKernel");
  return DERP_OK;
}

int derp_ping_pong(DerpCtx* c, int dst, int iterations) {
  int rc = checkDst(c, dst, "derp_ping_pong", true);
  if (rc) return rc;
  if ((rc = checkMasks(c, "derp_ping_pong: masks not set"))) return rc;
  const int W = c->W, H = c->H;
  const size_t n = c->plane;
  float* disp = c->dDisp.p + (size_t)dst * n;
  float* cost = c->dCost.p + (size_t)dst * n;
  if ((rc = resetCounters(c))) return rc;
  if ((rc = ensureTablesU16(c))) return rc;
  // dstArgs after ensureTablesU16 (see dstArgs); changed / changedNext are set per iteration
  PingPongArgs a{c->dstArgs(dst), disp, nullptr, c->dScratchA.p, c->dScratchB.p, nullptr, c->dList.p, listCountPtr(c),
                 c->dCounters.p, c->profiling ? c->dCountersPP.p : nullptr};
  // active pixels: interior, in FOV, foreground, variance >= noise floor (Derp.cpp:420-437)
  if ((rc = buildActiveList(c, a.fov, a.fg, a.v.variance, c->varNoiseFloor))) return rc;
  fillKernel<uint8_t><<<grid1(n), 256, 0, c->stream>>>(n, c->dChangedA.p, (uint8_t)1);
  LAUNCHED("fillKernel");
  uint8_t* chIn = c->dChangedA.p;
  uint8_t* chOut = c->dChangedB.p;
  if ((rc = checkSmem(c->patchSmem(kPingThreads), "pingPongKernel"))) return rc;
  for (int it = 1; it <= iterations; ++it) {
    pingPongInitKernel<<<grid2(W, H), block2(), 0, c->stream>>>(W, H, a.fov, a.fg, a.bg, disp, c->dScratchA.p, c->dScratchB.p,
                                                                chOut);
    LAUNCHED("pingPongInitKernel");
    a.changed = chIn;
    a.changedNext = chOut;
    if (c->profiling && (rc = c->pingLog.begin(c->stream))) return rc;
    c->k.pingPong<<<listGrid(W, H, kPingThreads), kPingThreads, c->patchSmem(kPingThreads), c->stream>>>(a);
    LAUNCHED("pingPongKernel");
    if (c->profiling && (rc = c->pingLog.end(c->stream))) return rc;
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
  CU(c->dDispNext.ensure(n * c->Sd));
  for (int d = 0; d < c->Sd; ++d) {
    const int self = c->dst2src[d];
    const MismatchArgs a{c->W, c->H, c->S, self, c->dCams.p, dispAll, c->dVariance.p + (size_t)self * n, c->dFov.p + (size_t)d * n,
                         c->fgFor(d), c->varNoiseFloor, c->lp.var_high_thresh, c->dDispNext.p + (size_t)d * n,
                         c->dMismatch.p + (size_t)d * n};
    mismatchKernel<<<grid2(c->W, c->H), block2(), (size_t)c->S * sizeof(DevCamera), c->stream>>>(a);  // cameras only
    LAUNCHED("mismatchKernel");
  }
  CU(cudaMemcpyAsync(c->dDisp.p, c->dDispNext.p, n * c->Sd * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));
  // return with the planes written: peers read them through derp_disparity_device_ptr on streams of their own
  CU(cudaStreamSynchronize(c->stream));
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
  float* disp = c->dDisp.p + (size_t)dst * n;
  const float sigma = 0.005f;
  DivConst three, denom;
  CU(makeDivConst(3.0f, c->stream, &three));
  CU(makeDivConst(2.0f * (sigma * sigma), c->stream, &denom));
  bilateralKernel<GuideU16><<<grid2(c->W, c->H), block2(), bilateralSmem(spaceRadius), c->stream>>>(
      c->W, c->H, disp, GuideU16{c->dColor.p + (size_t)self * n}, c->dFov.p + (size_t)dst * n, c->fgFor(dst), spaceRadius,
      three, denom, 0.5f, 1.0f, 1.0f, c->dScratchA.p);
  LAUNCHED("bilateralKernel");
  CU(cudaMemcpyAsync(disp, c->dScratchA.p, n * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));
  return DERP_OK;
}

int derp_median(DerpCtx* c, int dst) {
  int rc = checkDst(c, dst, "derp_median", false);
  if (rc) return rc;
  const size_t n = c->plane;
  float* disp = c->dDisp.p + (size_t)dst * n;
  // The background is passed whenever one is set, also with use_foreground_masks off (unlike dstArgs' background), and
  // the kernel writes it to every pixel outside the FOV (and foreground) mask.
  medianKernel<<<grid2(c->W, c->H), block2(), 0, c->stream>>>(c->W, c->H, disp, c->bgOf(dst), c->dFov.p + (size_t)dst * n,
                                                             c->fgFor(dst), c->dScratchA.p);
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

// upsampleDisparityInPlace (UpsampleDisparityLib.cpp:98-147) on device buffers, on stream st.  dCoarse: cw*ch floats;
// with useFg, s.maskC / s.maskUp hold the masks fovAndMasks prepared.  Counts its kernels in `launches`.
int upsampleDevice(cudaStream_t st, const float* dCoarse, int cw, int ch, const float* dBgUp, int W, int H, bool useFg,
                   float* dOut, UpsampleScratch& s, uint64_t& launches) {
  int rc = DERP_OK;
  if (useFg) {
    const float scale = float(W) / float(cw);  // getRadius (UpsampleDisparityLib.cpp:93-96)
    const int radius = (int)(scale * scale + 1);
    std::vector<int> xo, yo;
    nearestAxis(cw, W, xo);
    nearestAxis(ch, H, yo);
    std::vector<int> ofs(xo);
    ofs.insert(ofs.end(), yo.begin(), yo.end());
    std::vector<short2> sp;
    spiralOffsets(radius * 2 + 1, sp);
    if ((rc = upload(s.ofs, ofs.data(), ofs.size(), st)) || (rc = upload(s.spiral, sp.data(), sp.size(), st))) return rc;
    CU(cudaStreamSynchronize(st));
    CU(s.tmpA.ensure((size_t)W * H));
    nearestMaskedKernel<<<grid2(W, H), block2(), 0, st>>>(cw, ch, W, H, dCoarse, s.maskC.p, s.maskUp.p, s.ofs.p,
                                                          s.ofs.p + W, s.tmpA.p);
    replaceNansKernel<<<grid2(W, H), block2(), 0, st>>>(W, H, s.tmpA.p, dBgUp, s.maskUp.p, s.spiral.p, (int)sp.size(), dOut);
    launches += 2;
  } else {
    std::vector<int> xo, yo;
    std::vector<float> al, be;
    lanczosAxis(cw, W, xo, al);
    lanczosAxis(ch, H, yo, be);
    std::vector<int> ofs(xo);
    ofs.insert(ofs.end(), yo.begin(), yo.end());
    std::vector<float> taps(al);
    taps.insert(taps.end(), be.begin(), be.end());
    if ((rc = upload(s.ofs, ofs.data(), ofs.size(), st)) || (rc = upload(s.taps, taps.data(), taps.size(), st))) return rc;
    CU(cudaStreamSynchronize(st));
    CU(s.tmpA.ensure((size_t)cw * ch));
    CU(s.tmpB.ensure((size_t)W * ch));
    nanToKernel<<<grid1((size_t)cw * ch), 256, 0, st>>>((size_t)cw * ch, dCoarse, 1e-4f, s.tmpA.p);
    lanczosHKernel<<<grid2(W, ch), block2(), 0, st>>>(cw, ch, W, s.tmpA.p, s.ofs.p, s.taps.p, s.tmpB.p);
    lanczosVKernel<<<grid2(W, H), block2(), 0, st>>>(ch, W, H, s.tmpB.p, s.ofs.p + W, s.taps.p + (size_t)W * 8, dOut);
    launches += 3;
  }
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) return fail(DERP_ECUDA, std::string("upsample kernels: ") + cudaGetErrorString(e));
  return DERP_OK;
}

__global__ void andMaskKernel(size_t n, const uint8_t* a, const uint8_t* b, uint8_t* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (a[i] && b[i]) ? 1 : 0;
}

// The caller's foreground masks AND-ed with the FOV masks of `cam` at both sizes (UpsampleDisparityLib.cpp:163-176), into
// s.maskC / s.maskUp on stream st.  fovUp: the fine FOV mask when the caller has it, else it is built in s.fovUp.
int fovAndMasks(cudaStream_t st, const DevCamera* cam, const uint8_t* coarseMask, int cw, int ch, const uint8_t* fineMask,
                const uint8_t* fovUp, int W, int H, UpsampleScratch& s, uint64_t& launches) {
  const size_t nc = (size_t)cw * ch, n = (size_t)W * H;
  CU(s.maskC.ensure(nc));
  CU(s.maskUp.ensure(n));
  CU(s.fovC.ensure(nc));
  CU(cudaMemcpyAsync(s.maskC.p, coarseMask, nc, cudaMemcpyDefault, st));
  CU(cudaMemcpyAsync(s.maskUp.p, fineMask, n, cudaMemcpyDefault, st));
  fovMaskKernel<<<grid2(cw, ch), block2(), 0, st>>>(cam, cw, ch, s.fovC.p);
  if (!fovUp) {
    CU(s.fovUp.ensure(n));
    fovMaskKernel<<<grid2(W, H), block2(), 0, st>>>(cam, W, H, s.fovUp.p);
    fovUp = s.fovUp.p;
    launches++;
  }
  andMaskKernel<<<grid1(nc), 256, 0, st>>>(nc, s.fovC.p, s.maskC.p, s.maskC.p);
  andMaskKernel<<<grid1(n), 256, 0, st>>>(n, fovUp, s.maskUp.p, s.maskUp.p);
  launches += 3;
  return DERP_OK;
}

}  // namespace

extern "C" {

// shared body of derp_upsample_from / derp_upsample_from_kept: dCoarse is a device plane; every temporary belongs to the
// context (no allocation, no host synchronisation per call)
static int upsampleIntoLevel(DerpCtx* c, int dst, const float* dCoarse, int cw, int ch, const uint8_t* coarse_mask,
                             const uint8_t* fine_mask, const char* who) {
  const bool useFg = c->lp.use_foreground_masks != 0;
  if (useFg) {
    if (!coarse_mask || !fine_mask) return fail(DERP_EINVAL, std::string(who) + ": masks required");
    if (!c->haveBg) return fail(DERP_ESTATE, std::string(who) + ": background disparity not set");
    const int rc = fovAndMasks(c->stream, c->dCams.p + c->dst2src[dst], coarse_mask, cw, ch, fine_mask,
                               c->dFov.p + (size_t)dst * c->plane, c->W, c->H, c->up, c->launches);
    if (rc) return rc;
  }
  return upsampleDevice(c->stream, dCoarse, cw, ch, c->bgOf(dst), c->W, c->H, useFg, c->dDisp.p + (size_t)dst * c->plane,
                        c->up, c->launches);
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

// computeResizeAreaTab (resize.cpp) as per-destination tap ranges; scale = 1. / (dsize / ssize), as cv::resize derives it
static void areaTaps(int ssize, int dsize, double scale, std::vector<int>& ofs, std::vector<int>& si, std::vector<float>& alpha) {
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

// The taps of INTER_AREA's bilinear variant on one axis (cv::resize when an axis grows).  On the x axis a column whose
// second tap would pass the last one takes the last column alone (xmax: the first such column); rows are clipped by the
// kernel instead, with the weights as computed.
static void linearTaps(int ssize, int dsize, bool xAxis, std::vector<LinearTap>& tab, int* xmax) {
  const double inv = (double)dsize / ssize, scale = 1. / inv;
  tab.resize(dsize);
  if (xmax) *xmax = dsize;
  for (int d = 0; d < dsize; ++d) {
    int s = floorD(d * scale);
    float f = (float)((d + 1) - (s + 1) * inv);
    f = f <= 0 ? 0.f : f - (float)floorD(f);
    if (xAxis && s + 1 >= ssize) {
      *xmax = std::min(*xmax, d);
      if (s >= ssize - 1) {
        f = 0.f;
        s = ssize - 1;
      }
    }
    const float w0 = 1.f - f;
    tab[d] = LinearTap{s, w0, f, (int)std::lrintf(w0 * (float)kResizeCoefScale), (int)std::lrintf(f * (float)kResizeCoefScale)};
  }
}

}  // extern "C"

namespace {
// grow-only tap tables per host thread
struct ResizeTables {
  DevBuf<int> xo, xs, yo, ys;
  DevBuf<float> xa, ya;
  DevBuf<LinearTap> xl, yl;
};

// cv::resize(INTER_AREA) [+ threshold] of device image sp into device image dp on the legacy default stream.  *synced: the
// call waited for the kernel (a general ratio: its tables live in thread scratch).
template <typename T, int C>
int resizeAreaDevice(const T* sp, int sw, int sh, T* dp, int dw, int dh, int thr, ResizeTables& sc, bool* synced) {
  *synced = false;
  const size_t nd = (size_t)dw * dh * C;
  const dim3 grid((unsigned)(((size_t)dw * C + 255) / 256), (unsigned)std::min(dh, 65535));
  if (sw == dw && sh == dh && thr < 0) {  // cv::resize copies an image of the same size
    CU(cudaMemcpyAsync(dp, sp, nd * sizeof(T), cudaMemcpyDeviceToDevice, 0));
    return DERP_OK;
  }
  const double scaleX = 1. / ((double)dw / sw), scaleY = 1. / ((double)dh / sh);
  int rc;
  if (scaleX >= 1 && scaleY >= 1) {
    const int kx = (int)std::lrint(scaleX), ky = (int)std::lrint(scaleY);  // saturate_cast<int>
    if (std::fabs(scaleX - kx) < 2.220446049250313e-16 && std::fabs(scaleY - ky) < 2.220446049250313e-16) {
      areaResizeFastKernel<T, C><<<grid, 256>>>(sp, sw, dp, dw, dh, kx, ky, thr);
    } else {
      std::vector<int> xo, xs, yo, ys;
      std::vector<float> xa, ya;
      areaTaps(sw, dw, scaleX, xo, xs, xa);
      areaTaps(sh, dh, scaleY, yo, ys, ya);
      if ((rc = upload(sc.xo, xo.data(), xo.size())) || (rc = upload(sc.xs, xs.data(), xs.size())) ||
          (rc = upload(sc.xa, xa.data(), xa.size())) || (rc = upload(sc.yo, yo.data(), yo.size())) ||
          (rc = upload(sc.ys, ys.data(), ys.size())) || (rc = upload(sc.ya, ya.data(), ya.size())))
        return rc;
      areaResizeKernel<T, C><<<grid, 256>>>(sp, sw, dp, dw, dh, sc.xo.p, sc.xs.p, sc.xa.p, sc.yo.p, sc.ys.p, sc.ya.p, thr);
      CU(cudaDeviceSynchronize());
      *synced = true;
    }
  } else {
    std::vector<LinearTap> xt, yt;
    int xmax = 0;
    linearTaps(sw, dw, true, xt, &xmax);
    linearTaps(sh, dh, false, yt, nullptr);
    if ((rc = upload(sc.xl, xt.data(), xt.size())) || (rc = upload(sc.yl, yt.data(), yt.size()))) return rc;
    areaEnlargeKernel<T, C><<<grid, 256>>>(sp, sw, sh, dp, dw, dh, sc.xl.p, xmax, sc.yl.p, thr);
    CU(cudaDeviceSynchronize());
    *synced = true;
  }
  CU(cudaGetLastError());
  return DERP_OK;
}

// derp_resize_area for one sample type and channel count: stage, resize, copy back, return with dst written
template <typename T, int C>
int resizeAreaCall(const void* src, int sw, int sh, void* dst, int dw, int dh, int thr) {
  static thread_local struct {
    DevBuf<T> src, dst;
    ResizeTables tables;
  } sc;
  const T* sp = static_cast<const T*>(src);
  T* dp = static_cast<T*>(dst);
  const size_t ns = (size_t)sw * sh * C, nd = (size_t)dw * dh * C;
  bool synced = false;
  int rc = stageIn(sp, ns, sc.src);
  if (rc || (rc = outBuffer(dp, nd, sc.dst)) || (rc = resizeAreaDevice<T, C>(sp, sw, sh, dp, dw, dh, thr, sc.tables, &synced)) ||
      (rc = stageOut(static_cast<T*>(dst), dp, nd)))
    return rc;
  CU(cudaDeviceSynchronize());
  return DERP_OK;
}
}  // namespace

extern "C" {

int derp_downscale_area(int device, const uint16_t* src, int src_w, int src_h, uint16_t* dst, int dst_w, int dst_h) {
  if (!src || !dst || src_w < 1 || src_h < 1 || dst_w < 1 || dst_h < 1 || dst_w > src_w || dst_h > src_h)
    return fail(DERP_EINVAL, "derp_downscale_area: bad arguments (INTER_AREA is only used to shrink on this path)");
  CU(cudaSetDevice(device));
  const size_t ns = (size_t)src_w * src_h * 3, nd = (size_t)dst_w * dst_h * 3;
  // grow-only scratch per host thread: staged images and the tap tables of a general ratio
  static thread_local struct {
    DevBuf<uint16_t> src, dst;
    ResizeTables tables;
  } sc;
  // device-resident images are used in place; host images are staged
  const uint16_t* sp = src;
  uint16_t* dp = dst;
  int rc = stageIn(sp, ns, sc.src);
  if (rc || (rc = outBuffer(dp, nd, sc.dst))) return rc;
  // an integer ratio is stream-ordered on the legacy default stream when both images are device memory (a pyramid built
  // on the device); a general ratio returns with dst written
  bool synced = false;
  if ((rc = resizeAreaDevice<uint16_t, 3>(sp, src_w, src_h, dp, dst_w, dst_h, -1, sc.tables, &synced))) return rc;
  if ((rc = stageOut(dst, dp, nd))) return rc;
  // a staged image returns with the copies done: the caller may reuse its buffer (a copy to another GPU does not wait)
  if (sp != src || dp != dst) CU(cudaDeviceSynchronize());
  return DERP_OK;
}

int derp_resize_area(int device, const void* src, int sample_bits, int channels, int src_w, int src_h, void* dst, int dst_w,
                     int dst_h, int threshold) {
  if (!src || !dst || (sample_bits != 8 && sample_bits != 16 && sample_bits != 32) ||
      (channels != 1 && channels != 3 && channels != 4) || src_w < 1 || src_h < 1 || dst_w < 1 || dst_h < 1)
    return fail(DERP_EINVAL, "derp_resize_area: bad arguments (8-, 16- or 32-bit samples, 1, 3 or 4 channels, sizes > 0)");
  // rows of samples are indexed with int and whole images with size_t
  size_t bytes;
  for (const auto& [w, h] : {std::pair<int, int>{src_w, src_h}, {dst_w, dst_h}})
    if ((size_t)w * channels > (size_t)INT_MAX ||
        __builtin_mul_overflow((size_t)w * channels * (sample_bits / 8), (size_t)h, &bytes))
      return fail(DERP_EINVAL, "derp_resize_area: image too large");
  CU(cudaSetDevice(device));
  switch (sample_bits * 8 + channels) {
    case 8 * 8 + 1: return resizeAreaCall<uint8_t, 1>(src, src_w, src_h, dst, dst_w, dst_h, threshold);
    case 8 * 8 + 3: return resizeAreaCall<uint8_t, 3>(src, src_w, src_h, dst, dst_w, dst_h, threshold);
    case 8 * 8 + 4: return resizeAreaCall<uint8_t, 4>(src, src_w, src_h, dst, dst_w, dst_h, threshold);
    case 16 * 8 + 1: return resizeAreaCall<uint16_t, 1>(src, src_w, src_h, dst, dst_w, dst_h, threshold);
    case 16 * 8 + 3: return resizeAreaCall<uint16_t, 3>(src, src_w, src_h, dst, dst_w, dst_h, threshold);
    case 16 * 8 + 4: return resizeAreaCall<uint16_t, 4>(src, src_w, src_h, dst, dst_w, dst_h, threshold);
    case 32 * 8 + 1: return resizeAreaCall<float, 1>(src, src_w, src_h, dst, dst_w, dst_h, threshold);
    case 32 * 8 + 3: return resizeAreaCall<float, 3>(src, src_w, src_h, dst, dst_w, dst_h, threshold);
    default: return resizeAreaCall<float, 4>(src, src_w, src_h, dst, dst_w, dst_h, threshold);
  }
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
  // grow-only scratch per host thread (the app masks one camera after the other)
  static thread_local struct {
    DevBuf<uint16_t> dT, dF, dTb, dFb;
    DevBuf<uint8_t> dM, dM2;
  } sc;
  const uint16_t *pt = templ, *pf = frame;
  int rc = stageIn(pt, n * 3, sc.dT);
  if (rc || (rc = stageIn(pf, n * 3, sc.dF))) return rc;
  CU(sc.dM.ensure(n));
  if (blur_radius == 1) {
    CU(sc.dTb.ensure(n * 3));
    CU(sc.dFb.ensure(n * 3));
    const dim3 g((width * 3 + 255) / 256, height);
    gaussian3Kernel<<<g, 256>>>(pt, width, height, sc.dTb.p);
    gaussian3Kernel<<<g, 256>>>(pf, width, height, sc.dFb.p);
    pt = sc.dTb.p;
    pf = sc.dFb.p;
  }
  foregroundDiffKernel<<<grid1(n), 256>>>(n, pt, pf, threshold, sc.dM.p);
  if (morph_closing_size > 0) {  // MORPH_CLOSE = dilate, then erode
    CU(sc.dM2.ensure(n));
    morphRectKernel<<<grid2(width, height), block2()>>>(sc.dM.p, width, height, morph_closing_size, 1, sc.dM2.p);
    morphRectKernel<<<grid2(width, height), block2()>>>(sc.dM2.p, width, height, morph_closing_size, 0, sc.dM.p);
  }
  CU(cudaGetLastError());
  CU(cudaMemcpy(mask, sc.dM.p, n, cudaMemcpyDefault));
  CU(cudaDeviceSynchronize());  // return with mask written, also when it is device memory (that copy does not wait)
  return DERP_OK;
}

// The taps of cv::GaussianBlur((2 r + 1)^2, sigma 0) as OpenCV's bit-exact path builds them (getGaussianKernelBitExact,
// then getGaussianKernelFixedPoint_ED with 16 fraction bits): its table kernels for sizes 3, 5, 7 and 9; above those the
// sampled Gaussian with sigma = 0.15 n + 0.35 (one rounding), normalised to sum 1, scaled to 2^16 with error diffusion
// over the left half and mirrored, the centre tap taking what is left of 2^16.
static GaussTaps gaussTaps(int r) {
  GaussTaps t{};
  t.r = r;
  const int n = 2 * r + 1;
  if (r <= 4) {  // left halves and centres of {1 2 1} / 4, {1 4 6 4 1} / 16, {2 7 14 18 14 7 2} / 64, {4 13 30 51 60 ...} / 256
    static const uint32_t kTable[5][5] = {{1}, {1, 2}, {1, 4, 6}, {2, 7, 14, 18}, {4, 13, 30, 51, 60}};
    for (int i = 0; i <= r; ++i) t.k[i] = t.k[n - 1 - i] = kTable[r][i] << (16 - 2 * r);
    return t;
  }
  const double sigma = std::fma((double)n, 0.15, 0.35), scale = -0.125 / (sigma * sigma);
  double half[kGaussMaxRadius], sum = 0;
  for (int i = 0, x = 1 - n; i < r; ++i, x += 2) {
    half[i] = std::exp((double)(x * x) * scale);
    sum += half[i];
  }
  const double mul = 1.0 / (sum * 2 + 1);
  double err = 0;
  uint32_t side = 0;
  for (int i = 0; i < r; ++i) {
    const double a = half[i] * mul * 65536.0 + err, v = std::nearbyint(a);  // cvRound: to nearest, ties to even
    err = a - v;
    t.k[i] = t.k[n - 1 - i] = (uint32_t)v;
    side += (uint32_t)v;
  }
  t.k[r] = 65536u - 2 * side;
  return t;
}

int derp_gaussian_blur(int device, const uint16_t* src, int width, int height, int radius, uint16_t* dst) {
  if (!src || !dst || width < 1 || height < 1 || radius < 0 || radius > kGaussMaxRadius)
    return fail(DERP_EINVAL, "derp_gaussian_blur: bad arguments (radius 0 to " + std::to_string(kGaussMaxRadius) + ")");
  CU(cudaSetDevice(device));
  const size_t n = (size_t)width * height * 3;
  if (radius == 0) {  // a 1 x 1 kernel: a copy
    if (src != dst) CU(cudaMemcpy(dst, src, n * sizeof(uint16_t), cudaMemcpyDefault));
    CU(cudaDeviceSynchronize());  // also when both are device memory (that copy does not wait)
    return DERP_OK;
  }
  // grow-only scratch per host thread: staged images and the row pass's u32 sums
  static thread_local struct {
    DevBuf<uint16_t> src, dst;
    DevBuf<uint32_t> rows;
  } sc;
  const uint16_t* sp = src;
  uint16_t* dp = dst;
  int rc = stageIn(sp, n, sc.src);
  if (rc || (rc = outBuffer(dp, n, sc.dst))) return rc;
  CU(sc.rows.ensure(n));
  const GaussTaps taps = gaussTaps(radius);
  const dim3 rowGrid((width + kGaussRowPixels - 1) / kGaussRowPixels, std::min(height, 65535));
  gaussRowKernel<<<rowGrid, 256, 3 * (kGaussRowPixels + 2 * radius) * sizeof(uint32_t)>>>(sp, width, height, taps,
                                                                                          sc.rows.p);
  const dim3 colGrid((unsigned)((3 * (size_t)width + kGaussColElems - 1) / kGaussColElems),
                     (height + kGaussColRows - 1) / kGaussColRows);
  gaussColKernel<<<colGrid, dim3(kGaussColElems, kGaussColThreadsY),
                   (kGaussColRows + 2 * radius) * kGaussColElems * sizeof(uint32_t)>>>(sc.rows.p, width, height, taps, dp);
  CU(cudaGetLastError());
  if ((rc = stageOut(dst, dp, n))) return rc;
  CU(cudaDeviceSynchronize());  // return with dst written, also when it is device memory
  return DERP_OK;
}

int derp_upsample_disparity(int device, const DerpCameraDesc* cam, const float* coarse, int coarse_w, int coarse_h,
                            const float* background_up, const uint8_t* coarse_mask, const uint8_t* fine_mask, int out_w,
                            int out_h, int use_foreground_masks, float* out) {
  if (!cam || !coarse || !out || coarse_w < 1 || coarse_h < 1 || out_w < 1 || out_h < 1)
    return fail(DERP_EINVAL, "derp_upsample_disparity: bad arguments");
  CU(cudaSetDevice(device));
  if (use_foreground_masks && (!coarse_mask || !fine_mask || !background_up)) return fail(DERP_EINVAL, "derp_upsample_disparity: masks/background required");
  const size_t nc = (size_t)coarse_w * coarse_h, n = (size_t)out_w * out_h;
  // grow-only scratch per host thread (the app upsamples one camera after the other)
  static thread_local struct {
    UpsampleScratch up;
    DevBuf<float> coarse, bg, out;
    DevBuf<DevCamera> cam;
  } sc;
  cudaStream_t st = nullptr;  // legacy default stream
  uint64_t launches = 0;      // not reported: no context
  const float *dCoarse = coarse, *dBg = background_up;
  float* dOut = out;
  int rc = stageIn(dCoarse, nc, sc.coarse);
  if (rc || (rc = outBuffer(dOut, n, sc.out))) return rc;
  if (use_foreground_masks) {
    DevCamera hc;
    if (!host::makeCamera(*cam, &hc)) return fail(DERP_EINVAL, "derp_upsample_disparity: invalid camera");
    host::normalise(hc);
    if ((rc = upload(sc.cam, &hc, 1)) || (rc = stageIn(dBg, n, sc.bg)) ||
        (rc = fovAndMasks(st, sc.cam.p, coarse_mask, coarse_w, coarse_h, fine_mask, nullptr, out_w, out_h, sc.up, launches)))
      return rc;
  }
  if ((rc = upsampleDevice(st, dCoarse, coarse_w, coarse_h, dBg, out_w, out_h, use_foreground_masks != 0, dOut, sc.up,
                           launches)) ||
      (rc = stageOut(out, dOut, n)))
    return rc;
  CU(cudaDeviceSynchronize());  // synchronous: return with out written, also when it is device memory
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
  const size_t n = c->plane;
  return copyPlanes(c, n * sizeof(float), {{c->dDisp.p + (size_t)dst * n, disparity}, {c->dCost.p + (size_t)dst * n, cost},
                                           {c->dConf.p + (size_t)dst * n, confidence}});
}

int derp_get_disparity(DerpCtx* c, int dst, float* disparity, float* cost, float* confidence) {
  int rc = checkDst(c, dst, "derp_get_disparity", false);
  if (rc) return rc;
  const size_t n = c->plane;
  return copyPlanes(c, n * sizeof(float), {{disparity, c->dDisp.p + (size_t)dst * n}, {cost, c->dCost.p + (size_t)dst * n},
                                           {confidence, c->dConf.p + (size_t)dst * n}});
}

// destination dst's plane of the FOV or the mismatch masks
static int getMask(DerpCtx* c, int dst, uint8_t* mask, const char* who, bool mismatch) {
  if (!mask) return fail(DERP_EINVAL, "bad arguments");
  int rc = checkDst(c, dst, who, false);
  if (rc) return rc;
  return copyPlanes(c, c->plane, {{mask, (mismatch ? c->dMismatch.p : c->dFov.p) + (size_t)dst * c->plane}});
}
int derp_get_fov_mask(DerpCtx* c, int dst, uint8_t* mask) { return getMask(c, dst, mask, "derp_get_fov_mask", false); }
int derp_get_mismatch_mask(DerpCtx* c, int dst, uint8_t* mask) { return getMask(c, dst, mask, "derp_get_mismatch_mask", true); }

int derp_get_variance(DerpCtx* c, int src, float* variance) {
  if (!c || !variance) return fail(DERP_EINVAL, "bad arguments");
  if (!c->levelOpen || !c->haveColors) return fail(DERP_ESTATE, "derp_get_variance: colours not set");
  if (src < 0 || src >= c->S) return fail(DERP_EINVAL, "src out of range");
  int rc = useDevice(c);
  if (rc) return rc;
  return copyPlanes(c, c->plane * sizeof(float), {{variance, c->dVariance.p + (size_t)src * c->plane}});
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
  return copyPlanes(c, c->plane * sizeof(float2), {{warp_xy, c->warpOf(c->projDst) + (size_t)src * c->plane}});
}

// source src's plane of the float4 colour or bias table as u16 B, G, R texels
static int getTexels(DerpCtx* c, int src, uint16_t* bgr, const char* who, bool bias) {
  if (!bgr) return fail(DERP_EINVAL, "bad arguments");
  int rc = checkProj(c, src, who);
  if (rc) return rc;
  if ((rc = ensureTablesF32(c))) return rc;  // may reallocate the tables
  const size_t n = c->plane;
  uint16_t* st = reinterpret_cast<uint16_t*>(c->dStage.p);
  unpackTexelF32Kernel<<<grid1(n), 256, 0, c->stream>>>(n, (bias ? c->dProjBias.p : c->dProjColor.p) + (size_t)src * n, st);
  LAUNCHED("unpackTexelF32Kernel");
  return copyPlanes(c, n * 6, {{bgr, st}});
}
int derp_get_proj_color(DerpCtx* c, int src, uint16_t* bgr) { return getTexels(c, src, bgr, "derp_get_proj_color", false); }
int derp_get_proj_bias(DerpCtx* c, int src, uint16_t* bgr) { return getTexels(c, src, bgr, "derp_get_proj_bias", true); }

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
  // its own candidate table: the brute-force sweep's cached one in dDisparities stays as it is
  const std::vector<float> disparities = probeDisparities(num_depths, min_depth_m, max_depth_m);
  DevBuf<float> dTab;
  DevBuf<unsigned long long> dStats;
  if ((rc = upload(dTab, disparities.data(), num_depths, c->stream))) return rc;
  CU(dStats.ensure(5));
  CU(cudaMemsetAsync(dStats.p, 0, 5 * sizeof(unsigned long long), c->stream));
  if ((rc = ensureTablesF32(c))) return rc;
  if ((rc = resetCounters(c))) return rc;
  if ((rc = checkSmem(c->camSmem(), "lowerBoundCheckKernel"))) return rc;
  CU(c->dLb.ensure((size_t)num_depths * c->plane));
  CU(c->dSeed.ensure(c->plane));
  const DstArgs da = c->dstArgs(dst);  // after ensureTablesF32 (see dstArgs)
  if ((rc = boundPass(c, da, dTab.p, num_depths, SweepShape{kBlockY, 1, num_depths}))) return rc;
  const CheckArgs ca{da, dTab.p, num_depths, c->dLb.p, dStats.p};
  c->k.lowerBoundCheck<<<grid2(c->W, c->H), block2(), c->camSmem(), c->stream>>>(ca);
  LAUNCHED("lowerBoundCheckKernel");
  return copyPlanes(c, 5 * sizeof(uint64_t), {{stats, dStats.p}});
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
  static thread_local struct {
    DevBuf<uint2> dG;
    DevBuf<float> dD, dOut;
    DevBuf<uint8_t> dM, dStage;
  } sc;
  CU(sc.dG.ensure(n * num_frames));
  CU(sc.dD.ensure(n * num_frames));
  CU(sc.dM.ensure(n * num_frames));
  CU(sc.dOut.ensure(n));
  CU(sc.dStage.ensure(n * 6));
  for (int t = 0; t < num_frames; ++t) {  // frames may live in host or device memory (e.g. halo frames received over NVLink)
    CU(cudaMemcpy(sc.dStage.p, guides[t], n * 6, cudaMemcpyDefault));
    packColorKernel<<<grid1(n), 256>>>(n, reinterpret_cast<const uint16_t*>(sc.dStage.p), sc.dG.p + (size_t)t * n);
    CU(cudaMemcpy(sc.dD.p + (size_t)t * n, disps[t], n * sizeof(float), cudaMemcpyDefault));
    CU(cudaMemcpy(sc.dM.p + (size_t)t * n, masks[t], n, cudaMemcpyDefault));
  }
  TemporalArgs a;
  a.W = width;
  a.H = height;
  a.T = num_frames;
  a.frameOffset = frame_offset;
  a.radius = spatial_radius;
  a.guides = sc.dG.p;
  a.disps = sc.dD.p;
  a.masks = sc.dM.p;
  CU(makeDivConst(65535.0f, 0, &a.maxPix));
  CU(makeDivConst(sigma * sigma, 0, &a.sig2));
  a.w0 = weight0;
  a.w1 = weight1;
  a.w2 = weight2;
  a.out = sc.dOut.p;
  temporalKernel<<<grid2(width, height), block2()>>>(a);
  CU(cudaGetLastError());
  CU(cudaMemcpy(out, sc.dOut.p, n * sizeof(float), cudaMemcpyDefault));
  return DERP_OK;
}

int derp_joint_bilateral_f32(int device, int width, int height, const float* image, const float* guide_bgr,
                             const uint8_t* mask, int radius, float sigma, float weight0, float weight1, float weight2,
                             float* out) {
  if (!image || !guide_bgr || !mask || !out || radius < 0 || width < 1 || height < 1)
    return fail(DERP_EINVAL, "derp_joint_bilateral_f32: bad arguments");
  CU(cudaSetDevice(device));
  const size_t n = (size_t)width * height;
  // grow-only scratch per host thread (the app filters one camera after the other)
  static thread_local struct {
    DevBuf<float> dI, dG, dO;
    DevBuf<uint8_t> dM;
  } sc;
  const float *img = image, *guide = guide_bgr;
  const uint8_t* msk = mask;
  float* o = out;
  int rc = stageIn(img, n, sc.dI);
  if (rc || (rc = stageIn(guide, n * 3, sc.dG)) || (rc = stageIn(msk, n, sc.dM)) || (rc = outBuffer(o, n, sc.dO))) return rc;
  DivConst three, denom;
  CU(makeDivConst(3.0f, 0, &three));
  CU(makeDivConst(2.0f * (sigma * sigma), 0, &denom));
  if (bilateralSmem(radius) <= kBilMaxSmem)
    bilateralKernel<GuideF32><<<grid2(width, height), block2(), bilateralSmem(radius)>>>(
        width, height, img, GuideF32{guide}, msk, nullptr, radius, three, denom, weight0, weight1, weight2, o);
  else
    bilateralWideKernel<GuideF32><<<grid2(width, height), block2()>>>(width, height, img, GuideF32{guide}, msk, nullptr, radius,
                                                                    three, denom, weight0, weight1, weight2, o);
  CU(cudaGetLastError());
  if ((rc = stageOut(out, o, n))) return rc;
  CU(cudaDeviceSynchronize());  // synchronous: return with out written, also when it is device memory
  return DERP_OK;
}

}  // extern "C"

// ---- host-side test hooks ---------------------------------------------------------------------------
// The selection, RNG and camera code is __host__ __device__; these entry points run the HOST
// instantiation so that CPU-only tests (-m "not gpu") can check it against libstdc++ / the oracle.
static __global__ void appendRangeKernel(int n, UndecidedView<unsigned long long> undecided) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) undecided.append(i);
}

extern "C" {

// 1 if the three-instruction constant division (derp_divconst.cuh) was validated exact for divisor c on `device`
// (every dividend mantissa against __fdiv_rn), 0 if it failed and the kernels use the plain division, < 0 on error.
int derp_test_div_const(int device, float c) {
  if (cudaSetDevice(device) != cudaSuccess) return DERP_ECUDA;
  DivConst k;
  if (makeDivConst(c, 0, &k) != cudaSuccess) return DERP_ECUDA;
  return k.fast;
}

// UndecidedList::collect (derp_host.cuh) on a kernel that appends 0 .. n - 1, from a new list of start_capacity
// entries: the n items in list order into out; returns the number of launches it took, < 0 on error.
int derp_test_undecided_list(int device, int n, uint64_t start_capacity, uint64_t* out) {
  if (n < 0 || start_capacity < 1 || !out) return fail(DERP_EINVAL, "derp_test_undecided_list: bad arguments");
  CU(cudaSetDevice(device));
  UndecidedList<unsigned long long> list;
  std::vector<unsigned long long> items;
  int launches = 0;
  auto launch = [&](UndecidedView<unsigned long long> undecided) {
    ++launches;
    appendRangeKernel<<<grid1(std::max(n, 1)), 256>>>(n, undecided);
    return DERP_OK;
  };
  if (int rc = list.collect(launch, items, start_capacity)) return rc;
  std::copy(items.begin(), items.end(), out);
  return launches;
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
