// Filtered brute-force sweep: the same winner-takes-all result as sweepKernel (bit for bit), with the exact cost
// evaluated only where it can matter.
//
//   pass 1  sweepLowerKernel   every (pixel, candidate): L = a proven LOWER BOUND of computeCost (evalCost<..., LOWER>:
//                              exact visibility / projection / sample positions, cheap fused-multiply-add SSD with the
//                              error analysis in derp_cost.cuh).  Writes L to lb[candidate][pixel] and keeps, per pixel,
//                              the candidate with the smallest L (the seed).
//   pass 2a sweepSeedKernel    exact cost E* of the seed candidate of every pixel -> best[pixel] = (E*, seed).
//   pass 2b refineListKernel   every other candidate with L <= E* goes on a work list (warp-aggregated append, entries
//                              of one 32-pixel row segment and one candidate stay together).
//   pass 2c refineKernel       exact cost of every list entry, merged with atomicMin((cost bits << 32) | index).
//
// Why the result is the reference's: the reference's winner is the candidate with the lowest cost, lowest index among
// equals (strict-< scan in index order, Derp.cpp:323-333).  Its cost is <= E*, so its L is <= E*: it is the seed or on
// the list, is evaluated exactly, and the 64-bit atomicMin orders (cost, index) lexicographically.  Candidates whose L
// is FLT_MAX have no contributing source (visibility is exact in pass 1), cost FLT_MAX, and can never win.
// L = 0 marks "no bound formed" (a source took the generic border path): always refined.
#pragma once

#include "derp_cost.cuh"

namespace derp {

struct LowerArgs : DstArgs {
  const float* disparities;
  int D, chunk;
  float* lb;                   // [D][H][W]
  unsigned long long* seed;    // [H][W]  (L bits << 32 | candidate), atomicMin across candidate chunks
  unsigned long long* counters;
};

template <class Mask>
__global__ void __launch_bounds__(32 * kSweepMaxRows, kSweepMinCtas) sweepLowerKernel(const LowerArgs a) {
  extern __shared__ double smemRaw[];
  DevCamera* cams = reinterpret_cast<DevCamera*>(smemRaw);
  float* tile = reinterpret_cast<float*>(cams + a.v.S);
  stageCameras(cams, a.v.cams, a.v.S);
  loadDstTile(tile, a.v, blockIdx.x * kBlockX, blockIdx.y * blockDim.y, 0.5f);
  const int W = a.v.W, H = a.v.H;
  const int x = blockIdx.x * kBlockX + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  unsigned hits = 0, evals = 0;
  if (x >= 1 && x < W - 1 && y >= 1 && y < H - 1) {
    const size_t p = (size_t)y * W + x;
    const bool active = a.fov[p] && (!a.fg || a.fg[p]);
    if (active) {
      PixelState ps;
      loadPixelState(a.v, cams[a.v.self], tile, x, y, ps, 0.5f);
      const float bgd = a.bg ? a.bg[p] : 0.f;
      const int c0 = blockIdx.z * a.chunk;
      const int c1 = min(a.D, c0 + a.chunk);
      const size_t plane = (size_t)W * H;
      float bestL = FLT_MAX;
      int bestIdx = -1;
      for (int c = c0; c < c1; ++c) {
        const float d = __ldg(a.disparities + c);
        float L = FLT_MAX;
        if (!(a.bg && !(bgd < d))) {  // closerMask (Derp.cpp:240-243)
          L = evalCost<Mask, kTileW, 1, float4, true>(a.v, cams, ps, d, &hits);
          ++evals;
        }
        a.lb[c * plane + p] = L;
        if (L < bestL) {
          bestL = L;
          bestIdx = c;
        }
      }
      if (bestIdx >= 0) {
        const unsigned long long packed =
            ((unsigned long long)__float_as_uint(bestL) << 32) | (unsigned long long)(unsigned)bestIdx;
        atomicMin(a.seed + p, packed);
      }
    }
  }
  addCounters(a.counters, evals, hits);
}

// Not derived from DstArgs: its bg would take the parameter from 128 to 136 bytes, past the 128 bytes up to which nvcc
// (12.9) loads a kernel parameter field by field instead of addressing it in parameter space.  That changes this
// kernel's code and raises its spills (52 to 80 bytes with the 64-bit mask).
struct SeedArgs {
  CostView v;
  const uint8_t* fov;
  const uint8_t* fg;
  const float* disparities;
  const unsigned long long* seed;
  unsigned long long* best;
};

// exact cost of the seed candidate; same CTA shape and shared-memory layout as evalCostKernel
template <class Mask>
__global__ void __launch_bounds__(kBlockX* kBlockY, kCostMinCtas) sweepSeedKernel(const SeedArgs a) {
  extern __shared__ double smemRaw[];
  DevCamera* cams = reinterpret_cast<DevCamera*>(smemRaw);
  float* tile = reinterpret_cast<float*>(cams + a.v.S);
  stageCameras(cams, a.v.cams, a.v.S);
  loadDstTile(tile, a.v, blockIdx.x * kBlockX, blockIdx.y * kBlockY);
  const int W = a.v.W, H = a.v.H;
  const int x = blockIdx.x * kBlockX + threadIdx.x, y = blockIdx.y * kBlockY + threadIdx.y;
  if (x < 1 || x >= W - 1 || y < 1 || y >= H - 1) return;
  const size_t p = (size_t)y * W + x;
  if (!(a.fov[p] && (!a.fg || a.fg[p]))) return;
  const unsigned cstar = (unsigned)(a.seed[p] & 0xffffffffull);
  if (cstar == 0xffffffffu) return;  // no candidate has a source: best stays "none"
  PixelState ps;
  loadPixelState(a.v, cams[a.v.self], tile, x, y, ps);
  unsigned hits = 0;
  const float cost = evalCost<Mask, kTileW, 1>(a.v, cams, ps, __ldg(a.disparities + cstar), &hits);
  if (cost < FLT_MAX) a.best[p] = ((unsigned long long)__float_as_uint(cost) << 32) | (unsigned long long)cstar;
}

struct ListArgs {
  int W, H, D;
  const uint8_t* fov;
  const uint8_t* fg;
  const float* lb;
  const unsigned long long* seed;
  const unsigned long long* best;
  unsigned long long* list;  // entries: pixel index | candidate << 32
  unsigned long long capacity;
  unsigned long long* count;
};

__global__ void __launch_bounds__(kBlockX* kBlockY) refineListKernel(const ListArgs a) {
  const int x = blockIdx.x * kBlockX + threadIdx.x, y = blockIdx.y * kBlockY + threadIdx.y;
  const bool inside = x >= 1 && x < a.W - 1 && y >= 1 && y < a.H - 1;
  const size_t p = inside ? (size_t)y * a.W + x : 0;
  const bool active = inside && a.fov[p] && (!a.fg || a.fg[p]);
  unsigned cstar = 0xffffffffu;
  float estar = FLT_MAX;
  if (active) {
    cstar = (unsigned)(a.seed[p] & 0xffffffffull);
    estar = __uint_as_float((unsigned)(a.best[p] >> 32));  // 0x7f7fffff (FLT_MAX) when the seed had no finite cost
  }
  const bool any = __ballot_sync(0xffffffffu, active && cstar != 0xffffffffu) != 0;
  if (!any) return;
  const size_t plane = (size_t)a.W * a.H;
  const unsigned lane = threadIdx.x & 31u;
  for (int c = 0; c < a.D; ++c) {
    bool take = false;
    if (active && cstar != 0xffffffffu && (unsigned)c != cstar) {
      const float L = __ldg(a.lb + c * plane + p);
      take = L < FLT_MAX && L <= estar;
    }
    const unsigned m = __ballot_sync(0xffffffffu, take);
    if (!m) continue;
    unsigned long long base = 0;
    if (lane == (unsigned)(__ffs(m) - 1)) base = atomicAdd(a.count, (unsigned long long)__popc(m));
    base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
    if (take) {
      const unsigned long long slot = base + __popc(m & ((1u << lane) - 1u));
      if (slot < a.capacity) a.list[slot] = (unsigned long long)p | ((unsigned long long)(unsigned)c << 32);
    }
  }
}

struct RefineArgs {
  CostView v;
  const float* disparities;
  const unsigned long long* list;
  unsigned long long count;
  unsigned long long* best;
};

template <class Mask>
__global__ void __launch_bounds__(kPatchThreads, kPatchMinCtas) refineKernel(const RefineArgs a) {
  extern __shared__ double smemRaw[];
  DevCamera* cams = reinterpret_cast<DevCamera*>(smemRaw);
  float* patches = reinterpret_cast<float*>(cams + a.v.S);
  stageCameras(cams, a.v.cams, a.v.S);
  const unsigned long long i = (unsigned long long)blockIdx.x * kPatchThreads + threadIdx.x;
  if (i >= a.count) return;
  const unsigned long long e = a.list[i];
  const unsigned p = (unsigned)(e & 0xffffffffull), c = (unsigned)(e >> 32);
  const int y = (int)(p / (unsigned)a.v.W), x = (int)(p - (unsigned)y * (unsigned)a.v.W);
  PixelState ps;
  loadPixelStateCompactF32(a.v, cams[a.v.self], patches, x, y, ps);
  unsigned hits = 0;
  const float cost = evalCost<Mask, kPatchRP, kPatchCP, float4>(a.v, cams, ps, __ldg(a.disparities + c), &hits);
  if (cost < FLT_MAX) atomicMin(a.best + p, ((unsigned long long)__float_as_uint(cost) << 32) | (unsigned long long)c);
}

// Validation of the bound itself (derp_debug_lower_bound): exact cost of EVERY (pixel, candidate) against lb.
// stats: [0] evaluations compared, [1] violations (L > exact cost), [2] unknown (L == 0), [3] evaluations whose L is
// within 5 % of the exact cost, [4] candidates that a per-pixel threshold at the true minimum would keep.
struct CheckArgs : DstArgs {
  const float* disparities;
  int D;
  const float* lb;
  unsigned long long* stats;
};

template <class Mask>
__global__ void __launch_bounds__(kBlockX* kBlockY, kCostMinCtas) lowerBoundCheckKernel(const CheckArgs a) {
  extern __shared__ double smemRaw[];
  DevCamera* cams = reinterpret_cast<DevCamera*>(smemRaw);
  float* tile = reinterpret_cast<float*>(cams + a.v.S);
  stageCameras(cams, a.v.cams, a.v.S);
  loadDstTile(tile, a.v, blockIdx.x * kBlockX, blockIdx.y * kBlockY);
  const int W = a.v.W, H = a.v.H;
  const int x = blockIdx.x * kBlockX + threadIdx.x, y = blockIdx.y * kBlockY + threadIdx.y;
  if (x < 1 || x >= W - 1 || y < 1 || y >= H - 1) return;
  const size_t p = (size_t)y * W + x;
  if (!(a.fov[p] && (!a.fg || a.fg[p]))) return;
  PixelState ps;
  loadPixelState(a.v, cams[a.v.self], tile, x, y, ps);
  const float bgd = a.bg ? a.bg[p] : 0.f;
  const size_t plane = (size_t)W * H;
  unsigned long long n = 0, bad = 0, unk = 0, tight = 0, keep = 0;
  float minCost = FLT_MAX;
  for (int pass = 0; pass < 2; ++pass)
    for (int c = 0; c < a.D; ++c) {
      const float d = __ldg(a.disparities + c);
      if (a.bg && !(bgd < d)) continue;
      const float L = a.lb[c * plane + p];
      if (pass == 1) {
        keep += (L < FLT_MAX && L <= minCost) ? 1 : 0;
        continue;
      }
      unsigned hits = 0;
      const float cost = evalCost<Mask, kTileW, 1>(a.v, cams, ps, d, &hits);
      ++n;
      if (L > cost) ++bad;
      if (L == 0.0f) ++unk;
      if (cost < FLT_MAX && L >= 0.95f * cost) ++tight;
      minCost = fminf(minCost, cost);
    }
  atomicAdd(a.stats + 0, n);
  atomicAdd(a.stats + 1, bad);
  atomicAdd(a.stats + 2, unk);
  atomicAdd(a.stats + 3, tight);
  atomicAdd(a.stats + 4, keep);
}

}  // namespace derp
